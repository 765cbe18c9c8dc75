"""B200NewValueDetector -- the reference's detector plugin surface on top of libdmdetect.

Drop-in for ``detectmatelibrary.detectors.new_value_detector.NewValueDetector`` behind the
UNMODIFIED reference service:

  settings YAML   component_type: detectmateservice_b200.component.B200NewValueDetector
                  (the loader imports dotted paths as-is first,
                   /root/reference/src/service/features/component_loader.py:34-43,
                   calls ``cls(config=<ServiceConfig dump>)`` :47-50 and checks
                   ``isinstance(..., CoreComponent)`` :52-55)
  process()       ``process(data: bytes) -> bytes | None`` (docs/interfaces.md:23-35), called
                  from the single EngineLoop thread (features/engine.py:187)
  config YAML     the reference's own detector config (container/config/detector_config.yaml,
                  tests/config/detector_config.yaml): ``detectors: {<name>: {method_type,
                  data_use_training, auto_config, global: {...}, events: {...}, params: {...}}}``;
                  GPU options live under ``params`` (settings.py has extra="forbid").

Input formats, told apart per message (``params.input_format``: auto | raw_lines |
parser_schema | parser_schema_batch), or named (log_schema | log_schema_batch, never chosen by auto):

  record mode   one serialized ParserSchema per message -- what the upstream parser stage
                sends today.  The host decodes the protobuf framing, the monitored values go
                to the GPU (dm_process_values); an anomalous record yields ONE DetectorSchema
                (what container/fluentout/fluent.conf:4-17 parses), anything else None.
  raw mode      N '\\n'-terminated raw log records per message (the fused path: tokenizer +
                detector in one pass on the GPU, R-tok rules in DESIGN.md).  Output per
                ``params.output_format``: ``alerts`` = DetectorSchema messages of the anomalous
                records (a single bare message when the input held one record, else
                varint-length-delimited), None when there are none; ``compact`` =
                ``<u32 n><n x u8 flag><n x f32 score>`` for pipelines that want every score.
  LogSchema     what the reader stage sends (one serialized LogSchema per message, or a delimited
                batch): the device unwraps each record's ``log`` text and runs raw-mode detection on
                it, so that with a ``log_format`` this component stands where the parser stands.
                Replies as for ParserSchema input; alerts carry the record's logID.

Alerts of raw-line, LogSchema and ParserSchema batches with at least DEVICE_ALERTS_MIN anomalous records are encoded
on the device (dm_encode_alerts, rule R-alert in DESIGN.md), byte for byte what the host encoder here writes; on the
two-slot pipelined path of large raw-line messages each piece is such a batch.  The host encoder words the rest, every
batch the device declines and single ParserSchema records of B200NewValueDetector.

All detection decisions are taken on the device; there is no CPU path (DeviceDetector
raises without a GPU).

Learnt state across restarts (``params.state_path``, absent by default, rule R-state in DESIGN.md): the known-set
table's keys and the counters n_seen / n_alerts are written to that file (state.py) after the message that ends the
training window, on close(), at interpreter exit while a device handle is live, and after reset_state(), import_state()
and a reconfigure() that keeps the device configuration.  At construction a file whose key_signature and key_probe
match is restored: the counters at once, the keys into the device handle when it is created.  Nothing is saved per
message: after an exit that runs no Python exit handler (SIGKILL, a power loss) the state is that of the last save,
and alert IDs issued since then may be issued again.
"""
from __future__ import annotations

import logging
import os
import struct
import threading
import time
import weakref
from typing import Any, Dict, List, Optional, Tuple

import numpy as np

from . import alerts as _alerts
from . import state as _state
from . import wire
from .compat import install_shims

install_shims()
from detectmatelibrary.common.core import CoreComponent, CoreConfig  # noqa: E402

_FORBIDDEN = (0x20, 0x22, 0x27, 0x3D, 0x0A)
_log = logging.getLogger(__name__)


class B200NewValueDetectorConfig(CoreConfig):
    """Schema of the detector's config entry (found by the resolver as <Class>Config in the
    same module, features/component_resolver.py:98-123)."""
    method_type: str = "new_value_detector"
    data_use_training: Optional[int] = None
    auto_config: bool = False


class Monitor:
    __slots__ = ("event_id", "source", "pos", "label", "key")

    def __init__(self, event_id: Optional[int], source: str, pos: Any, label: str):
        self.event_id, self.source, self.pos, self.label = event_id, source, pos, label
        self.key = b""

    @property
    def alert_key(self) -> str:
        return f"Global - {self.label}" if self.event_id is None else f"EventID {self.event_id} - {self.label}"


def select_component_config(config: Optional[dict], name: str, fallback: str = "NewValueDetector",
                            section: str = "detectors") -> dict:
    """Pick this component's entry out of the ServiceConfig dump the loader passes
    (src/service/core.py:127-133,144-148) and flatten ``params`` (docs/interfaces.md:74-84).
    section: the top-level key holding the entries (``parsers`` for a parser)."""
    cfg = dict(config or {})
    if isinstance(cfg.get(section), dict):
        dets = cfg[section]
        pick = dets.get(name) or dets.get(fallback) or (next(iter(dets.values())) if dets else {})
        cfg = dict(pick or {})
    params = cfg.pop("params", None) or {}
    for k, v in params.items():
        cfg[k[4:] if k.startswith("all_") else k] = v
    return cfg


def parse_monitors(cfg: dict) -> List[Monitor]:
    mons: List[Monitor] = []

    def instances(scope: dict, event_id: Optional[int]) -> None:
        for _name, inst in (scope or {}).items():
            inst = inst or {}
            for hv in inst.get("header_variables") or []:
                mons.append(Monitor(event_id, "header", str(hv["pos"]), str(hv["pos"])))
            for var in inst.get("variables") or []:
                pos = int(var["pos"])
                mons.append(Monitor(event_id, "variable", pos, str(var.get("name", pos))))

    instances(cfg.get("global") or {}, None)
    for eid, scope in (cfg.get("events") or {}).items():
        instances(scope or {}, int(eid))
    if len(mons) > 32:
        raise ValueError(f"{len(mons)} monitored fields configured, the device table addresses at most 32")
    # device key of each monitor: global header variables are matched by name in raw records;
    # everything else only exists in record mode and gets a name no log can contain.
    used = set()
    for i, m in enumerate(mons):
        raw_ok = m.event_id is None and m.source == "header"
        kb = m.pos.encode("utf-8") if raw_ok else b""
        if not raw_ok or not kb or len(kb) > 32 or any(c in _FORBIDDEN for c in kb) or kb in used:
            kb = b"\x01m%d" % i
        used.add(kb)
        m.key = kb
    return mons


def key_signature(c) -> dict:
    """Everything a known-set table key of component c depends on, as JSON values: the ordered monitors (event scope,
    source, position, device key), the combinations, and the log_format with its templates, content capture and R-norm
    flags.  The device geometry (device, max_batch_bytes, table_log2_slots) changes no key and is not part of it."""
    lf = c.logformat
    return {"monitors": [[m.event_id, m.source, m.pos, m.key.hex()] for m in c.monitors],
            "combos": getattr(c, "combos", None),
            "log_format": None if lf is None else lf.source,
            "templates": None if lf is None else [bytes(t).hex() for t in lf.template_sources],
            "content_name": None if lf is None else lf.content_name,
            "norm_flags": None if lf is None else lf.flags}


def device_geometry(c) -> tuple:
    return (c.device, c.max_batch_bytes, c.table_log2_slots)


# log_schema / log_schema_batch are opt-in: protobuf's runtime parses any LogSchema as a ParserSchema (the string fields
# 1, 2, 3 and 5 are ParserSchema strings too), so `auto` cannot tell the two apart and keeps reading ParserSchema.
INPUT_FORMATS = ("auto", "raw_lines", "parser_schema", "parser_schema_batch", "log_schema", "log_schema_batch")


class B200NewValueDetector(CoreComponent):
    accepts_bytes_like = True      # process() takes bytes, bytearray or memoryview (see service.py)

    def __init__(self, name: str = "B200NewValueDetector", config: Optional[Any] = None,
                 _restore_state: bool = True) -> None:
        raw_cfg = config.model_dump() if hasattr(config, "model_dump") else config
        cfg = select_component_config(raw_cfg, name)
        super().__init__(name=name, config=B200NewValueDetectorConfig(
            method_type=cfg.get("method_type", "new_value_detector"),
            data_use_training=cfg.get("data_use_training"), auto_config=bool(cfg.get("auto_config", False))))
        if cfg.get("auto_config"):
            raise ValueError("auto_config: true (a configure phase) is not supported by the CUDA detector; "
                             "list the monitored fields under global/events")
        self.detector_id = cfg.get("detector_id", "NewValueDetector" if name.startswith("B200") else name)
        self.method_type = cfg.get("method_type", "new_value_detector")
        self.data_use_training = int(cfg.get("data_use_training") or 0)
        self.start_id = int(cfg.get("start_id", 10))
        self.input_format = cfg.get("input_format", "auto")
        self.output_format = cfg.get("output_format", "alerts")
        if self.input_format not in INPUT_FORMATS:
            raise ValueError(f"input_format {self.input_format!r} not in {'|'.join(INPUT_FORMATS)}")
        if self.output_format not in ("alerts", "compact"):
            raise ValueError(f"output_format {self.output_format!r} not in alerts|compact")
        self.monitors = parse_monitors(cfg)
        # MatcherParser fused in front of the detector (raw-line input): params.log_format
        # (+ params.templates: list, or params.path_templates: file, matched against the
        # capture params.content_name = "Content") -- the parser config of
        # tests/library_integration/test_pipe_filereader_matcher_nvd.py:74-88 moved here
        self.logformat = None
        if cfg.get("log_format"):
            from .logformat import LogFormat, load_templates
            templates = list(cfg.get("templates") or [])
            if cfg.get("path_templates"):
                templates += load_templates(str(cfg["path_templates"]))
            from .logformat import norm_flags
            # R-norm (params.remove_spaces / remove_punctuation / lowercase, ibid. lines 82-84)
            flags = norm_flags(bool(cfg.get("remove_spaces")), bool(cfg.get("remove_punctuation")), bool(cfg.get("lowercase")))
            self.logformat = LogFormat(cfg["log_format"], templates, str(cfg.get("content_name", "Content")), flags)
        self.device = int(cfg.get("device", 0))
        self.max_batch_bytes = int(cfg.get("max_batch_bytes", 64 << 20))
        self.table_log2_slots = int(cfg.get("table_log2_slots", 20))
        self._det = None                       # created on first use, on the EngineLoop thread
        self._frames = None                    # pinned receive slots, created on first alloc_frame()
        self._frame_lock = threading.Condition()
        self.n_seen = 0
        self.n_alerts = 0
        self.clock = time.time
        self._alert_sig = None                 # (handle, detector_id, method_type) the device's alert format was set for
        self.state_path = str(cfg["state_path"]) if cfg.get("state_path") else None
        self._state_lock = threading.RLock()   # held by process() and by every save
        self._pending_keys = None              # restored keys, imported when the device handle is created
        self._state_hold = False               # a reconfigure() rebuilt: no save until the new training window ends
        self._finalizer = None                 # saves at interpreter exit while a handle is live
        if _restore_state:
            self._restore_state()

    # ------------------------------------------------------------------ device handle
    @property
    def det(self):
        if self._det is None:
            from .detector import DeviceDetector
            self._det = DeviceDetector([m.key for m in self.monitors], device=self.device,
                                       max_batch_bytes=self.max_batch_bytes,
                                       table_log2_slots=self.table_log2_slots)
            self._det.set_monitors([{"event_id": m.event_id, "source": m.source, "pos": m.pos} for m in self.monitors])
            if self.logformat is not None:
                lf = self.logformat
                self._det.set_format(lf.source, lf.template_sources, lf.content_name, lf.flags)
            self._configure_device(self._det)
            if self.state_path:
                self._device_restored()
        return self._det

    def _configure_device(self, det) -> None:
        """Configuration a subclass adds to a new device handle."""

    # ------------------------------------------------------------------ receive buffers (lent to the transport)
    FRAME_SLOTS = 4

    def alloc_frame(self, nbytes: int):
        """Lend the transport a receive buffer for one large message: a slot of pinned host
        memory, so the message is DMA-able where it lands (no staging copy, no per-message
        allocation).  Returns a writable memoryview, or None when no slot is free / the
        message does not fit / there is no CUDA device (the transport then allocates itself).
        Called on the transport's reader thread; slots come back through release_frame()."""
        if nbytes > self.max_batch_bytes:
            return None
        with self._frame_lock:
            if self._frames is None:
                import torch
                if not torch.cuda.is_available():
                    self._frames = []
                else:
                    self._frames = []
                    from .numa import bound_to_gpu_node
                    with bound_to_gpu_node(self.device):       # pinned memory on the GPU's NUMA node
                        for _ in range(self.FRAME_SLOTS):
                            t = torch.empty(self.max_batch_bytes + 64, dtype=torch.uint8, pin_memory=True)
                            t.zero_()                           # first touch while bound
                            self._frames.append([t, memoryview(t.numpy()), False])
            deadline = time.monotonic() + 0.2
            while self._frames:
                for slot in self._frames:
                    if not slot[2]:
                        slot[2] = True
                        return slot[1][:nbytes]
                # every slot is queued or being processed: stall the reader (back-pressure on
                # the sender) rather than allocate; give up after 200 ms
                left = deadline - time.monotonic()
                if left <= 0:
                    break
                self._frame_lock.wait(left)
        return None

    def release_frame(self, frame) -> None:
        if not isinstance(frame, memoryview) or not self._frames:
            return
        base = frame.obj
        with self._frame_lock:
            for slot in self._frames:
                if slot[1].obj is base:
                    slot[2] = False
                    self._frame_lock.notify()
                    return

    def close(self) -> None:
        with self._state_lock:
            if self._det is not None:
                self._save_logged("close()")
            self._drop_device()

    def _drop_device(self) -> None:
        if self._det is not None:
            self._det.close()
            self._det = None
        if self._finalizer is not None:
            self._finalizer.detach()
            self._finalizer = None
        self._alert_sig = None

    def reconfigure(self, config: Optional[Any]) -> bool:
        """Take a new detector configuration (what Service.reconfigure has just put into its config manager,
        /root/reference/src/service/core.py:299-345 -- the reference updates the manager and leaves the loaded
        component alone; the detector service subclass of service.py forwards it here).  Scalar parameters
        (data_use_training, output_format, start_id ...) apply in place and the known sets stay.  If the monitored
        fields, the log_format / templates or the device geometry change, the device handle is dropped and rebuilt
        on the next message: table keys are salted by the monitor's position, so the learnt state cannot be carried
        over and training starts again (n_seen = 0).  Returns True if the device configuration was rebuilt.
        Call it from the thread that calls process()."""
        new = type(self)(name=self.name, config=config, _restore_state=False)
        rebuild = key_signature(new) != key_signature(self) or device_geometry(new) != device_geometry(self)
        keep = ("_det", "_frames", "_frame_lock", "n_seen", "n_alerts", "clock", "_state_lock", "_pending_keys",
                "_state_hold", "_finalizer")
        with self._state_lock:
            if rebuild:
                # the state file keeps the old configuration's state until the new training window ends: a restart with
                # the old configuration (this one is not persisted by the service) still finds it
                self._state_hold = True
                self._pending_keys = None
            for k, v in vars(new).items():
                if k not in keep:
                    setattr(self, k, v)
            if rebuild:
                self._drop_device()
                self.n_seen = 0
                if self._frames and new.max_batch_bytes > len(self._frames[0][1]) - 64:
                    with self._frame_lock:
                        self._frames = None                      # re-created at the new size on the next alloc_frame()
            else:
                self._save_logged("reconfigure()")
        return rebuild

    # ------------------------------------------------------------------ the plugin entry point
    def process(self, data: bytes) -> Optional[bytes]:
        if not self.state_path:
            return self._process(data)
        with self._state_lock:
            seen = self.n_seen
            try:
                return self._process(data)
            finally:
                # the message that ended the training window, a dropped one (DM_ERR_TABLE_FULL) included
                if seen < self.data_use_training <= self.n_seen:
                    self._state_hold = False
                    self._save_logged("the end of training")

    def _process(self, data: bytes) -> Optional[bytes]:
        if not data:
            return None
        fmt = self.input_format
        if fmt == "auto" and self.logformat is not None:
            fmt = "raw_lines"                                    # a log_format is configured: the input is log text
        if isinstance(data, memoryview) and fmt != "raw_lines":
            # a lent receive buffer: raw lines are used in place; protobuf inputs (rare as
            # large frames) are decoded from a bytes copy
            if fmt == "auto" and data[0] == 0x74:                # 't' of "type=": cannot start a ParserSchema
                fmt = "raw_lines"
            else:
                data = bytes(data)
        if fmt == "auto":
            if wire.looks_like_parser_schema(data):
                fmt = "parser_schema"
            elif wire.looks_like_delimited_parser_schemas(data):
                fmt = "parser_schema_batch"
            else:
                fmt = "raw_lines"
        if fmt == "parser_schema":
            return self._process_record(data)
        if fmt == "parser_schema_batch":
            return self._process_record_batch(data)
        if fmt in ("log_schema", "log_schema_batch"):
            return self._process_logs(data, delimited=fmt == "log_schema_batch")
        return self._process_lines(data)

    # ------------------------------------------------------------------ record mode
    def _record_values(self, rec: Dict) -> List[Tuple[int, bytes]]:
        out = []
        eid, lfv, var = rec.get("EventID"), rec.get("logFormatVariables") or {}, rec.get("variables") or []
        for i, m in enumerate(self.monitors):
            if m.event_id is not None and m.event_id != eid:
                continue
            v = lfv.get(m.pos) if m.source == "header" else (var[m.pos] if 0 <= m.pos < len(var) else None)
            if v is not None:
                out.append((i, v.encode("utf-8") if isinstance(v, str) else bytes(v)))
        return out

    def _process_record(self, data: bytes) -> Optional[bytes]:
        rec = wire.decode_parser_schema(data, strict=False)
        vals = self._record_values(rec)
        train = self.n_seen < self.data_use_training
        self.n_seen += 1
        flags, scores, masks = self.det.process_values([[v for v in vals]], n_train_records=1 if train else 0,
                                                       record_bytes=len(data))
        if train or not flags[0]:
            return None
        return self._detector_schema(*self._record_alert(rec, vals, int(masks[0]), float(scores[0])))

    def _record_alert(self, rec: Dict, vals: List[Tuple[int, bytes]], mask: int, score: float) -> tuple:
        """(logID, score, alertsObtain, Time) of one anomalous ParserSchema record, vals its _record_values."""
        by_field = dict(vals)
        return (rec.get("logID", ""), score, self._alerts_of(mask, lambda i: by_field.get(i, b"")),
                (rec.get("logFormatVariables") or {}).get("Time"))

    def _bad_records(self) -> int:
        """The device's count of malformed records (0 for a device stand-in that keeps no statistics)."""
        stats = getattr(self.det, "stats", None)
        return int(stats()["bad_records"]) if stats else 0

    def _process_record_batch(self, data: bytes) -> Optional[bytes]:
        """A message holding many length-delimited ParserSchema records: field walk, monitor
        matching, hashing and scoring happen on the device; the host only decodes the (rare)
        anomalous records to word their alerts."""
        remaining = max(0, self.data_use_training - self.n_seen)
        bad0 = self._bad_records()
        flags, scores, masks = self._device_call(remaining, lambda: len(wire.split_delimited(data)),
                                                 self.det.process_records, data, n_train_records=remaining)
        n = int(flags.size)
        # malformed records take no training slot (as on the per-record path, where they raise before counting)
        self.last_n_malformed = self._bad_records() - bad0
        self.n_seen += n - self.last_n_malformed
        return self._reply(n, flags, scores, self.det.last_n_anomalies, False, 0,
                           self._record_batch_records, data, flags, scores, masks)

    def _record_batch_records(self, data: bytes, flags, scores, masks):
        """(logID, score, alertsObtain, Time) of the anomalous records of a ParserSchema batch."""
        frames = wire.split_delimited(data)
        for idx in np.flatnonzero(flags):
            try:
                rec = wire.decode_parser_schema(frames[int(idx)], strict=False)
            except wire.WireError:
                continue                     # (a frame the device could walk but the host cannot: skipped, not fatal)
            yield self._record_alert(rec, self._record_values(rec), int(masks[idx]), float(scores[idx]))

    # ------------------------------------------------------------------ LogSchema input (the reader stage's records)
    def _process_logs(self, data: bytes, delimited: bool) -> Optional[bytes]:
        """One bare LogSchema record, or a length-delimited batch of them: the device unwraps each record's `log` text
        and detects it as a raw line (key=value, or the log_format).  Replies as for ParserSchema input; the alert of a
        record carries its logID.  A malformed bare record raises WireError and takes no training slot."""
        if len(data) > self.max_batch_bytes:
            raise ValueError(f"a LogSchema message of {len(data)} bytes exceeds max_batch_bytes={self.max_batch_bytes}")
        remaining = max(0, self.data_use_training - self.n_seen)
        flags, scores, n_bad = self._device_call(remaining, lambda: len(wire.split_delimited(data)) if delimited else 1,
                                                 self.det.process_logs, data, n_train_records=remaining,
                                                 delimited=delimited)
        n = int(flags.size)
        self.last_n_malformed = n_bad
        self.n_seen += n - n_bad                                 # malformed and unusable records take no training slot
        if not delimited and n_bad:
            raise wire.WireError("malformed LogSchema record")
        return self._reply(n, flags, scores, self.det.last_n_anomalies, not delimited, 0,
                           self._log_records, data, delimited, scores)

    def _log_records(self, data: bytes, delimited: bool, scores):
        """(logID, score, alertsObtain, Time) of the anomalous records of the last LogSchema message."""
        frames = wire.split_delimited(data) if delimited else [data]
        for idx, mask, _offset in self.det.anomalies():
            rec = wire.decode_log_schema(frames[idx])
            alerts, t = self._text_alerts(wire.log_schema_line(rec), mask)
            yield rec["logID"], float(scores[idx]), alerts, t

    # ------------------------------------------------------------------ raw mode
    def _process_lines(self, data: bytes) -> Optional[bytes]:
        if len(data) > self.max_batch_bytes:
            return self._process_lines_chunked(data)
        return self._process_lines_one(data)

    def _process_lines_chunked(self, data: bytes) -> Optional[bytes]:
        """A message larger than the device batch: cut at record boundaries, process the pieces
        in order (training counter and record numbering carry over), merge the outputs."""
        outs, pos, n = [], 0, len(data)
        while pos < n:
            end = min(pos + self.max_batch_bytes, n)
            if end < n:
                cut = data.rfind(b"\n", pos, end)
                if cut < 0:
                    raise ValueError(f"a single record exceeds max_batch_bytes={self.max_batch_bytes}")
                end = cut + 1
            outs.append(self._process_lines_one(data[pos:end], force_delimited=True))
            pos = end
        if self.output_format == "compact":
            parts = [decode_compact(o) for o in outs]
            return _encode_compact(np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]))
        merged = b"".join(o for o in outs if o)
        return merged or None

    # Messages at least this large are cut into pieces that overlap copy and compute.  Every piece pays a fixed latency
    # (copy + kernel + two small copies back, each with a host synchronisation), so small pieces lose against one call;
    # scripts/e2e_pieces.py measures one call against 2 / 4 / 8 / 12 MiB pieces on the machine at hand.
    PIPE_MIN_BYTES = 24 << 20
    PIPE_PIECE_BYTES = 12 << 20
    # Batches with at least this many anomalous records have their alerts encoded on the device (dm_encode_alerts), raw
    # lines, LogSchema and ParserSchema alike.  On
    # one H100 (700 W), 64k-record messages, process() median [range] in ms, host encoder against device encoder: 1 alert
    # 0.60 against 0.59 [0.57-0.62], 4 alerts 0.65 [0.56-0.75] against 0.58 [0.55-0.61], 8 alerts 0.61 [0.59-0.76]
    # against 0.54 [0.53-0.60], 16 alerts 0.92 against 0.58 (scripts/alerts_bench.py, DESIGN.md section 5.3).  Below 8
    # the two overlap, and a record with a long value once made one alert slower on the device (0.77 against 0.60), so
    # the device takes over where it was ahead beyond the spread.  64k-record LogSchema / ParserSchema batches on the
    # same card were ahead on the device from 1 alert on (LogSchema 85 against 6.4 ms, ParserSchema 63 against 8.8 ms,
    # scripts/record_alerts_bench.py): there the host path splits the whole message first.  Small batches were not
    # measured, so the three inputs share this threshold.
    DEVICE_ALERTS_MIN = 8

    def _detect_pipelined(self, data, base: int):
        """Detection-only message, key=value records: cut it at record boundaries into PIPE_PIECE_BYTES pieces and run
        them through the library's two-slot path (dm_submit_lines / dm_collect): piece k+1 crosses PCIe while piece k is
        in the kernel.  Returns (flags, scores, pieces): flags and scores exactly as one dm_process_lines call would give
        them; pieces (None for compact output) has one entry per piece with anomalous records, in order.  A piece with at
        least DEVICE_ALERTS_MIN of them is encoded on the device between its collect and the next submit on its slot,
        which rewrites the slot: its entry is (varint-delimited DetectorSchemas, count).  Any other piece, or one the
        device declines, is left to the host encoder: its entry is the list of its anomalies as (record index in the
        message, mask, byte offset in the message).  base: the message's first record number; the device pieces are
        numbered as if every earlier piece's alerts were already counted in n_alerts, which the caller then does."""
        arr = np.frombuffer(data, dtype=np.uint8)
        n = int(arr.size)
        cuts = [0]
        while n - cuts[-1] > self.PIPE_PIECE_BYTES + (self.PIPE_PIECE_BYTES >> 1):
            p = cuts[-1] + self.PIPE_PIECE_BYTES
            nl = np.flatnonzero(arr[p:p + (1 << 16)] == 10)
            if nl.size == 0:                                  # a record longer than 64 KiB here: look further
                nl = np.flatnonzero(arr[p:] == 10)
                if nl.size == 0:
                    break
            cuts.append(p + int(nl[0]) + 1)
        cuts.append(n)
        k = len(cuts) - 1
        det = self.det
        want_alerts = self.output_format != "compact"
        parts_f, parts_s, pieces = [], [], []
        line_base, numbered = [0], [0]                     # records and alerts of the pieces collected so far

        def collect(i):
            f, s = det.collect(i & 1)
            n_anom = det.last_n_anomalies
            if want_alerts and n_anom:
                enc = None
                if n_anom >= self.DEVICE_ALERTS_MIN:
                    enc = self._device_alerts(base + line_base[0], int(f.size),
                                              first_alert_id=self.start_id + self.n_alerts + numbered[0])
                if enc is None:
                    enc = [(ln + line_base[0], mask, off + cuts[i]) for ln, mask, off in det.collect_anomalies(i & 1)]
                    numbered[0] += len(enc)
                else:
                    numbered[0] += enc[1]
                pieces.append(enc)
            parts_f.append(f.copy())
            parts_s.append(s.copy())
            line_base[0] += int(f.size)
        try:
            for i in range(k):
                if i >= 2:
                    collect(i - 2)
                det.submit(arr[cuts[i]:cuts[i + 1]], 0, i & 1)
            for i in range(max(0, k - 2), k):
                collect(i)
        except BaseException:
            for slot in (0, 1):                            # leave no slot in flight for the next message
                try:
                    det.collect(slot)
                except Exception:
                    pass
            raise
        return np.concatenate(parts_f), np.concatenate(parts_s), (pieces if want_alerts else None)

    def _process_lines_one(self, data: bytes, force_delimited: bool = False) -> Optional[bytes]:
        remaining = max(0, self.data_use_training - self.n_seen)
        pieces = None
        if (remaining == 0 and len(data) >= self.PIPE_MIN_BYTES and self.logformat is None and not getattr(self, "combos", None)
                and os.environ.get("DM_KERNEL", "stream") == "stream"):
            flags, scores, pieces = self._detect_pipelined(data, self.n_seen)
            n_anom = int(np.count_nonzero(flags))
        else:
            flags, scores = self._device_call(remaining, lambda: _alerts.count_records(data),
                                              self.det.process_lines, data, n_train_lines=remaining, copy=False)
            n_anom = self.det.last_n_anomalies
        n = int(flags.size)
        base = self.n_seen
        self.n_seen += n
        bare = n == 1 and not force_delimited
        if pieces is None:                                 # (always so for compact output)
            return self._reply(n, flags, scores, n_anom, bare, base, self._line_records, data, None, base, scores)
        # a pipelined message: the pieces' varint-delimited alerts in order, the host wording those the device did not
        blobs = []
        for p in pieces:
            if isinstance(p, tuple):
                blobs.append(p[0])
                self.n_alerts += p[1]
            else:
                blobs.append(self._host_alerts(self._line_records(data, p, base, scores)))
        return _reply_of(b"".join(blobs), bare)

    def _line_records(self, data, anomalies, base: int, scores):
        """(logID, score, alertsObtain, Time) of raw-line anomalies (record index, mask, byte offset in data), those of
        the last batch when anomalies is None; base: the number of the message's first record."""
        for line_idx, mask, offset in self.det.anomalies() if anomalies is None else anomalies:
            alerts, t = self._text_alerts(_alerts.record_at(data, offset), mask)
            yield str(base + line_idx), float(scores[line_idx]), alerts, t

    def _device_call(self, remaining: int, count, call, *args, **kwargs):
        """call(*args, **kwargs), the device call of a message that trains on up to `remaining` records; should it fail,
        count() is the message's record count for _count_dropped_training."""
        try:
            return call(*args, **kwargs)
        except Exception as e:
            self._count_dropped_training(e, remaining, count)
            raise

    def _count_dropped_training(self, err: Exception, remaining: int, count) -> None:
        """A training message the device refused because the known-set table is full (DM_ERR_TABLE_FULL) is dropped by
        the engine like any failing message (engine.py:192-194) -- but its records still count as seen, otherwise the
        training window would never end and every later message would fail the same way (the reference's Python sets
        are unbounded; a larger params.table_log2_slots is the cure)."""
        from ._lib import DM_ERR_TABLE_FULL
        if remaining > 0 and getattr(err, "code", None) == DM_ERR_TABLE_FULL:
            try:
                self.n_seen += int(count())
            except Exception:
                self.n_seen += remaining

    # ------------------------------------------------------------------ alert wording
    @staticmethod
    def _format_value(m: Monitor, variables: List[bytes], lfv: Dict[str, bytes]) -> bytes:
        """Value of monitor m in a record LogFormat.parse split (variables are slices of the normalised Content)."""
        return lfv.get(m.pos, b"") if m.source == "header" else (variables[m.pos] if m.pos < len(variables) else b"")

    def _text_alerts(self, line: bytes, mask: int) -> Tuple[Dict[str, str], Any]:
        """alertsObtain and Time value of one anomalous log text (a raw line, or a LogSchema record's `log`): values and
        Time from the log_format's split, else from the key=value fields (R-tok)."""
        if self.logformat is not None:
            _eid, variables, lfv = self.logformat.parse(line) or (-1, [], {})
            return self._alerts_of(mask, lambda i: self._format_value(self.monitors[i], variables, lfv)), lfv.get("Time")
        fields = _alerts.record_fields(line, self._quoted_keys(mask))
        return self._alerts_of(mask, lambda i: fields.get(self.monitors[i].key, b"")), _alerts.record_time(line)

    def _quoted_keys(self, mask: int) -> List[bytes]:
        """The keys of the monitors whose values _alerts_of quotes for an unknown-field mask."""
        return [m.key for i, m in enumerate(self.monitors) if mask >> i & 1]

    def _alerts_of(self, mask: int, value_of) -> Dict[str, str]:
        """alertsObtain of one anomalous record: one entry per monitor flagged in the device's unknown-field mask, with
        value_of(i) the value of monitor i in the record (b"" when it has none).  Of two flagged monitors that share an
        alert key the last one in config order wins."""
        return {m.alert_key: _alerts.alert_text(value_of(i)) for i, m in enumerate(self.monitors) if mask >> i & 1}

    # ------------------------------------------------------------------ output
    def _reply(self, n: int, flags, scores, n_anomalies: int, bare: bool, first_log_id: int, host_records, *args):
        """The reply to a batch of n records: compact output, or None without anomalous records, or their alerts.  From
        DEVICE_ALERTS_MIN anomalous records on the device encodes the alerts; below that, or when the device declines, the
        host encodes host_records(*args), which yields (logID, score, alertsObtain, Time) per anomalous record in reply
        order.  bare: reply with the one DetectorSchema without its length prefix (one record came in).  first_log_id:
        the number of the batch's first record (raw lines; the record inputs carry their logIDs and pass 0)."""
        if self.output_format == "compact":
            return _encode_compact(flags, scores)
        if n_anomalies == 0:
            return None
        if n_anomalies >= self.DEVICE_ALERTS_MIN:
            enc = self._device_alerts(first_log_id, n)
            if enc is not None:
                self.n_alerts += enc[1]
                return _reply_of(enc[0], bare)
        return _reply_of(self._host_alerts(host_records(*args)), bare)

    def _host_alerts(self, records) -> bytes:
        """The host encoder: one DetectorSchema per (logID, score, alertsObtain, Time), numbered as it is written,
        varint-delimited."""
        return wire.frame_delimited([self._detector_schema(*r) for r in records])

    def _alert_keys(self) -> List[Tuple[str, List[int]]]:
        """alertsObtain keys in the order the host encoder writes them (sorted), each with the mask bits that supply it
        in config order (two monitors may share a key: the last one flagged wins, as in _alerts_of)."""
        by_key: Dict[str, List[int]] = {}
        for i, m in enumerate(self.monitors):
            by_key.setdefault(m.alert_key, []).append(i)
        return sorted(by_key.items())

    def _device_alerts(self, first_log_id: int, n_records: int,
                       first_alert_id: Optional[int] = None) -> Optional[Tuple[bytes, int]]:
        """The alerts of the last batch -- raw lines (a collected pipeline slot too), LogSchema or ParserSchema records --
        encoded on the device (DESIGN.md R-alert): (varint-delimited DetectorSchemas, count), or None when the host
        encodes them -- the device declined the batch, the handle has no encoder (a stand-in), or an ID does not fit the
        device's 64-bit integers.  first_log_id numbers raw lines; the other two carry their records' logIDs and pass 0.
        first_alert_id: the first alert's number (default start_id + n_alerts)."""
        det = self.det
        if not hasattr(det, "encode_alerts"):
            return None
        now = int(self.clock())
        if first_alert_id is None:
            first_alert_id = self.start_id + self.n_alerts
        if not (-(1 << 63) <= now < (1 << 63) and -(1 << 63) <= first_alert_id and first_alert_id + n_records < (1 << 63)
                and 0 <= first_log_id and first_log_id + n_records < (1 << 64)):
            return None
        sig = (det, self.detector_id, self.method_type)
        if self._alert_sig != sig:
            combos = getattr(self, "combos", None) or []
            names = self.logformat.header.names if self.logformat is not None else []
            det.set_alert_format("1.0.0", self.detector_id, self.method_type, self._description(), self._alert_keys(), combos,
                                 time_capture=names.index("Time") if "Time" in names else None)
            self._alert_sig = sig
        return det.encode_alerts(first_log_id, first_alert_id, now)

    def _description(self) -> str:
        return f"{self.detector_id} detects values not encountered in training as anomalies."

    def _detector_schema(self, log_id: str, score: float, alerts: Dict[str, str], time_value) -> bytes:
        now = int(self.clock())
        try:
            ts = int(float(time_value))
        except (TypeError, ValueError):
            ts = now
        alert_id = str(self.start_id + self.n_alerts)
        self.n_alerts += 1
        return wire.encode_detector_schema(
            detector_id=self.detector_id, detector_type=self.method_type, alert_id=alert_id, detection_ts=now,
            log_ids=[log_id], score=score, extracted_ts=[ts],
            description=self._description(),
            received_ts=now, alerts=alerts)

    # ------------------------------------------------------------------ state
    def stats(self) -> dict:
        return self.det.stats()

    def export_state(self) -> dict:
        """Learnt keys + counters (the reference loses detector state on restart)."""
        return {"known": self.det.export_known().tolist(), "n_seen": self.n_seen, "n_alerts": self.n_alerts}

    def reset_state(self) -> None:
        """Forget everything learnt and restart the training window."""
        with self._state_lock:
            self.det.reset()
            self.n_seen = 0
            self.n_alerts = 0
            self._save_logged("reset_state()")

    def import_state(self, state: dict) -> None:
        with self._state_lock:
            self.det.import_known(np.array(state.get("known", []), dtype=np.uint64))
            self.n_seen = int(state.get("n_seen", 0))
            self.n_alerts = int(state.get("n_alerts", 0))
            self._save_logged("import_state()")

    # ------------------------------------------------------------------ the state file (params.state_path)
    def _state_header(self) -> dict:
        return {"component": type(self).__name__, "key_signature": key_signature(self),
                "key_probe": _state.probe_key(), "n_seen": int(self.n_seen), "n_alerts": int(self.n_alerts)}

    def _restore_state(self) -> None:
        """Read params.state_path if it exists (ValueError if it is not a valid state file).  A file of this component
        class, key signature and key fingerprint restores n_seen and n_alerts now and its keys when the device handle is
        created; any other is ignored with a warning, and replaced at the next save."""
        if not self.state_path or not os.path.exists(self.state_path):
            return
        hdr, keys = _state.read_state(self.state_path)
        want = self._state_header()
        for field in ("component", "key_signature", "key_probe"):
            if hdr[field] != want[field]:
                _log.warning("%s: state file %s was written for another %s; ignored, training starts from scratch "
                             "and the file is replaced at the next save", self.name, self.state_path, field)
                return
        self.n_seen = hdr["n_seen"]
        self.n_alerts = hdr["n_alerts"]
        self._pending_keys = keys

    def _device_restored(self) -> None:
        """A new device handle: import the restored keys, and save at interpreter exit while the handle is live."""
        keys, self._pending_keys = self._pending_keys, None
        if keys is not None and keys.size:
            from ._lib import DM_ERR_TABLE_FULL
            try:
                self._det.import_known(keys)
            except Exception as e:
                if getattr(e, "code", None) != DM_ERR_TABLE_FULL:
                    raise
                _log.warning("%s: the %d restored keys take the table past its load limit; raise table_log2_slots",
                             self.name, keys.size)
        if self._finalizer is None:
            self._finalizer = weakref.finalize(self, _save_at_exit, weakref.ref(self))

    def save_state(self) -> bool:
        """Write the learnt keys and counters to params.state_path now.  Returns False when there is nothing to write: no
        state_path, no device handle, or a reconfigure() rebuilt the device configuration and its training window has
        not ended.  Raises what the write raises; the previous file is then left as it was."""
        with self._state_lock:
            if not self.state_path or self._det is None:
                return False
            if self._state_hold and self.n_seen < self.data_use_training:
                return False
            _state.write_state(self.state_path, self._state_header(), self._det.export_known())
            return True

    def _save_logged(self, when: str) -> None:
        if not self.state_path:
            return
        try:
            self.save_state()
        except Exception:
            _log.exception("%s: saving the detector state to %s at %s failed", self.name, self.state_path, when)


def _save_at_exit(ref) -> None:
    comp = ref()
    if comp is None or not comp._state_lock.acquire(timeout=30.0):
        return
    try:
        comp._save_logged("interpreter exit")
    finally:
        comp._state_lock.release()


class B200NewValueComboDetectorConfig(B200NewValueDetectorConfig):
    method_type: str = "new_value_combo_detector"


def parse_combos(cfg: dict) -> Tuple[List[Monitor], List[List[int]]]:
    """NewValueComboDetector config (same tree as NewValueDetector,
    tests/test_reconfigure_params.py:149-169): every instance is one combination = the
    ordered tuple of its fields, header_variables first, then variables."""
    mons = parse_monitors(cfg)                    # same instance / field order as below
    combos: List[List[int]] = []
    k = 0

    def instances(scope: dict) -> None:
        nonlocal k
        for _name, inst in (scope or {}).items():
            inst = inst or {}
            n = len(inst.get("header_variables") or []) + len(inst.get("variables") or [])
            if n:
                combos.append(list(range(k, k + n)))
            k += n

    instances(cfg.get("global") or {})
    for _eid, scope in (cfg.get("events") or {}).items():
        instances(scope or {})
    assert k == len(mons)
    if len(mons) + len(combos) > 32:
        raise ValueError(f"{len(mons)} fields + {len(combos)} combinations configured, the device mask holds 32")
    if len(mons) > 64:
        raise ValueError("at most 64 combination members in total")
    return mons, combos


def check_format_combos(cfg: dict, lf) -> None:
    """With a log_format, a combination one of whose members no record can ever have is dead configuration (one
    missing member silences the whole tuple): a header variable that names no capture of the log_format, or a
    template variable when no templates are configured.  Raises ValueError naming the instance."""
    captures = set(lf.header.names)
    scopes = [("global", cfg.get("global"))] + [("events.%s" % eid, sc) for eid, sc in (cfg.get("events") or {}).items()]
    for where, scope in scopes:
        for inst_name, inst in (scope or {}).items():
            inst = inst or {}
            for hv in inst.get("header_variables") or []:
                if str(hv["pos"]) not in captures:
                    raise ValueError(f"combination {where}.{inst_name}: header variable {str(hv['pos'])!r} is not a capture "
                                     f"of the log_format, so the combination can never be complete")
            if inst.get("variables") and not lf.templates:
                raise ValueError(f"combination {where}.{inst_name}: template variables but no templates are configured, "
                                 f"so the combination can never be complete")


class B200NewValueComboDetector(B200NewValueDetector):
    """NewValueComboDetector on the device (SURVEY.md section 8f-4; semantics R-combo in DESIGN.md /
    oracle/nvcd.py): tuples of field values instead of single values.  The member
    fingerprints are folded in order into one 64-bit key and learnt / probed in the same
    table (`dm_set_combos`).  Input: ParserSchema (one per message or a delimited batch), raw
    key=value records for combinations of global header variables, or raw log lines split by
    ``params.log_format`` / ``templates`` / ``path_templates`` (and the R-norm switches), where a
    combination may mix header captures and the variables of its event's template.  A tuple
    has the same key in all three, so known sets carry over (export_state / import_state)."""

    def __init__(self, name: str = "B200NewValueComboDetector", config: Optional[Any] = None,
                 _restore_state: bool = True) -> None:
        raw_cfg = config.model_dump() if hasattr(config, "model_dump") else config
        cfg = select_component_config(raw_cfg, name, fallback="NewValueComboDetector")
        cfg.setdefault("method_type", "new_value_combo_detector")
        cfg.setdefault("detector_id", "NewValueComboDetector" if name.startswith("B200") else name)
        super().__init__(name=name, config={"detectors": {name: cfg}}, _restore_state=False)
        self.monitors, self.combos = parse_combos(cfg)
        if self.logformat is not None:
            check_format_combos(cfg, self.logformat)
        if _restore_state:
            self._restore_state()

    def _configure_device(self, det) -> None:
        det.set_combos(self.combos, member_only_mask=(1 << len(self.monitors)) - 1)

    def _description(self) -> str:
        return f"{self.detector_id} detects value combinations not encountered in training as anomalies."

    def _alert_keys(self) -> List[Tuple[str, List[int]]]:
        n = len(self.monitors)
        by_key: Dict[str, List[int]] = {}
        for c, members in enumerate(self.combos):
            by_key.setdefault(self._combo_alert(members, [b""] * len(members))[0], []).append(n + c)
        return sorted(by_key.items())

    def _combo_alert(self, members: List[int], values: List[bytes]) -> Tuple[str, str]:
        """("<scope> - (<label>, ...)", "Unknown value combination: ('v1', ...)") of one combination."""
        m0 = self.monitors[members[0]]
        scope = "Global" if m0.event_id is None else f"EventID {m0.event_id}"
        key = "%s - (%s)" % (scope, ", ".join(self.monitors[i].label for i in members))
        return key, "Unknown value combination: (%s)" % ", ".join("'%s'" % v.decode("utf-8", "replace") for v in values)

    def _quoted_keys(self, mask: int) -> List[bytes]:
        n = len(self.monitors)
        return [self.monitors[i].key for c, members in enumerate(self.combos) if mask >> (n + c) & 1 for i in members]

    def _alerts_of(self, mask: int, value_of) -> Dict[str, str]:
        """One entry per combination flagged in the mask (bit len(monitors) + c), quoting its members' values."""
        n = len(self.monitors)
        return dict(self._combo_alert(members, [value_of(i) for i in members])
                    for c, members in enumerate(self.combos) if mask >> (n + c) & 1)

    def _process_record(self, data: bytes) -> Optional[bytes]:
        out = self._process_record_batch(wire.frame_delimited([data]))     # the device walks the record
        if self.last_n_malformed:
            raise wire.WireError("malformed ParserSchema record")          # as B200NewValueDetector's per-record path
        if out is None or self.output_format == "compact":
            return out
        return _reply_of(out, bare=True)                                    # one record in, one bare alert out


def _reply_of(blob: bytes, bare: bool) -> Optional[bytes]:
    """The alerts reply made of varint-delimited DetectorSchemas: None without any, the one DetectorSchema without its
    length prefix when one record came in bare, else the blob."""
    if not blob:
        return None
    if bare:
        _ln, pos = wire._read_varint(blob, 0)
        return blob[pos:]
    return blob


def _encode_compact(flags: np.ndarray, scores: np.ndarray) -> bytes:
    """The ``compact`` output format: ``<u32 n><n x u8 flag><n x f32 score>``."""
    return struct.pack("<I", flags.size) + flags.tobytes() + scores.tobytes()


def decode_compact(blob: bytes) -> Tuple[np.ndarray, np.ndarray]:
    """Inverse of the ``compact`` output format."""
    (n,) = struct.unpack_from("<I", blob, 0)
    flags = np.frombuffer(blob, dtype=np.uint8, count=n, offset=4)
    scores = np.frombuffer(blob, dtype=np.float32, count=n, offset=4 + n)
    return flags, scores
