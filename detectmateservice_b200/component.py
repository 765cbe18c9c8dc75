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

Two input formats, told apart per message (``params.input_format``: auto | raw_lines |
parser_schema):

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

All detection decisions are taken on the device; there is no CPU path (DeviceDetector
raises without a GPU).
"""
from __future__ import annotations

import os
import struct
import threading
import time
from typing import Any, Dict, List, Optional, Tuple

import numpy as np

from . import alerts as _alerts
from . import wire
from .compat import install_shims

install_shims()
from detectmatelibrary.common.core import CoreComponent, CoreConfig  # noqa: E402

_FORBIDDEN = (0x20, 0x22, 0x27, 0x3D, 0x0A)


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


def select_component_config(config: Optional[dict], name: str, fallback: str = "NewValueDetector") -> dict:
    """Pick this component's entry out of the ServiceConfig dump the loader passes
    (src/service/core.py:127-133,144-148) and flatten ``params`` (docs/interfaces.md:74-84)."""
    cfg = dict(config or {})
    if isinstance(cfg.get("detectors"), dict):
        dets = cfg["detectors"]
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


class B200NewValueDetector(CoreComponent):
    accepts_bytes_like = True      # process() takes bytes, bytearray or memoryview (see service.py)

    def __init__(self, name: str = "B200NewValueDetector", config: Optional[Any] = None) -> None:
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
        if self.input_format not in ("auto", "raw_lines", "parser_schema", "parser_schema_batch"):
            raise ValueError(f"input_format {self.input_format!r} not in auto|raw_lines|parser_schema|parser_schema_batch")
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
        return self._det

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
        if self._det is not None:
            self._det.close()
            self._det = None

    def reconfigure(self, config: Optional[Any]) -> bool:
        """Take a new detector configuration (what Service.reconfigure has just put into its config manager,
        /root/reference/src/service/core.py:299-345 -- the reference updates the manager and leaves the loaded
        component alone; the detector service subclass of service.py forwards it here).  Scalar parameters
        (data_use_training, output_format, start_id ...) apply in place and the known sets stay.  If the monitored
        fields, the log_format / templates or the device geometry change, the device handle is dropped and rebuilt
        on the next message: table keys are salted by the monitor's position, so the learnt state cannot be carried
        over and training starts again (n_seen = 0).  Returns True if the device configuration was rebuilt.
        Call it from the thread that calls process()."""
        new = type(self)(name=self.name, config=config)
        sig = lambda c: ([(m.event_id, m.source, m.pos, m.key) for m in c.monitors],
                         None if c.logformat is None else (c.logformat.source, c.logformat.template_sources,
                                                           c.logformat.content_name, c.logformat.flags),
                         c.device, c.max_batch_bytes, c.table_log2_slots, getattr(c, "combos", None))
        rebuild = sig(new) != sig(self)
        keep = ("_det", "_frames", "_frame_lock", "n_seen", "n_alerts", "clock")
        for k, v in vars(new).items():
            if k not in keep:
                setattr(self, k, v)
        if rebuild:
            self.close()
            self.n_seen = 0
            if self._frames and new.max_batch_bytes > len(self._frames[0][1]) - 64:
                with self._frame_lock:
                    self._frames = None                          # re-created at the new size on the next alloc_frame()
        return rebuild

    # ------------------------------------------------------------------ the plugin entry point
    def process(self, data: bytes) -> Optional[bytes]:
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
        mask = int(masks[0])
        by_field = dict(vals)
        alerts = {self.monitors[i].alert_key: _alerts.alert_text(by_field[i])
                  for i in range(len(self.monitors)) if mask >> i & 1}
        t = (rec.get("logFormatVariables") or {}).get("Time")
        return self._detector_schema(rec.get("logID", ""), float(scores[0]), alerts, t)

    def _record_alerts(self, rec: Dict, mask: int) -> Dict[str, str]:
        """alertsObtain of one anomalous record from the device's unknown-field mask."""
        by_field = dict(self._record_values(rec))
        return {self.monitors[i].alert_key: _alerts.alert_text(by_field.get(i, b""))
                for i in range(len(self.monitors)) if mask >> i & 1}

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
        try:
            flags, scores, masks = self.det.process_records(data, n_train_records=remaining)
        except Exception as e:
            self._count_dropped_training(e, remaining, lambda: len(wire.split_delimited(data)))
            raise
        n = int(flags.size)
        # malformed records take no training slot (as on the per-record path, where they raise before counting)
        self.last_n_malformed = self._bad_records() - bad0
        self.n_seen += n - self.last_n_malformed
        if self.output_format == "compact":
            return struct.pack("<I", n) + flags.tobytes() + scores.tobytes()
        if self.det.last_n_anomalies == 0:
            return None
        frames = wire.split_delimited(data)
        out = []
        for idx in np.flatnonzero(flags):
            try:
                rec = wire.decode_parser_schema(frames[int(idx)], strict=False)
            except wire.WireError:
                continue                     # (a frame the device could walk but the host cannot: skipped, not fatal)
            alerts = self._record_alerts(rec, int(masks[idx]))
            t = (rec.get("logFormatVariables") or {}).get("Time")
            out.append(self._detector_schema(rec.get("logID", ""), float(scores[idx]), alerts, t))
        return wire.frame_delimited(out) if out else None

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
            flags = np.concatenate([p[0] for p in parts])
            scores = np.concatenate([p[1] for p in parts])
            return struct.pack("<I", flags.size) + flags.tobytes() + scores.tobytes()
        merged = b"".join(o for o in outs if o)
        return merged or None

    # Messages at least this large are cut into pieces that overlap copy and compute.  Every piece pays a fixed latency
    # (copy + kernel + two small copies back, each with a host synchronisation), so small pieces lose against one call;
    # scripts/e2e_pieces.py measures one call against 2 / 4 / 8 / 12 MiB pieces on the machine at hand.
    PIPE_MIN_BYTES = 24 << 20
    PIPE_PIECE_BYTES = 12 << 20

    def _detect_pipelined(self, data):
        """Detection-only message, key=value records: cut it at record boundaries into ~4 MiB pieces and run them
        through the library's two-slot path (dm_submit_lines / dm_collect): piece k+1 crosses PCIe while piece k is
        in the kernel.  Returns (flags, scores, anomalies or None) exactly as one dm_process_lines call would."""
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
        want_anoms = self.output_format != "compact"
        parts_f, parts_s, anoms, line_base = [], [], [], [0]

        def collect(i):
            f, s = det.collect(i & 1)
            if want_anoms and det.last_n_anomalies:
                anoms.extend((ln + line_base[0], mask, off + cuts[i]) for ln, mask, off in det.collect_anomalies(i & 1))
            parts_f.append(f.copy())
            parts_s.append(s.copy())
            line_base[0] += int(f.size)
        for i in range(k):
            if i >= 2:
                collect(i - 2)
            det.submit(arr[cuts[i]:cuts[i + 1]], 0, i & 1)
        for i in range(max(0, k - 2), k):
            collect(i)
        return np.concatenate(parts_f), np.concatenate(parts_s), (anoms if want_anoms else None)

    def _process_lines_one(self, data: bytes, force_delimited: bool = False) -> Optional[bytes]:
        remaining = max(0, self.data_use_training - self.n_seen)
        anomalies = None
        if (remaining == 0 and len(data) >= self.PIPE_MIN_BYTES and self.logformat is None and not getattr(self, "combos", None)
                and os.environ.get("DM_KERNEL", "stream") == "stream"):
            flags, scores, anomalies = self._detect_pipelined(data)
            n_anom = int(np.count_nonzero(flags))
        else:
            try:
                flags, scores = self.det.process_lines(data, n_train_lines=remaining, copy=False)
            except Exception as e:
                self._count_dropped_training(e, remaining, lambda: _alerts.count_records(data))
                raise
            n_anom = self.det.last_n_anomalies
        n = int(flags.size)
        base = self.n_seen
        self.n_seen += n
        if self.output_format == "compact":
            return struct.pack("<I", n) + flags.tobytes() + scores.tobytes()
        if n_anom == 0:
            return None
        if anomalies is None:
            anomalies = self.det.anomalies()
        out = []
        raw_keys = [m.key for m in self.monitors]
        for line_idx, mask, offset in anomalies:
            rec = _alerts.record_at(data, offset)
            if self.logformat is not None:
                _eid, variables, lfv = self.logformat.parse(rec) or (-1, [], {})
                alerts = {}
                for i, m in enumerate(self.monitors):
                    if mask >> i & 1:
                        v = lfv.get(m.pos, b"") if m.source == "header" else (variables[m.pos] if m.pos < len(variables) else b"")
                        alerts[m.alert_key] = _alerts.alert_text(v)
                out.append(self._detector_schema(str(base + line_idx), float(scores[line_idx]), alerts, lfv.get("Time")))
                continue
            alerts = self._line_alerts(rec, mask, raw_keys)
            out.append(self._detector_schema(str(base + line_idx), float(scores[line_idx]), alerts,
                                             _alerts.record_time(rec)))
        if not out:
            return None
        return out[0] if (n == 1 and not force_delimited) else wire.frame_delimited(out)

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

    def _line_alerts(self, rec: bytes, mask: int, raw_keys: List[bytes]) -> Dict[str, str]:
        """alertsObtain of one anomalous raw record from the device's unknown-field mask."""
        wanted = [raw_keys[i] for i in range(len(raw_keys)) if mask >> i & 1]
        vals = _alerts.record_fields(rec, wanted)
        return {self.monitors[i].alert_key: _alerts.alert_text(vals.get(raw_keys[i], b""))
                for i in range(len(raw_keys)) if mask >> i & 1}

    # ------------------------------------------------------------------ output
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
        self.det.reset()
        self.n_seen = 0
        self.n_alerts = 0

    def import_state(self, state: dict) -> None:
        self.det.import_known(np.array(state.get("known", []), dtype=np.uint64))
        self.n_seen = int(state.get("n_seen", 0))
        self.n_alerts = int(state.get("n_alerts", 0))


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


class B200NewValueComboDetector(B200NewValueDetector):
    """NewValueComboDetector on the device (SURVEY.md section 8f-4; semantics R-combo in DESIGN.md /
    oracle/nvcd.py): tuples of field values instead of single values.  The member
    fingerprints are folded in order into one 64-bit key and learnt / probed in the same
    table (`dm_set_combos`).  Input: ParserSchema (one per message or a delimited batch), or raw
    key=value records for combinations of global header variables."""

    def __init__(self, name: str = "B200NewValueComboDetector", config: Optional[Any] = None) -> None:
        raw_cfg = config.model_dump() if hasattr(config, "model_dump") else config
        cfg = select_component_config(raw_cfg, name, fallback="NewValueComboDetector")
        cfg.setdefault("method_type", "new_value_combo_detector")
        cfg.setdefault("detector_id", "NewValueComboDetector" if name.startswith("B200") else name)
        if cfg.get("log_format"):
            raise ValueError("combination monitors are not evaluated in log_format mode; feed key=value records "
                             "or ParserSchema messages")
        super().__init__(name=name, config={"detectors": {name: cfg}})
        self.monitors, self.combos = parse_combos(cfg)

    @property
    def det(self):
        fresh = self._det is None
        d = B200NewValueDetector.det.fget(self)
        if fresh:
            d.set_combos(self.combos, member_only_mask=(1 << len(self.monitors)) - 1)
        return d

    def _description(self) -> str:
        return f"{self.detector_id} detects value combinations not encountered in training as anomalies."

    def _record_alerts(self, rec: Dict, mask: int) -> Dict[str, str]:
        by_field = dict(self._record_values(rec))
        n = len(self.monitors)
        out = {}
        for c, members in enumerate(self.combos):
            if mask >> (n + c) & 1:
                m0 = self.monitors[members[0]]
                scope = "Global" if m0.event_id is None else f"EventID {m0.event_id}"
                key = "%s - (%s)" % (scope, ", ".join(self.monitors[i].label for i in members))
                out[key] = "Unknown value combination: (%s)" % ", ".join(
                    "'%s'" % by_field.get(i, b"").decode("utf-8", "replace") for i in members)
        return out

    def _process_record(self, data: bytes) -> Optional[bytes]:
        out = self._process_record_batch(wire.frame_delimited([data]))     # the device walks the record
        if self.last_n_malformed:
            raise wire.WireError("malformed ParserSchema record")          # as B200NewValueDetector's per-record path
        if out is None or self.output_format == "compact":
            return out
        return wire.split_delimited(out)[0]                                 # one record in, one bare alert out

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

    def _line_alerts(self, rec: bytes, mask: int, raw_keys: List[bytes]) -> Dict[str, str]:
        """Raw key=value records (one thread per record on the device, dm_kernels_lanes.cuh): a
        combination of global header variables is the tuple of those fields of the record."""
        n = len(self.monitors)
        out = {}
        for c, members in enumerate(self.combos):
            if mask >> (n + c) & 1:
                vals = _alerts.record_fields(rec, [raw_keys[i] for i in members])
                m0 = self.monitors[members[0]]
                scope = "Global" if m0.event_id is None else f"EventID {m0.event_id}"
                key = "%s - (%s)" % (scope, ", ".join(self.monitors[i].label for i in members))
                out[key] = "Unknown value combination: (%s)" % ", ".join(
                    "'%s'" % vals.get(raw_keys[i], b"").decode("utf-8", "replace") for i in members)
        return out


def decode_compact(blob: bytes) -> Tuple[np.ndarray, np.ndarray]:
    """Inverse of the ``compact`` output format."""
    (n,) = struct.unpack_from("<I", blob, 0)
    flags = np.frombuffer(blob, dtype=np.uint8, count=n, offset=4)
    scores = np.frombuffer(blob, dtype=np.float32, count=n, offset=4 + n)
    return flags, scores
