"""DeviceDetector -- thin ctypes wrapper of one libdmdetect handle (one GPU).

Host code stays Python; all tokenizing, hashing, set membership and scoring run in the
sm_90a kernels behind include/dmdetect.h.  PyTorch tensors are used only as device /
pinned-host buffer containers whose raw pointers are handed to the C ABI.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib

BytesLike = Union[bytes, bytearray, memoryview, np.ndarray]


def _as_key_bytes(k: Union[str, bytes]) -> bytes:
    return k if isinstance(k, bytes) else k.encode("utf-8")


def parser_format_strings(version: str, parser_type: str, parser_id: str, templates: Sequence[bytes],
                          names: Sequence[str]) -> Tuple[List[bytes], List[int]]:
    """dm_set_parser_format's strings and capture_order: the capture names go out sorted by their UTF-8 bytes, as
    wire.encode_parser_schema sorts the logFormatVariables keys."""
    order = sorted(range(len(names)), key=lambda i: names[i].encode("utf-8"))
    strs = [s.encode("utf-8") for s in (version, parser_type, parser_id)] + [bytes(t) for t in templates]
    return strs + [names[i].encode("utf-8") for i in order], order


class DeviceDetector:
    """NewValueDetector state (known-value table + running statistics) on one H100.

    keys: the monitored field names, in monitor order (field k <-> bit k of the masks).
    """

    def __init__(self, keys: Sequence[Union[str, bytes]], device: int = 0,
                 max_batch_bytes: int = 32 << 20, max_lines: int = 0, table_log2_slots: int = 20):
        self._lib = _lib.load()
        self.keys: List[bytes] = [_as_key_bytes(k) for k in keys]
        self.device = int(device)
        self.max_batch_bytes = int(max_batch_bytes)
        blob = b"".join(self.keys)
        lens = (C.c_uint32 * max(1, len(self.keys)))(*[len(k) for k in self.keys])
        h = C.c_void_p()
        _lib.check(self._lib.dm_create(self.device, len(self.keys), blob, lens, self.max_batch_bytes,
                                       int(max_lines), int(table_log2_slots), C.byref(h)))
        self._h = h
        self.max_lines = int(max_lines) if max_lines else max(self.max_batch_bytes // 8, 1024)
        self._pin_flags = None
        self._pin_scores = None
        self._pin_in = None

    # ------------------------------------------------------------------ lifecycle
    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.dm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False

    # ------------------------------------------------------------------ helpers
    def _pinned_outputs(self):
        if self._pin_flags is None:
            import torch
            self._pin_flags = torch.empty(self.max_lines, dtype=torch.uint8, pin_memory=True)
            self._pin_scores = torch.empty(self.max_lines, dtype=torch.float32, pin_memory=True)
        return self._pin_flags, self._pin_scores

    @staticmethod
    def _host_ptr(buf: BytesLike) -> Tuple[int, int, object]:
        """(address, nbytes, keepalive) of a host buffer without copying."""
        if isinstance(buf, np.ndarray):
            a = np.ascontiguousarray(buf).view(np.uint8).reshape(-1)
            return a.ctypes.data, a.size, a
        if isinstance(buf, bytes):
            return C.cast(C.c_char_p(buf), C.c_void_p).value or 0, len(buf), buf
        mv = memoryview(buf).cast("B")
        a = np.frombuffer(mv, dtype=np.uint8)
        return a.ctypes.data, a.size, a

    # ------------------------------------------------------------------ hot path, host buffers
    def process_lines(self, buf: BytesLike, n_train_lines: int = 0, copy: bool = True
                      ) -> Tuple[np.ndarray, np.ndarray]:
        """One message of '\\n'-terminated raw records in host memory.  The first
        n_train_lines records are training data.  Returns (flags uint8[n], scores float32[n])."""
        ptr, n, keep = self._host_ptr(buf)
        pf, ps = self._pinned_outputs()
        n_lines = C.c_uint64()
        n_anom = C.c_uint64()
        _lib.check(self._lib.dm_process_lines(self._h, ptr, n, 0, int(n_train_lines), pf.data_ptr(), ps.data_ptr(),
                                              self.max_lines, 0, C.byref(n_lines), C.byref(n_anom), None))
        del keep
        k = n_lines.value
        f = pf.numpy()[:k]
        s = ps.numpy()[:k]
        self.last_n_anomalies = n_anom.value
        return (f.copy(), s.copy()) if copy else (f, s)

    def stage_pinned(self, buf: BytesLike):
        """Copy a host message into the detector's pinned staging buffer; returns a uint8
        numpy view usable as input of process_lines (fast H2D path)."""
        import torch
        if self._pin_in is None:
            self._pin_in = torch.empty(self.max_batch_bytes + 64, dtype=torch.uint8, pin_memory=True)
        ptr, n, keep = self._host_ptr(buf)
        view = self._pin_in.numpy()[:n]
        C.memmove(view.ctypes.data, ptr, n)
        del keep
        return view

    # ------------------------------------------------------------------ hot path, device buffers
    def enqueue_device(self, data_ptr: int, nbytes: int, n_train_lines: int = 0, flags_ptr: int = 0,
                       scores_ptr: int = 0, out_cap_lines: int = 0, stream: int = 0) -> None:
        """Enqueue one device-resident message on `stream` (a raw cudaStream_t, 0 = the
        handle's own stream) without synchronising.  Pointers are raw device addresses
        (e.g. torch.Tensor.data_ptr()); the message buffer needs 16 bytes of slack."""
        _lib.check(self._lib.dm_process_lines(self._h, data_ptr, int(nbytes), 1, int(n_train_lines),
                                              flags_ptr or None, scores_ptr or None, int(out_cap_lines), 1,
                                              None, None, stream or None))

    # ------------------------------------------------------------------ pipelined host path
    def submit(self, buf: BytesLike, n_train_lines: int = 0, slot: int = 0) -> None:
        """Enqueue one host message on `slot` (0 or 1) without waiting: H2D copy, kernels and
        the header copy back overlap with the other slot's work.  `buf` must stay alive and
        unchanged until collect(slot); pinned memory (stage_pinned / torch pin_memory) gives
        real copy/compute overlap."""
        ptr, n, keep = self._host_ptr(buf)
        if not hasattr(self, "_inflight"):
            self._inflight = {}
        self._inflight[slot] = keep
        _lib.check(self._lib.dm_submit_lines(self._h, ptr, n, int(n_train_lines), int(slot)))

    def collect(self, slot: int = 0) -> Tuple[np.ndarray, np.ndarray]:
        """Wait for `slot`; returns (flags, scores) as views of the handle's pinned result
        buffers (valid until the slot is submitted again).  The slot's batch becomes the last
        batch: encode_alerts() words it until the next submit()."""
        pf, ps = C.c_void_p(), C.c_void_p()
        n_lines, n_anom = C.c_uint64(), C.c_uint64()
        _lib.check(self._lib.dm_collect(self._h, int(slot), C.byref(pf), C.byref(ps), C.byref(n_lines), C.byref(n_anom)))
        self._inflight.pop(slot, None)
        k = n_lines.value
        self.last_n_anomalies = n_anom.value
        if k == 0:
            return np.zeros(0, np.uint8), np.zeros(0, np.float32)
        f = np.ctypeslib.as_array(C.cast(pf, C.POINTER(C.c_uint8)), shape=(k,))
        s = np.ctypeslib.as_array(C.cast(ps, C.POINTER(C.c_float)), shape=(k,))
        return f, s

    def collect_anomalies(self, slot: int = 0, cap: int = 1 << 20) -> List[Tuple[int, int, int]]:
        n = C.c_uint32()
        _lib.check(self._lib.dm_collect_anomalies(self._h, int(slot), None, 0, C.byref(n)))
        k = min(n.value, cap)
        if k == 0:
            return []
        arr = (_lib.Anomaly * k)()
        _lib.check(self._lib.dm_collect_anomalies(self._h, int(slot), arr, k, C.byref(n)))
        return [(arr[i].line, arr[i].mask, arr[i].offset) for i in range(min(k, n.value))]

    # ------------------------------------------------------------------ record mode
    def process_values(self, records, n_train_records: int = 0, record_bytes: int = 0
                       ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """records: one list of (monitored-field index, value bytes) per record (the values a
        ParserSchema holds for the configured monitors).  The first n_train_records records
        are training data.  Returns (flags u8, scores f32, unknown-field masks u32)."""
        n_rec = len(records)
        blob = bytearray()
        offsets, fields, rec_of = [0], [], []
        for r, vals in enumerate(records):
            for f, v in vals:
                blob += v
                offsets.append(len(blob))
                fields.append(int(f))
                rec_of.append(r)
        n_val = len(fields)
        off_a = (C.c_uint32 * (n_val + 1))(*offsets)
        fld_a = (C.c_uint32 * max(1, n_val))(*fields)
        rec_a = (C.c_uint32 * max(1, n_val))(*rec_of)
        flags = np.zeros(max(1, n_rec), dtype=np.uint8)
        scores = np.zeros(max(1, n_rec), dtype=np.float32)
        masks = np.zeros(max(1, n_rec), dtype=np.uint32)
        n_anom = C.c_uint64()
        _lib.check(self._lib.dm_process_values(self._h, bytes(blob), len(blob), off_a, fld_a, rec_a, n_val, n_rec,
                                               int(n_train_records), int(record_bytes), flags.ctypes.data,
                                               scores.ctypes.data, masks.ctypes.data, C.byref(n_anom)))
        self.last_n_anomalies = n_anom.value
        return flags[:n_rec], scores[:n_rec], masks[:n_rec]

    # ------------------------------------------------------------------ record mode on the device
    def set_monitors(self, monitors) -> None:
        """monitors: one dict per monitored field, in field order:
        {"event_id": int|None, "source": "header"|"variable", "pos": key str/bytes | index}."""
        arr = (_lib.Monitor * max(1, len(monitors)))()
        for i, m in enumerate(monitors):
            arr[i].event_id = int(m["event_id"]) if m.get("event_id") is not None else 0
            arr[i].has_event = 0 if m.get("event_id") is None else 1
            if m["source"] == "header":
                kb = m["pos"] if isinstance(m["pos"], bytes) else str(m["pos"]).encode("utf-8")
                if not 0 < len(kb) <= 64:
                    raise ValueError(f"header key {kb!r}: length not in 1..64")
                arr[i].source, arr[i].var_index, arr[i].key_len = 0, 0, len(kb)
                for j, c in enumerate(kb):
                    arr[i].key[j] = c
            else:
                arr[i].source, arr[i].var_index, arr[i].key_len = 1, int(m["pos"]), 0
        _lib.check(self._lib.dm_set_monitors(self._h, len(monitors), arr))

    def set_combos(self, combos, member_only_mask: int = 0) -> None:
        """combos: lists of monitor indices (ordered tuples of fields, NewValueComboDetector);
        combination c reports in mask bit n_monitors + c.  Call after set_monitors."""
        off, flat = [0], []
        for members in combos:
            flat.extend(int(i) for i in members)
            off.append(len(flat))
        a_off = (C.c_uint32 * len(off))(*off)
        a_mem = (C.c_uint32 * max(1, len(flat)))(*flat)
        _lib.check(self._lib.dm_set_combos(self._h, len(combos), a_off, a_mem, int(member_only_mask)))

    def set_format(self, log_format: Optional[str], templates=(), content_name: str = "Content", norm_flags: int = 0) -> None:
        """Tokenise process_lines() input with a MatcherParser log_format (+ `<*>` templates
        matched against the capture `content_name`) instead of key=value fields.  The
        monitors of set_monitors() bind to it by capture name / wildcard index / EventID.
        norm_flags: logformat.NORM_* (remove_spaces / remove_punctuation / lowercase).
        None switches back."""
        if log_format is None:
            _lib.check(self._lib.dm_set_format(self._h, None, None, 0, None))
            return
        ts = [t.encode("utf-8") if isinstance(t, str) else bytes(t) for t in templates]
        arr = (C.c_char_p * max(1, len(ts)))(*ts)
        _lib.check(self._lib.dm_set_format_ex(self._h, log_format.encode("utf-8"), content_name.encode("utf-8"), len(ts), arr,
                                              int(norm_flags)))

    def process_records(self, buf: bytes, n_train_records: int = 0) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """A batch of varint-length-delimited ParserSchema records, decoded and scored on the
        device.  Returns (flags u8, scores f32, unknown-field masks u32), one entry per record."""
        # a record takes its length prefix and, nearly always, at least one more byte; a batch of (mostly) EMPTY records --
        # one zero byte each -- gets a second try with room for one record per byte
        for cap in (max(1, len(buf) // 2 + 1), len(buf) + 1):
            flags = np.zeros(cap, dtype=np.uint8)
            scores = np.zeros(cap, dtype=np.float32)
            masks = np.zeros(cap, dtype=np.uint32)
            n_rec, n_anom = C.c_uint64(), C.c_uint64()
            rc = self._lib.dm_process_records(self._h, bytes(buf), len(buf), int(n_train_records), flags.ctypes.data,
                                              scores.ctypes.data, masks.ctypes.data, cap, C.byref(n_rec), C.byref(n_anom))
            if rc != _lib.DM_ERR_CAPACITY or cap == len(buf) + 1:
                break
        _lib.check(rc)
        self.last_n_anomalies = n_anom.value
        k = n_rec.value
        return flags[:k], scores[:k], masks[:k]

    def process_logs(self, buf: bytes, n_train_records: int = 0, delimited: bool = True
                     ) -> Tuple[np.ndarray, np.ndarray, int]:
        """LogSchema records -- one bare record (delimited=False) or a varint-length-delimited batch -- whose `log`
        texts are unwrapped on the device and detected as raw lines (key=value, or the log_format of set_format).
        The first n_train_records usable records train.  Returns (flags u8, scores f32, records malformed or
        unusable), one flag and score per record; anomalies() then names records and their payload offsets."""
        cap = max(1, len(buf)) if delimited else 1              # (a delimited record takes at least its length byte)
        flags = np.empty(cap, dtype=np.uint8)                   # (the library writes the first n_records entries)
        scores = np.empty(cap, dtype=np.float32)
        n_rec, n_bad, n_anom = C.c_uint64(), C.c_uint64(), C.c_uint64()
        _lib.check(self._lib.dm_process_logs(self._h, bytes(buf), len(buf), int(bool(delimited)), int(n_train_records),
                                             flags.ctypes.data, scores.ctypes.data, cap, C.byref(n_rec), C.byref(n_bad),
                                             C.byref(n_anom)))
        self.last_n_anomalies = n_anom.value
        k = n_rec.value
        return flags[:k], scores[:k], int(n_bad.value)

    # ------------------------------------------------------------------ DetectorSchema alerts on the device
    def set_alert_format(self, version: str, detector_id: str, detector_type: str, description: str,
                         alert_keys: Sequence[Tuple[str, Sequence[int]]], combos: Sequence[Sequence[int]] = (),
                         capacity: int = 0, time_capture: Optional[int] = None) -> None:
        """What encode_alerts() writes besides the record's own values (dm_set_alert_format): the constant strings, the
        alertsObtain keys in output order, each with the mask bits that supply it in config order (bit k < n monitors =
        monitor k, bit n + c = combination c, whose monitors `combos[c]` lists), the capacity of the output buffer in
        bytes (0: a quarter of max_batch_bytes, at least 1 MiB) and, in log_format mode, the index of the header capture
        that holds the record's Time (None: none).  Allocates the buffers once."""
        strs = [s.encode("utf-8") for s in (version, detector_id, detector_type, description)]
        strs += [k.encode("utf-8") for k, _bits in alert_keys]
        lens = (C.c_uint32 * len(strs))(*[len(s) for s in strs])
        off, flat = [0], []
        for _k, bits in alert_keys:
            flat.extend(int(b) for b in bits)
            off.append(len(flat))
        c_off, c_mem = [0], []
        for members in combos:
            c_mem.extend(int(i) for i in members)
            c_off.append(len(c_mem))
        cap = int(capacity) or max(1 << 20, self.max_batch_bytes // 4)
        _lib.check(self._lib.dm_set_alert_format(
            self._h, len(strs), b"".join(strs), lens, (C.c_uint32 * len(off))(*off), (C.c_uint32 * max(1, len(flat)))(*flat),
            len(combos), (C.c_uint32 * len(c_off))(*c_off), (C.c_uint32 * max(1, len(c_mem)))(*c_mem),
            0xFFFFFFFF if time_capture is None else int(time_capture), cap))
        if getattr(self, "_pin_alerts", None) is None or self._pin_alerts.numel() != cap:
            import torch
            self._pin_alerts = torch.empty(cap, dtype=torch.uint8, pin_memory=True)

    def encode_alerts(self, first_log_id: int, first_alert_id: int, now: int) -> Optional[Tuple[bytes, int]]:
        """The varint-delimited DetectorSchemas of the last process_lines(), process_logs(), process_records() or
        collect() batch (dm_encode_alerts) and their count, or None when the device declines the batch (the caller then
        encodes it on the host).  first_log_id numbers raw lines only; LogSchema and ParserSchema alerts carry the
        record's logID.  A collected slot must be encoded before it is submitted again."""
        out_len, n, declined = C.c_uint64(), C.c_uint64(), C.c_int()
        buf = self._pin_alerts
        _lib.check(self._lib.dm_encode_alerts(self._h, int(first_log_id), int(first_alert_id), int(now), buf.data_ptr(),
                                              buf.numel(), C.byref(out_len), C.byref(n), C.byref(declined)))
        if declined.value:
            return None
        return bytes(buf.numpy()[:out_len.value]), int(n.value)

    # ------------------------------------------------------------------ the MatcherParser stage on the device
    def set_parser_format(self, version: str, parser_type: str, parser_id: str, templates: Sequence[bytes],
                          names: Sequence[str]) -> None:
        """What parse_logs() writes besides the record's own text (dm_set_parser_format), after set_format(): the
        constant strings, the template texts verbatim in EventID order and the log_format's capture names in capture
        order (written sorted by their UTF-8 bytes)."""
        strs, order = parser_format_strings(version, parser_type, parser_id, templates, names)
        lens = (C.c_uint32 * len(strs))(*[len(s) for s in strs])
        _lib.check(self._lib.dm_set_parser_format(self._h, len(strs), b"".join(strs), lens,
                                                  (C.c_uint32 * max(1, len(order)))(*order)))

    def parse_logs(self, buf: BytesLike, delimited: bool, first_parsed_id: int, now: int) -> Tuple[bytes, int, int, int]:
        """LogSchema records -- one bare record (delimited=False) or a varint-length-delimited batch -- parsed on the
        device into ParserSchemas (dm_parse_logs, rule R-parse in DESIGN.md).  Returns (the varint-delimited
        ParserSchemas, records, ParserSchemas emitted, records malformed or unusable)."""
        ptr, n, keep = self._host_ptr(buf)
        out, out_len = C.c_void_p(), C.c_uint64()
        n_rec, n_emit, n_bad = C.c_uint64(), C.c_uint64(), C.c_uint64()
        _lib.check(self._lib.dm_parse_logs(self._h, ptr, n, int(bool(delimited)), int(first_parsed_id), int(now),
                                           C.byref(out), C.byref(out_len), C.byref(n_rec), C.byref(n_emit), C.byref(n_bad)))
        del keep
        blob = C.string_at(out.value, out_len.value) if out_len.value else b""
        return blob, n_rec.value, n_emit.value, n_bad.value

    def sync(self) -> Tuple[int, int]:
        n_lines = C.c_uint64()
        n_anom = C.c_uint64()
        _lib.check(self._lib.dm_sync(self._h, C.byref(n_lines), C.byref(n_anom)))
        return n_lines.value, n_anom.value

    # ------------------------------------------------------------------ results / state
    def anomalies(self, cap: int = 1 << 20) -> List[Tuple[int, int, int]]:
        n = C.c_uint32()
        _lib.check(self._lib.dm_get_anomalies(self._h, None, 0, C.byref(n)))
        k = min(n.value, cap)
        if k == 0:
            return []
        arr = (_lib.Anomaly * k)()
        _lib.check(self._lib.dm_get_anomalies(self._h, arr, k, C.byref(n)))
        k = min(k, n.value)
        return [(arr[i].line, arr[i].mask, arr[i].offset) for i in range(k)]

    def stats(self) -> dict:
        st = _lib.Stats()
        _lib.check(self._lib.dm_get_stats(self._h, C.byref(st)))
        return st.as_dict(len(self.keys))

    def global_stats(self) -> dict:
        st = _lib.Stats()
        _lib.check(self._lib.dm_get_global_stats(self._h, C.byref(st)))
        return st.as_dict(len(self.keys))

    def export_known(self) -> np.ndarray:
        n = C.c_uint64()
        _lib.check(self._lib.dm_export_known(self._h, None, 0, C.byref(n)))
        out = np.zeros(max(1, n.value), dtype=np.uint64)
        _lib.check(self._lib.dm_export_known(self._h, out.ctypes.data_as(C.POINTER(C.c_uint64)), n.value, C.byref(n)))
        return out[:n.value]

    def import_known(self, keys: np.ndarray) -> None:
        a = np.ascontiguousarray(keys, dtype=np.uint64)
        _lib.check(self._lib.dm_import_known(self._h, a.ctypes.data_as(C.POINTER(C.c_uint64)), a.size))

    def reset(self) -> None:
        _lib.check(self._lib.dm_reset(self._h))

    def table_key(self, field: int, value: bytes) -> int:
        return int(self._lib.dm_table_key(int(field), value, len(value)))

    # ------------------------------------------------------------------ measurement
    def set_overlap(self, on: bool = True) -> None:
        """Let consecutive device-resident detection calls on one stream overlap (dm_set_overlap:
        the caller promises not to rewrite a call's input with a kernel enqueued between calls)."""
        _lib.check(self._lib.dm_set_overlap(self._h, int(on)))

    def stream_recheck_chained(self) -> bool:
        """Did the last key=value message go through the stream kernel's batch-wise re-check of candidates?"""
        rc = self._lib.dm_stream_recheck_chained(self._h)
        if rc < 0:
            _lib.check(rc)
        return rc == 1

    def profile_enable(self, on: bool = True) -> None:
        _lib.check(self._lib.dm_profile_enable(self._h, int(on)))

    def profile_read(self) -> Tuple[float, int, int]:
        """(summed dominant-kernel ms, launches timed, kernels launched since creation)."""
        ms = C.c_double()
        n = C.c_uint64()
        tot = C.c_uint64()
        _lib.check(self._lib.dm_profile_read(self._h, C.byref(ms), C.byref(n), C.byref(tot)))
        return ms.value, n.value, tot.value

    # ------------------------------------------------------------------ multi-GPU window
    def window_words(self, world: int, with_keys: bool) -> int:
        return int(self._lib.dm_window_words(self._h, int(world), int(with_keys)))

    def window_export(self, dev_ptr: int, rank: int, world: int, with_keys: bool, stream: int = 0) -> None:
        _lib.check(self._lib.dm_window_export(self._h, dev_ptr, rank, world, int(with_keys), stream or None))

    @staticmethod
    def nccl_unique_id() -> bytes:
        """128-byte NCCL id (call on rank 0, hand the bytes to every rank's nccl_init)."""
        buf = C.create_string_buffer(128)
        _lib.check(_lib.load().dm_nccl_unique_id(buf))
        return buf.raw

    def nccl_init(self, unique_ids: bytes, rank: int, world: int) -> None:
        """Give the handle its own NCCL communicator(s) for window_allreduce(): one or two
        128-byte ids (two: consecutive windows alternate between them)."""
        if len(unique_ids) not in (128, 256):
            raise ValueError("one or two 128-byte NCCL unique ids")
        _lib.check(self._lib.dm_nccl_init(self._h, unique_ids, len(unique_ids) // 128, int(rank), int(world)))

    def window_allreduce(self, with_keys: bool, stream: int = 0) -> None:
        """export + ncclAllReduce + import of one window, enqueued on `stream` by one call."""
        _lib.check(self._lib.dm_window_allreduce(self._h, int(with_keys), stream or None))

    def window_import(self, dev_ptr: int, rank: int, world: int, with_keys: bool, stream: int = 0) -> None:
        _lib.check(self._lib.dm_window_import(self._h, dev_ptr, rank, world, int(with_keys), stream or None))
