"""Loader for the CPU emulation of the kernels (tests/emu).  TEST INFRASTRUCTURE.

The emulator compiles the product's kernel SOURCES (detectmateservice_b200/csrc/
dm_kernels_*.cuh) with g++ -DDM_EMU and runs one thread block at a time on OS threads; it lets the
CPU test tier check the kernels' logic against the oracle.  It is not a CPU implementation of the
product: nothing outside tests/ can reach it.  One library, tests/emu/_build/libemu.so, holds every
emu_* entry point; lib() declares their signatures.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMU = os.path.join(HERE, "emu")
SO = os.path.join(EMU, "_build", "libemu.so")
CSRC = os.path.join(ROOT, "detectmateservice_b200", "csrc")
TILE_BYTES = 32768


def build():
    srcs = [os.path.join(EMU, "emu.cpp"), os.path.join(EMU, "cuda_emu.h")] + [
        os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "dmdetect.h")]
    if os.path.exists(SO) and all(os.path.getmtime(s) <= os.path.getmtime(SO) for s in srcs):
        return SO
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-DDM_EMU", "-I" + EMU, "-I" + CSRC, "-shared", "-fPIC",
                           "-pthread", "-o", SO, os.path.join(EMU, "emu.cpp")])
    return SO


class Anomaly(C.Structure):
    _fields_ = [("line", C.c_uint32), ("mask", C.c_uint32), ("offset", C.c_uint64)]


_P32, _P64 = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
_LINES = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, _P64, _P64, _P32]
_SIGNATURES = {                                                   # name: (restype, argtypes)
    "emu_create": (C.c_void_p, [C.c_uint32, C.c_char_p, _P32, C.c_uint32, C.c_uint64, C.c_uint64]),
    "emu_destroy": (None, [C.c_void_p]),
    "emu_set_monitors": (None, [C.c_void_p, C.c_void_p, C.c_uint32]),
    "emu_set_combos": (None, [C.c_void_p, C.c_uint32, _P32, _P32, C.c_uint32]),
    "emu_set_format": (C.c_char_p, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_char_p), C.c_uint32]),
    "emu_stream_ctas": (None, [C.c_uint32]),
    "emu_process_stream": (C.c_int, _LINES),
    "emu_process_stream_chain": (C.c_int, _LINES),
    "emu_stream_hint": (C.c_uint64, []),
    "emu_chain_stats": (None, [_P64, C.c_int]),
    "emu_process_lanes": (C.c_int, _LINES),
    "emu_process_format": (C.c_int, _LINES),
    "emu_frame_split": (C.c_int64, [C.c_char_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, _P64]),
    "emu_process_records": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_uint64, _P64, _P64]),
    "emu_set_anomaly_cap": (None, [C.c_void_p, C.c_uint32]),
    "emu_logs_unwrap": (C.c_int64, [C.c_char_p, C.c_uint64, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                    C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "emu_process_logs": (C.c_int, [C.c_void_p, C.c_int, C.c_char_p, C.c_uint64, C.c_int, C.c_uint32, C.c_void_p,
                                   C.c_void_p, C.c_uint64, _P64, _P64, _P64]),
    "emu_set_alert_format": (C.c_char_p, [C.c_void_p, C.c_uint32, C.c_char_p, _P32, _P32, _P32, C.c_uint32, _P32, _P32,
                                          C.c_uint32]),
    "emu_encode_alerts": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int64, C.c_int64, C.c_void_p, C.c_uint64, _P64, _P64,
                                    C.POINTER(C.c_int)]),
    "emu_utf8_replace": (C.c_uint32, [C.c_char_p, C.c_uint32, C.c_void_p]),
    "emu_alert_time": (C.c_int, [C.c_char_p, C.c_uint32, C.c_longlong, C.POINTER(C.c_longlong)]),
    "emu_alert_time_str": (C.c_int, [C.c_char_p, C.c_uint32, C.c_longlong, C.POINTER(C.c_longlong)]),
    "emu_set_parser_format": (C.c_char_p, [C.c_void_p, C.c_uint32, C.c_char_p, _P32, _P32]),
    "emu_parse_logs": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_uint64,
                                 _P64, _P64, _P64]),
    "emu_get_anomalies": (C.c_uint32, [C.c_void_p, C.POINTER(Anomaly), C.c_uint32]),
    "emu_get_stats": (None, [C.c_void_p, _P64]),
    "emu_export_known": (C.c_uint64, [C.c_void_p, _P64, C.c_uint64]),
    "emu_import_known": (C.c_uint32, [C.c_void_p, C.c_void_p, C.c_uint64]),
    "emu_window_words": (C.c_uint64, [C.c_uint32, C.c_int, C.c_uint64]),
    "emu_window_export": (None, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint64]),
    "emu_window_pending_keys": (C.c_uint64, [C.c_void_p]),
    "emu_window_import": (C.c_uint32, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint64]),
    "emu_get_global_stats": (None, [C.c_void_p, _P64]),
}


def lib():
    """The emulator library (built when a source is newer), every emu_* signature declared."""
    L = C.CDLL(build())
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    return L


def _u32(v):
    return (C.c_uint32 * max(1, len(v)))(*v)


class EmuDetector:
    """One emulated handle.  variant: the kernel process_lines runs -- "stream", "chain" (the stream kernel's chained
    re-check), "lanes" (one thread per record) or "format" (log_format mode: set_format first)."""

    def __init__(self, keys, table_log2=12, max_bytes=4 << 20, max_lines=1 << 20, variant="stream"):
        self.lib = lib()
        self.variant = variant
        self.keys = [k if isinstance(k, bytes) else k.encode() for k in keys]
        lens = _u32([len(k) for k in self.keys])
        self.h = self.lib.emu_create(len(self.keys), b"".join(self.keys), lens, table_log2,
                                     max_bytes // TILE_BYTES + 2, max_lines)
        self.max_lines = max_lines
        self.table_log2 = table_log2

    def close(self):
        if self.h:
            self.lib.emu_destroy(self.h)
            self.h = None

    def set_monitors(self, arr, n):
        """arr: n dm_monitor_t (detectmateservice_b200._lib.Monitor); clears the combinations, as dm_set_monitors."""
        self.lib.emu_set_monitors(self.h, arr, n)

    def set_combos(self, combos, member_only):
        """combos: member lists of monitor indices; () turns combinations off."""
        off, flat = [0], []
        for members in combos:
            flat += members
            off.append(len(flat))
        self.lib.emu_set_combos(self.h, len(combos), _u32(off), _u32(flat), member_only)

    def set_format(self, log_format, templates=(), flags=0, content_name=b"Content"):
        """Binds the monitors of set_monitors; raises ValueError with dm_format_build's reason."""
        ts = [t if isinstance(t, bytes) else t.encode() for t in templates]
        fmt = log_format if isinstance(log_format, bytes) else log_format.encode()
        err = self.lib.emu_set_format(self.h, fmt, content_name, len(ts), (C.c_char_p * max(1, len(ts)))(*ts), flags)
        if err:
            raise ValueError(err.decode())

    def process_lines(self, msg: bytes, n_train: int = 0, out=None):
        """out: (flags u8, scores f32) arrays owned by the caller, written in place (capacity = their length), as a
        device-resident caller passes the same buffers to call after call; default: fresh ones pre-filled with 7 / -1."""
        if out is None:
            cap = msg.count(b"\n") + 2
            flags = np.full(cap, 7, dtype=np.uint8)
            scores = np.full(cap, -1, dtype=np.float32)
        else:
            flags, scores = out
            cap = min(flags.size, scores.size)
        n_lines, n_anom, err = C.c_uint64(), C.c_uint64(), C.c_uint32()
        fn = {"lanes": self.lib.emu_process_lanes, "stream": self.lib.emu_process_stream,
              "chain": self.lib.emu_process_stream_chain, "format": self.lib.emu_process_format}[self.variant]
        rc = fn(self.h, msg, len(msg), n_train, flags.ctypes.data, scores.ctypes.data, cap,
                C.byref(n_lines), C.byref(n_anom), C.byref(err))
        assert rc == 0 and err.value == 0, (rc, err.value)
        self.last_n_anomalies = n_anom.value
        return flags[:n_lines.value], scores[:n_lines.value]

    def process_records(self, batch: bytes, n_train: int, flags, scores, masks, cap):
        """dm_process_records on the caller's arrays: (return code, records, anomalous records)."""
        n_rec, n_an = C.c_uint64(), C.c_uint64()
        rc = self.lib.emu_process_records(self.h, batch, len(batch), n_train, flags.ctypes.data, scores.ctypes.data,
                                          masks.ctypes.data, cap, C.byref(n_rec), C.byref(n_an))
        return rc, n_rec.value, n_an.value

    def anomalies(self):
        arr = (Anomaly * 65536)()
        n = self.lib.emu_get_anomalies(self.h, arr, 65536)
        return [(arr[i].line, arr[i].mask, arr[i].offset) for i in range(n)]

    def _stats(self, fn):
        w = (C.c_uint64 * 40)()
        fn(self.h, w)
        return {"lines": w[0], "train_lines": w[1], "detect_lines": w[2], "anomalies": w[3], "score_sum": w[4],
                "bytes": w[5], "known_keys": w[6], "bad_records": w[7], "unknown_per_key": [w[8 + i] for i in range(len(self.keys))]}

    def stats(self):
        return self._stats(self.lib.emu_get_stats)

    def global_stats(self):
        """The statistics summed over the ranks by the window imports so far (dm_get_global_stats)."""
        return self._stats(self.lib.emu_get_global_stats)

    def export_known(self):
        """Every key of the table, sorted (dm_export_known)."""
        out = (C.c_uint64 * (1 << self.table_log2))()
        n = self.lib.emu_export_known(self.h, out, 1 << self.table_log2)
        return [out[i] for i in range(n)]

    def import_known(self, keys):
        """dm_import_known; returns the DM_DEVERR_* bits of the insert."""
        a = np.ascontiguousarray(keys, dtype=np.uint64)
        return self.lib.emu_import_known(self.h, a.ctypes.data, a.size)

    # the window exchange, seg_keys keys per rank segment (libdmdetect: 65536); buffers are uint64 numpy arrays
    def window_words(self, world, with_keys, seg_keys):
        return int(self.lib.emu_window_words(world, int(with_keys), seg_keys))

    def window_export(self, rank, world, with_keys, seg_keys):
        """dm_window_export into a fresh buffer filled with hostile words first; the buffer."""
        buf = np.full(self.window_words(world, with_keys, seg_keys), 0xDEADBEEFDEADBEEF, dtype=np.uint64)
        self.lib.emu_window_export(self.h, buf.ctypes.data, rank, world, int(with_keys), seg_keys)
        return buf

    def window_pending_keys(self):
        return int(self.lib.emu_window_pending_keys(self.h))

    def window_import(self, buf, rank, world, with_keys, seg_keys):
        """dm_window_import of an all-reduced buffer; returns the DM_DEVERR_* bits it leaves for the next sync."""
        a = np.ascontiguousarray(buf).view(np.uint64)
        assert a.size == self.window_words(world, with_keys, seg_keys)
        return self.lib.emu_window_import(self.h, a.ctypes.data, rank, world, int(with_keys), seg_keys)
