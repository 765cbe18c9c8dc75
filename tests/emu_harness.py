"""Loader for the CPU emulation of the fused kernel (tests/emu).  TEST INFRASTRUCTURE.

The emulator compiles the product's kernel SOURCES (detectmateservice_b200/csrc/
dm_kernels_*.cuh) with g++ -DDM_EMU and runs one thread block on OS threads; it lets the
CPU test tier check the kernel's tokenizer / detector logic against the oracle.  It is not a
CPU implementation of the product: nothing outside tests/ can reach it.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMU = os.path.join(HERE, "emu")
SO = os.path.join(EMU, "_build", "libemu_tile.so")
CSRC = os.path.join(ROOT, "detectmateservice_b200", "csrc")
TILE_BYTES = 32768


def build():
    srcs = [os.path.join(EMU, "emu_tile.cpp"), os.path.join(EMU, "cuda_emu.h")] + [
        os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "dmdetect.h")]
    if os.path.exists(SO) and all(os.path.getmtime(s) <= os.path.getmtime(SO) for s in srcs):
        return SO
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-DDM_EMU", "-I" + EMU, "-I" + CSRC, "-shared", "-fPIC",
                           "-pthread", "-o", SO, os.path.join(EMU, "emu_tile.cpp")])
    return SO


class Anomaly(C.Structure):
    _fields_ = [("line", C.c_uint32), ("mask", C.c_uint32), ("offset", C.c_uint64)]


class EmuDetector:
    def __init__(self, keys, table_log2=12, max_bytes=4 << 20, max_lines=1 << 20, variant="stream"):
        self.lib = C.CDLL(build())
        self.variant = variant
        L = self.lib
        L.emu_process_lanes.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64,
                                        C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
        L.emu_process_stream.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64,
                                         C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
        L.emu_process_stream_chain.argtypes = L.emu_process_stream.argtypes
        L.emu_stream_hint.restype = C.c_uint64
        L.emu_create.restype = C.c_void_p
        L.emu_create.argtypes = [C.c_uint32, C.c_char_p, C.POINTER(C.c_uint32), C.c_uint32, C.c_uint64, C.c_uint64]
        L.emu_destroy.argtypes = [C.c_void_p]
        L.emu_get_anomalies.restype = C.c_uint32
        L.emu_get_anomalies.argtypes = [C.c_void_p, C.POINTER(Anomaly), C.c_uint32]
        L.emu_get_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.emu_export_known.restype = C.c_uint64
        L.emu_export_known.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint64]
        self.keys = [k if isinstance(k, bytes) else k.encode() for k in keys]
        lens = (C.c_uint32 * len(self.keys))(*[len(k) for k in self.keys])
        self.h = L.emu_create(len(self.keys), b"".join(self.keys), lens, table_log2,
                              max_bytes // TILE_BYTES + 2, max_lines)
        self.max_lines = max_lines

    def close(self):
        if self.h:
            self.lib.emu_destroy(self.h)
            self.h = None

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
              "chain": self.lib.emu_process_stream_chain}[self.variant]
        rc = fn(self.h, msg, len(msg), n_train, flags.ctypes.data, scores.ctypes.data, cap,
                                  C.byref(n_lines), C.byref(n_anom), C.byref(err))
        assert rc == 0 and err.value == 0, (rc, err.value)
        self.last_n_anomalies = n_anom.value
        return flags[:n_lines.value], scores[:n_lines.value]

    def anomalies(self):
        arr = (Anomaly * 65536)()
        n = self.lib.emu_get_anomalies(self.h, arr, 65536)
        return [(arr[i].line, arr[i].mask, arr[i].offset) for i in range(n)]

    def stats(self):
        w = (C.c_uint64 * 40)()
        self.lib.emu_get_stats(self.h, w)
        return {"lines": w[0], "train_lines": w[1], "detect_lines": w[2], "anomalies": w[3], "score_sum": w[4],
                "bytes": w[5], "known_keys": w[6], "bad_records": w[7], "unknown_per_key": [w[8 + i] for i in range(len(self.keys))]}

    def export_known(self):
        out = (C.c_uint64 * (1 << 16))()
        n = self.lib.emu_export_known(self.h, out, 1 << 16)
        return [out[i] for i in range(n)]
