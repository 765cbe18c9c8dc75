"""Build and load libdmdetect.so (the sm_90a CUDA library behind include/dmdetect.h).

There is no CPU fallback: if the library is missing or cannot be loaded this module
raises, and every compute entry point of the library itself fails without a CUDA device
(``DM_ERR_NO_DEVICE``).
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
from typing import List

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
SO_PATH = os.environ.get("DM_LIB_PATH") or os.path.join(PKG_DIR, "libdmdetect.so")   # (DM_LIB_PATH: A/B builds side by side)
HEADER = os.path.join(os.path.dirname(PKG_DIR), "include", "dmdetect.h")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]

DM_MAX_KEYS = 32
DM_MAX_KEYLEN = 32
DM_OK = 0
DM_ERR_ARG, DM_ERR_CUDA, DM_ERR_NO_DEVICE, DM_ERR_CAPACITY, DM_ERR_TABLE_FULL, DM_ERR_STATE = -1, -2, -3, -4, -5, -6


class DmError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"libdmdetect error {code}: {message}")
        self.code = code


def _sources() -> List[str]:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))) + [HEADER]


def needs_build() -> bool:
    if os.environ.get("DM_LIB_PATH"):
        return False                                              # a hand-built variant: never rebuilt behind the user's back
    if not os.path.exists(SO_PATH):
        return True
    so_m = os.path.getmtime(SO_PATH)
    return any(os.path.exists(s) and os.path.getmtime(s) > so_m for s in _sources())


def build(force: bool = False, verbose: bool = False) -> str:
    """nvcc -gencode arch=compute_90a,code=sm_90a ... -> detectmateservice_b200/libdmdetect.so
    (in-tree, so the built library travels with the repo snapshot)."""
    if not force and not needs_build():
        return SO_PATH
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libdmdetect.so (no CPU fallback exists)")
    extra = os.environ.get("DM_NVCC_EXTRA", "").split()          # development knob (e.g. -DDMX_MIN_CTAS=3)
    cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + [
        "-o", SO_PATH, os.path.join(CSRC, "dmdetect.cu")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return SO_PATH


class Stats(C.Structure):
    _fields_ = [("lines", C.c_uint64), ("train_lines", C.c_uint64), ("detect_lines", C.c_uint64),
                ("anomalies", C.c_uint64), ("score_sum", C.c_uint64), ("bytes", C.c_uint64),
                ("known_keys", C.c_uint64), ("bad_records", C.c_uint64), ("unknown_per_key", C.c_uint64 * DM_MAX_KEYS)]

    def as_dict(self, n_keys: int = DM_MAX_KEYS) -> dict:
        return {"lines": self.lines, "train_lines": self.train_lines, "detect_lines": self.detect_lines,
                "anomalies": self.anomalies, "score_sum": self.score_sum, "bytes": self.bytes,
                "known_keys": self.known_keys, "bad_records": self.bad_records, "unknown_per_key": list(self.unknown_per_key)[:n_keys]}


class Monitor(C.Structure):
    _fields_ = [("event_id", C.c_int32), ("has_event", C.c_uint32), ("source", C.c_uint32), ("var_index", C.c_uint32),
                ("key_len", C.c_uint32), ("key", C.c_uint8 * 64)]


class Anomaly(C.Structure):
    _fields_ = [("line", C.c_uint32), ("mask", C.c_uint32), ("offset", C.c_uint64)]


# every symbol include/dmdetect.h declares: name -> (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "dm_last_error": (C.c_char_p, []),
    "dm_abi_version": (C.c_int, []),
    "dm_create": (C.c_int, [C.c_int, C.c_uint32, C.c_char_p, C.POINTER(C.c_uint32), C.c_uint64, C.c_uint64,
                            C.c_uint32, C.POINTER(_P)]),
    "dm_destroy": (C.c_int, [_P]),
    "dm_process_lines": (C.c_int, [_P, _P, C.c_uint64, C.c_int, C.c_uint64, _P, _P, C.c_uint64, C.c_int,
                                   C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), _P]),
    "dm_process_values": (C.c_int, [_P, C.c_char_p, C.c_uint64, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                    C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64,
                                    _P, _P, _P, C.POINTER(C.c_uint64)]),
    "dm_set_monitors": (C.c_int, [_P, C.c_uint32, C.POINTER(Monitor)]),
    "dm_set_combos": (C.c_int, [_P, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_uint32]),
    "dm_host_cache_flush": (C.c_int, [_P, C.c_uint64]),
    "dm_debug_rows_timeline": (C.c_int, [_P, C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint32)]),
    "dm_set_format": (C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_char_p)]),
    "dm_stream_recheck_chained": (C.c_int, [_P]),
    "dm_set_format_ex": (C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_char_p), C.c_uint32]),
    "dm_process_records": (C.c_int, [_P, C.c_char_p, C.c_uint64, C.c_uint32, _P, _P, _P, C.c_uint64,
                                     C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "dm_submit_lines": (C.c_int, [_P, _P, C.c_uint64, C.c_uint64, C.c_uint32]),
    "dm_collect": (C.c_int, [_P, C.c_uint32, C.POINTER(_P), C.POINTER(_P), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "dm_collect_anomalies": (C.c_int, [_P, C.c_uint32, C.POINTER(Anomaly), C.c_uint32, C.POINTER(C.c_uint32)]),
    "dm_sync": (C.c_int, [_P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "dm_get_anomalies": (C.c_int, [_P, C.POINTER(Anomaly), C.c_uint32, C.POINTER(C.c_uint32)]),
    "dm_get_stats": (C.c_int, [_P, C.POINTER(Stats)]),
    "dm_export_known": (C.c_int, [_P, C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint64)]),
    "dm_import_known": (C.c_int, [_P, C.POINTER(C.c_uint64), C.c_uint64]),
    "dm_reset": (C.c_int, [_P]),
    "dm_table_key": (C.c_uint64, [C.c_uint32, C.c_char_p, C.c_uint32]),
    "dm_window_words": (C.c_uint64, [_P, C.c_uint32, C.c_int]),
    "dm_window_export": (C.c_int, [_P, _P, C.c_uint32, C.c_uint32, C.c_int, _P]),
    "dm_window_import": (C.c_int, [_P, _P, C.c_uint32, C.c_uint32, C.c_int, _P]),
    "dm_nccl_unique_id": (C.c_int, [C.c_char_p]),
    "dm_nccl_init": (C.c_int, [_P, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32]),
    "dm_window_allreduce": (C.c_int, [_P, C.c_int, _P]),
    "dm_get_global_stats": (C.c_int, [_P, C.POINTER(Stats)]),
    "dm_profile_enable": (C.c_int, [_P, C.c_int]),
    "dm_set_overlap": (C.c_int, [_P, C.c_int]),
    "dm_window_pending_keys": (C.c_int, [_P, C.POINTER(C.c_uint64)]),
    "dm_profile_read": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
}

_lib = None


def load() -> C.CDLL:
    """Load the library (building it first if the sources are newer).  Raises if it
    cannot be built or loaded -- the product has no other implementation."""
    global _lib
    if _lib is not None:
        return _lib
    if needs_build():
        build()
    lib = C.CDLL(SO_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)          # AttributeError if the ABI lost a symbol
        fn.restype = res
        fn.argtypes = args
    if lib.dm_abi_version() != 4:
        raise RuntimeError(f"libdmdetect ABI version {lib.dm_abi_version()} != 4")
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != DM_OK:
        raise DmError(rc, load().dm_last_error().decode("utf-8", "replace"))
