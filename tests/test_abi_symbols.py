"""The C-ABI library builds, loads and exports every symbol include/dmdetect.h declares.
No compute calls here (there is no GPU in the build container)."""
import ctypes as C
import os
import re

import pytest

from detectmateservice_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "dmdetect.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dm_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_all_exported():
    lib = _lib.load()
    names = _declared_symbols()
    assert len(names) >= 16
    for n in names:
        assert hasattr(lib, n), f"{n} declared in dmdetect.h but not exported"
        assert n in _lib.SYMBOLS, f"{n} has no ctypes prototype"
    assert set(_lib.SYMBOLS) == set(names)
    assert lib.dm_abi_version() == 4


def test_sass_is_sm90a_only():
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", _lib.SO_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out and "sm_80" not in out


def test_host_side_table_key_matches_spec():
    """dm_table_key is a pure host function (no device): it must follow DESIGN.md's dm_fp64."""
    from oracle import fingerprint
    lib = _lib.load()
    for f, v in [(0, b""), (0, b"USER_ACCT"), (1, b'"/usr/sbin/cron"'), (4, b"success'"), (31, bytes(range(200)))]:
        assert lib.dm_table_key(f, v, len(v)) == fingerprint.table_key(f, v)


def test_create_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    lib = _lib.load()
    h = C.c_void_p()
    lens = (C.c_uint32 * 1)(4)
    rc = lib.dm_create(0, 1, b"type", lens, 1 << 20, 0, 16, C.byref(h))
    assert rc == _lib.DM_ERR_NO_DEVICE and not h.value
    assert b"no CPU path" in lib.dm_last_error()
    from detectmateservice_b200.detector import DeviceDetector
    with pytest.raises(_lib.DmError):
        DeviceDetector(["type"])


def test_bad_arguments_rejected_before_touching_device():
    lib = _lib.load()
    h = C.c_void_p()
    lens = (C.c_uint32 * 1)(4)
    assert lib.dm_create(0, 1, b"type", lens, 0, 0, 16, C.byref(h)) == _lib.DM_ERR_ARG
    assert lib.dm_create(0, 1, b"type", lens, 1 << 20, 0, 5, C.byref(h)) == _lib.DM_ERR_ARG
    assert lib.dm_create(0, 40, b"type", lens, 1 << 20, 0, 16, C.byref(h)) == _lib.DM_ERR_ARG
    assert lib.dm_process_lines(None, None, 0, 0, 0, None, None, 0, 0, None, None, None) == _lib.DM_ERR_ARG


def test_host_cache_flush_is_harmless():
    """dm_host_cache_flush is a host-only utility (clflush): contents are unchanged."""
    import numpy as np
    from detectmateservice_b200 import _lib
    a = np.arange(1 << 16, dtype=np.uint8).copy()
    before = a.copy()
    assert _lib.load().dm_host_cache_flush(a.ctypes.data + 3, a.size - 7) == 0      # unaligned start / length
    assert (a == before).all()
    assert _lib.load().dm_host_cache_flush(None, 0) == 0
