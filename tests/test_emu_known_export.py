"""dm_export_known's device kernels (compaction of the table's slots, LSD radix sort of the keys) on the CPU emulator,
against numpy.sort of the table's non-zero slots.  tests/emu/emu_known.cpp runs them, built here into its own
library."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from emu_harness import CSRC, EMU, ROOT

SO = os.path.join(EMU, "_build", "libemu_known.so")
_P64 = C.POINTER(C.c_uint64)


@pytest.fixture(scope="module")
def lib():
    srcs = [os.path.join(EMU, "emu_known.cpp"), os.path.join(EMU, "cuda_emu.h"),
            os.path.join(ROOT, "include", "dmdetect.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not (os.path.exists(SO) and all(os.path.getmtime(s) <= os.path.getmtime(SO) for s in srcs)):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-DDM_EMU", "-I" + EMU, "-I" + CSRC, "-shared",
                               "-fPIC", "-pthread", "-o", SO, os.path.join(EMU, "emu_known.cpp")])
    L = C.CDLL(SO)
    for name, res, args in (("emu_known_create", C.c_void_p, [C.c_uint32]),
                            ("emu_known_destroy", None, [C.c_void_p]),
                            ("emu_known_insert", C.c_uint32, [C.c_void_p, _P64, C.c_uint64]),
                            ("emu_known_count", C.c_uint64, [C.c_void_p]),
                            ("emu_known_export", C.c_uint64, [C.c_void_p, _P64, C.c_uint64, C.POINTER(C.c_uint32)])):
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    return L


class Table:
    """An emulated known-set table of 2^log2 slots."""

    def __init__(self, L, log2):
        self.L, self.log2, self.h = L, log2, L.emu_known_create(log2)

    def __del__(self):
        self.L.emu_known_destroy(self.h)

    def insert(self, keys):
        a = np.ascontiguousarray(keys, dtype=np.uint64)
        return self.L.emu_known_insert(self.h, a.ctypes.data_as(_P64), a.size) if a.size else 0

    def count(self):
        return int(self.L.emu_known_count(self.h))

    def export(self, cap=None):
        """(the keys copied, their count, the radix passes run); cap defaults to the table's slots."""
        cap = (1 << self.log2) if cap is None else cap
        out = np.zeros(max(1, cap), dtype=np.uint64)
        passes = C.c_uint32()
        n = self.L.emu_known_export(self.h, out.ctypes.data_as(_P64), cap, C.byref(passes))
        assert n != (1 << 64) - 1, "the compaction's count disagrees with the table's"
        return out[:min(n, cap)], int(n), passes.value


def _table(L, log2, keys):
    t = Table(L, log2)
    return t, t.insert(keys)


def _random_keys(rng, n, top_bit=None):
    k = np.unique(rng.integers(1, 2**64 - 1, size=n + 64, dtype=np.uint64, endpoint=True))
    if top_bit is True:
        k = np.unique(k | np.uint64(1 << 63))
    k = k[k != 0]
    rng.shuffle(k)
    return k[:n]


def _check(d, keys):
    got, n, passes = d.export()
    want = np.sort(np.asarray(keys, dtype=np.uint64))
    assert n == want.size == d.count()
    assert got.dtype == np.uint64 and np.array_equal(got, want)
    assert np.all(got[1:] > got[:-1])
    return passes


def test_empty_table_copies_nothing(lib):
    d, _ = _table(lib, 10, [])
    got, n, passes = d.export()
    assert n == 0 and got.size == 0 and passes == 0


def test_one_key(lib):
    d, _ = _table(lib, 10, [0xFEDCBA9876543210])
    assert _check(d, [0xFEDCBA9876543210]) == 0          # one key: every digit is shared, no pass runs


@pytest.mark.parametrize("top_bit", [None, True])
def test_half_load_limit(lib, top_bit):
    rng = np.random.default_rng(7 if top_bit else 8)
    keys = _random_keys(rng, 1 << 11, top_bit)           # 2^12 slots at their 1/2 load limit
    d, err = _table(lib, 12, keys)
    assert err == 0
    assert _check(d, keys) == 8


def test_keys_either_side_of_the_top_bit(lib):
    keys = [1, 2, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, 2**64 - 1, 2**64 - 2, 0x8000000000000100, 0x00000000000000FF]
    d, _ = _table(lib, 10, keys)
    _check(d, keys)


def test_more_keys_than_a_tile_and_more_slots_than_the_grid_has_threads(lib):
    # 2^14 slots: the compaction's 2 CTAs stride over 4 tiles of slots; 8192 keys make 2 sort tiles
    rng = np.random.default_rng(9)
    keys = _random_keys(rng, 1 << 13)
    d, err = _table(lib, 14, keys)
    assert err == 0
    assert _check(d, keys) == 8


def test_shared_digits_skip_their_passes(lib):
    # keys differ in bits 8..23 only: the six other digits are the same for every key
    keys = [0xAB00000000000055 | (i << 8) for i in range(1, 3000)]
    d, _ = _table(lib, 13, keys)
    assert _check(d, keys) == 2


def test_cap_below_the_count_copies_the_smallest(lib):
    rng = np.random.default_rng(10)
    keys = _random_keys(rng, 1000)
    d, _ = _table(lib, 11, keys)
    got, n, _ = d.export(cap=100)
    assert n == 1000 and np.array_equal(got, np.sort(keys)[:100])
    got, n, passes = d.export(cap=0)
    assert n == 1000 and got.size == 0 and passes == 0


def test_table_past_its_load_limit(lib):
    # an insert past the limit reports DM_DEVERR_TABLE_FULL but keeps the key: the export still returns every key
    rng = np.random.default_rng(11)
    keys = _random_keys(rng, 700)
    d, err = _table(lib, 10, keys)
    assert err & 1
    _check(d, keys)
