"""The stream kernel's level-1 lookup rounds (dm_kernels_stream.cuh, CPU emulator) against the oracle.

A row's '=' are ranked across the warp in message order and looked up DMX_ROUND (128) ranks per round, 32 per slot:
rows with 33-64 '=' take two slots, 65-128 three or four, more than 128 several rounds with the field queue drained
in between.  The messages here are built to hold each of those rows, a row made only of '=', rows in which every
32-byte lane holds five '=' or more, and a dense partial last row; quoted look-alikes and repeated keys make the
re-check (one by one, and chained) decide many candidates.
"""
import random

import numpy as np
import pytest

import emu_harness
from oracle.native import NativeOracle

KEYS = [b"k", b"type", b"acct"]
ROW = 1024


def _record(rng, field_bytes, n_fields):
    """One record of n_fields fields of about field_bytes bytes each (separator included)."""
    out = []
    for _ in range(n_fields):
        key = rng.choice([b"k", b"type", b"acct", b"x", b"zz"])
        val = b"%d" % rng.randrange(5)
        r = rng.random()
        if r < 0.06:
            f = b'q="w ' + key + b"=" + val + b'"'               # look-alike inside double quotes
        elif r < 0.08:
            f = b"'" + key + b"=" + val                          # field start after a quote delimiter
        else:
            f = key + b"=" + val
        pad = field_bytes - 1 - len(f)
        if pad > 0:
            f += b"p" * pad                                      # lengthens the value
        out.append(f)
    return b" ".join(out) + b"\n"


def _message(seed, tail=True):
    rng = random.Random(seed)
    parts = []
    for field_bytes, nbytes in [(18, 3 * ROW), (10, 3 * ROW), (4, 3 * ROW), (7, 2 * ROW), (3, 2 * ROW), (24, 2 * ROW)]:
        seg = b""
        while len(seg) < nbytes:
            seg += _record(rng, field_bytes, rng.randrange(8, 60))
        parts.append(seg)
    parts.append(b"k=" + b"=" * (2 * ROW + 100) + b" type=1\n")         # holds a whole row of '='
    parts.append(b"k=" * 700 + b"1\n")                                  # '=' every other byte
    if tail:
        want = ROW - sum(len(p) for p in parts) % ROW + 900
        seg = b""
        while len(seg) < want:
            seg += _record(rng, 4, rng.randrange(8, 40))
        parts.append(seg[:want])                                        # ends 900 bytes into a dense row, inside a record
    return b"".join(parts)


def _row_classes(msg):
    """'=' per 1 KiB row and the fewest '=' of any 32-byte lane of it."""
    arr = np.frombuffer(msg, dtype=np.uint8)
    n_rows = (arr.size + ROW - 1) // ROW
    pad = np.zeros(n_rows * ROW, dtype=np.uint8)
    pad[:arr.size] = arr
    eq = (pad == ord("=")).reshape(n_rows, ROW // 32, 32).sum(axis=2)
    return eq.sum(axis=1), eq.min(axis=1)


def _check(det, oracle, msg, n_train):
    f, s = det.process_lines(msg, n_train)
    of, os_, om = oracle.process(msg, n_train, want_masks=True)
    assert f.shape == of.shape, (f.shape, of.shape)
    bad = np.nonzero(f != of)[0]
    assert bad.size == 0, f"flags differ at records {bad[:10]} (emu {f[bad[:10]]}, oracle {of[bad[:10]]})"
    assert (s == os_).all()
    an = det.anomalies()
    idx = np.nonzero(of)[0]
    assert [a[0] for a in an] == idx.tolist()
    assert [a[1] for a in an] == om[idx].tolist()
    arr = np.frombuffer(msg, dtype=np.uint8)
    starts = np.concatenate([[0], np.nonzero(arr == 10)[0] + 1])
    assert [a[2] for a in an] == starts[idx].tolist()
    return f


def test_messages_hold_every_round_shape():
    for seed in (1, 2):
        msg = _message(seed)
        per_row, lane_min = _row_classes(msg)
        assert ((per_row >= 33) & (per_row <= 64)).any()
        assert ((per_row >= 65) & (per_row <= 128)).any()
        assert (per_row > 128).any()
        assert (per_row == ROW).any()                                   # a row made only of '='
        assert (lane_min >= 5).sum() >= 3                               # every lane with five or more
        assert len(msg) % ROW and per_row[-1] > 128                     # a dense partial last row


@pytest.mark.parametrize("variant", ["stream", "chain"])
def test_emu_lookup_rounds(variant):
    o = NativeOracle(KEYS)
    det = emu_harness.EmuDetector(KEYS, variant=variant)
    train = _message(1)
    _check(det, o, train, train.count(b"\n") // 2)
    f = _check(det, o, _message(2), 0)
    assert 0 < f.sum() < f.size
    _check(det, o, _message(3, tail=False), 0)
    lib = det.lib
    lib.emu_stream_ctas(40)                                             # a few rows per warp
    try:
        _check(det, o, _message(4), 0)
    finally:
        lib.emu_stream_ctas(3)
    det.close()
