"""The key=value kernels' SOURCES (dm_kernels_stream.cuh, dm_kernels_lanes.cuh), compiled for the CPU emulator in
tests/emu, against the oracle.  Runs in the CPU tier; the same cases run on the H100
through the C ABI in test_gpu_parity.py.  (Emulation is test infrastructure: one thread
block on OS threads -- it checks logic, not memory-model or multi-CTA behaviour.)
"""
import json
import os

import numpy as np
import pytest

import emu_harness
from oracle import fingerprint
from oracle.native import NativeOracle
import util
from util import FUZZ_KEYS, FUZZ_KEYS_FEW, fuzz_lines, lookalike_lines


@pytest.fixture(params=["stream", "chain", "lanes"], autouse=True)
def emu_variant(request):
    """Every test runs against the key=value kernels: stream (DM_KERNEL=stream; both of its instantiations, candidates
    re-checked one by one = "stream" and batch-wise = "chain") and lanes."""
    global VARIANT
    VARIANT = request.param
    return request.param


VARIANT = "stream"


def EmuDetector(keys, **kw):
    return emu_harness.EmuDetector(keys, variant=VARIANT, **kw)


def _default_variant_only():
    """The chained instantiation differs from "stream" only in how candidates are re-checked: it skips the tests
    that hold few candidates (the CPU tier has to stay within minutes)."""
    if VARIANT == "chain":
        pytest.skip("covered by the stream variant; the chained re-check has its own tests")


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
    assert det.last_n_anomalies == int(of.sum())
    return f, s


def test_emu_audit_sample_golden(golden_dir):
    exp = json.load(open(os.path.join(golden_dir, "audit_sample.expected.json")))
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read()
    det = EmuDetector(exp["keys"])
    f, s = det.process_lines(buf, exp["n_train"])
    assert f.tolist() == exp["flags"] and s.tolist() == exp["scores"]
    assert [a[1] for a in det.anomalies()] == [m for m in exp["masks"] if m]
    st = det.stats()
    assert st["lines"] == exp["n_records"] and st["train_lines"] == exp["n_train"]
    assert st["anomalies"] == sum(exp["flags"]) and st["score_sum"] == int(sum(exp["scores"]))
    assert st["known_keys"] == sum(exp["known_counts"]) and st["bytes"] == len(buf)
    det.close()


@pytest.mark.parametrize("seed,keys", [(1, FUZZ_KEYS), (2, FUZZ_KEYS_FEW)])
def test_emu_fuzz_tokenizer(seed, keys):
    FUZZ_KEYS = keys
    o = NativeOracle(FUZZ_KEYS)
    det = EmuDetector(FUZZ_KEYS)
    _check(det, o, fuzz_lines(seed, 1500), 600)
    _check(det, o, fuzz_lines(seed + 100, 1500), 0)
    want = sorted(fingerprint.table_key(i, v) for i in range(len(FUZZ_KEYS)) for v in o.known_values(i))
    assert det.export_known() == want
    det.close()


def test_emu_edge_cases():
    keys = [b"k", b"type", b"longer_key_name_0123456789abcdef"]
    cases = [
        b"", b"\n", b"\n\n\n", b"type=A", b"type=A\ntype=B", b"k=1 k=2\n", b"type=\n", b"=x k=\n",
        b"x" * 5000 + b" k=v\n", b"k=" + b"v" * 5000 + b"\n", b'q="a b k=1" k=2\n', b'q="unbalanced k=1\nk=1\n',
        b"longer_key_name_0123456789abcdef=1 xlonger_key_name_0123456789abcdef=2\n", b"a'k=5 b'type=Z\n",
        b" k=1\n  k=2\n", b"k=1\n" * 1000, (b"y" * 126 + b" k=edge\n") * 50, (b"y" * 123 + b" type=edge\n") * 50,
        b" k=" * 600 + b"\n" + b"=" * 700 + b"\n" + b"k=2 " * 300 + b"\n",   # rows dense in '=' (queue overflow path)
        b"k=2",                                            # '=' at position 1 (q < 4), no newline
        b"k=9\n" + b"z" * 4090 + b"\nk=3\n",               # record starting exactly at a segment boundary
        b"z" * 4095 + b"\nk=4\n",                          # newline as the last byte of a segment
        b"z" * 4094 + b"\nk=5\n",
        (b"w" * 37 + b"\n") * 900 + b"k=6",                # tail record without newline after many tiles
        b"k=7 " + b"m" * 40000 + b" type=Q\n" + b"k=8\n",  # one record spanning more than a tile
        b"\n" * 5000 + b"k=10\n",                          # thousands of empty records
    ]
    o = NativeOracle(keys)
    det = EmuDetector(keys)
    _check(det, o, b"k=1\ntype=A\nk=v\n", 3)
    for c in cases:
        _check(det, o, c, 0)
    # training values that need the exact re-check: duplicates and quoted look-alikes
    o2 = NativeOracle(keys)
    det2 = EmuDetector(keys)
    train = b'k=first k=second\nq="x k=inquote" k=real\ntype=T type=U\n'
    _check(det2, o2, train, 3)
    _check(det2, o2, b"k=second\nk=inquote\nk=first\nk=real\ntype=U\ntype=T\n", 0)
    det.close()
    det2.close()
    # '<' right behind an '=': the stream kernel's '=' mask flags such bytes too (dmx_eq_bits); they must never turn into
    # fields, not even with keys made of '<'
    keys3 = [b"<", b"<<", b"k", b"a<<"]
    o3 = NativeOracle(keys3)
    det3 = EmuDetector(keys3)
    _check(det3, o3, b"k=<1 <=2 <<=3 a<<=4\n", 1)
    for c in [b"k=<< <=<\n", b"k==< <<=<< a<<=<<<\n", b"x=<=5 =<<=6 k=<<<<=7\n", b"<=<=<=< k=<\n" * 40,
              b"a<<=<<< a<<=1\n", b"'<=9 '<<=9 'a<<=9\n", b"=<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<<=1 <=u\n"]:
        _check(det3, o3, c, 0)
    det3.close()
    # 0x0B right behind a newline (the loose newline test's only false positive), runs of newlines, 0x0B alone
    o4 = NativeOracle(keys)
    det4 = EmuDetector(keys)
    _check(det4, o4, b"k=1\ntype=A\n", 2)
    for c in [b"k=2\n\x0bk=3\n\x0b\x0b\x0bk=4\n", b"\x0b\x0b\x0b\n\x0bk=5\x0b\n\n\n\x0b\n", (b"k=7\n\x0b" * 700), b"\n\x0b" * 3000 + b"k=9\n",
              b"type=B\x0b\nk=\x0b\n"]:
        _check(det4, o4, c, 0)
    det4.close()


def test_emu_synthetic_and_split():
    _default_variant_only()
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    g = AuditSynth(seed=5)
    a, _ = g.batch(1500, inject=False)
    b, inj = g.batch(2500, inject=True)
    keys = [k.encode() for k in MONITORED_KEYS]
    o = NativeOracle(keys)
    det = EmuDetector(keys)
    _check(det, o, a + b, 1500)
    f, _ = _check(det, o, b, 0)
    assert f.sum() >= inj.sum() > 0
    st = det.stats()
    assert st["unknown_per_key"] == [o.unknown_count(i) for i in range(len(keys))]
    assert st["lines"] == 4000 + 2500 and st["train_lines"] == 1500
    if VARIANT != "lanes":
        hint = det.lib.emu_stream_hint()
        assert (hint >> 32) * 4 < (hint & 0xFFFFFFFF), hint              # rare anomalies: the host stays with the one-by-one re-check
    det.close()


def test_emu_varlen():
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    g = AuditSynth(seed=20260924)
    n1, n2 = (700, 1100) if VARIANT == "chain" else (1500, 2500)      # (the emulated chain path is slow)
    train, _ = g.batch_varlen(n1, inject=False)
    g.anomaly_rate = 0.02
    msg, _ = g.batch_varlen(n2, inject=True)
    keys = [k.encode() for k in MONITORED_KEYS]
    o = NativeOracle(keys)
    det = EmuDetector(keys)
    _check(det, o, train, n1)
    f, _ = _check(det, o, msg, 0)
    assert f.sum() > 5
    det.close()


@pytest.mark.parametrize("seed", [11])
def test_emu_lookalikes_and_duplicates(seed):
    """Long records with dozens of candidates each: quoted look-alikes, duplicates, parity flips (the chained
    re-check of the stream kernel and its fall-backs)."""
    keys = [b"key", b"type", b"res"]
    o = NativeOracle(keys)
    det = EmuDetector(keys)
    _check(det, o, lookalike_lines(seed, 200), 80)
    import ctypes as C
    lib = det.lib
    st = (C.c_uint64 * 8)()
    lib.emu_chain_stats(st, 1)
    f, _ = _check(det, o, lookalike_lines(seed + 50, 300), 0)
    assert 20 < f.sum() < f.size
    if VARIANT == "chain":
        lib.emu_chain_stats(st, 1)
        chain, fallback, unordered = st[0], st[1], st[2]
        assert chain > 10 * fallback and chain > 600 and unordered > 0, (chain, fallback, unordered)
    if VARIANT != "lanes":
        # many short warp segments (the GPU's geometry: a few rows per warp): nearly every batch starts without carried state
        for ctas in (40, 150):
            lib.emu_stream_ctas(ctas)
            try:
                _check(det, o, lookalike_lines(seed + 70 + ctas, 150), 0)
            finally:
                lib.emu_stream_ctas(3)
        _check(det, o, lookalike_lines(seed + 50, 300), 0)
        # what the host's choice of instantiation rests on: most batches of this message held a candidate
        hint = lib.emu_stream_hint()
        rows, slow = hint & 0xFFFFFFFF, hint >> 32
        assert rows > 100 and slow * 4 >= rows, (rows, slow)
    det.close()


def test_emu_everything_unknown():
    """No training at all: every monitored field alerts (stresses the pending-alert flush)."""
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    g = AuditSynth(seed=3)
    msg, _ = g.batch(1200, inject=False)
    keys = [k.encode() for k in MONITORED_KEYS]
    o = NativeOracle(keys)
    det = EmuDetector(keys)
    f, s = _check(det, o, msg, 0)
    assert f.all() and (s == 5).all()
    det.close()


def test_emu_byte_position_sweep():
    """'=' on every residue mod 32 and at the 1 KiB row edges, the first '=' at bytes 1-4, values ending before, at and
    behind the 32-byte window and the 64 bytes behind a row, quoted spaces around the window's end, messages ending
    inside a value for every nbytes % 16; about half of the values learnt.  Stream variants also with many short warp
    segments (40 CTAs)."""
    train, _ = util.sweep_training(0)
    msgs = util.sweep_messages(0)
    o = NativeOracle(util.SWEEP_KEYS)
    det = EmuDetector(util.SWEEP_KEYS)
    _check(det, o, train, train.count(b"\n"))
    alerts = 0
    for m in msgs:
        f, _ = _check(det, o, m, 0)
        alerts += int(f.sum())
    assert alerts > len(msgs) // 2
    if VARIANT != "lanes":
        lib = det.lib
        lib.emu_stream_ctas(40)
        try:
            for m in msgs:
                _check(det, o, m, 0)
        finally:
            lib.emu_stream_ctas(3)
    det.close()


def test_emu_keys32():
    """One key of every length 1..32 (last four bytes shared along a chain, a suffix key, a byte >= 0x80): records
    with all 32 fields and look-alikes; then nothing learnt: mask 0xFFFFFFFF and score 32."""
    keys = util.KEYS32
    assert sorted(len(k) for k in keys) == list(range(1, 33))
    train, known = util.keys32_training(1)
    o = NativeOracle(keys)
    det = EmuDetector(keys)
    _check(det, o, train, train.count(b"\n"))
    f, _ = _check(det, o, util.keys32_lines(2, 60, known=known), 0)
    assert 0 < f.sum() < f.size
    det.close()
    o2 = NativeOracle(keys)
    det2 = EmuDetector(keys)
    msg = util.keys32_lines(3, 12)
    f, s = _check(det2, o2, msg, 0)
    assert f.all() and (s == 32).all()
    assert {a[1] for a in det2.anomalies()} == {0xFFFFFFFF}
    st = det2.stats()
    assert st["unknown_per_key"] == [12] * 32 and st["score_sum"] == 12 * 32
    det2.close()


def test_emu_keys32_three_byte_level1_table():
    """32 distinct 3-byte keys: 96 level-1 patterns, the 512-slot table."""
    _default_variant_only()
    keys = util.KEYS32_3BYTE
    train, known = util.keys32_training(4, keys=keys)
    o = NativeOracle(keys)
    det = EmuDetector(keys)
    _check(det, o, train, train.count(b"\n"))
    f, _ = _check(det, o, util.keys32_lines(5, 40, keys=keys, known=known), 0)
    assert 0 < f.sum() < f.size
    det.close()


def test_emu_train_detect_split_sweep():
    """Every split point of a ~3 KB message of 40 records (several 512-byte rows of dm_k_bound, no newline at the
    end), each with a fresh detector."""
    _default_variant_only()
    keys = [b"type", b"res", b"acct"]
    msg = util.split_message(6)
    n = msg.count(b"\n") + 1
    assert len(msg) > 4 * 512 and n == 40
    for n_train in range(n + 3):
        o = NativeOracle(keys)
        det = EmuDetector(keys)
        _check(det, o, msg, n_train)
        st = det.stats()
        assert st["train_lines"] == min(n_train, n) and st["lines"] == n
        assert st["unknown_per_key"] == [o.unknown_count(i) for i in range(len(keys))]
        assert st["known_keys"] == sum(o.known_count(i) for i in range(len(keys)))
        det.close()


def test_emu_train_detect_split_per_group():
    """More than 256 rows of 512 bytes: dm_k_bound finds the split through its per-thread groups of rows; n_train at
    records that hold a group edge."""
    _default_variant_only()
    keys = [b"type", b"res", b"acct"]
    msg = util.split_message(7, n_records=2000, mean_len=90)
    rows = (len(msg) + 511) // 512
    assert rows > 256
    per = (rows + 255) // 256
    arr = np.frombuffer(msg, dtype=np.uint8)
    nl = np.nonzero(arr == 10)[0]
    for grp in (1, 2, 100, 255):
        edge = grp * per * 512
        rec = int(np.searchsorted(nl, edge))                           # the record holding byte `edge`
        for n_train in (rec - 1, rec, rec + 1):
            o = NativeOracle(keys)
            det = EmuDetector(keys)
            _check(det, o, msg, n_train)
            det.close()


def test_emu_shared_output_buffer():
    """One caller-owned output buffer, pre-filled with 7 / -1 once, through messages whose record counts grow and shrink
    across the 4-set rotation: the zero-fill bound left by the call four back, the epilogue's rest and its take-out of
    the previous call's alerts."""
    keys = [b"type", b"res", b"acct"]
    msgs = [util.split_message(s, n_records=n) for s, n in
            [(10, 300), (11, 5), (12, 1), (13, 250), (14, 40), (15, 400), (16, 2), (17, 350), (18, 30), (19, 120)]]
    msgs.insert(3, b"")
    msgs.insert(6, b"\n")
    o = NativeOracle(keys)
    det = EmuDetector(keys)
    flags = np.full(512, 7, dtype=np.uint8)
    scores = np.full(512, -1, dtype=np.float32)
    _check(det, o, msgs[0], 200)
    for m in msgs[1:]:
        f, s = det.process_lines(m, 0, out=(flags, scores))
        wf, ws, _ = o.process(m, 0)
        assert f.tolist() == wf.tolist() and s.tolist() == ws.tolist()
    det.close()
