"""Parity of the CUDA path (through the C ABI) with the oracle.  Needs an H100.

Bars: flags bit-exact; scores within 1e-5 (they are small integers, so in practice exact);
unknown-field masks, anomaly lists and statistics exact; learnt key sets equal to the
oracle's known strings mapped through dm_fp64.
"""
import json
import os

import numpy as np
import pytest

from oracle import fingerprint
from oracle.native import NativeOracle
from util import FUZZ_KEYS, FUZZ_KEYS_FEW, fuzz_lines

pytestmark = pytest.mark.gpu

# stream = the default kernel with candidates re-checked one by one, chain = the same kernel's batch-wise re-check
# (DM_STREAM_RECHECK; left alone the library picks per message), lanes = one thread per record
VARIANTS = ["stream", "chain", "lanes"]
SCORE_TOL = 1e-5


@pytest.fixture(params=VARIANTS)
def variant(request, monkeypatch):
    monkeypatch.setenv("DM_KERNEL", "lanes" if request.param == "lanes" else "stream")
    if request.param != "lanes":
        monkeypatch.setenv("DM_STREAM_RECHECK", "chain" if request.param == "chain" else "thread")
    return request.param


def _det(keys, **kw):
    from detectmateservice_b200.detector import DeviceDetector
    kw.setdefault("max_batch_bytes", 32 << 20)
    kw.setdefault("table_log2_slots", 16)
    return DeviceDetector(keys, **kw)


def _check(det, oracle, msg, n_train, check_masks=True):
    f, s = det.process_lines(msg, n_train)
    of, os_, om = oracle.process(msg, n_train, want_masks=True)
    assert f.shape == of.shape, (f.shape, of.shape)
    bad = np.nonzero(f != of)[0]
    assert bad.size == 0, f"flags differ at records {bad[:10]} (gpu {f[bad[:10]]}, oracle {of[bad[:10]]})"
    assert np.max(np.abs(s - os_), initial=0.0) <= SCORE_TOL
    if check_masks:
        an = det.anomalies()
        idx = np.nonzero(of)[0]
        assert [a[0] for a in an] == idx.tolist()
        assert [a[1] for a in an] == om[idx].tolist()
        # offsets point at the record starts
        arr = np.frombuffer(msg, dtype=np.uint8)
        starts = np.concatenate([[0], np.nonzero(arr == 10)[0] + 1])
        assert [a[2] for a in an] == starts[idx].tolist()
    return f, s


def test_audit_sample_golden(variant, golden_dir):
    exp = json.load(open(os.path.join(golden_dir, "audit_sample.expected.json")))
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read()
    with _det(exp["keys"]) as det:
        f, s = det.process_lines(buf, exp["n_train"])
        assert f.tolist() == exp["flags"]
        assert np.allclose(s, np.array(exp["scores"], dtype=np.float32), atol=SCORE_TOL)
        an = det.anomalies()
        assert [a[1] for a in an] == [m for m in exp["masks"] if m]
        st = det.stats()
        assert st["lines"] == exp["n_records"] and st["train_lines"] == exp["n_train"]
        assert st["anomalies"] == sum(exp["flags"]) and st["score_sum"] == int(sum(exp["scores"]))
        assert st["known_keys"] == sum(exp["known_counts"])
        assert st["bytes"] == len(buf)


def test_synthetic_64k_x_256(variant):
    """BASELINE config 2 shape: 64k records of 256 B; window 1 trains, window 2 detects."""
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    g = AuditSynth()
    train, _ = g.batch(65536, inject=False)
    det_msg, inj = g.batch(65536, inject=True)
    keys = [k.encode() for k in MONITORED_KEYS]
    o = NativeOracle(keys)
    with _det(keys) as det:
        _check(det, o, train, 65536)
        f, s = _check(det, o, det_msg, 0)
        assert f.sum() >= inj.sum() > 0
        # learnt set == oracle's strings through dm_fp64
        want = sorted(fingerprint.table_key(i, v) for i in range(len(keys)) for v in o.known_values(i))
        assert det.export_known().tolist() == want
        st = det.stats()
        assert st["unknown_per_key"] == [o.unknown_count(i) for i in range(len(keys))]
        # idempotence: detection never inserts (R-spec 2)
        f2, s2 = det.process_lines(det_msg, 0)
        assert (f2 == f).all() and (s2 == s).all()


def test_train_detect_split_inside_one_message(variant):
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    g = AuditSynth(seed=5)
    a, _ = g.batch(3000, inject=False)
    b, _ = g.batch(5000, inject=True)
    keys = [k.encode() for k in MONITORED_KEYS]
    o = NativeOracle(keys)
    with _det(keys) as det:
        _check(det, o, a + b, 3000)
        _check(det, o, b, 100)         # more training on top, then detect


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_fuzz_tokenizer_prefilter_on(variant, seed):
    """Same fuzz with keys that share 3 last bytes: the row phase's candidate pre-filter is active."""
    o = NativeOracle(FUZZ_KEYS_FEW)
    with _det(FUZZ_KEYS_FEW) as det:
        _check(det, o, fuzz_lines(seed + 7, 4000), 1500)
        _check(det, o, fuzz_lines(seed + 107, 4000), 0)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_fuzz_tokenizer(variant, seed):
    """Random records rich in '=', spaces and both quote characters: empty records,
    unbalanced quotes, duplicate keys, keys at record start, values at record end."""
    o = NativeOracle(FUZZ_KEYS)
    with _det(FUZZ_KEYS) as det:
        _check(det, o, fuzz_lines(seed, 4000), 1500)
        _check(det, o, fuzz_lines(seed + 100, 4000), 0)


def test_edge_cases(variant):
    keys = [b"k", b"type", b"longer_key_name_0123456789abcdef"]
    cases = [
        b"",                                              # empty message
        b"\n",                                            # one empty record
        b"\n\n\n",
        b"type=A",                                        # no trailing newline
        b"type=A\ntype=B",                                # tail record
        b"k=1 k=2\n",                                     # duplicate key: first wins
        b"type=\n",                                       # empty value
        b"=x k=\n",
        b"x" * 5000 + b" k=v\n",                          # long record, key late
        b"k=" + b"v" * 5000 + b"\n",                      # long value
        b'q="a b k=1" k=2\n',                             # key inside quotes is not a field
        b'q="unbalanced k=1\nk=1\n',                      # quote parity resets per record
        b"longer_key_name_0123456789abcdef=1 xlonger_key_name_0123456789abcdef=2\n",
        b"a'k=5 b'type=Z\n",                              # single quote starts a field
        b" k=1\n  k=2\n",                                 # leading spaces
        b"k=1\n" * 1000,
        (b"y" * 126 + b" k=edge\n") * 50,                 # key straddling the 128-byte steps
        (b"y" * 123 + b" type=edge\n") * 50,
        b" k=" * 600 + b"\n" + b"=" * 700 + b"\n" + b"k=2 " * 300 + b"\n",   # rows dense in '=' (queue overflow path)
    ]
    o = NativeOracle(keys)
    with _det(keys) as det:
        train = b"k=1\ntype=A\nk=v\n"
        _check(det, o, train, 3)
        for c in cases:
            _check(det, o, c, 0)


def test_varlen_config5(variant):
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    g = AuditSynth(seed=20260924)
    train, _ = g.batch_varlen(20000, inject=False)
    msg, _ = g.batch_varlen(30000, inject=True)
    keys = [k.encode() for k in MONITORED_KEYS]
    o = NativeOracle(keys)
    with _det(keys) as det:
        _check(det, o, train, 20000)
        f, _ = _check(det, o, msg, 0)
        assert f.sum() > 0


def test_recheck_mode_follows_the_stream(monkeypatch):
    """Left alone (DM_STREAM_RECHECK unset) the library re-checks one by one while candidates are rare and switches to the
    batch-wise re-check when most batches hold one (config-5 look-alikes) -- with the oracle's results either way."""
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    from util import lookalike_lines
    monkeypatch.setenv("DM_KERNEL", "stream")
    monkeypatch.delenv("DM_STREAM_RECHECK", raising=False)
    keys = [k.encode() for k in MONITORED_KEYS]
    g = AuditSynth(seed=77)
    o = NativeOracle(keys)
    with _det(keys) as det:
        _check(det, o, g.batch(20000, inject=False)[0], 20000)
        modes = []
        for i in range(3):
            _check(det, o, g.batch(20000, inject=True)[0], 0)
            modes.append(det.stream_recheck_chained())
        for i in range(4):
            _check(det, o, g.batch_varlen(20000, inject=True)[0], 0)
            modes.append(det.stream_recheck_chained())
        for i in range(3):
            _check(det, o, g.batch(20000, inject=True)[0], 0)
            modes.append(det.stream_recheck_chained())
        # (the choice for a message rests on the message before it)
        assert modes == [False, False, False, False, True, True, True, True, False, False], modes
    keys2 = [b"key", b"type", b"res"]
    o2 = NativeOracle(keys2)
    with _det(keys2) as det:
        _check(det, o2, lookalike_lines(5, 3000), 1000)
        for seed in (6, 7, 8):
            _check(det, o2, lookalike_lines(seed, 3000), 0)
        assert det.stream_recheck_chained()


def test_full_size_properties(variant):
    """BASELINE config 2 at full size (1M x 256 B, 16 messages of 64k): count identities
    and agreement with the oracle on every message."""
    from detectmateservice_b200.synth import MONITORED_KEYS, config2_stream
    keys = [k.encode() for k in MONITORED_KEYS]
    o = NativeOracle(keys)
    total = anomalies = 0
    with _det(keys) as det:
        for msg, n_train in config2_stream(1_000_000):
            f, s = _check(det, o, msg, n_train, check_masks=False)
            assert f.size == msg.count(b"\n")
            assert ((s > 0) == (f == 1)).all()
            total += f.size
            anomalies += int(f.sum())
        st = det.stats()
        assert st["lines"] == total == 1_000_000 and st["anomalies"] == anomalies
        assert st["train_lines"] == 65536 and st["detect_lines"] == total - 65536
        assert st["score_sum"] == sum(st["unknown_per_key"])


def test_device_resident_enqueue(variant):
    """The no-sync device path used by bench.py gives the same flags as the host path."""
    import torch
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    g = AuditSynth(seed=9)
    train, _ = g.batch(8192, inject=False)
    msg, _ = g.batch(8192, inject=True)
    with _det(MONITORED_KEYS) as det:
        det.process_lines(train, 8192)
        f_host, s_host = det.process_lines(msg, 0)
        t = torch.zeros(len(msg) + 64, dtype=torch.uint8, device="cuda")
        t[:len(msg)] = torch.frombuffer(bytearray(msg), dtype=torch.uint8).cuda()
        flags = torch.full((8192,), 7, dtype=torch.uint8, device="cuda")
        scores = torch.full((8192,), -1.0, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        stream = torch.cuda.Stream()
        st = stream.cuda_stream
        assert st != 0                      # NULL would mean "the handle's own stream"
        det.enqueue_device(t.data_ptr(), len(msg), 0, flags.data_ptr(), scores.data_ptr(), 8192, st)
        n_lines, n_anom = det.sync()
        assert n_lines == 8192 and n_anom == int(f_host.sum())
        assert (flags.cpu().numpy() == f_host).all() and (scores.cpu().numpy() == s_host).all()


def test_known_set_export_import_roundtrip(variant):
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    g = AuditSynth(seed=11)
    train, _ = g.batch(4096, inject=False)
    msg, _ = g.batch(4096, inject=True)
    with _det(MONITORED_KEYS) as a, _det(MONITORED_KEYS) as b:
        a.process_lines(train, 4096)
        keys = a.export_known()
        b.import_known(keys)
        fa, sa = a.process_lines(msg, 0)
        fb, sb = b.process_lines(msg, 0)
        assert (fa == fb).all() and (sa == sb).all() and fa.sum() > 0
        assert b.export_known().tolist() == keys.tolist()
        b.reset()
        fr, _ = b.process_lines(msg, 0)
        assert fr.all()                      # nothing known any more: every record alerts


def test_capacity_errors_are_loud(variant):
    from detectmateservice_b200 import _lib
    with _det([b"k"], max_batch_bytes=4096, max_lines=16, table_log2_slots=10) as det:
        with pytest.raises(_lib.DmError) as e:
            det.process_lines(b"x" * 5000, 0)
        assert e.value.code == _lib.DM_ERR_CAPACITY
        with pytest.raises(_lib.DmError) as e:
            det.process_lines(b"k=1\n" * 100, 0)
        assert e.value.code == _lib.DM_ERR_CAPACITY
        many = b"".join(b"k=%d\n" % i for i in range(16))
        det.process_lines(many, 16)
    with _det([b"k"], max_batch_bytes=1 << 16, table_log2_slots=10) as det:
        many = b"".join(b"k=%d\n" % i for i in range(2000))
        with pytest.raises(_lib.DmError) as e:
            det.process_lines(many, 2000)
        assert e.value.code == _lib.DM_ERR_TABLE_FULL


def test_window_exchange_two_ranks_on_one_gpu(variant):
    """dm_window_export / dm_window_import with two handles standing in for two ranks: the SUM
    of their buffers (what the NCCL all-reduce computes) teaches each rank the other's keys and
    yields the global statistics."""
    import torch
    from detectmateservice_b200 import window
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    g = AuditSynth(seed=21)
    train, _ = g.batch(6000, inject=False)
    detect, _ = g.batch(6000, inject=True)
    cuts = window.shard_bounds(train, 2)
    dcuts = window.shard_bounds(detect, 2)
    keys = [k.encode() for k in MONITORED_KEYS]
    one = NativeOracle(keys)
    one.process(train, 6000)
    wf, ws, _ = one.process(detect, 0)
    with _det(MONITORED_KEYS) as d0, _det(MONITORED_KEYS) as d1:
        dets = [d0, d1]
        bufs = []
        for r, d in enumerate(dets):
            shard = train[cuts[r]:cuts[r + 1]]
            d.process_lines(shard, shard.count(b"\n"))
            b = torch.zeros(d.window_words(2, True), dtype=torch.int64, device="cuda")
            d.window_export(b.data_ptr(), r, 2, True)
            d.sync()
            bufs.append(b)
        total = bufs[0] + bufs[1]                               # the all-reduce
        torch.cuda.synchronize()
        for r, d in enumerate(dets):
            d.window_import(total.data_ptr(), r, 2, True)
            d.sync()
        assert d0.export_known().tolist() == d1.export_known().tolist()
        got = []
        for r, d in enumerate(dets):
            f, s = d.process_lines(detect[dcuts[r]:dcuts[r + 1]], 0)
            got.append((f, s))
        assert np.concatenate([g_[0] for g_ in got]).tolist() == wf.tolist()
        assert np.concatenate([g_[1] for g_ in got]).tolist() == ws.tolist()
        # statistics-only window: global = sum over ranks
        sb = [torch.zeros(d.window_words(2, False), dtype=torch.int64, device="cuda") for d in dets]
        for r, d in enumerate(dets):
            d.window_export(sb[r].data_ptr(), r, 2, False)
            d.sync()
        tot = sb[0] + sb[1]
        torch.cuda.synchronize()
        for r, d in enumerate(dets):
            d.window_import(tot.data_ptr(), r, 2, False)
        gs = d0.global_stats()
        assert gs["lines"] == 12000 and gs["train_lines"] == 6000 and gs["anomalies"] == int(wf.sum())
        assert gs["score_sum"] == int(ws.sum()) and gs == d1.global_stats()


def test_pipelined_submit_collect(monkeypatch, kernel="stream"):
    """dm_submit_lines / dm_collect (two slots in flight) give the same flags, scores and
    anomaly lists as the synchronous call, in submission order, training included."""
    import torch
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    monkeypatch.setenv("DM_KERNEL", kernel)
    g = AuditSynth(seed=31)
    msgs = [g.batch(5000, inject=False)[0]] + [g.batch(5000, inject=True)[0] for _ in range(6)] + [b"", b"type=A\n"]
    n_train = [3000] + [0] * (len(msgs) - 1)
    keys = [k.encode() for k in MONITORED_KEYS]
    o = NativeOracle(keys)
    want = [o.process(m, t, want_masks=True) for m, t in zip(msgs, n_train)]
    pinned = []
    for m in msgs:
        t = torch.empty(max(len(m), 1), dtype=torch.uint8, pin_memory=True)
        t[:len(m)].copy_(torch.frombuffer(bytearray(m), dtype=torch.uint8)) if m else None
        pinned.append(t.numpy()[:len(m)])
    with _det(keys) as det:
        got = {}
        for i in range(len(msgs)):
            slot = i & 1
            if i >= 2:
                f, s = det.collect(slot)
                got[i - 2] = (f.copy(), s.copy(), det.collect_anomalies(slot))
            det.submit(pinned[i], n_train[i], slot)
        for i in range(len(msgs) - 2, len(msgs)):
            f, s = det.collect(i & 1)
            got[i] = (f.copy(), s.copy(), det.collect_anomalies(i & 1))
        for i, (wf, ws, wm) in enumerate(want):
            f, s, an = got[i]
            assert f.tolist() == wf.tolist() and s.tolist() == ws.tolist(), i
            idx = np.nonzero(wf)[0]
            assert [a[0] for a in an] == idx.tolist() and [a[1] for a in an] == wm[idx].tolist()
        from detectmateservice_b200 import _lib
        with pytest.raises(_lib.DmError):
            det.collect(0)                                   # nothing in flight
        det.submit(pinned[1], 0, 0)
        with pytest.raises(_lib.DmError):
            det.submit(pinned[2], 0, 0)                      # slot busy
        det.collect(0)
        st = det.stats()
        assert st["lines"] == sum(w[0].size for w in want) + 5000 and st["train_lines"] == 3000


def _check_device(det, oracle, msg, n_train, stream):
    """_check through the device-resident path: the message in a device buffer with exactly 16 bytes of hostile
    slack, outputs in device buffers pre-filled with 7 / -1."""
    import torch
    host = np.concatenate([np.frombuffer(msg, dtype=np.uint8), np.frombuffer(b"=\n" * 8, dtype=np.uint8)])
    x = torch.from_numpy(host).cuda()
    cap = msg.count(b"\n") + 1
    flags = torch.full((cap,), 7, dtype=torch.uint8, device="cuda")
    scores = torch.full((cap,), -1.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    det.enqueue_device(x.data_ptr(), len(msg), n_train, flags.data_ptr(), scores.data_ptr(), cap, stream.cuda_stream)
    n, _ = det.sync()
    of, os_, om = oracle.process(msg, n_train, want_masks=True)
    assert n == of.size
    f, s = flags.cpu().numpy()[:n], scores.cpu().numpy()[:n]
    bad = np.nonzero(f != of)[0]
    assert bad.size == 0, f"flags differ at records {bad[:10]} (gpu {f[bad[:10]]}, oracle {of[bad[:10]]})"
    assert (s == os_).all()
    an = det.anomalies()
    idx = np.nonzero(of)[0]
    assert [a[0] for a in an] == idx.tolist() and [a[1] for a in an] == om[idx].tolist()
    return f, s


def test_byte_position_sweep(variant):
    """tests/util.sweep_messages: '=' on every residue mod 32 and at the 1 KiB row edges, first '=' at bytes 1-4,
    value lengths around the 32-byte window and the 64 bytes behind a row, quoted spaces at the window's end, messages
    ending inside a value for every nbytes % 16.  Host path and device buffers with exactly 16 bytes of slack."""
    import torch
    import util
    train, _ = util.sweep_training(0)
    msgs = util.sweep_messages(0)
    stream = torch.cuda.Stream()
    for device in (False, True):
        o = NativeOracle(util.SWEEP_KEYS)
        with _det(util.SWEEP_KEYS) as det:
            _check(det, o, train, train.count(b"\n"))
            for m in msgs:
                if device:
                    _check_device(det, o, m, 0, stream)
                else:
                    _check(det, o, m, 0)


def test_keys32(variant):
    """One key of every length 1..32 (shared last four bytes, a suffix key, a byte >= 0x80) with look-alikes; then
    nothing learnt: every record alerts on all 32 fields."""
    import util
    keys = util.KEYS32
    train, known = util.keys32_training(1)
    o = NativeOracle(keys)
    with _det(keys) as det:
        _check(det, o, train, train.count(b"\n"))
        f, _ = _check(det, o, util.keys32_lines(2, 2000, known=known), 0)
        assert 0 < f.sum() < f.size
        st = det.stats()
        assert st["unknown_per_key"] == [o.unknown_count(i) for i in range(32)]
    o2 = NativeOracle(keys)
    with _det(keys) as det:
        f, s = _check(det, o2, util.keys32_lines(3, 500), 0)
        assert f.all() and (s == 32).all()
        assert {a[1] for a in det.anomalies()} == {0xFFFFFFFF}
        st = det.stats()
        assert st["unknown_per_key"] == [500] * 32 and st["score_sum"] == 500 * 32


def test_keys32_three_byte_level1_table_full_message(variant):
    """32 distinct 3-byte keys (96 level-1 patterns: the 512-slot table, 4 KiB more shared memory per CTA) on a full
    64k x 256 B message."""
    import util
    keys = util.KEYS32_3BYTE
    train, known = util.keys32_training(4, keys=keys)
    o = NativeOracle(keys)
    with _det(keys) as det:
        _check(det, o, train, train.count(b"\n"))
        rng = np.random.Generator(np.random.PCG64(8))
        recs = []
        for i in range(65536):
            js = rng.choice(32, 12, replace=False)
            toks = [keys[j] + b"=" + (known[j][int(rng.integers(0, len(known[j])))] if rng.random() < 0.99 else b"n%d" % i)
                    for j in js]
            rec = b" ".join(toks)
            recs.append(rec + b" " + b"p" * max(0, 255 - len(rec) - 1) if len(rec) < 254 else rec[:255])
        msg = b"\n".join(recs) + b"\n"
        assert msg.count(b"\n") == 65536
        f, _ = _check(det, o, msg, 0)
        assert 0 < f.sum() < f.size


def test_train_detect_split_sweep(variant):
    """Every split point 0 .. n+2 of a ~3 KB message of 40 records crossing several 512-byte rows of dm_k_bound (tail
    record without a newline), each with a fresh detector; then a message of more than 256 such rows (dm_k_bound's
    per-group path) split at records that hold a group edge."""
    import util
    keys = [b"type", b"res", b"acct"]
    msg = util.split_message(6)
    n = msg.count(b"\n") + 1
    for n_train in range(n + 3):
        o = NativeOracle(keys)
        with _det(keys, max_batch_bytes=1 << 20, table_log2_slots=12) as det:
            _check(det, o, msg, n_train)
            st = det.stats()
            assert st["train_lines"] == min(n_train, n) and st["lines"] == n
            assert st["unknown_per_key"] == [o.unknown_count(i) for i in range(len(keys))]
            assert st["known_keys"] == sum(o.known_count(i) for i in range(len(keys)))
    big = util.split_message(7, n_records=2000, mean_len=90)
    rows = (len(big) + 511) // 512
    per = (rows + 255) // 256
    nl = np.nonzero(np.frombuffer(big, dtype=np.uint8) == 10)[0]
    for grp in (1, 2, 100, 255):
        rec = int(np.searchsorted(nl, grp * per * 512))
        for n_train in (rec - 1, rec, rec + 1):
            o = NativeOracle(keys)
            with _det(keys, max_batch_bytes=1 << 20, table_log2_slots=12) as det:
                _check(det, o, big, n_train)
