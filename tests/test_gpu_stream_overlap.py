"""Device-resident detection with overlapping launches (dm_set_overlap(1)) against the oracle, and errors of enqueued
messages.  Needs an H100.

With overlap on, consecutive launches on one stream start before their predecessor has finished (programmatic
dependent launch), their scratch rotates over four sets, each launch's CTAs zero-fill the outputs up to the record
count of the launch four calls earlier, and each epilogue first takes the previous call's late alerts out of the
output buffers.  These tests enqueue long runs of messages without a sync in between, so that the rotation wraps
several times, and compare every call's outputs with the oracle run over the same messages in the same order.
"""
import numpy as np
import pytest

from oracle.native import NativeOracle
from util import lookalike_lines

pytestmark = pytest.mark.gpu

SLACK = np.frombuffer(b"=\n" * 8, dtype=np.uint8)          # the 16 bytes of slack dmdetect.h asks for, hostile


def _det(keys, **kw):
    from detectmateservice_b200.detector import DeviceDetector
    kw.setdefault("max_batch_bytes", 32 << 20)
    kw.setdefault("table_log2_slots", 18)
    return DeviceDetector(keys, **kw)


def _dev_msg(msg: bytes):
    """The message in its own device tensor with exactly 16 bytes of slack behind it."""
    import torch
    host = np.concatenate([np.frombuffer(msg, dtype=np.uint8), SLACK])
    return torch.from_numpy(host).cuda()


class _Out:
    """One call's output buffers, pre-filled with 7 / -1.0: `cap` entries, at element offset `off` into the tensors
    (offset 1 leaves the pointers off 16-byte alignment)."""

    def __init__(self, cap: int, off: int = 0):
        import torch
        self.flags_t = torch.full((cap + off,), 7, dtype=torch.uint8, device="cuda")
        self.scores_t = torch.full((cap + off,), -1.0, dtype=torch.float32, device="cuda")
        self.flags, self.scores, self.cap = self.flags_t[off:], self.scores_t[off:], cap

    def host(self):
        return self.flags.cpu().numpy(), self.scores.cpu().numpy()


def _messages():
    """(message, n_train) in call order: one training message, then 20 detection messages whose record counts grow
    and shrink across the 4-set rotation, a training message in the middle, and config-5 look-alikes."""
    from detectmateservice_b200.synth import AuditSynth
    g = AuditSynth(seed=4711)
    train, _ = g.batch(8192, inject=False)
    taught = b"".join(b"type=TAUGHT_%d res=r%d exe=/usr/bin/t%d\n" % (i, i % 7, i) for i in range(300))
    probe = b"".join(b"type=TAUGHT_%d res=r%d exe=/usr/bin/t%d\n" % (i, i % 7, i) for i in range(0, 600, 2))
    seq = [
        (train, 8192),
        (g.batch(65536, inject=True)[0], 0),
        (b"type=USER_LOGIN res=success", 0),                  # one record, no trailing newline
        (b"", 0),
        (b"\n", 0),
        (g.batch(5000, inject=True)[0], 0),
        (g.batch(65536, inject=True)[0], 0),
        (g.batch(200, inject=True)[0], 0),
        (probe, 0),                                          # TAUGHT_* not learnt yet: alerts
        (taught + probe, 300),                               # training in mid-run (launched without overlap)
        (probe, 0),                                          # the first half of TAUGHT_* is known now
        (g.batch(3, inject=True)[0], 0),
        (g.batch_varlen(8000, inject=True)[0], 0),
        (lookalike_lines(3, 3000, keys=(b"type", b"res", b"acct")), 0),
        (lookalike_lines(4, 3000, keys=(b"type", b"res", b"acct")), 0),
        (g.batch_varlen(8000, inject=True)[0], 0),
        (g.batch(65536, inject=True)[0], 0),                 # (re-check choice switches back)
        (b"", 0),
        (g.batch(7, inject=True)[0] + b"type=tail_without_newline", 0),
        (g.batch(40000, inject=True)[0], 0),
        (b"\n\n\n", 0),
        (g.batch(12000, inject=True)[0], 0),
    ]
    return seq


def _oracle(keys, seq):
    o = NativeOracle(keys)
    want = [o.process(m, t, want_masks=True) for m, t in seq]
    return o, want


def _want_stats(o, keys, seq, want):
    n = [w[0].size for w in want]
    tr = [min(t, k) for (_, t), k in zip(seq, n)]
    return {"lines": sum(n), "train_lines": sum(tr), "detect_lines": sum(n) - sum(tr),
            "anomalies": int(sum(int(w[0].sum()) for w in want)), "score_sum": int(sum(float(w[1].sum()) for w in want)),
            "bytes": sum(len(m) for m, _ in seq), "unknown_per_key": [o.unknown_count(i) for i in range(len(keys))]}


def _run(keys, seq, overlap: bool):
    """Enqueue every message of seq on one non-default stream (call 14 on a second stream), sync once; returns the
    per-call output buffers (host copies of their full capacity), the statistics and the last anomaly list."""
    import torch
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    ins = [_dev_msg(m) for m, _ in seq]
    outs = []
    for i, (m, _) in enumerate(seq):
        n = m.count(b"\n") + (1 if m and not m.endswith(b"\n") else 0)
        outs.append(_Out(max(n, 1) + (0 if i % 2 else 37), off=1 if i % 3 == 1 else 0))
    torch.cuda.synchronize()
    with _det(keys) as det:
        det.set_overlap(overlap)
        for i, ((m, t), x, o) in enumerate(zip(seq, ins, outs)):
            st = s2 if i == 14 else s1
            det.enqueue_device(x.data_ptr(), len(m), t, o.flags.data_ptr(), o.scores.data_ptr(), o.cap, st.cuda_stream)
        n_last, _ = det.sync()
        torch.cuda.synchronize()
        assert n_last == seq[-1][0].count(b"\n")
        got = [o.host() for o in outs]
        return got, det.stats(), det.anomalies()


def _check_calls(got, want):
    for i, ((f, s), (wf, ws, _)) in enumerate(zip(got, want)):
        n = wf.size
        bad = np.nonzero(f[:n] != wf)[0]
        assert bad.size == 0, f"call {i}: flags differ at records {bad[:10]} (gpu {f[bad[:10]]}, oracle {wf[bad[:10]]})"
        assert (s[:n] == ws).all(), f"call {i}: scores differ"


def test_overlapped_stream_matches_oracle(monkeypatch):
    from detectmateservice_b200.synth import MONITORED_KEYS
    monkeypatch.setenv("DM_KERNEL", "stream")
    monkeypatch.delenv("DM_STREAM_RECHECK", raising=False)
    keys = [k.encode() for k in MONITORED_KEYS]
    seq = _messages()
    assert len(seq) - 1 >= 16
    o, want = _oracle(keys, seq)
    got, st, an = _run(keys, seq, overlap=True)
    _check_calls(got, want)
    ws = _want_stats(o, keys, seq, want)
    assert {k: st[k] for k in ws} == ws
    wf, _, wm = want[-1]
    idx = np.nonzero(wf)[0]
    assert [a[0] for a in an] == idx.tolist() and [a[1] for a in an] == wm[idx].tolist()
    assert sum(int(w[0].sum()) for w in want[1:]) > 100               # the run holds alerts to get wrong
    # the same sequence without overlap: byte-identical buffers, slack included
    got_off, st_off, an_off = _run(keys, seq, overlap=False)
    for i, ((f, s), (f2, s2)) in enumerate(zip(got, got_off)):
        assert f.tobytes() == f2.tobytes() and s.tobytes() == s2.tobytes(), i
    assert st_off == st and an_off == an


def test_overlapped_stream_shared_output_buffer(monkeypatch):
    """Every call writes into the SAME flags / scores buffer, read after one sync: the calls before the last one alert
    at record indices where the last one does not, so the last call's result is only right if its epilogue takes the
    late alerts of the call before it out of the buffer."""
    import torch
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    monkeypatch.setenv("DM_KERNEL", "stream")
    monkeypatch.delenv("DM_STREAM_RECHECK", raising=False)
    keys = [k.encode() for k in MONITORED_KEYS]
    g = AuditSynth(seed=99)
    train, _ = g.batch(20000, inject=False)
    other = AuditSynth(seed=100)
    seq = [(train, 20000)]
    for n in (65536, 3000, 65536, 30000, 65536, 1, 50000, 65536, 20000, 65536, 40000):
        m = other.batch(n, inject=False)[0]
        seq.append((m.replace(b" res=", b" res=never_"), 0))            # a value never learnt: every record alerts
    seq.append((train, 0))                                             # clean: no record alerts
    o, want = _oracle(keys, seq)
    assert want[-1][0].sum() == 0 and all(w[0].sum() > 0 for w in want[1:-1])
    ins = [_dev_msg(m) for m, _ in seq]
    out = _Out(65536 + 16, off=1)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with _det(keys) as det:
        det.set_overlap(True)
        for (m, t), x in zip(seq, ins):
            det.enqueue_device(x.data_ptr(), len(m), t, out.flags.data_ptr(), out.scores.data_ptr(), out.cap, s.cuda_stream)
        det.sync()
        f, sc = out.host()
        n = want[-1][0].size
        assert (f[:n] == 0).all(), np.nonzero(f[:n])[0][:10]
        assert (sc[:n] == 0).all()
        ws = _want_stats(o, keys, seq, want)
        st = det.stats()
        assert {k: st[k] for k in ws} == ws
        assert det.anomalies() == []


# ---------------------------------------------------------------------------------------------------------------------
# errors of enqueued messages reach dm_sync
# ---------------------------------------------------------------------------------------------------------------------
def _enqueue(det, msg, n_train, cap, stream):
    x, o = _dev_msg(msg), _Out(cap)
    det.enqueue_device(x.data_ptr(), len(msg), n_train, o.flags.data_ptr(), o.scores.data_ptr(), cap, stream)
    return x, o


@pytest.mark.parametrize("overlap", [False, True])
def test_enqueued_capacity_error_reaches_sync(monkeypatch, overlap):
    """A message with more records than its out_cap, then a good one: dm_sync reports DM_ERR_CAPACITY, once."""
    import torch
    from detectmateservice_b200 import _lib
    monkeypatch.setenv("DM_KERNEL", "stream")
    s = torch.cuda.Stream()
    with _det([b"k"], max_batch_bytes=1 << 16) as det:
        det.set_overlap(overlap)
        keep = [_enqueue(det, b"k=1\n" * 100, 0, 50, s.cuda_stream), _enqueue(det, b"k=1\n" * 10, 0, 10, s.cuda_stream)]
        with pytest.raises(_lib.DmError) as e:
            det.sync()
        assert e.value.code == _lib.DM_ERR_CAPACITY
        assert det.sync() == (10, 10)                                # reported once, then cleared
        del keep


def test_enqueued_training_table_full_reaches_sync(monkeypatch):
    import torch
    from detectmateservice_b200 import _lib
    monkeypatch.setenv("DM_KERNEL", "stream")
    s = torch.cuda.Stream()
    many = b"".join(b"k=%d\n" % i for i in range(2000))
    with _det([b"k"], max_batch_bytes=1 << 16, table_log2_slots=10) as det:
        det.set_overlap(True)
        keep = [_enqueue(det, many, 2000, 2000, s.cuda_stream), _enqueue(det, b"k=1\n", 0, 1, s.cuda_stream)]
        with pytest.raises(_lib.DmError) as e:
            det.sync()
        assert e.value.code == _lib.DM_ERR_TABLE_FULL
        del keep


def test_enqueued_anomaly_list_overflow_reaches_sync(monkeypatch):
    """32 keys, nothing learnt: every record adds 32 entries to an anomaly list of max_lines = 64 entries."""
    import torch
    from detectmateservice_b200 import _lib
    from util import KEYS32
    monkeypatch.setenv("DM_KERNEL", "stream")
    s = torch.cuda.Stream()
    rec = b" ".join(k + b"=u" for k in KEYS32) + b"\n"
    with _det(KEYS32, max_batch_bytes=1 << 16, max_lines=64) as det:
        det.set_overlap(True)
        keep = [_enqueue(det, rec * 3, 0, 64, s.cuda_stream), _enqueue(det, b"\n", 0, 64, s.cuda_stream)]
        with pytest.raises(_lib.DmError) as e:
            det.sync()
        assert e.value.code == _lib.DM_ERR_CAPACITY
        del keep


def test_anomaly_list_capacity_boundary(monkeypatch):
    """The anomaly list holds one entry per unknown (record, field) and max_lines entries: exactly that many alerts
    work, one more is an error (synchronous path)."""
    from detectmateservice_b200 import _lib
    from util import KEYS32
    monkeypatch.setenv("DM_KERNEL", "stream")
    rec = b" ".join(k + b"=u" for k in KEYS32) + b"\n"
    with _det(KEYS32, max_batch_bytes=1 << 16, max_lines=64) as det:
        f, s = det.process_lines(rec * 2, 0)                         # 64 alerts
        assert f.tolist() == [1, 1] and s.tolist() == [32.0, 32.0]
        assert det.anomalies() == [(0, 0xFFFFFFFF, 0), (1, 0xFFFFFFFF, len(rec))]
        with pytest.raises(_lib.DmError) as e:
            det.process_lines(rec * 2 + KEYS32[0] + b"=u\n", 0)     # 65
        assert e.value.code == _lib.DM_ERR_CAPACITY
        f, _ = det.process_lines(b"\n" + rec, 0)                     # the handle is usable again
        assert f.tolist() == [0, 1]
