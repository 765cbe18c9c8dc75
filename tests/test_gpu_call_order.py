"""A handle's calls take effect in call order, whatever stream each one is enqueued on.  Needs an H100.

Every case first enqueues work on a stream that a bounded device spin (torch.cuda._sleep) holds back, with no sync, and
asserts that the stream is still busy right before the call under test.  So a call that does not wait for the earlier
work sees the handle without it, deterministically: no case repeats a run to make a race appear.  Results are compared
with the oracle run over the same calls in call order.  ParserSchema, bare-record and LogSchema inputs carry the
values of raw lines under monitors in the same order as the handle's keys, so their keys are those of the raw lines
(DESIGN.md R-combo) and the raw-line oracle gives their expected flags, scores and masks too.
"""
import numpy as np
import pytest

from detectmateservice_b200 import wire
from oracle.native import NativeOracle

pytestmark = pytest.mark.gpu

KEYS = [b"type", b"res", b"exe"]
MONITORS = [{"source": "header", "pos": k} for k in KEYS]
HOLD_CYCLES = 200_000_000                 # ~0.1 s at the H100's ~2 GHz SM clock
SLACK = np.frombuffer(b"=\n" * 8, dtype=np.uint8)

# (type, res, exe) of each record: training learns 50 types, 7 results and 3000 programs; detection mixes known and
# unknown values of every field, so that both wrong ways (nothing learnt yet, too much learnt) change the result
TRAIN = [(b"T%d" % (i % 50), b"r%d" % (i % 7), b"/bin/e%d" % i) for i in range(3000)]


def _detect(shift: int, n: int = 2000):
    return [(b"T%d" % ((j + shift) % 60), b"r%d" % ((j + shift) % 9), b"/bin/e%d" % (3 * j + shift)) for j in range(n)]


def _lines(vals) -> bytes:
    return b"".join(b"type=%s res=%s exe=%s\n" % v for v in vals)


def _records(vals) -> bytes:
    """A ParserSchema batch holding the values as logFormatVariables."""
    return wire.frame_delimited([wire.encode_parser_schema(
        {"logFormatVariables": {k.decode(): x.decode() for k, x in zip(KEYS, v)}}) for v in vals])


def _logs(vals) -> bytes:
    """A LogSchema batch holding the raw lines as texts."""
    return wire.frame_delimited([wire.encode_log_schema({"logID": str(i), "log": ln.decode() + "\n"})
                                 for i, ln in enumerate(_lines(vals).splitlines())])


VARIANTS = ["stream", "chain", "lanes"]


@pytest.fixture(params=VARIANTS)
def variant(request, monkeypatch):
    """stream / chain: the default kernel, re-checking candidates one by one / batch-wise; lanes: a thread per record."""
    monkeypatch.setenv("DM_KERNEL", "lanes" if request.param == "lanes" else "stream")
    if request.param != "lanes":
        monkeypatch.setenv("DM_STREAM_RECHECK", "chain" if request.param == "chain" else "thread")
    return request.param


@pytest.fixture
def default_kernel(monkeypatch):
    monkeypatch.setenv("DM_KERNEL", "stream")
    monkeypatch.delenv("DM_STREAM_RECHECK", raising=False)


@pytest.fixture(autouse=True)
def _drained():
    yield
    import torch
    torch.cuda.synchronize()                                          # no held stream outlives its case


def _det(keys=KEYS, **kw):
    from detectmateservice_b200.detector import DeviceDetector
    kw.setdefault("max_batch_bytes", 1 << 20)
    kw.setdefault("table_log2_slots", 16)
    return DeviceDetector(keys, **kw)


def _hold(stream) -> None:
    import torch
    with torch.cuda.stream(stream):
        torch.cuda._sleep(HOLD_CYCLES)


def _dev_msg(msg: bytes):
    import torch
    return torch.from_numpy(np.concatenate([np.frombuffer(msg, dtype=np.uint8), SLACK])).cuda()


class _Out:
    """Device output buffers of one enqueued call, pre-filled with 7 / -1.0."""

    def __init__(self, cap: int):
        import torch
        self.flags = torch.full((cap,), 7, dtype=torch.uint8, device="cuda")
        self.scores = torch.full((cap,), -1.0, dtype=torch.float32, device="cuda")
        self.cap = cap

    def host(self):
        return self.flags.cpu().numpy(), self.scores.cpu().numpy()


def _enqueue(det, x, msg: bytes, n_train: int, stream, out: "_Out" = None) -> None:
    det.enqueue_device(x.data_ptr(), len(msg), n_train, out.flags.data_ptr() if out else 0,
                       out.scores.data_ptr() if out else 0, out.cap if out else 0, stream.cuda_stream)


def _oracle(calls):
    o = NativeOracle(KEYS)
    return o, [o.process(m, t, want_masks=True) for m, t in calls]


def _check(f, s, want, masks=None, anomalies=None):
    wf, ws, wm = want
    assert f.shape == wf.shape, (f.shape, wf.shape)
    bad = np.nonzero(f != wf)[0]
    assert bad.size == 0, f"flags differ at records {bad[:10]} (gpu {f[bad[:10]]}, oracle {wf[bad[:10]]})"
    assert (s == ws).all(), "scores differ"
    assert 0 < int(wf.sum()) < wf.size                                # known and unknown records both
    if masks is not None:
        assert masks.tolist() == wm.tolist()
    if anomalies is not None:
        idx = np.nonzero(wf)[0]
        assert [a[0] for a in anomalies] == idx.tolist() and [a[1] for a in anomalies] == wm[idx].tolist()


def _want_stats(o, calls, want):
    n = [w[0].size for w in want]
    tr = [min(t, k) for (_, t), k in zip(calls, n)]
    return {"lines": sum(n), "train_lines": sum(tr), "detect_lines": sum(n) - sum(tr),
            "anomalies": int(sum(int(w[0].sum()) for w in want)), "score_sum": int(sum(float(w[1].sum()) for w in want)),
            "bytes": sum(len(m) for m, _ in calls), "known_keys": sum(o.known_count(k) for k in range(len(KEYS))),
            "unknown_per_key": [o.unknown_count(k) for k in range(len(KEYS))]}


def _check_stats(det, o, calls, want):
    st = det.stats()
    ws = _want_stats(o, calls, want)
    assert {k: st[k] for k in ws} == ws


# ---------------------------------------------------------------------------------------------------------------------
# raw lines: every kernel
# ---------------------------------------------------------------------------------------------------------------------
def test_sync_call_after_training_on_held_stream(variant):
    """Training enqueued on a held stream, then a synchronous process_lines on the handle's own stream."""
    import torch
    train, msg = _lines(TRAIN), _lines(_detect(0))
    calls = [(msg, 0), (train, len(TRAIN)), (msg, 0)]
    o, want = _oracle(calls)
    s = torch.cuda.Stream()
    x = _dev_msg(train)
    torch.cuda.synchronize()
    with _det() as det:
        det.process_lines(msg, 0)                 # first use before the hold, as in _after_held_training
        _hold(s)
        _enqueue(det, x, train, len(TRAIN), s)
        assert not s.query()
        f, sc = det.process_lines(msg, 0)
        assert s.query(), "process_lines returned while the training it is ordered behind was still held"
        _check(f, sc, want[2], anomalies=det.anomalies())
        _check_stats(det, o, calls, want)


def test_enqueue_on_second_stream_after_training(variant):
    """Training enqueued on a held stream, detection enqueued on a second stream, then sync()."""
    import torch
    train, msg = _lines(TRAIN), _lines(_detect(0))
    o, want = _oracle([(train, len(TRAIN)), (msg, 0)])
    s, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    x, y, out = _dev_msg(train), _dev_msg(msg), _Out(want[1][0].size)
    torch.cuda.synchronize()
    with _det() as det:
        _hold(s)
        _enqueue(det, x, train, len(TRAIN), s)
        assert not s.query()
        _enqueue(det, y, msg, 0, s2, out)
        n_lines, n_anom = det.sync()
        assert s.query() and s2.query(), "sync() returned while the handle's work on the first stream was still held"
        assert (n_lines, n_anom) == (want[1][0].size, int(want[1][0].sum()))
        _check(*out.host(), want[1], anomalies=det.anomalies())


def test_detection_on_two_streams_then_sync(variant):
    """Detection enqueued on a held stream and more detection on a second stream: sync() waits for both, both outputs
    are complete, and the statistics count both messages."""
    import torch
    train, a, b = _lines(TRAIN), _lines(_detect(0)), _lines(_detect(7, 1500))
    calls = [(train, len(TRAIN)), (a, 0), (b, 0)]
    o, want = _oracle(calls)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    xa, xb, out_a, out_b = _dev_msg(a), _dev_msg(b), _Out(want[1][0].size), _Out(want[2][0].size)
    torch.cuda.synchronize()
    with _det() as det:
        det.process_lines(train, len(TRAIN))
        _hold(s1)
        _enqueue(det, xa, a, 0, s1, out_a)
        _enqueue(det, xb, b, 0, s2, out_b)
        assert not s1.query()
        n_lines, _ = det.sync()
        assert s1.query() and s2.query(), "sync() returned while the handle's work on the first stream was still held"
        assert n_lines == want[2][0].size
        _check(*out_a.host(), want[1])
        _check(*out_b.host(), want[2], anomalies=det.anomalies())
        _check_stats(det, o, calls, want)


def test_reset_after_work_on_two_streams(variant):
    """Training on a held stream and detection on a second one, then reset(): nothing learnt survives it, and the
    next detection alerts on every record."""
    import torch
    train, msg = _lines(TRAIN), _lines(_detect(0))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    x, y, out = _dev_msg(train), _dev_msg(msg), _Out(2000)
    torch.cuda.synchronize()
    with _det() as det:
        _hold(s1)
        _enqueue(det, x, train, len(TRAIN), s1)
        _enqueue(det, y, msg, 0, s2, out)
        assert not s1.query()
        det.reset()
        assert s1.query() and s2.query(), "reset() returned while the handle's training was still held"
        assert det.export_known().size == 0
        st = det.stats()
        assert st["lines"] == 0 and st["known_keys"] == 0
        f, sc = det.process_lines(msg, 0)
        wf, ws, _ = NativeOracle(KEYS).process(msg, 0)
        assert f.all() and f.tolist() == wf.tolist() and sc.tolist() == ws.tolist()


def test_export_and_stats_after_work_on_two_streams(variant):
    """Training on a held stream and detection on a second one, then export_known() and stats(): the held stream's
    keys and counts are in them."""
    import torch
    train, msg = _lines(TRAIN), _lines(_detect(0))
    calls = [(train, len(TRAIN)), (msg, 0)]
    o, want = _oracle(calls)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    x, y, out = _dev_msg(train), _dev_msg(msg), _Out(want[1][0].size)
    torch.cuda.synchronize()
    with _det() as det:
        _hold(s1)
        _enqueue(det, x, train, len(TRAIN), s1)
        _enqueue(det, y, msg, 0, s2, out)
        assert not s1.query()
        keys = det.export_known()
        assert s1.query() and s2.query(), "export_known() returned while the handle's training was still held"
        want_keys = sorted(det.table_key(k, v) for k in range(len(KEYS)) for v in o.known_values(k))
        assert keys.tolist() == want_keys
        _check_stats(det, o, calls, want)
        _check(*out.host(), want[1])


# ---------------------------------------------------------------------------------------------------------------------
# the other entry points, behind training enqueued on a held stream
# ---------------------------------------------------------------------------------------------------------------------
def _after_held_training(det, call):
    """Makes the detection-only call once -- so that loading its kernels and allocating its scratch, both of which
    synchronise the device, happen before the hold -- then enqueues the training message on a held stream, makes the
    call again and checks that it waited for the training.  Returns what the second call returned."""
    import torch
    call()
    train = _lines(TRAIN)
    s, x = torch.cuda.Stream(), _dev_msg(train)
    torch.cuda.synchronize()
    _hold(s)
    _enqueue(det, x, train, len(TRAIN), s)
    assert not s.query()
    got = call()
    assert s.query(), "the call returned while the training it is ordered behind was still held"
    return got


def _want_detect(vals):
    _, want = _oracle([(_lines(TRAIN), len(TRAIN)), (_lines(vals), 0)])
    return want[1]


def test_records_after_training_on_held_stream(default_kernel):
    vals = _detect(0)
    batch = _records(vals)
    with _det() as det:
        det.set_monitors(MONITORS)
        f, sc, m = _after_held_training(det, lambda: det.process_records(batch, 0))
        _check(f, sc, _want_detect(vals), masks=m)


def test_values_after_training_on_held_stream(default_kernel):
    vals = [(b"T3", b"r99", b"/bin/e5")]                               # res unknown, the other two known
    with _det() as det:
        f, sc, m = _after_held_training(det, lambda: det.process_values([list(enumerate(vals[0]))], 0))
        wf, ws, wm = _want_detect(vals)
        assert (f.tolist(), sc.tolist(), m.tolist()) == (wf.tolist(), ws.tolist(), wm.tolist()) == ([1], [1.0], [2])


def test_logs_after_training_on_held_stream(default_kernel):
    vals = _detect(0)
    batch = _logs(vals)
    with _det() as det:
        f, sc, n_bad = _after_held_training(det, lambda: det.process_logs(batch, 0))
        assert n_bad == 0
        _check(f, sc, _want_detect(vals), anomalies=det.anomalies())


def test_submit_collect_after_training_on_held_stream(default_kernel):
    import torch
    vals = _detect(0)
    msg = _lines(vals)
    pinned = torch.empty(len(msg), dtype=torch.uint8, pin_memory=True)
    pinned.copy_(torch.frombuffer(bytearray(msg), dtype=torch.uint8))

    def submit_collect():
        det.submit(pinned.numpy(), 0, 0)
        f, sc = det.collect(0)
        return f.copy(), sc.copy()

    with _det() as det:
        f, sc = _after_held_training(det, submit_collect)
        _check(f, sc, _want_detect(vals), anomalies=det.collect_anomalies(0))


def test_table_full_of_held_training_is_reported(default_kernel):
    """Training that overfills the table, enqueued on a held stream, then a synchronous process_records and sync():
    DM_ERR_TABLE_FULL is reported once, by one of the two."""
    import torch
    from detectmateservice_b200 import _lib
    many = b"".join(b"k=%d\n" % i for i in range(2000))
    batch = wire.frame_delimited([wire.encode_parser_schema({"logFormatVariables": {"k": "1"}})])
    s, x = torch.cuda.Stream(), _dev_msg(many)
    torch.cuda.synchronize()
    with _det([b"k"], table_log2_slots=10) as det:
        det.set_monitors([{"source": "header", "pos": "k"}])
        det.process_records(batch, 0)                                 # first use, before the hold
        _hold(s)
        _enqueue(det, x, many, 2000, s)
        assert not s.query()
        errors = []
        for call in (lambda: det.process_records(batch, 0), det.sync):
            try:
                call()
            except _lib.DmError as e:
                errors.append(e.code)
            assert s.query()
        assert errors == [_lib.DM_ERR_TABLE_FULL]
