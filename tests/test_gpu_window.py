"""The multi-GPU window exchange on the H100 (dm_window_export / dm_window_import / dm_window_allreduce, DeviceWindow),
with the library's real per-rank key cap (window.WINDOW_KEYS = 65536).  N DeviceDetector handles on one GPU stand in
for N ranks and the sum of their export buffers for the sum all-reduce; the native NCCL route runs in process at world 1
and, when two GPUs are visible, at world 2.  References as in test_emu_window.py (which runs the same kernel sources on
the CPU emulator with a 64-key cap): the single-rank NativeOracle, window.pack_window_host and the sum of the per-rank
statistics."""
import os
import socket

import numpy as np
import pytest

from detectmateservice_b200 import window
from test_emu_window import detect_msg, keys_of, kv, oracle_detect, shards, train_set

pytestmark = pytest.mark.gpu

KEYS = [b"k", b"t"]
WK = window.WINDOW_KEYS
BIG = 70000                                  # distinct k=<i> values one rank learns: WK + 4464


@pytest.fixture(params=["stream", "lanes"])
def variant(request, monkeypatch):
    monkeypatch.setenv("DM_KERNEL", request.param)
    return request.param


def _det(log2=18, max_bytes=4 << 20):
    from detectmateservice_b200.detector import DeviceDetector
    return DeviceDetector(KEYS, max_batch_bytes=max_bytes, table_log2_slots=log2)


def words(st):
    """The dm_stats_t words of a stats() dict, known_keys as the export sends it: 0."""
    w = [st["lines"], st["train_lines"], st["detect_lines"], st["anomalies"], st["score_sum"], st["bytes"], 0,
         st["bad_records"]] + list(st["unknown_per_key"])
    return np.array(w + [0] * (40 - len(w)), dtype=np.uint64)


def big_msg(n=BIG):
    return b"".join(b"k=%d\n" % i for i in range(n))


class Ranks:
    """`world` handles on one GPU, one per rank; every call synchronises."""

    def __init__(self, world, log2=18):
        self.world = world
        self.dets = [_det(log2) for _ in range(world)]

    def close(self):
        for d in self.dets:
            d.close()

    def export(self, with_keys):
        import torch
        bufs = [torch.full((d.window_words(self.world, with_keys),), -1, dtype=torch.int64, device="cuda") for d in self.dets]
        torch.cuda.synchronize()                                     # (the handles' streams do not wait for torch's)
        for r, (d, b) in enumerate(zip(self.dets, bufs)):
            d.window_export(b.data_ptr(), r, self.world, with_keys)
            d.sync()
        return bufs

    def import_(self, bufs, with_keys):
        import torch
        total = torch.stack(bufs).sum(0)                              # the all-reduce (two's complement = uint64 sum)
        torch.cuda.synchronize()
        for r, d in enumerate(self.dets):
            d.window_import(total.data_ptr(), r, self.world, with_keys)
            d.sync()
        return total.cpu().numpy()

    def window(self, with_keys):
        bufs = self.export(with_keys)
        self.import_(bufs, with_keys)
        return [b.cpu().numpy().view(np.uint64) for b in bufs]

    def pending(self):
        return [d.window_pending_keys() for d in self.dets]

    def summed(self):
        return sum(words(d.stats()) for d in self.dets)

    def detect(self, msg):
        f, s, an, base = [], [], [], 0
        for d, m in zip(self.dets, shards(msg, self.world)):
            fr, sr = d.process_lines(m, 0)
            f.append(fr); s.append(sr)
            an += [(base + a[0], a[1]) for a in d.anomalies()]
            base += fr.size
        return np.concatenate(f), np.concatenate(s), an


def segment(buf, world, r):
    return window.unpack_window_host(buf, world, True)[1][r]


def check_detection(R, train, detect):
    wf, ws, wan = oracle_detect(train, detect)
    f, s, an = R.detect(detect)
    assert f.tolist() == wf.tolist() and s.tolist() == ws.tolist() and an == wan and wf.sum() > 0


@pytest.mark.parametrize("world", [2, 4, 8])
def test_gpu_export_bytes_and_detection(world, variant):
    """Each rank's buffer is pack_window_host(its delta, its keys) word for word; after the import every rank knows
    the union and detects its shard as the oracle does; a statistics-only window sums the statistics."""
    R = Ranks(world)
    trains = [train_set(r) for r in range(world)]
    for d, m in zip(R.dets, trains):
        d.process_lines(m, m.count(b"\n"))
    want = [words(d.stats()) for d in R.dets]
    bufs = R.export(True)
    for r, b in enumerate(bufs):
        b = b.cpu().numpy()
        seg = segment(b, world, r)
        assert sorted(seg.tolist()) == sorted(keys_of(trains[r]))
        assert b.view(np.uint64).tolist() == window.pack_window_host(want[r], seg, r, world, True).view(np.uint64).tolist()
    R.import_(bufs, True)
    train = b"".join(trains)
    union = sorted(keys_of(train))
    for d in R.dets:
        assert d.export_known().tolist() == union and d.stats()["known_keys"] == len(union)
    check_detection(R, train, detect_msg(world))
    assert [b.size for b in R.window(False)] == [40] * world
    for d in R.dets:
        assert words(d.global_stats()).tolist() == R.summed().tolist()
    R.close()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_gpu_rank_learning_70000_keys_drains_in_two_windows(world, variant):
    """Rank 0 learns 70 000 distinct k=<i> values in one training window: the first export reports exactly 4 464
    pending, the second 0; then every rank detects its shard as the single-rank oracle does."""
    R = Ranks(world)
    big = big_msg()
    trains = [big] + [train_set(r) for r in range(1, world)]
    for d, m in zip(R.dets, trains):
        d.process_lines(m, m.count(b"\n"))
    b1 = R.window(True)
    assert R.pending() == [BIG - WK] + [0] * (world - 1)
    b2 = R.window(True)
    assert R.pending() == [0] * world
    s1, s2 = segment(b1[0], world, 0), segment(b2[0], world, 0)
    assert s1.size == WK and s2.size == BIG - WK and set(s1.tolist()) | set(s2.tolist()) == keys_of(big)
    assert all(segment(b, world, r).size == 0 for r, b in enumerate(b2) if r)
    train = b"".join(trains)
    union = sorted(keys_of(train))
    for d in R.dets:
        assert d.export_known().tolist() == union
    check_detection(R, train, detect_msg(world, seed=3) + b"".join(b"k=%d t=0\n" % i for i in range(0, 2 * BIG, 997)))
    R.close()


@pytest.mark.parametrize("world", [4])
def test_gpu_several_training_windows_and_two_in_flight(world):
    """Three training windows with statistics-only windows between: each keys window carries only what each rank
    learnt since the previous one, a key two ranks learn in the same window is inserted once.  Then windows A and B
    exported before either is imported, B first: the global statistics are the sum, and a third window's delta is
    exactly what changed since B's export."""
    R = Ranks(world)
    known, all_train = set(), b""
    for w in range(3):
        trains = [train_set(r, n=30, seed=w) + kv([("new%d" % w, "both%d" % w)]) for r in range(world)]
        novel = []
        for d, m in zip(R.dets, trains):
            d.process_lines(m, m.count(b"\n"))
            novel.append(keys_of(m) - known)
        all_train += b"".join(trains)
        for _ in range(w):
            R.window(False)
        bufs = R.window(True)
        assert [set(segment(b, world, r).tolist()) for r, b in enumerate(bufs)] == novel
        known |= set().union(*novel)
        for d in R.dets:
            assert d.export_known().tolist() == sorted(known) and d.stats()["known_keys"] == len(known)
    check_detection(R, all_train, detect_msg(world, seed=4))
    a = R.export(False)
    for d, m in zip(R.dets, shards(detect_msg(world, seed=5), world)):
        d.process_lines(m, 0)
    before_c = [words(d.stats()) for d in R.dets]
    b = R.export(False)
    R.import_(b, False)
    R.import_(a, False)
    for d in R.dets:
        assert words(d.global_stats()).tolist() == R.summed().tolist()
    for d, m in zip(R.dets, shards(detect_msg(world, seed=6), world)):
        d.process_lines(m, 0)
    c = R.export(False)
    for r, d in enumerate(R.dets):
        assert c[r].cpu().numpy().view(np.uint64).tolist() == (words(d.stats()) - before_c[r]).tolist()
    R.close()


def test_gpu_imported_keys_are_not_reshipped():
    """Keys received from a peer or through import_known never appear in the rank's next export."""
    R = Ranks(2)
    trains = [train_set(r) for r in range(2)]
    for d, m in zip(R.dets, trains):
        d.process_lines(m, m.count(b"\n"))
    R.window(True)
    restored = kv([("restored%d" % i, "old") for i in range(10)])
    R.dets[0].import_known(np.array(sorted(keys_of(restored)), dtype=np.uint64))
    fresh = kv([("fresh%d" % i, 1) for i in range(5)])
    again = trains[1] + restored + fresh
    R.dets[0].process_lines(again, again.count(b"\n"))
    bufs = R.window(True)
    assert set(segment(bufs[0], 2, 0).tolist()) == keys_of(fresh) - keys_of(b"".join(trains) + restored)
    assert R.dets[1].export_known().tolist() == sorted(keys_of(b"".join(trains) + fresh))
    R.close()


# ------------------------------------------------------------------------------------------ the native route
def test_gpu_native_route_world1():
    """dm_nccl_init with two communicators at world 1, no torch.distributed: windows alternate between them (and
    between two streams); window_allreduce(True) sets the pending count, a second one drains it; after several
    statistics-only windows the global statistics equal the handle's own."""
    import torch
    from detectmateservice_b200.detector import DeviceDetector
    det = _det()
    det.nccl_init(DeviceDetector.nccl_unique_id() + DeviceDetector.nccl_unique_id(), 0, 1)
    big = big_msg()
    det.process_lines(big, BIG)
    det.window_allreduce(True)
    assert det.window_pending_keys() == BIG - WK
    det.window_allreduce(True)
    assert det.window_pending_keys() == 0
    det.sync()
    assert words(det.global_stats()).tolist() == words(det.stats()).tolist()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for i in range(6):
        det.process_lines(detect_msg(1, seed=10 + i), 0)
        det.window_allreduce(False, streams[i % 2].cuda_stream)
    streams[0].synchronize()                                        # (the wait covers the last import only)
    g = det.global_stats()
    assert words(g).tolist() == words(det.stats()).tolist() and g["lines"] == BIG + 6 * 300
    det.close()


def test_gpu_device_window_world1_drains_without_a_collective():
    """DeviceWindow at world 1 on the torch route: exchange(True) drains the pending keys in two exchanges with no
    process group at all."""
    import torch
    import torch.distributed as dist
    assert not dist.is_initialized()
    det = _det()
    det.process_lines(big_msg(), BIG)
    dw = window.DeviceWindow(det, 0, 1, torch.device("cuda"))
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    assert dw.exchange(True, st.cuda_stream) == 2 and det.window_pending_keys() == 0
    assert dw.exchange(False, st.cuda_stream) == 1
    assert words(det.global_stats()).tolist() == words(det.stats()).tolist()
    det.close()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_main(rank, world, port, trains, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from detectmateservice_b200.detector import DeviceDetector
        det = DeviceDetector(KEYS, device=rank, max_batch_bytes=4 << 20, table_log2_slots=18)
        dw = window.DeviceWindow(det, rank, world, torch.device("cuda", rank))
        dw.init_native(n_comms=2)
        st = torch.cuda.Stream(device=rank)
        m = trains[rank]
        det.process_lines(m, m.count(b"\n"))
        n = dw.exchange(True, st.cuda_stream)
        det.sync()
        q.put((rank, n, det.export_known().tolist()))
        det.close()
    finally:
        dist.destroy_process_group()


def test_gpu_native_route_two_processes():
    """Two processes on two GPUs, DeviceWindow on the native route: rank 0's 70 000 keys reach rank 1 after the
    drain (two exchanges on both ranks)."""
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    trains = [big_msg(), train_set(1)]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(r, 2, port, trains, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = sorted(q.get(timeout=300) for _ in range(2))
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    assert [p.exitcode for p in procs] == [0, 0]
    union = sorted(keys_of(b"".join(trains)))
    assert res[0][1] == res[1][1] == 2 and res[0][2] == res[1][2] == union


# ------------------------------------------------------------------------------------------ the fixes
def test_gpu_import_error_reaches_the_next_call():
    """An import that pushes a 2^10-slot table over its load limit, then process_lines with no sync in between: the
    call raises DM_ERR_TABLE_FULL (the next launch rewrites the batch header, so the import reports into the handle's
    accumulating error word)."""
    import torch
    from detectmateservice_b200 import _lib
    det = _det(log2=10)
    peer = np.arange(1, 601, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    buf = torch.from_numpy(window.pack_window_host([0] * 40, peer, 1, 2, True)).cuda()
    torch.cuda.synchronize()
    det.window_import(buf.data_ptr(), 0, 2, True)
    with pytest.raises(_lib.DmError) as e:
        det.process_lines(b"k=1\n", 0)
    assert e.value.code == _lib.DM_ERR_TABLE_FULL
    det.close()


def test_gpu_global_stats_wait_for_a_side_stream_import():
    """The import enqueued on a side stream held back by a spin: global_stats() called at once returns the imported
    sums, not the statistics from before the import."""
    import torch
    det = _det()
    msg = train_set(0)
    det.process_lines(msg, msg.count(b"\n"))
    want = words(det.stats())
    buf = torch.zeros(det.window_words(1, False), dtype=torch.int64, device="cuda")
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(1 << 30)                                 # ~0.5 s at H100 clocks
        det.window_export(buf.data_ptr(), 0, 1, False, side.cuda_stream)
        det.window_import(buf.data_ptr(), 0, 1, False, side.cuda_stream)
    g = det.global_stats()
    assert words(g).tolist() == want.tolist() and g["lines"] == msg.count(b"\n")
    torch.cuda.synchronize()
    det.close()
