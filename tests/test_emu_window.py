"""The multi-GPU window exchange's kernel SOURCES (dm_kernels_window.cuh: dm_k_window_export / dm_k_window_import) on
the CPU emulator.  N emulated handles stand in for N ranks, and the sum of their export buffers for the sum all-reduce.
A rank segment carries SEG = 64 keys here (libdmdetect: 65536, the same code with another cap), so that a few hundred
keys take several windows of carry-over.  References: the single-rank NativeOracle trained on every training record,
window.pack_window_host for the buffer, and the sum of the per-rank statistics for the global ones (known_keys aside:
the export sends it as 0).  The same scenarios run on the H100 with the real cap in test_gpu_window.py."""
import numpy as np
import pytest

import emu_harness
from detectmateservice_b200 import window
from oracle import fingerprint
from oracle.native import NativeOracle

SEG = 64
KEYS = [b"k", b"t"]
WORLDS = [1, 2, 3, 5, 8]
DEVERR_TABLE_FULL = 1


@pytest.fixture(params=["stream", "lanes"])
def variant(request):
    """The key=value kernels: the stream kernel (default) and one thread per record."""
    return request.param


def kv(pairs):
    """key=value records: one per (k, t) pair."""
    return b"".join(b"k=%s t=%s\n" % (str(a).encode(), str(b).encode()) for a, b in pairs)


def keys_of(msg, keys=KEYS):
    """The table keys training on every record of msg learns."""
    o = NativeOracle(keys)
    o.process(msg, msg.count(b"\n"))
    return {fingerprint.table_key(i, v) for i in range(len(keys)) for v in o.known_values(i)}


def words(d, glob=False):
    """The 40 dm_stats_t words of a handle's statistics (every unknown-value counter, combinations' included) or of its
    global statistics; known_keys (word 6) as the export sends it: 0."""
    w = np.zeros(40, np.uint64)
    (d.lib.emu_get_global_stats if glob else d.lib.emu_get_stats)(d.h, w.ctypes.data_as(emu_harness._P64))
    if glob:
        assert w[6] == 0
    w[6] = 0
    return w


def summed(dets):
    """The sum of the ranks' statistics words: what the global statistics must be."""
    return sum((words(d) for d in dets), np.zeros(40, np.uint64))


class Ranks:
    """`world` emulated handles, one per rank."""

    def __init__(self, world, variant, keys=KEYS, table_log2=12, dets=None, seg=SEG):
        self.world, self.seg = world, seg
        self.dets = dets or [emu_harness.EmuDetector(keys, table_log2=table_log2, variant=variant) for _ in range(world)]

    def close(self):
        for d in self.dets:
            d.close()

    def export(self, with_keys):
        return [d.window_export(r, self.world, with_keys, self.seg) for r, d in enumerate(self.dets)]

    def import_(self, bufs, with_keys):
        total = np.sum(np.stack(bufs), axis=0, dtype=np.uint64)                  # the all-reduce
        errs = [d.window_import(total, r, self.world, with_keys, self.seg) for r, d in enumerate(self.dets)]
        assert errs == [0] * self.world
        return total

    def window(self, with_keys):
        """One exchange; returns the export buffers."""
        bufs = self.export(with_keys)
        self.import_(bufs, with_keys)
        return bufs

    def segment(self, buf, r):
        return window.unpack_window_host(buf, self.world, True, self.seg)[1][r]

    def detect(self, msgs):
        """Each rank detects its message; flags, scores and (record, mask) of the anomalies, concatenated in rank
        order."""
        f, s, an, base = [], [], [], 0
        for d, m in zip(self.dets, msgs):
            fr, sr = d.process_lines(m, 0)
            f.append(fr.copy()); s.append(sr.copy())
            an += [(base + a[0], a[1]) for a in d.anomalies()]
            base += fr.size
        return np.concatenate(f), np.concatenate(s), an


def shards(msg, world):
    cuts = window.shard_bounds(msg, world)
    return [msg[cuts[r]:cuts[r + 1]] for r in range(world)]


def oracle_detect(train, detect, keys=KEYS):
    o = NativeOracle(keys)
    o.process(train, train.count(b"\n"))
    f, s, m = o.process(detect, 0, want_masks=True)
    return f, s, [(i, int(m[i])) for i in np.nonzero(f)[0]]


def check_detection(ranks, train, detect, keys=KEYS):
    wf, ws, wan = oracle_detect(train, detect, keys)
    f, s, an = ranks.detect(shards(detect, ranks.world))
    assert f.tolist() == wf.tolist() and s.tolist() == ws.tolist() and an == wan
    assert wf.sum() > 0


def train_set(r, n=48, seed=0):
    """A training shard: values shared by every rank and values only rank r sees (fewer than SEG keys in all)."""
    rng = np.random.default_rng(seed * 100 + r)
    return kv([(int(rng.integers(0, 6)), "r%d_%d" % (r, i % 17)) if i % 3 else ("x%d_%d" % (r, i % 9), i % 4)
               for i in range(n)])


def detect_msg(world, seed=0, n=300):
    """Records mixing every rank's values, the shared ones and values nobody trained on."""
    rng = np.random.default_rng(1000 + seed)
    out = []
    for i in range(n):
        r = int(rng.integers(0, world))
        a = int(rng.integers(0, 8)) if i % 2 else "x%d_%d" % (r, int(rng.integers(0, 11)))
        b = "r%d_%d" % (r, int(rng.integers(0, 19))) if i % 5 else int(rng.integers(0, 5))
        out.append((a, b))
    return kv(out)


@pytest.mark.parametrize("world", WORLDS)
def test_export_bytes_equal_host_mirror_and_detection_matches_oracle(world, variant):
    """Every rank's export buffer is pack_window_host(its delta, its learnt keys) word for word: 0 outside its own
    segment, so the sum is a concatenation.  After the import, every rank knows the union and detects its shard as
    the single-rank oracle detects the whole message; a statistics-only window then sums the detection statistics."""
    trains = [train_set(r) for r in range(world)]
    train = b"".join(trains)
    R = Ranks(world, variant)
    for d, m in zip(R.dets, trains):
        d.process_lines(m, m.count(b"\n"))
    want_stats = [words(d) for d in R.dets]
    bufs = R.export(True)
    for r, (d, buf) in enumerate(zip(R.dets, bufs)):
        seg = R.segment(buf, r)
        assert sorted(seg.tolist()) == sorted(keys_of(trains[r])) and d.window_pending_keys() == 0
        assert buf.tolist() == window.pack_window_host(want_stats[r], seg, r, world, True, SEG).view(np.uint64).tolist()
    R.import_(bufs, True)
    union = sorted(keys_of(train))
    for d in R.dets:
        assert d.export_known() == union and d.stats()["known_keys"] == len(union)
        assert d.global_stats() == R.dets[0].global_stats()
    assert words(R.dets[0], True).tolist() == sum(want_stats).tolist()
    detect = detect_msg(world)
    check_detection(R, train, detect)
    bufs = R.window(False)
    assert all(b.size == 40 for b in bufs)
    g = R.dets[0].global_stats()
    assert words(R.dets[0], True).tolist() == summed(R.dets).tolist()
    assert g["lines"] == train.count(b"\n") + detect.count(b"\n") and g["known_keys"] == 0
    R.close()


@pytest.mark.parametrize("world", WORLDS)
def test_rank_learning_more_than_the_cap_drains_over_several_windows(world, variant):
    """Rank 0 learns 3 * SEG + 21 keys in one training window: the first export reports exactly learnt - SEG pending,
    each later keys window carries the next SEG (the last one the rest), none twice; then every rank knows the union
    and detects as the oracle does."""
    big = kv([(i, "big%d" % (i % 50)) for i in range(3 * SEG + 21 - 50)])
    trains = [big] + [train_set(r) for r in range(1, world)]
    train = b"".join(trains)
    learnt = keys_of(big)
    assert len(learnt) == 3 * SEG + 21
    R = Ranks(world, variant)
    for d, m in zip(R.dets, trains):
        d.process_lines(m, m.count(b"\n"))
    shipped, n_windows = [], 0
    while True:
        bufs = R.export(True)
        n_windows += 1
        seg = R.segment(bufs[0], 0).tolist()
        left = len(learnt) - len(shipped)
        assert len(seg) == min(SEG, left) and R.dets[0].window_pending_keys() == left - len(seg)
        assert all(d.window_pending_keys() == 0 for d in R.dets[1:])
        if n_windows > 1:
            assert all(R.segment(b, r).size == 0 for r, b in enumerate(bufs) if r)
        shipped += seg
        R.import_(bufs, True)
        if max(d.window_pending_keys() for d in R.dets) == 0:
            break
    assert n_windows == 4 and len(set(shipped)) == len(shipped) and set(shipped) == learnt
    union = sorted(keys_of(train))
    for d in R.dets:
        assert d.export_known() == union
    # the drained windows carried no statistics twice
    assert words(R.dets[-1], True).tolist() == summed(R.dets).tolist()
    check_detection(R, train, detect_msg(world, seed=1) + kv([(i, "big%d" % i) for i in range(0, 400, 7)]))
    # a window with keys after the drain carries nothing
    bufs = R.window(True)
    assert all(R.segment(b, r).size == 0 for r, b in enumerate(bufs))
    R.close()


@pytest.mark.parametrize("world", WORLDS)
def test_several_training_windows(world, variant):
    """Three training windows with statistics-only windows between them.  Each keys window carries only the keys each
    rank learnt since the previous one; statistics-only windows carry no keys and do not move the export position; a
    key that two ranks learn in the same window is inserted once, so known_keys is the size of the union."""
    R = Ranks(world, variant)
    known = set()
    all_train = b""
    for w in range(3):
        trains = [train_set(r, n=30, seed=w) + kv([("new%d" % w, "both%d" % w)]) for r in range(world)]
        novel = []
        for d, m in zip(R.dets, trains):
            d.process_lines(m, m.count(b"\n"))
            novel.append(keys_of(m) - known)
        all_train += b"".join(trains)
        for _ in range(w):                                       # statistics-only windows in between
            assert [b.size for b in R.window(False)] == [40] * world
        bufs = R.export(True)
        segs = [set(R.segment(b, r).tolist()) for r, b in enumerate(bufs)]
        assert segs == novel
        total = R.import_(bufs, True)
        per_rank = window.unpack_window_host(total, world, True, SEG)[1]
        assert sum(p.size for p in per_rank) == sum(len(n) for n in novel)
        known |= set().union(*novel)
        assert known == keys_of(all_train)
        for d in R.dets:
            assert d.export_known() == sorted(known) and d.stats()["known_keys"] == len(known)
        assert words(R.dets[0], True).tolist() == summed(R.dets).tolist()
    check_detection(R, all_train, detect_msg(world, seed=2) + kv([("new1", "both2"), ("new2", "both2")]))
    R.close()


@pytest.mark.parametrize("world", [2, 5])
def test_two_windows_in_flight_imported_out_of_order(world, variant):
    """Windows A and B exported on every rank before either is imported, B imported before A: the global statistics
    are still the sum of the per-rank ones, and a third window's delta is exactly what changed since B's export."""
    R = Ranks(world, variant)
    trains = [train_set(r) for r in range(world)]
    for d, m in zip(R.dets, trains):
        d.process_lines(m, m.count(b"\n"))
    R.window(True)
    msgs = [shards(detect_msg(world, seed=s), world) for s in range(3)]
    for d, m in zip(R.dets, msgs[0]):
        d.process_lines(m, 0)
    a = R.export(False)
    for d, m in zip(R.dets, msgs[1]):
        d.process_lines(m, 0)
    before_c = [words(d) for d in R.dets]
    b = R.export(True)                                            # (B with keys: none are pending)
    R.import_(b, True)
    R.import_(a, False)
    assert words(R.dets[0], True).tolist() == summed(R.dets).tolist()
    for d in R.dets[1:]:
        assert d.global_stats() == R.dets[0].global_stats()
    for d, m in zip(R.dets, msgs[2]):
        d.process_lines(m, 0)
    c = R.export(False)
    for r, d in enumerate(R.dets):
        assert c[r].tolist() == (words(d) - before_c[r]).tolist()
    R.import_(c, False)
    assert words(R.dets[0], True).tolist() == summed(R.dets).tolist()
    R.close()


@pytest.mark.parametrize("world", [2, 3])
def test_imported_keys_are_not_reshipped(world, variant):
    """Keys a rank received from its peers or through import_known never appear in its next export, even when its own
    records then carry those values: only the keys new to its table travel."""
    R = Ranks(world, variant)
    trains = [train_set(r) for r in range(world)]
    for d, m in zip(R.dets, trains):
        d.process_lines(m, m.count(b"\n"))
    R.window(True)
    restored = kv([("restored%d" % i, "old") for i in range(10)])
    assert R.dets[0].import_known(sorted(keys_of(restored))) == 0
    fresh = kv([("fresh%d" % i, 1) for i in range(5)])
    again = trains[-1] + restored + fresh                         # a peer's records, the restored ones, new values
    R.dets[0].process_lines(again, again.count(b"\n"))
    bufs = R.export(True)
    assert set(R.segment(bufs[0], 0).tolist()) == keys_of(fresh) - keys_of(b"".join(trains) + restored)
    assert all(R.segment(b, r).size == 0 for r, b in enumerate(bufs) if r)
    R.import_(bufs, True)
    # the peers learn the new keys, not the restored ones
    for d in R.dets[1:]:
        assert d.export_known() == sorted(keys_of(b"".join(trains) + fresh))
    R.close()


def test_import_over_the_load_limit_reports_table_full():
    """An import that pushes the table over its load limit (half its slots) reports DM_DEVERR_TABLE_FULL."""
    d = emu_harness.EmuDetector(KEYS, table_log2=10)
    peer = np.arange(1, 601, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    buf = window.pack_window_host([0] * 40, peer, 1, 2, True, 1024).view(np.uint64)
    assert d.window_import(buf, 0, 2, True, 1024) == DEVERR_TABLE_FULL
    d.close()


# ------------------------------------------------------------------------------------------ log_format and combinations
@pytest.mark.parametrize("combos", [False, True], ids=["log_format", "log_format_combos"])
@pytest.mark.parametrize("world", [2, 3])
def test_log_format_and_combination_keys_travel_like_values(world, combos, golden_dir):
    """The golden audit sample in log_format mode with the audit templates, single monitors and (second case) the
    NewValueComboDetector instances of AUDIT_COMBO_CFG: the ranks train on shards of its first 250 records, exchange
    their keys (16 per rank segment: several windows) and detect shards of the rest as FormatComboOracle does on one
    rank."""
    import os
    from test_format_combos import AUDIT, AUDIT_COMBO_CFG, NAME, EmuFormatCombo, FormatComboOracle, _mons_combos
    from detectmateservice_b200.logformat import load_templates
    tm = load_templates(os.path.join(golden_dir, "audit_templates.txt"))
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read()
    lines = buf.split(b"\n")[:-1]
    n_train = 250
    train = b"".join(ln + b"\n" for ln in lines[:n_train])
    detect = b"".join(ln + b"\n" for ln in lines[n_train:])
    mons, cmb = _mons_combos(AUDIT_COMBO_CFG)
    cmb = cmb if combos else []
    member_only = ((1 << len(mons)) - 1) & ~1 if combos else 0   # with combinations, only `type` alerts on its own
    cfg = {"detectors": {NAME: dict(AUDIT_COMBO_CFG["detectors"][NAME], data_use_training=n_train)}}
    wf, ws, wm, _, _ = FormatComboOracle(cfg, AUDIT, tm, combos=cmb, member_only=member_only).process_lines(buf)
    one = EmuFormatCombo(mons, cmb, member_only, AUDIT, tm)
    one.process(train, n_train)
    union = one.det.export_known()
    one.det.close()
    ranks = [EmuFormatCombo(mons, cmb, member_only, AUDIT, tm) for _ in range(world)]
    R = Ranks(world, None, dets=[e.det for e in ranks], seg=16)
    for e, m in zip(ranks, shards(train, world)):
        e.process(m, m.count(b"\n"))
    n_windows = 1
    R.window(True)
    while max(d.window_pending_keys() for d in R.dets):
        R.window(True)
        n_windows += 1
    assert n_windows > 1
    for d in R.dets:
        assert d.export_known() == union
    f, s, an = [], [], {}
    for e, m in zip(ranks, shards(detect, world)):
        fr, sr, ar, _ = e.process(m, 0)
        an.update({len(f) + i: mk for i, (mk, _) in ar.items()})
        f += fr; s += sr
    assert f == wf[n_train:] and s == ws[n_train:] and sum(f) > 0
    assert an == {i: m for i, m in enumerate(wm[n_train:]) if m}
    R.window(False)                                                # combination counters travel as well
    assert words(R.dets[0], True).tolist() == summed(R.dets).tolist()
    R.close()
