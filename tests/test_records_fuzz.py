"""Record mode against protobuf's own parser: the device walker (dm_k_records, on the CPU emulator here and on the
H100 in the GPU tier), the host framing and training split of dm_process_records, and wire.decode_parser_schema,
all fed with what tests/pbgen.py writes -- non-canonical, mutated and malformed ParserSchema records -- and compared
record by record with oracle/pbrecords.py (upb decides what is well-formed and what each record holds)."""
import random

import numpy as np
import pytest

import pbgen
from detectmateservice_b200 import wire
from oracle import pbrecords

T = 150                                                           # data_use_training of every config below


def _nvd(glob=None, events=None, t=T):
    return {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": t,
                                               "global": glob or {}, "events": events or {}}}}


def _hv(*keys):
    return [{"pos": k} for k in keys]


def _vars(*idx):
    return [{"pos": i} for i in idx]


K64 = "K" * 64
CONFIGS = {
    "global headers": _nvd({"g": {"header_variables": _hv("k", "use", "user", "users", K64, "clé")}}),
    # EventID 0 (records without an EventID must not match it), negative, and 2^31 + 5 as protobuf reads it
    "event scoped": _nvd(events={0: {"e": {"header_variables": _hv("k"), "variables": _vars(0)}},
                                 -7: {"n": {"header_variables": _hv("user"), "variables": _vars(1)}},
                                 -2147483643: {"big": {"header_variables": _hv("k")}},
                                 4: {"f": {"header_variables": _hv("users")}}}),
    "variables": _nvd({"g": {"variables": _vars(0, 1, 31, 39)}}),
    "32 monitors": _nvd({"g": {"header_variables": _hv("k", "use", "user", "users", K64, "clé", "Time", "level"),
                               "variables": _vars(*range(12))}},
                        {4: {"a": {"header_variables": _hv("k", "users"), "variables": _vars(0, 1, 31, 39)}},
                         0: {"b": {"header_variables": _hv("k", "user"), "variables": _vars(0, 2)}},
                         -7: {"c": {"header_variables": _hv("use"), "variables": _vars(39)}}}),
}
COMBO_CFG = {"detectors": {"NewValueComboDetector": {
    "method_type": "new_value_combo_detector", "data_use_training": T,
    "global": {"ku": {"header_variables": _hv("k", "user")}, "uv": {"header_variables": _hv("use"), "variables": _vars(0)}},
    "events": {4: {"kv": {"header_variables": _hv("k"), "variables": _vars(1)}},
               0: {"one": {"header_variables": _hv("users")}},
               -7: {"three": {"header_variables": _hv(K64, "clé"), "variables": _vars(39)}}}}}}
ALL = list(CONFIGS) + ["combos"]


def config(name):
    return (COMBO_CFG, True) if name == "combos" else (CONFIGS[name], False)


def monitors_and_combos(cfg, combo):
    from detectmateservice_b200.component import parse_combos, parse_monitors, select_component_config
    if combo:
        return parse_combos(select_component_config(cfg, "NewValueComboDetector"))
    return parse_monitors(select_component_config(cfg, "NewValueDetector")), []


def monitor_dicts(mons):
    return [{"event_id": m.event_id, "source": m.source, "pos": m.pos} for m in mons]


class EmuRecords:
    """dm_process_records on the CPU emulator: the host framing, the train/bound/detect launches of the library."""

    def __init__(self, cfg, combo):
        import emu_harness
        from detectmateservice_b200 import _lib
        self.mons, self.combos = monitors_and_combos(cfg, combo)
        self.det = emu_harness.EmuDetector([b"\x01m%d" % i for i in range(len(self.mons))], table_log2=14)
        arr = (_lib.Monitor * len(self.mons))()
        for i, m in enumerate(self.mons):
            arr[i].event_id = m.event_id if m.event_id is not None else 0
            arr[i].has_event = 0 if m.event_id is None else 1
            if m.source == "header":
                kb = m.pos.encode()
                arr[i].source, arr[i].key_len = 0, len(kb)
                for j, c in enumerate(kb):
                    arr[i].key[j] = c
            else:
                arr[i].source, arr[i].var_index = 1, m.pos
        self.det.set_monitors(arr, len(self.mons))
        self.det.set_combos(self.combos, (1 << len(self.mons)) - 1 if self.combos else 0)

    def process(self, batch: bytes, n_train: int):
        """-> flags, scores, masks, and the deltas of (bad_records, train_lines, detect_lines, lines)"""
        cap = len(batch) + 1
        f = np.full(cap, 9, np.uint8); s = np.full(cap, -1, np.float32); m = np.full(cap, 0xDEAD, np.uint32)
        st0 = self.det.stats()
        rc, k, n_an = self.det.process_records(batch, n_train, f, s, m, cap)
        assert rc == 0
        st1 = self.det.stats()
        assert n_an == int(f[:k].sum())
        d = {w: st1[w] - st0[w] for w in ("bad_records", "train_lines", "detect_lines", "lines")}
        return f[:k], s[:k], m[:k], d

    def close(self):
        self.det.close()


def split_sizes(r: random.Random, n: int):
    """100, 120 (the training window of T well-formed records ends inside it), then 0..97-record batches."""
    sizes, left = [100, 120], n - 220
    while left > 0:
        k = min(left, r.choice([0, 1, 2, 17, 60, 97]))
        sizes.append(k)
        left -= k
    return sizes


def describe(frames, tags, i):
    return "record %d %r tags=%s" % (i, frames[i][:80], sorted(tags[i]))


def check_stream(run_batch, frames, tags, run, seed):
    """Feeds `frames` in batches through run_batch(batch_bytes, n_train) -> (f, s, m, deltas), as the component does
    (n_train = what is left of the window, counted in well-formed records), and compares each batch with the oracle."""
    r = random.Random(seed + 1000)
    seen_ok, lo, boundary_batches = 0, 0, 0
    for size in split_sizes(r, len(frames)):
        part = frames[lo:lo + size]
        remaining = max(0, T - seen_ok)
        f, s, m, d = run_batch(pbgen.frame(part, r, overlong_p=0.1), remaining)
        n0 = len(run.ok)
        run.feed(part)
        ok = run.ok[n0:]
        assert f.size == size
        for i in range(size):
            want = (run.flags[n0 + i], run.scores[n0 + i], run.masks[n0 + i])
            got = (int(f[i]), float(s[i]), int(m[i]))
            assert got == want, (got, want, describe(frames, tags, lo + i))
        n_ok = sum(ok)
        trained = min(remaining, n_ok)
        assert d["bad_records"] == size - n_ok and d["train_lines"] == trained and d["lines"] == size
        if 0 < remaining < n_ok:                                  # the window ends inside this batch
            bound = [j for j in range(size) if ok[j]][remaining - 1] + 1
            assert d["detect_lines"] == size - bound
            if not all(ok[:bound]) and bound < size:
                boundary_batches += 1
        seen_ok += n_ok
        lo += size
    return boundary_batches


SEEDS = list(range(20))


@pytest.mark.parametrize("seed", SEEDS)
def test_emu_records_match_protobuf(seed):
    name = ALL[seed % len(ALL)]
    cfg, combo = config(name)
    frames, tags = pbgen.Gen(seed).records(600)
    run = pbrecords.new_run(cfg, combo)
    emu = EmuRecords(cfg, combo)
    try:
        n_boundary = check_stream(emu.process, frames, tags, run, seed)
    finally:
        emu.close()
    assert n_boundary == 1, "the training window should end inside a batch, behind malformed records"
    assert sum(run.flags) >= 10 and 0 < run.n_bad < len(frames) // 2


@pytest.mark.parametrize("seed", SEEDS)
def test_host_decoder_matches_protobuf(seed):
    """decode_parser_schema(strict=False) refuses exactly what upb refuses (and groups) and reads the same values."""
    frames, tags = pbgen.Gen(seed).records(600)
    for i, fr in enumerate(frames):
        want = pbrecords.parse(fr)
        try:
            got = wire.decode_parser_schema(fr, strict=False)
        except wire.WireError:
            got = None
        if want is None or got is None:
            assert want is None and got is None, (want, got, describe(frames, tags, i))
            continue
        assert (got["EventID"], got["variables"], got["logFormatVariables"], got["logID"]) == (
            want["EventID"], want["variables"], want["logFormatVariables"], want["logID"]), describe(frames, tags, i)


def test_generator_covers_the_encodings():
    """The fuzz corpus holds every encoding it is meant to exercise, and both outcomes of each mutation."""
    bad, good = set(), set()
    long_lens = set()
    for seed in SEEDS:
        frames, tags = pbgen.Gen(seed).records(600)
        for fr, tg in zip(frames, tags):
            ok = pbrecords.parse(fr) is not None
            for t in tg:
                key = t.split(" at ")[0].split(" byte ")[0].split(" (")[0]
                (good if ok else bad).add(key)
            for n in (127, 128, 16383, 16384):
                if b"L" * (n - 4) in fr:
                    long_lens.add(n)
    for t in ["shuffled", "EventID overlong", "EventID repeated", "EventID 10th-byte overflow", "entry: key only",
              "entry: value only", "entry: value before key", "entry: repeated key/value", "entry: empty",
              "entry: foreign field", "unknown wt0", "unknown wt1", "unknown wt2", "unknown wt5", "mistyped known field",
              "empty record", "singular string repeated"]:
        assert t in good, t
    for t in ["cut", "flip", "invalid UTF-8", "field 0", "11-byte varint", "fixed64 cut short", "fixed32 cut short",
              "LEN past the record", "group", "6-byte tag", "wire type 4/6/7"]:
        assert t in bad, t
    assert "tag" in bad                                           # a tag of 2^32 or more aliasing a monitored field
    assert long_lens >= {127, 128, 16383}


# ------------------------------------------------------------------ the findings, one test each
FIND_CFG = _nvd({"g": {"header_variables": _hv("k"), "variables": _vars(0)}}, {4: {"e": {"header_variables": _hv("k")}}}, t=1)
BASE = wire.encode_parser_schema({"EventID": 4, "variables": ["a"], "logFormatVariables": {"k": "v"}})


def finding(frame):
    """(device, oracle, host) outcome of `frame` after BASE trained: device = (flag, score, mask, bad_records delta),
    oracle = (flag, score, mask, malformed), host = decode_parser_schema(strict=False) or None if it raised."""
    emu = EmuRecords(FIND_CFG, False)
    run = pbrecords.new_run(FIND_CFG)
    try:
        emu.process(pbgen.frame([BASE]), 1)
        run.feed([BASE])
        f, s, m, d = emu.process(pbgen.frame([frame]), 0)
    finally:
        emu.close()
    run.feed([frame])
    try:
        host = wire.decode_parser_schema(frame, strict=False)
    except wire.WireError:
        host = None
    return (int(f[0]), float(s[0]), int(m[0]), d["bad_records"]), (run.flags[-1], run.scores[-1], run.masks[-1], not run.ok[-1]), host


MALFORMED = (0, 0.0, 0, 1)


@pytest.mark.parametrize("tail", [b"\x69\x00\x00\x00", b"\x6d\x00"], ids=["fixed64", "fixed32"])
def test_fixed_width_field_cut_short_is_malformed(tail):
    dev, orc, host = finding(BASE + tail)
    assert orc == (0, 0.0, 0, True) and dev == MALFORMED and host is None


def test_field_number_zero_is_malformed():
    dev, orc, host = finding(b"\x00\x01" + BASE)
    assert orc == (0, 0.0, 0, True) and dev == MALFORMED and host is None


def test_tag_above_2_32_does_not_alias_variables():
    # 0x32 | 1 << 35: truncated to 32 bits it is field 6, and variables[0] = "z" would raise an alert
    dev, orc, host = finding(b"\xb2\x80\x80\x80\x80\x01\x01z" + BASE)
    assert orc == (0, 0.0, 0, True) and dev == MALFORMED and host is None


@pytest.mark.parametrize("frame", [wire.encode_parser_schema({"EventID": 4, "variables": [b"\xff"], "logFormatVariables": {"k": "v"}}),
                                   BASE + b"\x4a\x01\xff"], ids=["monitored-variable", "log"])
def test_invalid_utf8_in_string_field_is_malformed(frame):
    dev, orc, host = finding(frame)
    assert orc == (0, 0.0, 0, True) and dev == MALFORMED and host is None


def test_invalid_utf8_values_are_not_merged_on_the_single_record_path():
    """b"\\xff" and b"\\xfe" used to become the same U+FFFD value on the host and two values on the device; both are
    now refused on both paths."""
    for b in (b"\xff", b"\xfe"):
        with pytest.raises(wire.WireError):
            wire.decode_parser_schema(wire.encode_parser_schema({"variables": [b]}), strict=False)


def test_map_entry_with_foreign_len_field_is_dropped():
    # upb drops the entry, so k stays "v" (known): no alert
    dev, orc, host = finding(BASE + b"\x52\x09\x0a\x01k\x1a\x01q\x12\x01z")
    assert orc == (0, 0.0, 0, False) and dev == (0, 0.0, 0, 0) and host["logFormatVariables"] == {"k": "v"}


@pytest.mark.parametrize("entry", [b"\x0a\x01k\x18\x05\x12\x01z", b"\x08\x05\x0a\x01k\x12\x01z"], ids=["varint-field-3", "varint-key"])
def test_map_entry_with_foreign_varint_field_is_dropped(entry):
    dev, orc, host = finding(BASE + b"\x52" + bytes([len(entry)]) + entry)
    assert orc == (0, 0.0, 0, False) and dev == (0, 0.0, 0, 0) and host["logFormatVariables"] == {"k": "v"}


def test_group_is_malformed_by_design():
    """upb skips a group as an unknown field; the product refuses it (proto3 cannot declare groups)."""
    frame = BASE + b"\x6b\x08\x01\x6c"
    from oracle.schemas import ParserSchema
    ParserSchema().ParseFromString(frame)                         # upb accepts it ...
    assert pbrecords.parse(frame) is None                         # ... the oracle harness counts it malformed
    dev, orc, host = finding(frame)
    assert dev == MALFORMED and host is None


def test_malformed_record_takes_no_training_slot():
    """A malformed record inside the training window: the batch path trains on the same records as the per-record
    path (which raises before counting) and the oracle (which raises before step())."""
    cfg = _nvd({"g": {"variables": _vars(0)}}, t=2)
    recs = [wire.encode_parser_schema({"variables": [v]}) for v in ("a", "b", "c")]
    frames = [recs[0], b"\x32\x01\xff", recs[1], recs[2]]        # the second record is malformed
    emu = EmuRecords(cfg, False)
    try:
        f, s, m, d = emu.process(pbgen.frame(frames), 2)
    finally:
        emu.close()
    run = pbrecords.new_run(cfg).feed(frames)
    assert run.flags == [0, 0, 0, 1]                              # "b" is trained, "c" is new
    assert f.tolist() == run.flags and d == {"bad_records": 1, "train_lines": 2, "detect_lines": 1, "lines": 4}


# ------------------------------------------------------------------ GPU tier: the library on the H100
class DeviceRecords:
    def __init__(self, cfg, combo, max_batch_bytes=4 << 20, max_lines=1 << 16):
        from detectmateservice_b200.detector import DeviceDetector
        self.mons, self.combos = monitors_and_combos(cfg, combo)
        self.det = DeviceDetector([b"\x01m%d" % i for i in range(len(self.mons))], max_batch_bytes=max_batch_bytes,
                                  max_lines=max_lines, table_log2_slots=16)
        self.det.set_monitors(monitor_dicts(self.mons))
        if self.combos:
            self.det.set_combos(self.combos, member_only_mask=(1 << len(self.mons)) - 1)

    def process(self, batch: bytes, n_train: int):
        st0 = self.det.stats()
        f, s, m = self.det.process_records(batch, n_train_records=n_train)
        st1 = self.det.stats()
        assert self.det.last_n_anomalies == int(f.sum())
        return f, s, m, {w: st1[w] - st0[w] for w in ("bad_records", "train_lines", "detect_lines", "lines")}

    def close(self):
        self.det.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_gpu_records_match_protobuf(seed):
    name = ALL[seed % len(ALL)]
    cfg, combo = config(name)
    frames, tags = pbgen.Gen(seed).records(600)
    run = pbrecords.new_run(cfg, combo)
    dev = DeviceRecords(cfg, combo)
    try:
        assert check_stream(dev.process, frames, tags, run, seed) == 1
    finally:
        dev.close()


def _small_corpus(seed, n_distinct=300):
    g = pbgen.Gen(seed, novel=0.3, long_p=0.0, max_vars=3)
    return g.records(n_distinct)[0]


@pytest.mark.gpu
def test_gpu_grid_stride_message():
    """One message of more than twice as many records as the grid has threads (sm_count * 16 CTAs of 128), so that
    every launch's grid-stride loop makes at least three passes; training ends deep inside it."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 2 * sms * 16 * 128 + 4099
    cfg, _ = config("32 monitors")
    corpus = _small_corpus(5)
    r = random.Random(6)
    # training draws from two thirds of the corpus, detection from all of it
    frames = [corpus[r.randrange(200 if i < 50000 else len(corpus))] for i in range(n)]
    msg = pbgen.frame(frames)
    run = pbrecords.new_run(_nvd(cfg["detectors"]["NewValueDetector"]["global"], cfg["detectors"]["NewValueDetector"]["events"],
                                 t=20000)).feed(frames)
    assert 0 < run.n_bad and sum(run.flags) > 0
    dev = DeviceRecords(cfg, False, max_batch_bytes=len(msg) + 4096, max_lines=n + 16)
    try:
        f, s, m, d = dev.process(msg, 20000)
    finally:
        dev.close()
    assert f.size == n
    assert (f == np.array(run.flags, np.uint8)).all() and (s == np.array(run.scores, np.float32)).all()
    assert (m == np.array(run.masks, np.uint32)).all()
    bound = [j for j in range(n) if run.ok[j]][20000 - 1] + 1
    assert d == {"bad_records": run.n_bad, "train_lines": 20000, "detect_lines": n - bound, "lines": n}


@pytest.mark.gpu
def test_gpu_large_record():
    """A single 8 MiB record (4-byte length prefix) among small ones, its variables[0] a 1 MiB value."""
    cfg, _ = config("variables")
    corpus = _small_corpus(8)
    big_val = ("€" * ((1 << 20) // 3)).encode() + b"v"            # 1 MiB of 3-byte UTF-8
    head = pbgen.ld(pbgen.VARIABLES, big_val) + pbgen.ld(pbgen.VARIABLES, b"a")
    n_log = (8 << 20) - len(head) - 5                             # field 9: 1-byte tag, 4-byte length
    filler = ("x" * 1000 + "é").encode()
    big = head + pbgen.ld(pbgen.LOG, filler * (n_log // len(filler)) + b"x" * (n_log % len(filler)))
    assert len(big_val) == 1 << 20 and len(big) == 8 << 20 and len(pbgen.frame([big])) - len(big) == 4
    assert pbrecords.parse(big) is not None
    train = corpus[:200]
    detect = corpus[200:] + [big] + corpus[:50]
    run = pbrecords.new_run(cfg)
    dev = DeviceRecords(cfg, False, max_batch_bytes=16 << 20, max_lines=1 << 12)
    try:
        for part, n_train in ((train, T), (detect, 0)):
            f, s, m, d = dev.process(pbgen.frame(part), n_train)
            n0 = len(run.ok)
            run.feed(part)
            assert f.tolist() == run.flags[n0:] and s.tolist() == run.scores[n0:] and m.tolist() == run.masks[n0:]
            assert d["bad_records"] == run.ok[n0:].count(False)
    finally:
        dev.close()
    assert run.masks[len(train) + len(corpus) - 200] & 1          # the 1 MiB value is new


def _component(combo, fmt):
    from detectmateservice_b200.component import B200NewValueComboDetector, B200NewValueDetector
    if combo:
        cfg = {"detectors": {"NewValueComboDetector": dict(COMBO_CFG["detectors"]["NewValueComboDetector"], input_format=fmt)}}
        comp = B200NewValueComboDetector(config=cfg)
    else:
        cfg = {"detectors": {"NewValueDetector": dict(CONFIGS["32 monitors"]["detectors"]["NewValueDetector"], input_format=fmt)}}
        comp = B200NewValueDetector(name="NewValueDetector", config=cfg)
    comp.clock = lambda: 1773848383
    return comp


def _alert_fields(blob):
    a = wire.decode_detector_schema(blob)
    return (a["alertsObtain"], a["score"], a["alertID"], a["logIDs"], a["extractedTimestamps"], a["detectorID"])


@pytest.mark.gpu
@pytest.mark.parametrize("combo", [False, True], ids=["NewValueDetector", "NewValueComboDetector"])
@pytest.mark.parametrize("path", ["single", "batch", "alternating"])
def test_gpu_component_delivery_paths(path, combo):
    """One record stream, malformed records inside and after the training window, delivered one record per message,
    in batches, or alternating: the same alerts as the oracle, and the same training split."""
    frames, _ = pbgen.Gen(31 + combo).records(600)
    frames = [f for f in frames if f]                             # (an empty message is no record on the per-message path)
    run = pbrecords.new_run(COMBO_CFG if combo else CONFIGS["32 monitors"], combo).feed(frames)
    ok_rank = np.cumsum(run.ok)
    assert not all(run.ok[:200]) and not all(run.ok[300:])
    comp = _component(combo, "parser_schema" if path == "single" else "parser_schema_batch")
    r = random.Random(7)
    got, lo, k = [], 0, 0
    try:
        while lo < len(frames):
            single = path == "single" or (path == "alternating" and k % 2 == 0)
            size = 1 if single else min(len(frames) - lo, r.choice([1, 17, 60, 97]))
            part = frames[lo:lo + size]
            n_seen0 = comp.n_seen
            if single:
                comp.input_format = "parser_schema"
                try:
                    out = comp.process(part[0])
                except wire.WireError:
                    assert not run.ok[lo], lo                     # malformed: raises, takes no training slot
                    assert comp.n_seen == n_seen0
                    out = None
                else:
                    assert run.ok[lo], lo
                outs = [out] if out else []
            else:
                comp.input_format = "parser_schema_batch"
                out = comp.process(pbgen.frame(part))
                outs = wire.split_delimited(out) if out else []
                assert len(outs) == sum(run.flags[lo:lo + size])   # every flagged record worded, none skipped
            assert comp.n_seen == ok_rank[lo + size - 1]
            got += outs
            lo += size
            k += 1
        st = comp.stats()
    finally:
        comp.close()
    want = run.outputs
    assert len(got) == len(want) == sum(run.flags) > 0
    for g, w in zip(got, want):
        assert _alert_fields(g) == _alert_fields(w)
    assert st["train_lines"] == T
    if path == "batch" or combo:                                  # (the per-record path decodes on the host)
        assert st["bad_records"] == run.n_bad
