"""NewValueComboDetector (SURVEY.md section 8f-4): tuples of field values.  Oracle semantics (R-combo,
oracle/nvcd.py -- parity unpinned, defined by us), the kernel source on the CPU emulator,
the component's alert wording against the oracle, and (GPU tier) the real library."""

import numpy as np
import pytest

from detectmateservice_b200 import wire
from oracle.nvcd import NewValueComboDetectorOracle
from oracle import schemas as oschemas

CFG = {"detectors": {"NewValueComboDetector": {
    "method_type": "new_value_combo_detector", "data_use_training": 400, "auto_config": False, "params": {},
    "global": {"who_where": {"header_variables": [{"pos": "user"}, {"pos": "host"}]}},
    "events": {1: {"instance_1": {"params": {}, "variables": [{"pos": 0, "name": "var_0"}, {"pos": 1, "name": "var_1"}]},
                   "instance_2": {"params": {}, "variables": [{"pos": 1, "name": "var_1"}], "header_variables": [{"pos": "user"}]}},
               2: {"single": {"variables": [{"pos": 0}]}}}}}}


def make_records(n, seed=11):
    r = np.random.Generator(np.random.PCG64(seed))
    recs = []
    for i in range(n):
        late = i >= n // 2
        lfv = {"Time": str(1634567890 + i)}
        if r.random() < 0.9:
            lfv["user"] = "u%d" % r.integers(0, 6 if late else 4)
        if r.random() < 0.9:
            lfv["host"] = "h%d" % r.integers(0, 5 if late else 3)
        rec = {"EventID": [1, 2, 3][int(r.integers(0, 3))], "logID": str(i),
               "variables": ["v%d" % r.integers(0, 5 if late else 3) for _ in range(int(r.integers(0, 4)))],
               "logFormatVariables": lfv}
        recs.append(rec)
    return recs


def oracle_run(recs):
    orc = NewValueComboDetectorOracle(config=CFG, clock=lambda: 1773848383)
    n = len(orc.monitors)
    from oracle.nvcd import combo_alert_key
    keys = [combo_alert_key(orc.monitors, m) for m in orc.combos]
    flags, scores, masks, outs = [], [], [], []
    for rec in recs:
        out = orc.process(wire.encode_parser_schema(rec))
        outs.append(out)
        if out is None:
            flags.append(0); scores.append(0.0); masks.append(0)
            continue
        m = oschemas.DetectorSchema()
        m.ParseFromString(out)
        mask = 0
        for c, k in enumerate(keys):
            if k in m.alertsObtain:
                mask |= 1 << (n + c)
        flags.append(1); scores.append(float(m.score)); masks.append(mask)
    return flags, scores, masks, outs, orc


def test_oracle_semantics_by_hand():
    cfg = {"detectors": {"NewValueComboDetector": {
        "method_type": "new_value_combo_detector", "data_use_training": 3,
        "global": {"g": {"header_variables": [{"pos": "a"}, {"pos": "b"}]}}}}}
    orc = NewValueComboDetectorOracle(config=cfg, clock=lambda: 7)
    recs = [{"a": "1", "b": "x"}, {"a": "2", "b": "y"}, {"a": "1"},          # training: (1,x) (2,y); third lacks b
            {"a": "1", "b": "x"},                                             # known tuple
            {"a": "1", "b": "y"},                                             # both values known, the PAIR is new
            {"a": "1"},                                                       # member missing: skipped
            {"a": "1", "b": "y"}]                                             # detection never inserts
    got = [orc.step({"EventID": None, "variables": [], "logFormatVariables": r}) for r in recs]
    assert [g[0] for g in got] == [False, False, False, False, True, False, True]
    assert got[4] == (True, 1.0, {"Global - (a, b)": "Unknown value combination: ('1', 'y')"})
    out = orc.make_output({"logID": "9"}, 1.0, got[4][2])
    assert out.detectorType == "new_value_combo_detector" and out.alertID == "10"
    assert out.description == "NewValueComboDetector detects value combinations not encountered in training as anomalies."


def test_component_config_matches_oracle():
    from detectmateservice_b200.component import parse_combos, select_component_config
    mons, combos = parse_combos(select_component_config(CFG, "NewValueComboDetector"))
    orc = NewValueComboDetectorOracle(config=CFG)
    assert combos == orc.combos == [[0, 1], [2, 3], [4, 5], [6]]
    assert [(m.event_id, m.source, m.pos) for m in mons] == [(m.event_id, m.source, m.pos) for m in orc.monitors]


def _monitor_array(mons):
    from detectmateservice_b200 import _lib
    arr = (_lib.Monitor * len(mons))()
    for i, m in enumerate(mons):
        arr[i].event_id = m.event_id if m.event_id is not None else 0
        arr[i].has_event = 0 if m.event_id is None else 1
        if m.source == "header":
            kb = m.pos.encode()
            arr[i].source, arr[i].key_len = 0, len(kb)
            for j, c in enumerate(kb):
                arr[i].key[j] = c
        else:
            arr[i].source, arr[i].var_index = 1, m.pos
    return arr


def test_emu_combo_kernel():
    import emu_harness
    recs = make_records(1000)
    want_f, want_s, want_m, _, orc = oracle_run(recs)
    assert sum(want_f) > 40 and any(s > 1 for s in want_s)
    det = emu_harness.EmuDetector([b"\x01m%d" % i for i in range(len(orc.monitors))], table_log2=12)
    det.set_monitors(_monitor_array(orc.monitors), len(orc.monitors))
    det.set_combos(orc.combos, (1 << len(orc.monitors)) - 1)
    got_f, got_s, got_m, seen = [], [], [], 0
    for lo in range(0, len(recs), 300):
        batch = wire.frame_delimited([wire.encode_parser_schema(r) for r in recs[lo:lo + 300]])
        n_train = max(0, min(300, 400 - seen))
        f = np.full(300, 9, np.uint8); s = np.full(300, -1, np.float32); m = np.zeros(300, np.uint32)
        rc, k, _ = det.process_records(batch, n_train, f, s, m, 300)
        assert rc == 0
        seen += k
        got_f += f[:k].tolist(); got_s += s[:k].tolist(); got_m += m[:k].tolist()
    det.close()
    assert got_f == want_f and got_s == want_s and got_m == want_m


class FakeComboDevice:
    """Stands in for the device in the CPU tier: per-record masks from plain Python sets."""

    def __init__(self, monitors, combos):
        self.monitors, self.combos = monitors, combos
        self.known = [set() for _ in combos]
        self.last_n_anomalies = 0

    def process_records(self, data, n_train_records=0):
        flags, scores, masks = [], [], []
        for r, frame in enumerate(wire.split_delimited(data)):
            rec = wire.decode_parser_schema(frame, strict=False)
            vals = {}
            for i, m in enumerate(self.monitors):
                if m.event_id is not None and m.event_id != rec.get("EventID"):
                    continue
                v = (rec.get("logFormatVariables") or {}).get(m.pos) if m.source == "header" else (
                    rec["variables"][m.pos] if m.pos < len(rec.get("variables") or []) else None)
                if v is not None:
                    vals[i] = v
            mask = 0
            for c, mem in enumerate(self.combos):
                if all(i in vals for i in mem):
                    t = tuple(vals[i] for i in mem)
                    if r < n_train_records:
                        self.known[c].add(t)
                    elif t not in self.known[c]:
                        mask |= 1 << (len(self.monitors) + c)
            flags.append(1 if mask else 0); scores.append(float(bin(mask).count("1"))); masks.append(mask)
        self.last_n_anomalies = sum(flags)
        return np.array(flags, np.uint8), np.array(scores, np.float32), np.array(masks, np.uint32)


def _same_alerts(got_blobs, want_blobs):
    assert len(got_blobs) == len(want_blobs)
    for g, w in zip(got_blobs, want_blobs):
        a = wire.decode_detector_schema(g)
        b = oschemas.DetectorSchema()
        b.ParseFromString(w)
        assert a["alertsObtain"] == dict(b.alertsObtain) and a["score"] == b.score and a["alertID"] == b.alertID
        assert a["logIDs"] == list(b.logIDs) and a["extractedTimestamps"] == list(b.extractedTimestamps)
        assert a["detectorID"] == b.detectorID and a["detectorType"] == b.detectorType and a["description"] == b.description


def test_component_wording_matches_oracle_cpu():
    from detectmateservice_b200.component import B200NewValueComboDetector
    recs = make_records(900, seed=4)
    _, _, _, outs, _ = oracle_run(recs)
    comp = B200NewValueComboDetector(config=CFG)
    comp._det = FakeComboDevice(comp.monitors, comp.combos)
    comp.clock = lambda: 1773848383
    got = []
    for lo in range(0, 600, 200):                                               # batches ...
        out = comp.process(wire.frame_delimited([wire.encode_parser_schema(r) for r in recs[lo:lo + 200]]))
        got += wire.split_delimited(out) if out else []
    for r in recs[600:]:                                                         # ... then one record per message
        out = comp.process(wire.encode_parser_schema(r))
        got += [out] if out else []
    _same_alerts(got, [o for o in outs if o is not None])
    with pytest.raises(ValueError):                                              # not together with a log_format
        B200NewValueComboDetector(config={"detectors": {"NewValueComboDetector": dict(
            CFG["detectors"]["NewValueComboDetector"], params={"log_format": "<A> <B>"})}})


@pytest.mark.gpu
def test_gpu_combo_component_matches_oracle():
    from detectmateservice_b200.component import B200NewValueComboDetector, decode_compact
    recs = make_records(4000, seed=21)
    want_f, want_s, _, outs, _ = oracle_run(recs)
    comp = B200NewValueComboDetector(config=CFG)
    comp.clock = lambda: 1773848383
    got = []
    for lo in range(0, 3000, 500):
        out = comp.process(wire.frame_delimited([wire.encode_parser_schema(r) for r in recs[lo:lo + 500]]))
        got += wire.split_delimited(out) if out else []
    for r in recs[3000:]:
        out = comp.process(wire.encode_parser_schema(r))
        got += [out] if out else []
    _same_alerts(got, [o for o in outs if o is not None])
    st = comp.stats()
    assert st["lines"] == 4000 and st["anomalies"] == sum(want_f) and st["score_sum"] == int(sum(want_s))
    comp.close()
    comp2 = B200NewValueComboDetector(config={"detectors": {"NewValueComboDetector": dict(
        CFG["detectors"]["NewValueComboDetector"], params={"output_format": "compact"})}})
    f, s = decode_compact(comp2.process(wire.frame_delimited([wire.encode_parser_schema(r) for r in recs])))
    assert f.tolist() == want_f and s.tolist() == want_s
    comp2.close()


@pytest.mark.gpu
def test_gpu_set_combos_validation():
    from detectmateservice_b200.detector import DeviceDetector
    from detectmateservice_b200._lib import DmError
    det = DeviceDetector([b"\x01m0", b"\x01m1"], max_batch_bytes=1 << 20)
    with pytest.raises(DmError):
        det.set_combos([[0, 1]])                                                 # before set_monitors
    det.set_monitors([{"event_id": None, "source": "header", "pos": "a"}, {"event_id": None, "source": "variable", "pos": 0}])
    with pytest.raises(DmError):
        det.set_combos([[0, 2]])                                                 # not a monitor index
    with pytest.raises(DmError):
        det.set_combos([[]])                                                     # empty combination
    with pytest.raises(DmError):
        det.set_combos([[0, 1]] * 31)                                            # mask bits exhausted
    det.set_combos([[0, 1], [1, 0]], member_only_mask=1)                         # order matters: two distinct combos
    recs = [{"variables": ["x"], "logFormatVariables": {"a": "y"}}, {"variables": ["y"], "logFormatVariables": {"a": "x"}}]
    det.process_records(wire.frame_delimited([wire.encode_parser_schema(recs[0])]), n_train_records=1)
    f, s, m = det.process_records(wire.frame_delimited([wire.encode_parser_schema(recs[1])]))
    # (a=x, v=y): combo0 (a,v)=(x,y) new, combo1 (v,a)=(y,x) new, monitor 1 (v=y) new; monitor 0 is member-only
    assert f.tolist() == [1] and s.tolist() == [3.0] and m.tolist() == [0b1110]
    det.close()


# ------------------------------------------------------------------------------------------ raw key=value records
RAW_CFG = {"detectors": {"NewValueComboDetector": {
    "method_type": "new_value_combo_detector", "data_use_training": 1500, "auto_config": False,
    "global": {"exe_acct": {"header_variables": [{"pos": "exe"}, {"pos": "acct"}]},
               "type_res_term": {"header_variables": [{"pos": "type"}, {"pos": "res"}, {"pos": "terminal"}]},
               "lonely": {"header_variables": [{"pos": "hostname"}]},
               "never": {"header_variables": [{"pos": "nosuchkey"}, {"pos": "exe"}]}}}}}


def raw_lines(n, seed):
    """Synthetic audit records whose individual values are all seen in training, but whose
    pairs are not: the detection half draws (exe, acct) and (type, res, terminal) independently."""
    r = np.random.Generator(np.random.PCG64(seed))
    exes, accts, types, terms = ["/bin/a", "/bin/b", "/usr/c"], ["root", "bob", "eve"], ["LOGIN", "USER_ACCT", "CRED"], ["tty1", "ssh", "cron"]
    out = []
    for i in range(n):
        train = i < 1500
        e = int(r.integers(0, 3))
        a = e if train and r.random() < 0.9 else int(r.integers(0, 3))             # training: exe and acct mostly correlated
        t = int(r.integers(0, 3))
        ln = 'type=%s msg=audit(%d.000:%d): pid=%d acct="%s" exe="%s" hostname=%s terminal=%s res=%s' % (
            types[t], 1642723741 + i, i, r.integers(1, 999), accts[a], exes[e], "h1" if train or r.random() < 0.98 else "h%d" % r.integers(2, 5),
            terms[t if train else int(r.integers(0, 3))], "success" if train or r.random() < 0.7 else "failed")
        if r.random() < 0.05:
            ln = ln.replace(' acct="%s"' % accts[a], "")                           # a member missing: combination skipped
        out.append(ln.encode())
    return out


def raw_oracle(lines):
    orc = NewValueComboDetectorOracle(config=RAW_CFG, clock=lambda: 1773848383)
    from oracle.nvcd import combo_alert_key
    n = len(orc.monitors)
    keys = [combo_alert_key(orc.monitors, m) for m in orc.combos]
    flags, scores, masks, alerts = [], [], [], []
    for ln in lines:
        f, s, a = orc.step_line(ln)
        flags.append(int(f)); scores.append(float(s)); alerts.append(a)
        masks.append(sum(1 << (n + c) for c, k in enumerate(keys) if k in a))
    return flags, scores, masks, alerts, orc


def test_emu_raw_combo_kernel():
    import emu_harness
    lines = raw_lines(2600, seed=8)
    want_f, want_s, want_m, _, orc = raw_oracle(lines)
    assert sum(want_f) > 60 and any(s >= 2 for s in want_s)
    keys = [m.pos.encode() for m in orc.monitors]
    det = emu_harness.EmuDetector(keys, table_log2=12, variant="lanes")
    det.set_combos(orc.combos, (1 << len(keys)) - 1)
    buf = b"\n".join(lines) + b"\n"
    cut = buf.index(b"\n", len(buf) // 2) + 1
    f1, s1 = det.process_lines(buf[:cut], 1500)
    an = det.anomalies()
    n1 = len(f1)
    f2, s2 = det.process_lines(buf[cut:], max(0, 1500 - n1))
    an2 = det.anomalies()
    det.close()
    assert f1.tolist() + f2.tolist() == want_f and s1.tolist() + s2.tolist() == want_s
    got_m = {a[0]: a[1] for a in an}
    got_m.update({a[0] + n1: a[1] for a in an2})
    assert got_m == {i: m for i, m in enumerate(want_m) if m}


def test_component_raw_combo_wording_cpu():
    """Alert wording of raw records against the oracle, device replaced by per-record masks."""
    from detectmateservice_b200.component import B200NewValueComboDetector
    lines = raw_lines(2200, seed=9)
    _, _, want_m, want_alerts, orc = raw_oracle(lines)

    class FakeRaw:
        last_n_anomalies = 0

        def __init__(self):
            self.base = 0

        def process_lines(self, data, n_train_lines=0, copy=True):
            recs = bytes(data).split(b"\n")[:-1]
            ms = want_m[self.base:self.base + len(recs)]
            starts = np.concatenate([[0], np.cumsum([len(r) + 1 for r in recs])[:-1]]) if recs else []
            self._an = [(i, m, int(starts[i])) for i, m in enumerate(ms) if m]
            self.last_n_anomalies = len(self._an)
            self.base += len(recs)
            f = np.array([1 if m else 0 for m in ms], np.uint8)
            return f, np.array([bin(m).count("1") for m in ms], np.float32)

        def anomalies(self):
            return self._an

    comp = B200NewValueComboDetector(config=RAW_CFG)
    comp._det = FakeRaw()
    comp.clock = lambda: 1773848383
    got = []
    for lo in range(0, len(lines), 550):
        out = comp.process(b"\n".join(lines[lo:lo + 550]) + b"\n")
        got += [wire.decode_detector_schema(b) for b in wire.split_delimited(out)] if out else []
    want = [(i, a) for i, a in enumerate(want_alerts) if a]
    assert [(int(g["logIDs"][0]), g["alertsObtain"]) for g in got] == want
    assert all(g["detectorType"] == "new_value_combo_detector" for g in got)


@pytest.mark.gpu
def test_gpu_raw_combo_component_matches_oracle():
    from detectmateservice_b200.component import B200NewValueComboDetector, decode_compact
    lines = raw_lines(20000, seed=10)
    want_f, want_s, _, want_alerts, _ = raw_oracle(lines)
    comp = B200NewValueComboDetector(config=RAW_CFG)
    comp.clock = lambda: 1773848383
    got = []
    for lo in range(0, len(lines), 4100):
        out = comp.process(b"\n".join(lines[lo:lo + 4100]) + b"\n")
        got += [wire.decode_detector_schema(b) for b in wire.split_delimited(out)] if out else []
    want = [(i, a) for i, a in enumerate(want_alerts) if a]
    assert [(int(g["logIDs"][0]), g["alertsObtain"]) for g in got] == want
    assert [g["score"] for g in got] == [want_s[i] for i, _ in want]
    st = comp.stats()
    assert st["lines"] == 20000 and st["anomalies"] == sum(want_f)
    comp.close()
    comp = B200NewValueComboDetector(config={"detectors": {"NewValueComboDetector": dict(
        RAW_CFG["detectors"]["NewValueComboDetector"], params={"output_format": "compact"})}})
    f, s = decode_compact(comp.process(b"\n".join(lines) + b"\n"))
    assert f.tolist() == want_f and s.tolist() == want_s
    comp.close()
