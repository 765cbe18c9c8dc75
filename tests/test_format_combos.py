"""NewValueComboDetector on raw log lines in log_format / template mode (DESIGN.md R-combo with R-fmt / R-match /
R-norm): `dm_k_format_lanes<TRAIN, NORM, COMBO>` folds the fingerprints of a combination's members, re-hashed from the
captures the lane keeps, into the key the ParserSchema and key=value paths use.  FormatComboOracle (regex parser +
the R-combo rules) against the kernel source on the CPU emulator and (GPU tier) the library and the component."""
import ctypes as C
import os

import numpy as np
import pytest

from detectmateservice_b200 import wire
from detectmateservice_b200.logformat import LogFormat, load_templates, norm_flags
from oracle.nvcd import combo_alert_key, combo_alert_text, parse_combos
from oracle.nvd import NewValueDetectorOracle, select_component_config
from oracle.rfmt import FormatParser
from fmtgen import ALL_NORMS, format_case

AUDIT = "type=<type> msg=audit(<Time>): <Content>"
NAME = "NewValueComboDetector"


# ------------------------------------------------------------------------------------------ oracle
class FormatComboOracle:
    """FormatParser (regex) + the R-combo rules of oracle/nvcd.py.  `combos` (lists of monitor indices) replaces the
    config's one-combination-per-instance list; monitors outside `member_only` (default: all monitors) also alert on
    their own, by NewValueDetector's rule.  process_lines returns flags, scores, unknown-field masks (bit k: monitor k,
    bit n + c: combination c), alertsObtain dicts and the number of records the log_format rejects."""

    def __init__(self, cfg, log_format, templates=(), norm=(False, False, False), combos=None, member_only=None):
        self.parser = FormatParser(log_format, templates, remove_spaces=norm[0], remove_punctuation=norm[1], lowercase=norm[2])
        self.nvd = NewValueDetectorOracle(name=NAME, config=cfg)          # monitors, data_use_training, value lookup
        self.mons = self.nvd.monitors
        self.combos = parse_combos(select_component_config(cfg, NAME))[1] if combos is None else [list(m) for m in combos]
        n = len(self.mons)
        self.member_only = (1 << n) - 1 if member_only is None else member_only
        self.known = [set() for _ in self.mons]
        self.known_combos = [set() for _ in self.combos]
        self.unknown = [0] * (n + len(self.combos))                      # alerts per mask bit
        self.n_seen = 0
        self.eids = []

    def step(self, rec):
        self.n_seen += 1
        train = self.n_seen <= self.nvd.data_use_training
        vals = dict(self.nvd._values(rec))                               # monitor -> value, scope applied
        n, mask, alerts = len(self.mons), 0, {}
        for i, v in vals.items():
            if self.member_only >> i & 1:
                continue
            if train:
                self.known[i].add(v)
            elif v not in self.known[i]:
                mask |= 1 << i
                alerts[self.mons[i].alert_key] = "Unknown value: '%s'" % v.decode("utf-8", "replace")
        for c, members in enumerate(self.combos):
            if not all(i in vals for i in members):
                continue                                                 # a member is missing: no combination
            tup = tuple(vals[i] for i in members)
            if train:
                self.known_combos[c].add(tup)
            elif tup not in self.known_combos[c]:
                mask |= 1 << (n + c)
                alerts[combo_alert_key(self.mons, members)] = combo_alert_text(list(tup))
        for b in range(len(self.unknown)):
            self.unknown[b] += mask >> b & 1
        return mask, alerts

    def process_lines(self, buf):
        lines = buf.split(b"\n")
        if lines and lines[-1] == b"":
            lines.pop()
        flags, scores, masks, alerts, bad = [], [], [], [], 0
        for ln in lines:
            rec = self.parser.parse_line(ln)
            if rec is None:
                bad += 1
                rec = {"EventID": None, "variables": [], "logFormatVariables": {}}
            self.eids.append(rec["EventID"])
            m, a = self.step(rec)
            k = bin(m).count("1")
            flags.append(int(k > 0)); scores.append(float(k)); masks.append(m); alerts.append(a)
        return flags, scores, masks, alerts, bad


def _mons_combos(cfg):
    from detectmateservice_b200.component import parse_combos as comp_parse_combos
    return comp_parse_combos(select_component_config(cfg, NAME))


def test_oracle_by_hand():
    """R-combo on an nginx-shaped format, worked out by hand."""
    fmt = '<IP> - [<Time>] "<Method> <URL>" <Status> <Content>'
    cfg = {"detectors": {NAME: {"method_type": "new_value_combo_detector", "data_use_training": 3,
           "global": {"mu": {"header_variables": [{"pos": "Method"}, {"pos": "URL"}]}},
           "events": {-1: {"odd": {"header_variables": [{"pos": "Status"}, {"pos": "IP"}]}},
                      0: {"ua": {"variables": [{"pos": 0, "name": "agent"}, {"pos": 1, "name": "ver"}]}}}}}}
    line = lambda m, u, st=200, ip="1.2.3.4", c="agent=curl v=8": ('%s - [t] "%s %s" %d %s' % (ip, m, u, st, c)).encode()
    orc = FormatComboOracle(cfg, fmt, ["agent=<*> v=<*>"])
    buf = b"\n".join([
        line("GET", "/a"), line("POST", "/b", c="junk"), line("GET", "/b", c="agent=wget v="),    # training
        line("GET", "/a"),                      # every tuple known
        line("POST", "/a"),                     # both values known, the (Method, URL) pair is new
        b"not an access-log line",              # the log_format rejects it: bad, silent
        line("GET", "/a", c="agent=wget v=8"),  # (agent, ver) = (wget, 8) new; an empty capture ('v=') was learnt
        line("GET", "/b", c="agent=wget v="),   # known, the empty ver included
        line("GET", "/b", st=404, c="nothing"), # EventID -1: (Status, IP) = (404, ...) new
        line("POST", "/a")]) + b"\n"            # detection never inserts: alerts again
    f, s, m, a, bad = orc.process_lines(buf)
    assert f == [0, 0, 0, 0, 1, 0, 1, 0, 1, 1] and bad == 1 and orc.eids[5] is None
    assert a[4] == {"Global - (Method, URL)": "Unknown value combination: ('POST', '/a')"}
    assert a[6] == {"EventID 0 - (agent, ver)": "Unknown value combination: ('wget', '8')"}
    assert a[8] == {"EventID -1 - (Status, IP)": "Unknown value combination: ('404', '1.2.3.4')"}
    assert a[9] == a[4] and m[4] == 1 << 6 and m[6] == 1 << 8 and m[8] == 1 << 7
    # a missing member skips the combination: a record without a template match has no variables, so (agent, ver) is
    # neither learnt in training nor looked up in detection; the first record that has both alerts
    orc2 = FormatComboOracle(cfg, fmt, ["agent=<*> v=<*>"])
    f2, _, m2, _, _ = orc2.process_lines(b"\n".join([line("GET", "/a", c="x")] * 4 + [line("GET", "/a", c="agent=new v=1")]) + b"\n")
    assert f2 == [0, 0, 0, 0, 1] and m2[4] == 1 << 8 and orc2.known_combos[2] == set()


# ------------------------------------------------------------------------------------------ emulator tier
def _monitor_array(mons):
    from detectmateservice_b200 import _lib
    arr = (_lib.Monitor * max(1, len(mons)))()
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


class EmuFormatCombo:
    """The kernel source on the emulator: emu_set_monitors + emu_set_format + emu_set_combos + emu_process_format."""

    def __init__(self, mons, combos, member_only, log_format, templates=(), flags=0):
        import emu_harness
        self.mons, self.combos, self.member_only = mons, combos, member_only
        self.det = emu_harness.EmuDetector([b"\x01m%d" % i for i in range(len(mons))], table_log2=14)
        self.lib = self.det.lib
        self.det.set_monitors(_monitor_array(mons), len(mons))
        self.det.set_format(log_format, templates, flags)
        self.det.set_combos(combos, member_only)

    def process(self, buf, n_train):
        cap = buf.count(b"\n") + 2
        f = np.full(cap, 9, np.uint8); s = np.full(cap, -1, np.float32)
        n, na, err = C.c_uint64(), C.c_uint64(), C.c_uint32()
        rc = self.lib.emu_process_format(self.det.h, buf, len(buf), n_train, f.ctypes.data, s.ctypes.data, cap,
                                         C.byref(n), C.byref(na), C.byref(err))
        assert rc == 0 and err.value == 0
        k = n.value
        assert na.value == int(f[:k].sum())
        an = {a[0]: (a[1], a[2]) for a in self.det.anomalies()}
        return f[:k].tolist(), s[:k].tolist(), an, self.stats()

    def stats(self):
        w = (C.c_uint64 * 40)()
        self.lib.emu_get_stats(self.det.h, w)
        return {"lines": w[0], "train_lines": w[1], "detect_lines": w[2], "anomalies": w[3], "score_sum": w[4],
                "bytes": w[5], "known_keys": w[6], "bad_records": w[7], "unknown_per_key": [w[8 + i] for i in range(32)]}


def emu_run(mons, combos, member_only, log_format, templates, flags, buf, n_train):
    emu = EmuFormatCombo(mons, combos, member_only, log_format, templates, flags)
    out = emu.process(buf, n_train)
    emu.det.close()
    return out


def _record_starts(buf):
    starts, pos = [], 0
    for ln in buf.split(b"\n"):
        starts.append(pos)
        pos += len(ln) + 1
    return starts


def check_run(cfg, log_format, templates, norm, buf, n_train, run, combos=None, member_only=None):
    """One message through a fresh detector, compared with the oracle in everything it reports; returns the oracle."""
    cfg = {"detectors": {NAME: dict(cfg["detectors"][NAME], data_use_training=n_train)}}
    orc = FormatComboOracle(cfg, log_format, templates, norm, combos, member_only)
    wf, ws, wm, _, bad = orc.process_lines(buf)
    f, s, an, st = run(orc.mons, orc.combos, orc.member_only, log_format, templates, norm_flags(*norm), buf, n_train)
    ctx = (log_format, norm, n_train)
    assert f == wf and s == ws, ctx
    starts = _record_starts(buf)
    assert an == {i: (m, starts[i]) for i, m in enumerate(wm) if m}, ctx
    n, tr = len(wf), min(n_train, len(wf))
    assert (st["lines"], st["train_lines"], st["detect_lines"], st["bytes"]) == (n, tr, n - tr, len(buf)), ctx
    assert (st["anomalies"], st["score_sum"], st["bad_records"]) == (sum(wf), int(sum(ws)), bad), ctx
    assert st["unknown_per_key"][:len(orc.unknown)] == orc.unknown, ctx
    assert not any(st["unknown_per_key"][len(orc.unknown):]), ctx
    return orc


def audit_templates(golden_dir):
    return load_templates(os.path.join(golden_dir, "audit_templates.txt"))


AUDIT_COMBO_CFG = {"detectors": {NAME: {
    "method_type": "new_value_combo_detector", "data_use_training": 250, "auto_config": False,
    "global": {"type": {"header_variables": [{"pos": "type"}]}},
    "events": {0: {"pam": {"variables": [{"pos": 5, "name": "acct"}, {"pos": 6, "name": "exe"},
                                         {"pos": 9, "name": "terminal"}, {"pos": 10, "name": "res"}]},
                   "who": {"header_variables": [{"pos": "type"}], "variables": [{"pos": 4, "name": "op"}]}},
               1: {"unit": {"variables": [{"pos": 4, "name": "unit"}, {"pos": 6, "name": "exe"}]}},
               2: {"login": {"variables": [{"pos": 3, "name": "auid"}, {"pos": 7, "name": "res"}]}},
               -1: {"other": {"header_variables": [{"pos": "type"}, {"pos": "Content"}]}}}}}}
AUDIT_TAIL = (
    b"type=WEIRD msg=audit(1.0:1): totally unlike=any template\nnot an audit line at all\n\n"
    b"type=USER_ACCT msg=audit(1642723741.072:375): pid=10125   uid=0 AUID=4294967295 ses=4294967295 "
    b"msg='op=PAM:accounting acct=\"root\" exe=\"/usr/sbin/cron2\" hostname=? addr=? terminal=cron res=success'\n"
    b"type=LOGIN msg=audit(1642723741.076:377): pid=1 uid=0 old-auid=4294967295 auid=77777 tty=(none) old-ses=4294967295 ses=65 res=9")


def test_emu_audit_sample_every_switch(golden_dir):
    """The golden audit sample with the reference's audit templates, under all 8 R-norm switch combinations."""
    tm = audit_templates(golden_dir)
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read() + AUDIT_TAIL
    alerts = 0
    for norm in ALL_NORMS:
        orc = check_run(AUDIT_COMBO_CFG, AUDIT, tm, norm, buf, 250, emu_run)
        n = len(orc.mons)
        assert orc.unknown[n + 5] >= 1 and orc.unknown[n + 1] + orc.unknown[n + 4] >= 3, norm     # EventID -1; pam / login
        alerts += sum(orc.unknown)
    assert alerts >= 60


def combo_config(case):
    """NewValueComboDetector instances over a format_case: global header pairs and a 1-tuple, an EventID -1 pair, and per
    event (the 32-wildcard template first when there is one) variable pairs with index 0 and the last capture, a
    header + variable mix, a triple with index 31, and a pair with a member one past the last capture (never present).
    Returns the config and the combination index of every instance kind."""
    lf = LogFormat(case["log_format"], case["templates"], flags=norm_flags(*case["norm"]))
    caps = [t.n_captures for t in lf.templates]
    kinds = ["hc", "one", "u"]
    glob = {"hc": {"header_variables": [{"pos": "h"}, {"pos": "Content"}]}, "one": {"header_variables": [{"pos": "h"}]}}
    events = {-1: {"u": {"header_variables": [{"pos": "Content"}, {"pos": "h"}]}}}
    order = [e for e in case["cfg"]["detectors"]["NewValueDetector"]["events"] if e != -1]
    for t, shape in zip(order, (("vp", "hv", "v31"), ("vp", "oor"), ("hv",))):
        last = max(caps[t] - 1, 0)
        inst = {}
        for k in shape:
            inst[k] = {"vp": {"variables": [{"pos": 0}, {"pos": last}]},
                       "hv": {"header_variables": [{"pos": "h"}], "variables": [{"pos": last}]},
                       "v31": {"variables": [{"pos": 31}, {"pos": 0}, {"pos": last}]},
                       "oor": {"variables": [{"pos": 0}, {"pos": caps[t]}]}}[k]
            kinds.append(k)
        events[t] = inst
    cfg = {"detectors": {NAME: {"method_type": "new_value_combo_detector", "data_use_training": case["n_train"],
                                "global": glob, "events": events}}}
    return cfg, kinds


def check_combo_case(case, seed, run):
    cfg, kinds = combo_config(case)
    buf = b"\n".join(case["lines"]) + (b"\n" if seed % 2 == 0 else b"")
    orc = check_run(cfg, case["log_format"], case["templates"], case["norm"], buf, case["n_train"], run)
    n = len(orc.mons)
    for c, k in enumerate(kinds):
        if k == "oor":
            assert orc.unknown[n + c] == 0 and not orc.known_combos[c]
    return orc, kinds


def _tally(orc, kinds, tally):
    n = len(orc.mons)
    for c, k in enumerate(kinds):
        tally[k] = tally.get(k, 0) + orc.unknown[n + c]


def test_emu_generated_cases():
    """12 generated configurations (2 to 63 templates, literals up to 255 bytes, empty / malformed / odd-byte records)
    with combinations drawn over them, R-norm switches cycling, against the oracle."""
    tally = {}
    for seed in range(12):
        orc, kinds = check_combo_case(format_case(seed, ALL_NORMS[seed % 8]), seed, emu_run)
        _tally(orc, kinds, tally)
    assert tally["hc"] > 500 and tally["one"] > 10 and tally["u"] > 50
    assert tally["vp"] > 100 and tally["hv"] > 100 and tally["v31"] > 0 and tally["oor"] == 0


def test_emu_every_split_of_a_40_record_message():
    n_checked = 0
    for seed, norm in ((3, (True, True, True)), (4, (False, False, False))):
        case = format_case(seed, norm, n_records=40, n_templates=8)
        for n_train in range(41):
            check_combo_case(dict(case, n_train=n_train), seed, emu_run)
            n_checked += 1
    assert n_checked == 82


def cap32_case(n_train=40, n=600, seed=0):
    """A 32-capture log_format; 31 member-only header monitors (c0..c30) and one combination of all of them (mask
    bit 31).  Training records repeat a few tuples; detection records recombine known values."""
    fmt = "".join("<c%d>k%02dq" % (i, i) for i in range(32))   # distinct literals: the regex oracle stays linear
    cfg = {"detectors": {NAME: {"method_type": "new_value_combo_detector", "data_use_training": n_train,
           "global": {"all": {"header_variables": [{"pos": "c%d" % i} for i in range(31)]}}}}}
    r = np.random.Generator(np.random.PCG64(seed))
    rows = [[b"v%d" % int(x) for x in r.integers(0, 3, 32)] for _ in range(4)]
    lines = []
    for i in range(n):
        row = list(rows[int(r.integers(0, 4))])
        if i >= n_train and r.random() < 0.3:
            j = int(r.integers(0, 32))
            row[j] = rows[int(r.integers(0, 4))][j] if r.random() < 0.8 else b""      # a known value, or empty
        ln = b"".join(v + b"k%02dq" % j for j, v in enumerate(row))
        if r.random() < 0.05:
            ln = ln[:-1]                                         # the final literal cut short: bad record
        lines.append(ln)
    return fmt, cfg, b"\n".join(lines) + b"\n"


def test_emu_31_member_only_captures_one_combination():
    fmt, cfg, buf = cap32_case()
    orc = check_run(cfg, fmt, [], (False, False, False), buf, 40, emu_run)
    assert len(orc.mons) == 31 and orc.combos == [list(range(31))] and orc.unknown[31] > 50


EDGE_FMT = "<a>,<b>,<c>|<Content>"


def edge_lines(seed, n=300):
    r = np.random.Generator(np.random.PCG64(seed))
    out = []
    for i in range(n):
        v = [b"xyz"[int(j)] for j in r.integers(0, 2 if i < 100 else 3, 3)]
        content = b"k=%d" % int(r.integers(0, 3)) if r.random() < 0.8 else b"junk"
        out.append(b"%c,%c,%c|" % tuple(v) + content)
    return b"\n".join(out) + b"\n"


EDGE_CFG = {"detectors": {NAME: {"method_type": "new_value_combo_detector", "data_use_training": 100,
            "global": {"g": {"header_variables": [{"pos": "a"}, {"pos": "b"}, {"pos": "c"}]}},
            "events": {0: {"e": {"variables": [{"pos": 0}]}}}}}}
EDGES = [("reversed pair", [[0, 1], [1, 0]], None),                 # two keys for the same two monitors
         ("monitor in two combinations", [[0, 1], [0, 2], [3, 0]], None),
         ("partial member_only", [[0, 1], [2, 3]], 0b0101),         # monitors 1 and 3 also alert on their own
         ("no member_only", [[1, 2, 3]], 0)]


@pytest.mark.parametrize("label,combos,member_only", EDGES, ids=[e[0] for e in EDGES])
def test_emu_combination_edges(label, combos, member_only):
    buf = edge_lines(len(label))
    orc = check_run(EDGE_CFG, EDGE_FMT, ["k=<*>"], (False, False, False), buf, 100, emu_run, combos, member_only)
    n = len(orc.mons)
    assert all(orc.unknown[n + c] > 5 for c in range(len(combos))), label
    singles = [k for k in range(n) if orc.unknown[k]]
    allowed = [k for k in range(n) if not (orc.member_only >> k & 1)]     # member-only monitors never alert alone
    assert set(singles) <= set(allowed) and bool(singles) == bool(allowed), label
    if label == "partial member_only":
        _, _, wm, _, _ = FormatComboOracle(EDGE_CFG, EDGE_FMT, ["k=<*>"], combos=combos, member_only=member_only
                                           ).process_lines(buf)
        assert any(m & 0b1111 and m >> n for m in wm)           # single and combination alerts in one record


def test_emu_reversed_pair_gives_two_keys():
    """[[0, 1], [1, 0]]: one training record (x, y) learns two keys; (y, x) is new for both combinations."""
    cfg = {"detectors": {NAME: {"method_type": "new_value_combo_detector", "data_use_training": 1,
           "global": {"g": {"header_variables": [{"pos": "a"}, {"pos": "b"}]}}}}}
    mons, _ = _mons_combos(cfg)
    emu = EmuFormatCombo(mons, [[0, 1], [1, 0]], 0b11, "<a>,<b>")
    f, s, an, _ = emu.process(b"x,y\n", 1)
    assert len(emu.det.export_known()) == 2
    f, s, an, _ = emu.process(b"x,y\ny,x\nx,x\n", 0)
    assert f == [0, 1, 1] and s == [0.0, 2.0, 2.0] and an[1][0] == 0b1100
    emu.det.close()


def _schema_record(rec):
    return {"EventID": rec["EventID"], "variables": [v.decode() for v in rec["variables"]],
            "logFormatVariables": {k: v.decode() for k, v in rec["logFormatVariables"].items()}}


def test_emu_key_equivalence_with_parser_schema(golden_dir):
    """A tuple learnt from raw lines in format mode has the key it has when learnt from the same records as ParserSchema:
    the two known sets are equal, with and without R-norm (single monitors outside member_only included)."""
    import emu_harness
    tm = audit_templates(golden_dir)
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read()
    mons, combos = _mons_combos(AUDIT_COMBO_CFG)
    member_only = ((1 << len(mons)) - 1) & ~1                    # the global `type` monitor also learns on its own
    for norm in ((False, False, False), (True, True, True)):
        n = buf.count(b"\n")
        emu = EmuFormatCombo(mons, combos, member_only, AUDIT, tm, norm_flags(*norm))
        emu.process(buf, n)
        k_fmt = sorted(emu.det.export_known())
        emu.det.close()
        parser = FormatParser(AUDIT, tm, remove_spaces=norm[0], remove_punctuation=norm[1], lowercase=norm[2])
        recs = [parser.parse_line(ln) for ln in buf.split(b"\n")[:-1]]
        assert all(r is not None for r in recs)
        batch = wire.frame_delimited([wire.encode_parser_schema(_schema_record(r)) for r in recs])
        det = emu_harness.EmuDetector([b"\x01m%d" % i for i in range(len(mons))], table_log2=14)
        det.set_monitors(_monitor_array(mons), len(mons))
        det.set_combos(combos, member_only)
        f = np.zeros(n, np.uint8); s = np.zeros(n, np.float32); m = np.zeros(n, np.uint32)
        rc, nr, _ = det.process_records(batch, n, f, s, m, n)
        assert rc == 0
        k_rec = sorted(det.export_known())
        det.close()
        assert nr == n and len(k_fmt) > 40 and k_fmt == k_rec, norm


# ------------------------------------------------------------------------------------------ component, device faked
class EmuDevice:
    """The kernel source on the emulator behind the component's device interface."""

    def __init__(self, comp):
        lf = comp.logformat
        self.emu = EmuFormatCombo(comp.monitors, comp.combos, (1 << len(comp.monitors)) - 1, lf.source,
                                  lf.template_sources, lf.flags)
        self.last_n_anomalies = 0

    def process_lines(self, data, n_train_lines=0, copy=True):
        f, s, an, self._stats = self.emu.process(bytes(data), n_train_lines)
        self._an = sorted((ln, m, off) for ln, (m, off) in an.items())
        self.last_n_anomalies = len(self._an)
        return np.array(f, np.uint8), np.array(s, np.float32)

    def anomalies(self):
        return self._an

    def stats(self):
        return self._stats

    def close(self):
        self.emu.det.close()


def _combo_component(cfg, params):
    from detectmateservice_b200.component import B200NewValueComboDetector
    det = dict(cfg["detectors"][NAME])
    det["params"] = dict(det.get("params") or {}, **params)
    c = B200NewValueComboDetector(config={"detectors": {NAME: det}})
    c.clock = lambda: 1773848383
    return c


def _audit_params(golden_dir, **extra):
    return dict({"log_format": AUDIT, "path_templates": os.path.join(golden_dir, "audit_templates.txt"),
                 "remove_spaces": True, "remove_punctuation": True, "lowercase": True}, **extra)


def _alerts_of(out):
    return [wire.decode_detector_schema(b) for b in wire.split_delimited(out)] if out else []


def test_component_wording_chunked_and_compact_cpu(golden_dir):
    """The component's alert wording in format mode against the oracle (normalised variables), over messages cut into
    device batches (small max_batch_bytes), training ending inside one of them; then `compact` output."""
    from detectmateservice_b200.component import decode_compact
    tm = audit_templates(golden_dir)
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read() + AUDIT_TAIL + b"\n"
    orc = FormatComboOracle(AUDIT_COMBO_CFG, AUDIT, tm, (True, True, True))
    wf, ws, _, wa, _ = orc.process_lines(buf)
    comp = _combo_component(AUDIT_COMBO_CFG, _audit_params(golden_dir, max_batch_bytes=8192))
    comp._det = EmuDevice(comp)
    cut = buf.index(b"\n", len(buf) // 2) + 1
    got = _alerts_of(comp.process(buf[:cut])) + _alerts_of(comp.process(buf[cut:]))
    want = [(i, a) for i, a in enumerate(wa) if a]
    assert len(want) >= 8 and [(int(g["logIDs"][0]), g["alertsObtain"]) for g in got] == want
    assert [g["score"] for g in got] == [ws[i] for i, _ in want]
    assert all(g["detectorType"] == "new_value_combo_detector" and "combinations" in g["description"] for g in got)
    assert {"EventID 0 - (acct, exe, terminal, res)": "Unknown value combination: ('root', 'usrsbincron2', 'cron', 'success')"} in [
        a for _, a in want]
    comp._det.close()
    comp = _combo_component(AUDIT_COMBO_CFG, _audit_params(golden_dir, max_batch_bytes=8192, output_format="compact"))
    comp._det = EmuDevice(comp)
    f, s = decode_compact(comp.process(buf))
    assert f.tolist() == wf and s.tolist() == ws
    comp._det.close()


def test_component_rejects_dead_combinations():
    from detectmateservice_b200.component import B200NewValueComboDetector, B200NewValueDetector
    base = {"method_type": "new_value_combo_detector", "data_use_training": 5}
    dead_header = {"detectors": {NAME: dict(base, params={"log_format": AUDIT},
                   **{"global": {"tc": {"header_variables": [{"pos": "type"}, {"pos": "nosuch"}]}}})}}
    with pytest.raises(ValueError, match=r"global\.tc.*'nosuch'"):
        B200NewValueComboDetector(config=dead_header)
    dead_var = {"detectors": {NAME: dict(base, params={"log_format": AUDIT},
                events={3: {"pam": {"variables": [{"pos": 0}], "header_variables": [{"pos": "type"}]}}})}}
    with pytest.raises(ValueError, match=r"events\.3\.pam.*no templates"):
        B200NewValueComboDetector(config=dead_var)
    ok = {"detectors": {NAME: dict(base, params={"log_format": AUDIT, "templates": ["a=<*>"]},
          events={3: {"pam": {"variables": [{"pos": 0}], "header_variables": [{"pos": "type"}]}}})}}
    c = B200NewValueComboDetector(config=ok)
    assert c.combos == [[0, 1]] and c.logformat is not None
    # the single-value detector keeps monitors on absent captures as before
    B200NewValueDetector(config={"detectors": {"NewValueDetector": dict(dead_header["detectors"][NAME],
                                                                          method_type="new_value_detector")}})


# ------------------------------------------------------------------------------------------ GPU tier
def _gpu_stats(det):
    from detectmateservice_b200 import _lib
    st = _lib.Stats()
    _lib.check(det._lib.dm_get_stats(det._h, C.byref(st)))
    return st.as_dict(32)


def _device(mons, combos, member_only, log_format, templates, flags, combos_first=True, max_batch_bytes=1 << 20):
    from detectmateservice_b200.detector import DeviceDetector
    # (field names only matter to key=value records: the component's monitors carry theirs, the oracle's get placeholders)
    keys = [getattr(m, "key", b"") or b"\x01m%d" % i for i, m in enumerate(mons)]
    det = DeviceDetector(keys, max_batch_bytes=max_batch_bytes)
    det.set_monitors([{"event_id": m.event_id, "source": m.source, "pos": m.pos} for m in mons])
    lf = log_format.decode() if isinstance(log_format, bytes) else log_format
    if combos_first:
        det.set_combos(combos, member_only_mask=member_only)
        det.set_format(lf, list(templates), norm_flags=flags)
    else:
        det.set_format(lf, list(templates), norm_flags=flags)
        det.set_combos(combos, member_only_mask=member_only)
    return det


def _gpu_runner(combos_first):
    def run(mons, combos, member_only, log_format, templates, flags, buf, n_train):
        det = _device(mons, combos, member_only, log_format, templates, flags, combos_first)
        f, s = det.process_lines(buf, n_train_lines=n_train)
        an = {a[0]: (a[1], a[2]) for a in det.anomalies()}
        st = _gpu_stats(det)
        det.close()
        return f.tolist(), s.tolist(), an, st
    return run


@pytest.mark.gpu
def test_gpu_generated_cases_both_orders_then_key_value():
    tally = {}
    for seed in range(12):
        orc, kinds = check_combo_case(format_case(seed, ALL_NORMS[seed % 8]), seed, _gpu_runner(seed % 2 == 0))
        _tally(orc, kinds, tally)
    assert tally["hc"] > 500 and tally["vp"] > 100 and tally["v31"] > 0 and tally["oor"] == 0
    for seed, norm in ((3, (True, True, True)), (4, (False, False, False))):
        case = format_case(seed, norm, n_records=40, n_templates=8)
        for n_train in range(41):
            check_combo_case(dict(case, n_train=n_train), seed, _gpu_runner(n_train % 2 == 0))
    # set_format(None): the same handle goes back to key=value records and the dm_k_lanes combinations
    from oracle.nvcd import NewValueComboDetectorOracle
    cfg = {"detectors": {NAME: {"method_type": "new_value_combo_detector", "data_use_training": 2,
           "global": {"ab": {"header_variables": [{"pos": "a"}, {"pos": "b"}]}}}}}
    mons, combos = _mons_combos(cfg)
    det = _device(mons, combos, 0b11, "<a>,<b>", [], 0)
    assert det.process_lines(b"1,2\n1,3\n2,2\n1,2\n", n_train_lines=2)[0].tolist() == [0, 0, 1, 0]
    det.set_format(None)
    det.reset()
    lines = [b"a=1 b=2", b"a=1 b=3", b"a=2 b=2", b"a=1 b=2", b"a=2"]
    orc = NewValueComboDetectorOracle(config=cfg)
    want = [int(orc.step_line(ln)[0]) for ln in lines]
    assert det.process_lines(b"\n".join(lines) + b"\n", n_train_lines=2)[0].tolist() == want == [0, 0, 1, 0, 0]
    det.close()


@pytest.mark.gpu
def test_gpu_component_audit_sample_all_switches(golden_dir):
    """The reference's audit parser config (all three switches on) in front of NewValueComboDetector: two messages with
    training ending inside the first, then `compact` output."""
    from detectmateservice_b200.component import decode_compact
    tm = audit_templates(golden_dir)
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read() + AUDIT_TAIL + b"\n"
    wf, ws, _, wa, bad = FormatComboOracle(AUDIT_COMBO_CFG, AUDIT, tm, (True, True, True)).process_lines(buf)
    comp = _combo_component(AUDIT_COMBO_CFG, _audit_params(golden_dir))
    cut = buf.index(b"\n", len(buf) // 3) + 1
    got = _alerts_of(comp.process(buf[:cut])) + _alerts_of(comp.process(buf[cut:]))
    want = [(i, a) for i, a in enumerate(wa) if a]
    assert len(want) >= 8 and [(int(g["logIDs"][0]), g["alertsObtain"]) for g in got] == want
    assert [g["score"] for g in got] == [ws[i] for i, _ in want]
    st = comp.stats()
    assert st["bad_records"] == bad and st["anomalies"] == sum(wf) and st["lines"] == len(wf)
    comp.close()
    comp = _combo_component(AUDIT_COMBO_CFG, _audit_params(golden_dir, output_format="compact"))
    f, s = decode_compact(comp.process(buf))
    assert f.tolist() == wf and s.tolist() == ws
    comp.close()


def _grid_threads(threads_per_cta=64):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 32 * threads_per_cta


@pytest.mark.gpu
def test_gpu_stride_more_records_than_twice_the_grid():
    """One format-mode message with combinations and more than twice as many records as the grid has threads, training
    ending at a record index that is not a multiple of 32: both launches stride."""
    r = np.random.Generator(np.random.PCG64(41))
    n = 2 * _grid_threads() + 50001
    n_train = 300007
    pool = [b"%c,%c,%c|k=%d" % (b"xyz"[i % 2], b"xyz"[(i // 2) % 2], b"xyz"[(i // 4) % 2], (i // 8) % 2) for i in range(16)]
    extra = [b"%c,%c,%c|k=%d" % (b"xyz"[i % 3], b"xyz"[(i // 3) % 3], b"xyz"[(i // 9) % 3], (i // 27) % 3) for i in range(81)]
    extra += [b"x,y|k=1", b"x,y,z|junk", b"z,z,z|k="]              # malformed; no template; an empty variable
    lines = [pool[i] for i in r.integers(0, 16, n_train)] + [extra[i] for i in r.integers(0, len(extra), n - n_train)]
    buf = b"\n".join(lines) + b"\n"
    combos, member_only = [[0, 1], [2, 3], [0, 1, 2]], 0b0101
    cfg = {"detectors": {NAME: dict(EDGE_CFG["detectors"][NAME], data_use_training=n_train)}}
    memo = {}
    orc = FormatComboOracle(cfg, EDGE_FMT, ["k=<*>"], combos=combos, member_only=member_only)
    for ln in dict.fromkeys(lines[:n_train]):
        orc.process_lines(ln + b"\n")
    orc.n_seen = orc.nvd.data_use_training
    for ln in dict.fromkeys(lines[n_train:]):
        memo[ln] = orc.step(orc.parser.parse_line(ln) or {"EventID": None, "variables": [], "logFormatVariables": {}})[0]
    det = _device(orc.mons, combos, member_only, EDGE_FMT, ["k=<*>"], 0, max_batch_bytes=16 << 20)
    assert det.max_lines >= len(lines)
    f, s = det.process_lines(buf, n_train_lines=n_train)
    want = [memo[ln] for ln in lines[n_train:]]
    assert f[:n_train].sum() == 0 and f[n_train:].tolist() == [int(m != 0) for m in want]
    assert s[n_train:].tolist() == [float(bin(m).count("1")) for m in want]
    assert {a[0]: a[1] for a in det.anomalies()} == {n_train + i: m for i, m in enumerate(want) if m}
    st = det.stats()
    assert st["lines"] == n and st["bad_records"] > 1000 and st["anomalies"] == int(f.sum()) > 10000
    det.close()


@pytest.mark.gpu
def test_gpu_31_member_only_captures_one_combination():
    fmt, cfg, buf = cap32_case(n=4000, seed=3)
    orc = check_run(cfg, fmt, [], (False, False, False), buf, 40, _gpu_runner(True))
    assert orc.unknown[31] > 300


@pytest.mark.gpu
def test_gpu_device_resident_hostile_slack():
    """Messages in their own device tensors with exactly 16 bytes of slack made of the configured literals and '\\n',
    through enqueue_device + sync, with combinations."""
    import torch
    for seed, norm in ((21, (False, False, False)), (22, (True, True, True))):
        case = format_case(seed, norm, n_records=300, n_templates=16)
        cfg, _ = combo_config(dict(case, n_train=30))
        lits = b"".join(t.replace(b"<*>", b"") + b"\n" for t in case["templates"])
        slack = np.frombuffer((lits * (16 // max(1, len(lits)) + 1))[:16], dtype=np.uint8)
        orc = FormatComboOracle(cfg, case["log_format"], case["templates"], norm)
        det = _device(orc.mons, orc.combos, orc.member_only, case["log_format"], case["templates"], norm_flags(*norm))
        for k in range(10):
            m = b"\n".join(case["lines"][30 * k:30 * k + 30]) + (b"\n" if k % 2 else b"z")
            x = torch.from_numpy(np.concatenate([np.frombuffer(m, dtype=np.uint8), slack])).cuda()
            fo = torch.full((64,), 7, dtype=torch.uint8, device="cuda")
            so = torch.full((64,), -1.0, dtype=torch.float32, device="cuda")
            det.enqueue_device(x.data_ptr(), len(m), 30 if k == 0 else 0, fo.data_ptr(), so.data_ptr(), 64)
            n_lines, _ = det.sync()
            wf, ws, wm, _, _ = orc.process_lines(m)
            assert n_lines == len(wf) == 30
            assert fo[:30].cpu().tolist() == wf and so[:30].cpu().tolist() == ws, (seed, k)
            assert {a[0]: (a[1], a[2]) for a in det.anomalies()} == {
                i: (mm, _record_starts(m)[i]) for i, mm in enumerate(wm) if mm}, (seed, k)
        assert _gpu_stats(det)["unknown_per_key"][:len(orc.unknown)] == orc.unknown and sum(orc.unknown) > 20
        det.close()


@pytest.mark.gpu
def test_gpu_key_equivalence_with_parser_schema(golden_dir):
    tm = audit_templates(golden_dir)
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read()
    mons, combos = _mons_combos(AUDIT_COMBO_CFG)
    member_only = ((1 << len(mons)) - 1) & ~1
    n = buf.count(b"\n")
    for norm in ((False, False, False), (True, True, True)):
        det = _device(mons, combos, member_only, AUDIT, tm, norm_flags(*norm), combos_first=False)
        det.process_lines(buf, n_train_lines=n)
        k_fmt = sorted(det.export_known().tolist())
        det.close()
        parser = FormatParser(AUDIT, tm, remove_spaces=norm[0], remove_punctuation=norm[1], lowercase=norm[2])
        batch = wire.frame_delimited([wire.encode_parser_schema(_schema_record(parser.parse_line(ln)))
                                      for ln in buf.split(b"\n")[:-1]])
        det = _device(mons, combos, member_only, AUDIT, tm, 0)
        det.process_records(batch, n_train_records=n)
        k_rec = sorted(det.export_known().tolist())
        det.close()
        assert len(k_fmt) > 40 and k_fmt == k_rec, norm
