"""MatcherParser fused in front of the detector (SURVEY.md section 8f-3): log_format header
extraction + `<*>` template matching.  Regex oracle (oracle/rfmt.py) vs the host mirror vs
the kernel source on the CPU emulator, and (GPU tier) the real library / component.
Pinned known answer: the nginx example of docs/getting_started.md:395-435,498-510."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from detectmateservice_b200 import wire
from detectmateservice_b200.logformat import LogFormat, load_templates, norm_flags
from oracle.nvd import NewValueDetectorOracle
from oracle.rfmt import FormatParser
from fmtgen import (ALL_NORMS, NORMS, FormatOracle, format_case, fuzz_formats, fuzz_text, norm_fuzz_template,
                    norm_fuzz_text)

NGINX = '<IP> - - [<Time>] "<Method> <URL> <Protocol>" <Status> <Bytes> "<Referer>" "<UserAgent>"'
AUDIT = "type=<type> msg=audit(<Time>): <Content>"
NGINX_CFG = {"detectors": {"NewValueDetector": {                      # container/config/detector_config.yaml
    "method_type": "new_value_detector", "data_use_training": 2, "auto_config": False,
    "global": {"global_instance": {"header_variables": [{"pos": "URL"}]}}}}}


def nginx_line(url, ip="172.18.0.1", status=404):
    return ('%s - - [18/Mar/2026:15:39:43 +0000] "GET %s HTTP/1.1" %d 162 "-" "curl/8.5.0"' % (ip, url, status)).encode()


def audit_templates(golden_dir):
    return load_templates(os.path.join(golden_dir, "audit_templates.txt"))


# ------------------------------------------------------------------------------------------ CPU tier
def test_docs_nginx_golden_oracle_and_host():
    """docs/getting_started.md: train on /hello and /world, /foobar alerts with this exact text."""
    buf = b"\n".join(nginx_line(u) for u in ("/hello", "/world", "/foobar", "/hello")) + b"\n"
    orc = FormatOracle(NGINX_CFG, NGINX)
    flags, scores, alerts, bad = orc.process_lines(buf)
    assert flags == [0, 0, 1, 0] and scores == [0.0, 0.0, 1.0, 0.0] and bad == 0
    assert alerts[2] == {"Global - URL": "Unknown value: '/foobar'"}
    lf = LogFormat(NGINX)
    eid, variables, lfv = lf.parse(nginx_line("/foobar"))
    assert (eid, variables) == (-1, []) and lfv["URL"] == b"/foobar" and lfv["Time"] == b"18/Mar/2026:15:39:43 +0000"
    assert lfv == FormatParser(NGINX).parse_line(nginx_line("/foobar"))["logFormatVariables"]


def test_host_mirror_matches_regex_on_audit_log(golden_dir):
    tm = audit_templates(golden_dir)
    a, b = FormatParser(AUDIT, tm), LogFormat(AUDIT, tm)
    eids = []
    for ln in open(os.path.join(golden_dir, "audit_sample.log"), "rb").read().split(b"\n")[:-1]:
        r, s = a.parse_line(ln), b.parse(ln)
        assert (r["EventID"], r["variables"], r["logFormatVariables"]) == s
        eids.append(s[0])
    assert set(eids) >= {0, 1, 2} and -1 not in eids


def test_sequential_matcher_equals_regex_fuzz():
    r = np.random.Generator(np.random.PCG64(5))
    n_match = 0
    for lits, ends in fuzz_formats(r, 300):
        names = ["c%d" % i for i in range(len(lits) - (0 if ends else 1))]
        fmt = b"".join(l + (b"<%s>" % names[i].encode() if i < len(names) else b"") for i, l in enumerate(lits))
        tmpl = b"<*>".join(lits) + (b"<*>" if ends else b"")
        a, b = FormatParser(fmt), LogFormat(fmt)
        ta, tb = FormatParser("<Content>", [tmpl]), LogFormat("<Content>", [tmpl])
        for _ in range(40):
            text = fuzz_text(r, lits, ends)
            ra, rb = a.parse_line(text), b.parse(text)
            assert (ra is None) == (rb is None), (fmt, text)
            if ra is not None:
                n_match += 1
                assert ra["logFormatVariables"] == rb[2], (fmt, text)
            va, vb = ta.parse_line(text), tb.parse(text)
            assert (va["EventID"], va["variables"]) == (vb[0], vb[1]), (tmpl, text)
    assert n_match > 2000


def test_normalisation_switches_host_mirror_equals_regex(golden_dir):
    """R-norm (remove_spaces / remove_punctuation / lowercase): the sequential matcher on the normalised
    text against Python's re on the same; then the reference's audit templates with all three on."""
    from detectmateservice_b200.logformat import normalise
    assert normalise(b" A-b\tC\r\n.d_E ", norm_flags(True, True, True)) == b"abcde"
    assert normalise(b" A-b\tC ", norm_flags(True, False, False)) == b"A-bC"
    assert normalise(b" A-b\tC\x80\xc3\x84", norm_flags(False, True, True)) == b" ab\tc\x80\xc3\x84"
    r = np.random.Generator(np.random.PCG64(7))
    n_match = 0
    for it in range(300):
        lits, ends = norm_fuzz_template(r)
        norm = NORMS[it % len(NORMS)]
        tmpl = b"<*>".join(lits) + (b"<*>" if ends else b"")
        ta = FormatParser("<Content>", [tmpl], remove_spaces=norm[0], remove_punctuation=norm[1], lowercase=norm[2])
        tb = LogFormat("<Content>", [tmpl], flags=norm_flags(*norm))
        for _ in range(40):
            text = norm_fuzz_text(r, lits, ends)
            va, vb = ta.parse_line(text), tb.parse(text)
            assert (va["EventID"], va["variables"]) == (vb[0], vb[1]), (tmpl, text, norm)
            n_match += va["EventID"] == 0
    assert n_match > 3000
    tm = audit_templates(golden_dir)
    a, b = FormatParser(AUDIT, tm, remove_spaces=True, remove_punctuation=True, lowercase=True), LogFormat(AUDIT, tm, flags=7)
    plain = LogFormat(AUDIT, tm)
    for ln in open(os.path.join(golden_dir, "audit_sample.log"), "rb").read().split(b"\n")[:-1]:
        x, y = a.parse_line(ln), b.parse(ln)
        assert (x["EventID"], x["variables"], x["logFormatVariables"]) == y
        assert y[0] == plain.parse(ln)[0] and y[2] == plain.parse(ln)[2]     # same template, verbatim header
    first = b.parse(b"type=USER_ACCT msg=audit(1642723741.072:375): pid=10125 uid=0 auid=4294967295 ses=4294967295 "
                    b"msg='op=PAM:accounting acct=\"root\" exe=\"/usr/sbin/cron\" hostname=? addr=? terminal=cron res=success'")
    assert first[1] == [b"10125", b"0", b"4294967295", b"4294967295", b"pamaccounting", b"root", b"usrsbincron", b"", b"",
                        b"cron", b"success"]
    with pytest.raises(ValueError, match="nothing between"):
        LogFormat("<Content>", ["a<*> - <*>b"], flags=norm_flags(True, True, False))
    with pytest.raises(ValueError):
        FormatParser("<Content>", ["a<*> - <*>b"], remove_spaces=True, remove_punctuation=True)


def test_config_errors():
    with pytest.raises(ValueError):
        LogFormat("<A><B> x")
    with pytest.raises(ValueError):
        LogFormat("<A> <A>")
    with pytest.raises(ValueError):
        LogFormat("<A> x", ["a<*><*>b"])
    with pytest.raises(ValueError):
        LogFormat("<A> x", ["a<*>"])                             # templates need a <Content> capture
    assert LogFormat("a<b c>d <e>").header.names == ["e"]          # '<b c>' is literal text


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


EMU_KERNEL = "lanes"


@pytest.fixture(params=["lanes"])
def emu_kernel(request):
    """The matcher kernel: one thread per record."""
    global EMU_KERNEL
    EMU_KERNEL = request.param
    yield request.param
    EMU_KERNEL = "lanes"


class EmuFormat:
    def __init__(self, cfg, log_format, templates=(), name="NewValueDetector", norm=(False, False, False)):
        import emu_harness
        from detectmateservice_b200.component import parse_monitors, select_component_config
        self.mons = parse_monitors(select_component_config(cfg, name))
        self.det = emu_harness.EmuDetector([m.key for m in self.mons], table_log2=12)
        self.lib = self.det.lib
        self.det.set_monitors(_monitor_array(self.mons), len(self.mons))
        self.det.set_format(log_format, templates, norm_flags(*norm))

    def process(self, buf, n_train, with_offsets=False):
        cap = buf.count(b"\n") + 2
        f = np.full(cap, 9, np.uint8); s = np.full(cap, -1, np.float32)
        n, na, err = C.c_uint64(), C.c_uint64(), C.c_uint32()
        assert self.lib.emu_process_format(self.det.h, buf, len(buf), n_train, f.ctypes.data, s.ctypes.data, cap,
                                           C.byref(n), C.byref(na), C.byref(err)) == 0
        assert err.value == 0
        k = n.value
        assert na.value == int(f[:k].sum())
        an = self.det.anomalies()
        masks = {a[0]: a[1] for a in an}
        if with_offsets:
            return f[:k].tolist(), s[:k].tolist(), masks, {a[0]: a[2] for a in an}
        return f[:k].tolist(), s[:k].tolist(), masks

    def stats(self):
        return self.det.stats()


def _mask_of(alerts, mons):
    return sum(1 << i for i, m in enumerate(mons) if m.alert_key in alerts)


def test_emu_kernel_docs_nginx_golden(emu_kernel):
    buf = b"\n".join(nginx_line(u) for u in ("/hello", "/world", "/foobar", "/hello", "/x y")) + b"\n"
    emu = EmuFormat(NGINX_CFG, NGINX)
    f, s, masks = emu.process(buf, 2)
    assert f == [0, 0, 1, 0, 1] and s == [0.0, 0.0, 1.0, 0.0, 1.0] and masks == {2: 1, 4: 1}


AUDIT_CFG = {"detectors": {"NewValueDetector": {
    "method_type": "new_value_detector", "data_use_training": 250, "auto_config": False,
    "global": {"g": {"header_variables": [{"pos": "type"}]}},
    "events": {0: {"pam": {"variables": [{"pos": 4, "name": "op"}, {"pos": 6, "name": "exe"}, {"pos": 9, "name": "terminal"}],
                           "header_variables": [{"pos": "type"}]}},
               1: {"unit": {"variables": [{"pos": 4, "name": "unit"}, {"pos": 30}]}},
               2: {"login": {"variables": [{"pos": 3, "name": "auid"}, {"pos": 7, "name": "res"}]}},
               40: {"never": {"variables": [{"pos": 0}]}}}}}}


def test_emu_kernel_audit_templates(golden_dir, emu_kernel):
    tm = audit_templates(golden_dir)
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read()
    buf += b"type=WEIRD msg=audit(1.0:1): totally unlike=any template\nnot an audit line at all\n\n"
    buf += b"type=LOGIN msg=audit(1642723741.076:377): pid=1 uid=0 old-auid=4294967295 auid=77777 tty=(none) old-ses=4294967295 ses=65 res=9"
    orc = FormatOracle(AUDIT_CFG, AUDIT, tm)
    wf, ws, wa, bad = orc.process_lines(buf)
    emu = EmuFormat(AUDIT_CFG, AUDIT, tm)
    f, s, masks = emu.process(buf, 250)
    assert f == wf and s == ws
    assert masks == {i: _mask_of(a, emu.mons) for i, a in enumerate(wa) if a}
    assert sum(wf) >= 5 and bad == 2 and wf[-1] == 1 and ws[-1] == 2.0          # the unterminated last record counts
    assert emu.stats()["bad_records"] == bad


def test_emu_kernel_fuzz_formats(emu_kernel):
    r = np.random.Generator(np.random.PCG64(17))
    checked = 0
    for lits, ends in fuzz_formats(r, 25):
        names = ["c%d" % i for i in range(len(lits) - (0 if ends else 1))]
        if not names:
            continue
        fmt = b"".join(l + (b"<%s>" % names[i].encode() if i < len(names) else b"") for i, l in enumerate(lits))
        cfg = {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": 30,
                                                  "global": {"g": {"header_variables": [{"pos": n} for n in names]}}}}}
        lines = [fuzz_text(r, lits, ends).replace(b"\n", b"") for _ in range(90)]
        buf = b"\n".join(lines) + b"\n"
        wf, ws, wa, _ = FormatOracle(cfg, fmt).process_lines(buf)
        emu = EmuFormat(cfg, fmt)
        f, s, masks = emu.process(buf, 30)
        assert f == wf and s == ws, fmt
        assert masks == {i: _mask_of(a, emu.mons) for i, a in enumerate(wa) if a}, fmt
        checked += sum(wf)
    assert checked > 100


SYNTH_TMPL = "pid=<*> uid=<*> auid=<*> ses=<*> msg='op=<*> acct=<*> exe=<*> hostname=<*> addr=<*> terminal=<*> res=<*>' pad=<*>"
SYNTH_CFG = {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": 2000,
             "global": {"g": {"header_variables": [{"pos": "type"}]}},
             "events": {0: {"pam": {"variables": [{"pos": 5, "name": "acct"}, {"pos": 6, "name": "exe"},
                                                  {"pos": 9, "name": "terminal"}, {"pos": 10, "name": "res"}]}}}}}}


def test_emu_kernel_synthetic_header_and_variable_monitors(emu_kernel):
    """Header-capture and template-variable monitors side by side (different source lanes), on
    the config-2 synthetic records with their injected anomalies."""
    from detectmateservice_b200.synth import AuditSynth
    g = AuditSynth(seed=99)
    train, _ = g.batch(2000, inject=False)
    big, truth = g.batch(24000, inject=True)
    lines = big.split(b"\n")[:-1]
    sel = []
    for i in np.flatnonzero(truth):
        sel += lines[max(0, i - 1):i + 1]
    test = b"\n".join(sel) + b"\n"
    orc = FormatOracle(SYNTH_CFG, AUDIT, [SYNTH_TMPL])
    orc.process_lines(train)
    wf, ws, wa, bad = orc.process_lines(test)
    emu = EmuFormat(SYNTH_CFG, AUDIT, [SYNTH_TMPL])
    emu.process(train, 2000)
    f, s, masks = emu.process(test, 0)
    assert bad == 0 and f == wf and s == ws and sum(wf) >= 15
    assert masks == {i: _mask_of(a, emu.mons) for i, a in enumerate(wa) if a}
    assert len({m for m in masks.values()}) >= 3                  # several different monitors fired


AUDIT_NORM_CFG = {"detectors": {"NewValueDetector": {
    "method_type": "new_value_detector", "data_use_training": 250, "auto_config": False,
    "global": {"g": {"header_variables": [{"pos": "type"}]}},
    "events": {0: {"pam": {"variables": [{"pos": 4, "name": "op"}, {"pos": 6, "name": "exe"}, {"pos": 9, "name": "terminal"}]}},
               1: {"unit": {"variables": [{"pos": 4, "name": "unit"}]}},
               2: {"login": {"variables": [{"pos": 3, "name": "auid"}, {"pos": 7, "name": "res"}]}}}}}}
# records that differ from trained ones only in what R-norm removes (no alert) or in more (alert)
AUDIT_NORM_TAIL = (
    b"type=USER_ACCT msg=audit(1642723741.072:375): pid=10125 uid=0 auid=4294967295 ses=4294967295 "
    b"msg='op=pam:ACCOUNTING acct=\"root\" exe=\"/usr/sbin/CRON\" hostname=? addr=? terminal=cron res=success'\n"
    b"type=USER_ACCT msg=audit(1642723741.072:375): pid=10125   uid=0 AUID=4294967295 ses=4294967295 "
    b"msg='op=PAM:accounting acct=\"root\" exe=\"/usr/sbin/cron2\" hostname=? addr=? terminal=cron res=success'\n"
    b"type=LOGIN msg=audit(1642723741.076:377): pid=1 uid=0 old-auid=4294967295 auid=77777 tty=(none) old-ses=4294967295 ses=65 res=9")


def test_emu_kernel_normalisation_switches(golden_dir, emu_kernel):
    """R-norm on the device path: the reference's audit templates with all three switches on
    (tests/library_integration/test_pipe_filereader_matcher_nvd.py:82-84), then random templates
    under every switch combination, against the regular-expression oracle."""
    tm = audit_templates(golden_dir)
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read() + AUDIT_NORM_TAIL
    norm = (True, True, True)
    wf, ws, wa, bad = FormatOracle(AUDIT_NORM_CFG, AUDIT, tm, norm).process_lines(buf)
    emu = EmuFormat(AUDIT_NORM_CFG, AUDIT, tm, norm=norm)
    f, s, masks = emu.process(buf, 250)
    assert f == wf and s == ws and bad == 0
    assert masks == {i: _mask_of(a, emu.mons) for i, a in enumerate(wa) if a}
    assert wf[-3:] == [0, 1, 1] and wa[-2] == {"EventID 0 - exe": "Unknown value: 'usrsbincron2'"}
    r = np.random.Generator(np.random.PCG64(29))
    checked = 0
    for it in range(20):
        lits, ends = norm_fuzz_template(r)
        norm = NORMS[it % len(NORMS)]
        n_caps = len(lits) - (0 if ends else 1)
        tmpl = b"<*>".join(lits) + (b"<*>" if ends else b"")
        cfg = {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": 30,
               "global": {"g": {"header_variables": [{"pos": "h"}]}},
               "events": {0: {"e": {"variables": [{"pos": i} for i in range(n_caps)]}}}}}}
        lines = [b"%d|" % int(r.integers(0, 3)) + norm_fuzz_text(r, lits, ends) for _ in range(120)]
        buf = b"\n".join(lines) + b"\n"
        wf, ws, wa, _ = FormatOracle(cfg, "<h>|<Content>", [tmpl], norm).process_lines(buf)
        emu = EmuFormat(cfg, "<h>|<Content>", [tmpl], norm=norm)
        f, s, masks = emu.process(buf, 30)
        assert f == wf and s == ws, (tmpl, norm)
        assert masks == {i: _mask_of(a, emu.mons) for i, a in enumerate(wa) if a}, (tmpl, norm)
        checked += sum(wf)
    assert checked > 100


def test_emu_set_format_errors():
    with pytest.raises(ValueError, match="nothing between"):
        EmuFormat(NGINX_CFG, "<Content>", ["a<*> - <*>b"], norm=(True, True, False))
    with pytest.raises(ValueError, match="nothing between"):
        EmuFormat(NGINX_CFG, "<A><B>")
    with pytest.raises(ValueError, match="twice"):
        EmuFormat(NGINX_CFG, "<A> <A>")
    with pytest.raises(ValueError, match="Content"):
        EmuFormat(NGINX_CFG, "<A> x", ["y<*>"])
    with pytest.raises(ValueError, match="more than 32"):
        EmuFormat(NGINX_CFG, " ".join("<c%d>" % i for i in range(40)))


# ------------------------------------------------------------------------------------------ generated configurations
def _message(case, seed):
    """The case's records as one message; every other seed leaves the last record unterminated."""
    return b"\n".join(case["lines"]) + (b"\n" if seed % 2 == 0 else b"")


def _record_starts(buf):
    starts, pos = [], 0
    for ln in buf.split(b"\n"):
        starts.append(pos)
        pos += len(ln) + 1
    return starts


class FormatTally:
    """What a run of generated cases exercised, so that it cannot pass vacuously."""

    def __init__(self):
        self.alerts = self.bad = self.late = self.cap32 = self.var31 = self.unmatched_alerts = self.records = 0
        self.templates_hit = set()

    def add(self, case, orc, flags, mons):
        self.records += len(flags)
        self.alerts += sum(flags)
        self.bad += sum(e is None for e in orc.eids)
        for e in orc.eids:
            if e is not None and e >= 0:
                self.templates_hit.add((id(case), e))
                self.late += case["shadowed"][e]
                self.cap32 += case["templates"][e].count(b"<*>") == 32
        for k, m in enumerate(mons):
            self.var31 += orc.unknown[k] if m.source == "variable" and m.pos == 31 else 0
            self.unmatched_alerts += orc.unknown[k] if m.event_id == -1 else 0


def check_case(case, seed, run, tally=None):
    """run(cfg, log_format, templates, norm, buf, n_train) -> (flags, scores, {line: (mask, offset)}, stats): one
    message of the case through a fresh detector, compared with the oracle in everything it reports."""
    from detectmateservice_b200.component import parse_monitors, select_component_config
    norm = case["norm"]
    cfg = {"detectors": {"NewValueDetector": dict(case["cfg"]["detectors"]["NewValueDetector"], data_use_training=case["n_train"])}}
    mons = parse_monitors(select_component_config(cfg, "NewValueDetector"))
    buf = _message(case, seed)
    orc = FormatOracle(cfg, case["log_format"], case["templates"], norm)
    wf, ws, wa, bad = orc.process_lines(buf)
    f, s, an, st = run(cfg, case["log_format"], case["templates"], norm, buf, case["n_train"])
    ctx = (seed, norm, case["log_format"])
    assert f == wf and s == ws, ctx
    starts = _record_starts(buf)
    assert an == {i: (_mask_of(a, mons), starts[i]) for i, a in enumerate(wa) if a}, ctx
    n, tr = len(wf), min(case["n_train"], len(wf))
    assert (st["lines"], st["train_lines"], st["detect_lines"], st["bytes"]) == (n, tr, n - tr, len(buf)), ctx
    assert (st["anomalies"], st["score_sum"], st["bad_records"]) == (sum(wf), int(sum(ws)), bad), ctx
    assert st["unknown_per_key"] == orc.unknown, ctx
    if tally is not None:
        tally.add(case, orc, wf, mons)


def emu_run(cfg, log_format, templates, norm, buf, n_train):
    emu = EmuFormat(cfg, log_format, templates, norm=norm)
    f, s, masks, offs = emu.process(buf, n_train, with_offsets=True)
    st = emu.stats()
    st["unknown_per_key"] = st["unknown_per_key"][:len(emu.mons)]
    emu.det.close()
    return f, s, {i: (m, offs[i]) for i, m in masks.items()}, st


def test_emu_format_generated_templates_every_switch(emu_kernel):
    """2 to 63 templates in families sharing prefixes, literals of up to 255 bytes (periodic, self-overlapping, with
    near-misses in front), monitors of every scope, empty / malformed / \\r / 0x7F / >= 0x80 records and runs of tiny
    Contents: the kernel source under every R-norm switch combination against the regex oracle."""
    tally = FormatTally()
    for seed in range(12):
        for norm in ALL_NORMS:
            check_case(format_case(seed, norm), seed, emu_run, tally)
    assert tally.records > 30000 and tally.alerts > 8000 and tally.bad > 1500
    assert len(tally.templates_hit) > 800 and tally.late > 300
    assert tally.cap32 > 20 and tally.var31 > 0 and tally.unmatched_alerts > 100


def test_emu_format_every_split_of_a_40_record_message():
    """Training ends at every record of a 40-record message: the train launch's line_hi and the detect launch's
    line_lo at every position, including inside a warp."""
    n_checked = 0
    for seed, norm in ((3, (True, True, True)), (4, (False, False, False)), (7, (False, True, True))):
        case = format_case(seed, norm, n_records=40, n_templates=8)
        for n_train in range(41):
            check_case(dict(case, n_train=n_train), seed, emu_run)
            n_checked += 1
    assert n_checked == 123


# ------------------------------------------------------------------------------------------ configuration limits
def _lf_error(log_format, templates=(), flags=0):
    from detectmateservice_b200.logformat import LogFormat
    try:
        LogFormat(log_format, templates, flags=flags)
    except ValueError as e:
        return str(e)
    return None


def _emu_error(log_format, templates=(), flags=0):
    try:
        EmuFormat(NGINX_CFG, log_format, templates, norm=(bool(flags & 1), bool(flags & 2), bool(flags & 4)))
    except ValueError as e:
        return str(e)
    return None


def _limit_cases():
    """(name, log_format, templates, norm flags, accepted?) exactly at each device limit and one past it."""
    hdr = "<h>|<Content>"                                        # literals "" and "|": 2 literals, 1 word
    caps = lambda n, end: ",".join("<c%d>" % i for i in range(n)) + end
    wild = lambda n, end, sep=",": sep.join("<*>" for _ in range(n)) + end
    out = [
        ("32 header captures, final literal", caps(32, ";"), [], 0, True),
        ("33 header captures, final literal", caps(33, ";"), [], 0, False),
        ("32 header captures, final capture", caps(32, ""), [], 0, True),
        ("33 header captures, final capture", caps(33, ""), [], 0, False),
        ("32 wildcards, final literal", hdr, [wild(32, ";")], 0, True),
        ("33 wildcards, final literal", hdr, [wild(33, ";")], 0, False),
        ("32 wildcards, final literal R-norm empties", hdr, ["x" + wild(32, "'", "a")], 2, True),
        ("33 wildcards, final literal R-norm empties", hdr, ["x" + wild(33, "'", "a")], 2, False),
        ("255-byte literal", hdr, ["a" * 255 + "<*>"], 0, True),
        ("256-byte literal", hdr, ["a" * 256 + "<*>"], 0, False),
        ("256-byte header literal", "<h>" + "a" * 256 + "<Content>", [], 0, False),
        ("256 bytes, 255 after R-norm", hdr, ["a" * 128 + " " + "a" * 127 + "<*>"], 1, True),
        ("257 bytes, 256 after R-norm", hdr, ["a" * 128 + " " + "a" * 128 + "<*>"], 1, False),
        ("63 templates", hdr, ["t%d<*>" % i for i in range(63)], 0, True),
        ("64 templates", hdr, ["t%d<*>" % i for i in range(64)], 0, False),
    ]
    # 512 literals: the header's 2 + 15 templates of 33 + one of 15 (one more literal in the last template: 513)
    t33 = "a" + wild(32, "b")
    out.append(("512 literals", hdr, [t33] * 15 + ["a" + wild(14, "b")], 0, True))
    out.append(("513 literals", hdr, [t33] * 15 + ["a" + wild(15, "b")], 0, False))
    # 4096 bytes of literal text: the header's 1 word + 15 literals of 64 words + one of 63 words = 1024 words
    big = ["x" * 255 + "<*>"] * 15
    out.append(("4096 pool bytes", hdr, big + ["y" * 252 + "<*>"], 0, True))
    out.append(("4097 pool bytes", hdr, big + ["y" * 253 + "<*>"], 0, False))
    out.append(("4096 pool bytes, then a 1-byte literal (one more word)", hdr, big + ["y" * 252 + "<*>", "z<*>"], 0, False))
    # two limits broken at once: the first in the device's order wins
    out.append(("long literal in template 2 before the literal count", hdr, ["a<*>", "b<*>", "c" * 300 + "<*>"] + [t33] * 16, 0, False))
    out.append(("literal count before a later long literal", hdr, [t33] * 16 + ["c" * 300 + "<*>"], 0, False))
    out.append(("the 64th template before its long literal", hdr, ["t%d<*>" % i for i in range(63)] + ["c" * 300 + "<*>"], 0, False))
    return out


@pytest.mark.parametrize("case", _limit_cases(), ids=lambda c: c[0])
def test_format_limits_host_mirror_equals_device_builder(case):
    """LogFormat applies every limit of dm_format_build, in its order and with its reason, so that a configuration
    the device rejects fails where the component is constructed on every machine."""
    _, log_format, templates, flags, ok = case
    want = _emu_error(log_format, templates, flags)
    got = _lf_error(log_format, templates, flags)
    assert (want is None) == ok, want
    assert got == want


def test_format_limits_nul_byte():
    """The C ABI ends a configuration string at its first NUL: the host mirror rejects one anywhere."""
    for log_format, templates in (("<h>|\0<Content>", []), ("<h>|<Content>", ["a\0b<*>"]), ("<h>|<Content>", ["ok<*>", "\0"])):
        assert "NUL" in _lf_error(log_format, templates)
    from detectmateservice_b200.logformat import LogFormat
    with pytest.raises(ValueError, match="NUL"):
        LogFormat("<h>|<Content>", ["a<*>"], content_name="Con\0tent")


def test_component_rejects_device_limits_at_construction():
    from detectmateservice_b200.component import B200NewValueDetector
    det = dict(NGINX_CFG["detectors"]["NewValueDetector"], params={"log_format": "<h>|<Content>", "templates": ["a" * 256 + "<*>"]})
    with pytest.raises(ValueError, match="longer than 255"):
        B200NewValueDetector(config={"detectors": {"NewValueDetector": det}})


# 32 captures each, ending with a literal; distinct separators keep the regex oracle's backtracking linear
CAP32_NAMES = ["c%d" % i for i in range(31)] + ["Content"]
CAP32_FMT = "<c0>" + "".join(":%d=<%s>" % (i, n) for i, n in enumerate(CAP32_NAMES) if i) + ";"
CAP32_TMPL = b"[<*>" + b"".join(b"/%d/<*>" % i for i in range(1, 32)) + b"]"
CAP32_CFG = {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": 40,
             "global": {"g": {"header_variables": [{"pos": "c0"}, {"pos": "c30"}]}},
             "events": {0: {"v": {"variables": [{"pos": 0}, {"pos": 30}, {"pos": 31}, {"pos": 32}]}}}}}}


def cap32_message(seed, n=120):
    """Records of CAP32_FMT whose Content holds text for CAP32_TMPL; some miss the template's ']' (EventID -1), some
    the log_format's ';' (malformed)."""
    r = np.random.Generator(np.random.PCG64(seed))
    lines = []
    for i in range(n):
        val = lambda: b"%d" % int(r.integers(0, 3 if i < 40 else 4))
        content = b"[" + val() + b"".join(b"/%d/" % j + val() for j in range(1, 32)) + b"]"
        if r.random() < 0.1:
            content = content[:-1]
        ln = val() + b"".join(b":%d=" % j + (val() if j < 31 else content) for j in range(1, 32)) + b";"
        if r.random() < 0.05:
            ln = ln[:-1]
        lines.append(ln)
    return b"\n".join(lines) + b"\n"


def test_emu_32_captures_with_final_literal_end_to_end():
    """A log_format and a template of 32 captures each, both ending with a literal: accepted, and matched as the regex
    oracle matches them (variable 31 and header capture c30 monitored)."""
    fmt = CAP32_FMT
    buf = cap32_message(1)
    wf, ws, wa, bad = FormatOracle(CAP32_CFG, fmt, [CAP32_TMPL]).process_lines(buf)
    emu = EmuFormat(CAP32_CFG, fmt, [CAP32_TMPL])
    f, s, masks = emu.process(buf, 40)
    assert f == wf and s == ws and masks == {i: _mask_of(a, emu.mons) for i, a in enumerate(wa) if a}
    assert bad > 0 and sum(wf) > 20 and any("EventID 0 - 31" in a for a in wa)


# ------------------------------------------------------------------------------------------ GPU tier
def _component(cfg, params, name="NewValueDetector"):
    from detectmateservice_b200.component import B200NewValueDetector
    det = dict(cfg["detectors"]["NewValueDetector"])
    det["params"] = dict(det.get("params") or {}, **params)
    c = B200NewValueDetector(name=name, config={"detectors": {name: det}})
    c.clock = lambda: 1773848383
    return c


@pytest.mark.gpu
def test_gpu_docs_nginx_pipeline_golden(golden_dir):
    """docs/getting_started.md:395-435,498-510 with parser + detector fused: raw access-log lines in,
    the documented DetectorSchema out."""
    g = json.load(open(os.path.join(golden_dir, "docs_golden.json")))
    comp = _component(NGINX_CFG, {"log_format": NGINX})
    outs = [comp.process(nginx_line(u) + b"\n") for u in ("/hello", "/world", "/foobar")]
    assert outs[0] is None and outs[1] is None
    a = wire.decode_detector_schema(outs[2])
    e = g["expected"]
    assert a["alertsObtain"] == e["alertsObtain"] == {"Global - URL": "Unknown value: '/foobar'"}
    assert (a["detectorID"], a["detectorType"], a["alertID"], a["score"], a["description"]) == (
        e["detectorID"], e["detectorType"], e["alertID"], e["score"], e["description"])
    assert a["extractedTimestamps"] == [1773848383]              # the nginx Time is not epoch seconds: detection time
    # a whole message of lines, one of them not in the format
    buf = b"\n".join([nginx_line("/hello"), b"garbage line", nginx_line("/admin", ip="10.0.0.9"), nginx_line("/world")]) + b"\n"
    alerts = [wire.decode_detector_schema(b) for b in wire.split_delimited(comp.process(buf))]
    assert [x["alertsObtain"] for x in alerts] == [{"Global - URL": "Unknown value: '/admin'"}]
    assert alerts[0]["logIDs"] == ["5"] and comp.stats()["bad_records"] == 1
    comp.close()


@pytest.mark.gpu
def test_gpu_audit_templates_component_vs_oracle(golden_dir):
    tm = audit_templates(golden_dir)
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read()
    buf += b"type=WEIRD msg=audit(1.0:1): totally unlike=any template\nnot an audit line at all\n\n"
    buf += b"type=LOGIN msg=audit(1642723741.076:377): pid=1 uid=0 old-auid=4294967295 auid=77777 tty=(none) old-ses=4294967295 ses=65 res=9\n"
    wf, ws, wa, bad = FormatOracle(AUDIT_CFG, AUDIT, tm).process_lines(buf)
    comp = _component(AUDIT_CFG, {"log_format": AUDIT, "path_templates": os.path.join(golden_dir, "audit_templates.txt")})
    cut = buf.index(b"\n", len(buf) // 3) + 1                    # two messages; training ends inside the first or second
    got = []
    for part in (buf[:cut], buf[cut:]):
        out = comp.process(part)
        got += [wire.decode_detector_schema(b) for b in wire.split_delimited(out)] if out else []
    want = [(i, a) for i, a in enumerate(wa) if a]
    assert [(int(x["logIDs"][0]), x["alertsObtain"]) for x in got] == want
    assert [x["score"] for x in got] == [ws[i] for i, _ in want]
    st = comp.stats()
    assert st["bad_records"] == bad == 2 and st["anomalies"] == sum(wf) and st["lines"] == len(wf)
    comp.close()
    from detectmateservice_b200.component import decode_compact
    comp = _component(AUDIT_CFG, {"log_format": AUDIT, "templates": [t.decode() for t in tm], "output_format": "compact"})
    f, s = decode_compact(comp.process(buf))
    assert f.tolist() == wf and s.tolist() == ws
    comp.close()


@pytest.mark.gpu
def test_gpu_normalisation_switches(golden_dir):
    """The reference's audit parser config as it stands -- remove_spaces, remove_punctuation, lowercase all
    true (tests/library_integration/test_pipe_filereader_matcher_nvd.py:74-88) -- through the component,
    then random templates under every switch combination through the C-ABI, against the oracle."""
    from detectmateservice_b200.detector import DeviceDetector
    from detectmateservice_b200.component import parse_monitors, select_component_config
    tm = audit_templates(golden_dir)
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read() + AUDIT_NORM_TAIL + b"\n"
    norm = (True, True, True)
    wf, ws, wa, bad = FormatOracle(AUDIT_NORM_CFG, AUDIT, tm, norm).process_lines(buf)
    comp = _component(AUDIT_NORM_CFG, {"log_format": AUDIT, "path_templates": os.path.join(golden_dir, "audit_templates.txt"),
                                       "remove_spaces": True, "remove_punctuation": True, "lowercase": True})
    cut = buf.index(b"\n", len(buf) // 2) + 1
    got = []
    for part in (buf[:cut], buf[cut:]):
        out = comp.process(part)
        got += [wire.decode_detector_schema(b) for b in wire.split_delimited(out)] if out else []
    want = [(i, a) for i, a in enumerate(wa) if a]
    assert [(int(x["logIDs"][0]), x["alertsObtain"]) for x in got] == want and len(want) >= 5
    assert want[-2][1] == {"EventID 0 - exe": "Unknown value: 'usrsbincron2'"}
    assert comp.stats()["bad_records"] == bad == 0
    comp.close()
    r = np.random.Generator(np.random.PCG64(31))
    checked = 0
    for it in range(40):
        lits, ends = norm_fuzz_template(r)
        norm = NORMS[it % len(NORMS)]
        n_caps = len(lits) - (0 if ends else 1)
        tmpl = b"<*>".join(lits) + (b"<*>" if ends else b"")
        cfg = {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": 100,
               "global": {"g": {"header_variables": [{"pos": "h"}]}},
               "events": {0: {"e": {"variables": [{"pos": i} for i in range(n_caps)]}}}}}}
        mons = parse_monitors(select_component_config(cfg, "NewValueDetector"))
        lines = [b"%d|" % int(r.integers(0, 3)) + norm_fuzz_text(r, lits, ends) for _ in range(500)]
        buf = b"\n".join(lines) + b"\n"
        wf, ws, wa, _ = FormatOracle(cfg, "<h>|<Content>", [tmpl], norm).process_lines(buf)
        det = DeviceDetector([m.key for m in mons], max_batch_bytes=1 << 20)
        det.set_monitors([{"event_id": m.event_id, "source": m.source, "pos": m.pos} for m in mons])
        det.set_format("<h>|<Content>", [tmpl], norm_flags=norm_flags(*norm))
        f, s = det.process_lines(buf, n_train_lines=100)
        assert f.tolist() == wf and s.tolist() == ws, (tmpl, norm)
        assert {a[0]: a[1] for a in det.anomalies()} == {i: _mask_of(a, mons) for i, a in enumerate(wa) if a}
        checked += sum(wf)
        det.close()
    assert checked > 300


@pytest.mark.gpu
def test_gpu_fuzz_formats_and_switching():
    from detectmateservice_b200.detector import DeviceDetector
    from detectmateservice_b200._lib import DmError
    from detectmateservice_b200.component import parse_monitors, select_component_config
    r = np.random.Generator(np.random.PCG64(23))
    checked = 0
    for lits, ends in fuzz_formats(r, 60):
        names = ["c%d" % i for i in range(len(lits) - (0 if ends else 1))]
        if not names:
            continue
        fmt = b"".join(l + (b"<%s>" % names[i].encode() if i < len(names) else b"") for i, l in enumerate(lits))
        cfg = {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": 100,
                                                  "global": {"g": {"header_variables": [{"pos": n} for n in names]}}}}}
        mons = parse_monitors(select_component_config(cfg, "NewValueDetector"))
        lines = [fuzz_text(r, lits, ends).replace(b"\n", b"") for _ in range(400)]
        buf = b"\n".join(lines) + b"\n"
        wf, ws, wa, _ = FormatOracle(cfg, fmt).process_lines(buf)
        det = DeviceDetector([m.key for m in mons], max_batch_bytes=1 << 20)
        det.set_monitors([{"event_id": m.event_id, "source": m.source, "pos": m.pos} for m in mons])
        det.set_format(fmt.decode())
        f, s = det.process_lines(buf, n_train_lines=100)
        assert f.tolist() == wf and s.tolist() == ws, fmt
        assert {a[0]: a[1] for a in det.anomalies()} == {i: _mask_of(a, mons) for i, a in enumerate(wa) if a}
        checked += sum(wf)
        det.close()
    assert checked > 500
    # errors, and switching between log_format and key=value tokenisation on one handle
    det = DeviceDetector([b"type"], max_batch_bytes=1 << 20)
    with pytest.raises(DmError):
        det.set_format("<A> <B>")                                # before set_monitors
    det.set_monitors([{"event_id": None, "source": "header", "pos": "type"}])
    for bad in ("<A><B>", "<A> <A>"):
        with pytest.raises(DmError):
            det.set_format(bad)
    with pytest.raises(DmError):
        det.set_format("<A> x", ["y<*>"])
    lines = b"type=A msg=audit(1.0:1): k=v\ntype=B msg=audit(1.0:2): k=v\ntype=A msg=audit(1.0:3): k=v\n"
    det.set_format(AUDIT)
    assert det.process_lines(lines, n_train_lines=1)[0].tolist() == [0, 1, 0]
    with pytest.raises(DmError):
        det.submit(lines)                                        # the pipelined path is key=value only
    det.set_format(None)
    det.reset()
    assert det.process_lines(lines, n_train_lines=2)[0].tolist() == [0, 0, 0]
    det.close()


@pytest.mark.gpu
def test_gpu_format_mode_full_size_message():
    """BASELINE config-2 sized message (64k x 256 B) in log_format + template mode against the oracle."""
    from detectmateservice_b200.detector import DeviceDetector
    from detectmateservice_b200.component import parse_monitors, select_component_config
    from detectmateservice_b200.synth import AuditSynth
    tmpl, cfg = SYNTH_TMPL, SYNTH_CFG
    mons = parse_monitors(select_component_config(cfg, "NewValueDetector"))
    g = AuditSynth(seed=99)
    train, _ = g.batch(65536, inject=False)
    test, truth = g.batch(65536, inject=True)
    det = DeviceDetector([m.key for m in mons], max_batch_bytes=32 << 20)
    det.set_monitors([{"event_id": m.event_id, "source": m.source, "pos": m.pos} for m in mons])
    det.set_format(AUDIT, [tmpl])
    det.process_lines(train, n_train_lines=65536)
    f, s = det.process_lines(test)
    orc = FormatOracle(cfg, AUDIT, [tmpl])
    orc.nvd.data_use_training = 65536
    orc.process_lines(train)
    wf, ws, _, bad = orc.process_lines(test)
    assert bad == 0 and f.tolist() == wf and s.tolist() == ws
    assert int(f.sum()) == int(np.asarray(truth).astype(bool).sum()) > 20       # every injected anomaly, nothing else
    det.close()


# ------------------------------------------------------------------------------------------ GPU tier: generated configurations
def _device_detector(cfg, log_format, templates, norm, max_batch_bytes=1 << 20):
    from detectmateservice_b200.detector import DeviceDetector
    from detectmateservice_b200.component import parse_monitors, select_component_config
    mons = parse_monitors(select_component_config(cfg, "NewValueDetector"))
    det = DeviceDetector([m.key for m in mons], max_batch_bytes=max_batch_bytes)
    det.set_monitors([{"event_id": m.event_id, "source": m.source, "pos": m.pos} for m in mons])
    lf = log_format.decode() if isinstance(log_format, bytes) else log_format
    det.set_format(lf, list(templates), norm_flags=norm_flags(*norm))
    return det, mons


def gpu_run(cfg, log_format, templates, norm, buf, n_train):
    det, mons = _device_detector(cfg, log_format, templates, norm)
    f, s = det.process_lines(buf, n_train_lines=n_train)
    an = {a[0]: (a[1], a[2]) for a in det.anomalies()}
    st = det.stats()
    det.close()
    return f.tolist(), s.tolist(), an, st


def _grid_threads(threads_per_cta=64):
    """Threads of the record kernels' largest grid on this device: sm_count * 32 CTAs."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 32 * threads_per_cta


@pytest.mark.gpu
def test_gpu_format_generated_templates_every_switch():
    """The emulator tier's generated configurations, same seeds, through the library on the device."""
    tally = FormatTally()
    for seed in range(12):
        for norm in ALL_NORMS:
            check_case(format_case(seed, norm), seed, gpu_run, tally)
    assert tally.records > 30000 and tally.alerts > 8000 and tally.bad > 1500
    assert len(tally.templates_hit) > 800 and tally.late > 300
    assert tally.cap32 > 20 and tally.var31 > 0 and tally.unmatched_alerts > 100


@pytest.mark.gpu
def test_gpu_format_every_split_of_a_40_record_message():
    for seed, norm in ((3, (True, True, True)), (4, (False, False, False)), (7, (False, True, True))):
        case = format_case(seed, norm, n_records=40, n_templates=8)
        for n_train in range(41):
            check_case(dict(case, n_train=n_train), seed, gpu_run)


def _memo_oracle(make_oracle, step, lines, n_train):
    """Oracle results of the detection records of a long message drawn from a small set of distinct records: training
    only inserts into sets, and after it a distinct record always gives the same answer, so each is stepped once."""
    orc = make_oracle()
    for ln in dict.fromkeys(lines[:n_train]):
        step(orc, ln)
    getattr(orc, "nvd", orc).n_seen = n_train                    # training is over
    return {ln: step(orc, ln) for ln in dict.fromkeys(lines[n_train:])}


@pytest.mark.gpu
def test_gpu_format_stride_more_records_than_twice_the_grid():
    """One format-mode message with more than twice as many records as the grid has threads, R-norm on, 8 templates,
    training ending at a record index that is not a multiple of 32: both launches run their stride loop."""
    import collections
    from oracle.rfmt import FormatParser
    from fmtgen import monitor_config, n_captures, template_text
    norm = (True, True, True)
    r = np.random.Generator(np.random.PCG64(12))
    ts = [norm_fuzz_template(r) for _ in range(8)]
    templates = [template_text(l, e) for l, e in ts]
    pool = []
    while len(pool) < 3000:
        lits, ends = ts[int(r.integers(0, 8))]
        ln = b"h%d|" % int(r.integers(0, 5)) + norm_fuzz_text(r, lits, ends, 0.3)
        if len(ln) <= 24:
            pool.append(ln if r.random() < 0.95 else ln.replace(b"|", b""))   # no '|': malformed
    n = 2 * _grid_threads() + 60001
    n_train = 300001
    case = {"log_format": b"<h>|<Content>", "templates": templates,
            "cfg": monitor_config(r, [n_captures(l, e, 7) for l, e in ts], False, n_train)}
    idx = np.concatenate([r.integers(0, len(pool) * 3 // 5, n_train), r.integers(0, len(pool), n - n_train)])
    lines = [pool[i] for i in idx]                               # detection also draws records training never saw
    tiny = [b"h%d|" % (i % 4) + bytes(b"aB =:"[int(j)] for j in r.integers(0, 5, i % 4)) for i in range(5000)]
    lines[400000:400000 + len(tiny)] = tiny                      # thousands of 0-3 byte Contents in a row
    assert n_train % 32 and n_train > _grid_threads() and len(lines) > 2 * _grid_threads()
    buf = b"\n".join(lines) + b"\n"
    assert len(buf) <= 16 << 20
    cfg = {"detectors": {"NewValueDetector": dict(case["cfg"]["detectors"]["NewValueDetector"], data_use_training=n_train)}}

    def step(orc, ln):
        f, s, a, _ = orc.process_lines(ln + b"\n")
        return f[0], s[0], a[0]
    memo = _memo_oracle(lambda: FormatOracle(cfg, case["log_format"], case["templates"], norm), step, lines, n_train)
    det, mons = _device_detector(cfg, case["log_format"], case["templates"], norm, max_batch_bytes=16 << 20)
    assert det.max_lines >= len(lines)
    f, s = det.process_lines(buf, n_train_lines=n_train)
    want = [memo[ln] for ln in lines[n_train:]]
    assert f[:n_train].sum() == 0 and s[:n_train].sum() == 0
    assert f[n_train:].tolist() == [w[0] for w in want] and s[n_train:].tolist() == [w[1] for w in want]
    an = det.anomalies()
    assert {a[0]: a[1] for a in an} == {n_train + i: _mask_of(w[2], mons) for i, w in enumerate(want) if w[2]}
    parser = FormatParser(case["log_format"], case["templates"], remove_spaces=True, remove_punctuation=True, lowercase=True)
    counts = collections.Counter(lines)
    bad = sum(c for ln, c in counts.items() if parser.parse_line(ln) is None)
    st = det.stats()
    assert st["lines"] == len(lines) and st["bad_records"] == bad > 1000 and st["anomalies"] == int(f.sum()) > 500
    eids = collections.Counter(parser.parse_line(ln)["EventID"] for ln in set(pool) if parser.parse_line(ln))
    assert len([e for e in eids if e >= 0]) >= 3
    det.close()


@pytest.mark.gpu
def test_gpu_format_32_monitored_header_captures():
    """32 monitored header captures: max_slots = 32, the largest dynamic shared memory a format launch asks for
    (2 * 32 * 64 * 8 B = 32 KiB), with the 32-wildcard template matched on the last of them."""
    cfg = {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": 40,
           "global": {"g": {"header_variables": [{"pos": n} for n in CAP32_NAMES]}}}}}
    buf = cap32_message(0, n=40) + b"".join(cap32_message(s, n=1000) for s in range(1, 9))
    wf, ws, wa, bad = FormatOracle(cfg, CAP32_FMT, [CAP32_TMPL]).process_lines(buf)
    det, mons = _device_detector(cfg, CAP32_FMT, [CAP32_TMPL], (False, False, False), max_batch_bytes=4 << 20)
    assert len(mons) == 32
    f, s = det.process_lines(buf, n_train_lines=40)
    assert f.tolist() == wf and s.tolist() == ws
    assert {a[0]: a[1] for a in det.anomalies()} == {i: _mask_of(a, mons) for i, a in enumerate(wa) if a}
    assert bad > 100 and sum(wf) > 1000 and max(ws) >= 8
    det.close()


@pytest.mark.gpu
def test_gpu_32_captures_with_final_literal_end_to_end():
    buf = cap32_message(1)
    wf, ws, wa, bad = FormatOracle(CAP32_CFG, CAP32_FMT, [CAP32_TMPL]).process_lines(buf)
    det, mons = _device_detector(CAP32_CFG, CAP32_FMT, [CAP32_TMPL], (False, False, False))
    f, s = det.process_lines(buf, n_train_lines=40)
    assert f.tolist() == wf and s.tolist() == ws
    assert {a[0]: a[1] for a in det.anomalies()} == {i: _mask_of(a, mons) for i, a in enumerate(wa) if a}
    assert bad > 0 and any("EventID 0 - 31" in a for a in wa)
    det.close()


@pytest.mark.gpu
def test_gpu_format_1mib_record_with_512kib_capture():
    """Records of 1 MiB whose monitored variable is 512 KiB, among short ones, with and without R-norm."""
    tmpl = [b"k=<*>;v=<*>;"]
    cfg = {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": 3,
           "global": {"g": {"header_variables": [{"pos": "h"}]}},
           "events": {0: {"e": {"variables": [{"pos": 0}, {"pos": 1}]}}}}}}
    big_v = bytes(b"ab"[i % 2] for i in range(512 << 10))
    big = lambda k, v: b"h0|k=" + k + b";v=" + v + b";"
    pad = b"x" * ((1 << 20) - len(big(b"", big_v)))
    lines = [big(pad, big_v), b"h0|k=1;v=2;", big(pad, big_v[:-1] + b"c"), big(pad[:-3], big_v), b"h1|k=1;v=2;",
             big(pad, big_v[:-1] + b"c"), big(pad, big_v)]
    assert len(lines[0]) == 1 << 20
    buf = b"\n".join(lines) + b"\n"
    for norm in ((False, False, False), (True, True, True)):
        wf, ws, wa, bad = FormatOracle(cfg, "<h>|<Content>", tmpl, norm).process_lines(buf)
        det, mons = _device_detector(cfg, "<h>|<Content>", tmpl, norm, max_batch_bytes=8 << 20)
        f, s = det.process_lines(buf, n_train_lines=3)
        assert f.tolist() == wf and s.tolist() == ws, norm
        assert {a[0]: (a[1], a[2]) for a in det.anomalies()} == {
            i: (_mask_of(a, mons), _record_starts(buf)[i]) for i, a in enumerate(wa) if a}
        assert wf == [0, 0, 0, 1, 1, 0, 0]                          # a shorter key of 1 MiB - 3 bytes; header h1
        det.close()


@pytest.mark.gpu
def test_gpu_format_device_resident_hostile_slack():
    """Messages in their own device tensors with exactly 16 bytes of slack made of the configured literals and '\\n',
    through enqueue_device + sync, the last record ending at nbytes on every residue mod 4 (and terminated)."""
    import torch
    for seed, norm in ((21, (False, False, False)), (22, (True, True, True)), (23, (False, True, False))):
        case = format_case(seed, norm, n_records=300, n_templates=16)
        cfg = {"detectors": {"NewValueDetector": dict(case["cfg"]["detectors"]["NewValueDetector"], data_use_training=30)}}
        lits = b"".join(t.replace(b"<*>", b"") + b"\n" for t in case["templates"])
        slack = np.frombuffer((lits * (16 // max(1, len(lits)) + 1))[:16], dtype=np.uint8)
        orc = FormatOracle(cfg, case["log_format"], case["templates"], norm)
        det, mons = _device_detector(cfg, case["log_format"], case["templates"], norm)
        msgs, pos = [], 0
        for k in range(10):
            m = b"\n".join(case["lines"][pos:pos + 30])
            pos += 30
            if k % 5 == 4:
                m += b"\n"
            else:
                m += b"z"                                        # (the last record may be empty)
                while len(m) % 4 != k % 4:
                    m += b"z"
            msgs.append(m)
        assert {len(m) % 4 for m in msgs if not m.endswith(b"\n")} == {0, 1, 2, 3}
        for k, m in enumerate(msgs):
            x = torch.from_numpy(np.concatenate([np.frombuffer(m, dtype=np.uint8), slack])).cuda()
            fo = torch.full((64,), 7, dtype=torch.uint8, device="cuda")
            so = torch.full((64,), -1.0, dtype=torch.float32, device="cuda")
            n_train = 30 if k == 0 else 0
            det.enqueue_device(x.data_ptr(), len(m), n_train, fo.data_ptr(), so.data_ptr(), 64)
            n_lines, _ = det.sync()
            wf, ws, wa, _ = orc.process_lines(m)
            assert n_lines == len(wf) == 30
            assert fo[:30].cpu().tolist() == wf and so[:30].cpu().tolist() == ws, (seed, k)
            assert {a[0]: (a[1], a[2]) for a in det.anomalies()} == {
                i: (_mask_of(a, mons), _record_starts(m)[i]) for i, a in enumerate(wa) if a}, (seed, k)
        assert det.stats()["unknown_per_key"] == orc.unknown and sum(orc.unknown) > 20
        det.close()


@pytest.mark.gpu
def test_gpu_lanes_combos_stride_more_records_than_twice_the_grid():
    """Raw key=value records with combination monitors run on dm_k_lanes, whose grid has the same formula: one
    message with more than twice as many records as that grid has threads."""
    from detectmateservice_b200.detector import DeviceDetector
    from oracle.nvcd import NewValueComboDetectorOracle
    cfg = {"detectors": {"NewValueComboDetector": {"method_type": "new_value_combo_detector", "data_use_training": 0,
           "global": {"ta": {"header_variables": [{"pos": "t"}, {"pos": "a"}]},
                      "ex": {"header_variables": [{"pos": "e"}, {"pos": "x"}]},
                      "z": {"header_variables": [{"pos": "z"}]}}}}}
    r = np.random.Generator(np.random.PCG64(5))
    n = 2 * _grid_threads() + 40001
    n_train = 290017
    cols = [r.integers(0, 4, n), r.integers(0, 4, n), r.integers(0, 5, n), r.random(n)]
    lines = []
    for i in range(n):
        t, a, e, u = int(cols[0][i]), int(cols[1][i]), int(cols[2][i]), cols[3][i]
        if i < n_train:
            a, e = t, min(e, 3)                                  # training: a follows t, e never 4
        ln = b"t=%d a=%d e=%d x=%d z=%d" % (t, a, e, e % 2, t)
        if u < 0.05:
            ln = b"t=%d e=%d z=%d" % (t, e, e)                   # a member missing: its combination is skipped
        lines.append(ln)
    cfg["detectors"]["NewValueComboDetector"]["data_use_training"] = n_train
    orc0 = NewValueComboDetectorOracle(config=cfg)
    memo = _memo_oracle(lambda: NewValueComboDetectorOracle(config=cfg), lambda o, ln: o.step_line(ln), lines, n_train)
    from oracle.nvcd import combo_alert_key
    nm = len(orc0.monitors)
    keys = [combo_alert_key(orc0.monitors, m) for m in orc0.combos]
    from detectmateservice_b200.component import parse_combos, select_component_config
    mons, combos = parse_combos(select_component_config(cfg, "NewValueComboDetector"))
    assert combos == orc0.combos
    det = DeviceDetector([m.key for m in mons], max_batch_bytes=16 << 20)
    det.set_monitors([{"event_id": m.event_id, "source": m.source, "pos": m.pos} for m in mons])
    det.set_combos(combos, member_only_mask=(1 << nm) - 1)
    buf = b"\n".join(lines) + b"\n"
    f, s = det.process_lines(buf, n_train_lines=n_train)
    want = [memo[ln] for ln in lines[n_train:]]
    assert len(lines) > 2 * _grid_threads() and n_train > _grid_threads() and n_train % 32
    assert f[:n_train].sum() == 0
    assert f[n_train:].tolist() == [int(w[0]) for w in want] and s[n_train:].tolist() == [w[1] for w in want]
    got = {a[0]: a[1] for a in det.anomalies()}
    assert got == {n_train + i: sum(1 << (nm + c) for c, k in enumerate(keys) if k in w[2]) for i, w in enumerate(want) if w[2]}
    assert len(got) > 100000
    det.close()
