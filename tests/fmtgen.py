"""Generators and the oracle for the log_format / template matcher tests (csrc/dm_kernels_format.cuh).  TEST
INFRASTRUCTURE, shared by the emulator tier and the GPU tier of tests/test_format_matcher.py.

fuzz_formats / fuzz_text / norm_fuzz_template / norm_fuzz_text draw chains and texts; with their default arguments they
draw exactly what they always drew (the seeds of the older tests depend on it).  `long=True` draws literals of 1 to
about 40 bytes, a few up to 255, many of them periodic or self-overlapping; `near_miss_p` is the chance of a prefix of a
literal, or the literal with its last byte changed, in front of its real occurrence.  format_case() puts them together:
2 to 63 templates in families that share prefixes, a header log_format, monitors of every scope and record shapes the
kernel has to get right.
"""
from __future__ import annotations

import numpy as np

from oracle.nvd import NewValueDetectorOracle
from oracle.rfmt import FormatParser


class FormatOracle:
    """FormatParser (regex) + NewValueDetectorOracle: the CPU restatement of parser + detector."""

    def __init__(self, cfg, log_format, templates=(), norm=(False, False, False)):
        self.parser = FormatParser(log_format, templates, remove_spaces=norm[0], remove_punctuation=norm[1], lowercase=norm[2])
        self.nvd = NewValueDetectorOracle(config=cfg, clock=lambda: 1773848383)
        self.eids = []                                           # EventID of every record so far (None: malformed)
        self.unknown = [0] * len(self.nvd.monitors)             # alerts per monitor

    def process_lines(self, buf):
        lines = buf.split(b"\n")
        if lines and lines[-1] == b"":
            lines.pop()
        flags, scores, alerts, bad = [], [], [], 0
        keys = [m.alert_key for m in self.nvd.monitors]
        for ln in lines:
            rec = self.parser.parse_line(ln)
            if rec is None:
                bad += 1
                rec = {"EventID": None, "variables": [], "logFormatVariables": {}}
            self.eids.append(rec["EventID"])
            f, s, a = self.nvd.step(rec)
            for k, key in enumerate(keys):
                self.unknown[k] += key in a
            flags.append(int(f)); scores.append(float(s)); alerts.append(a)
        return flags, scores, alerts, bad


def _bytes(r, alpha, n):
    return bytes(alpha[int(i)] for i in r.integers(0, len(alpha), n))


def long_literal(r, alpha):
    """1 to about 40 bytes, rarely up to 255; periodic ("abab...", "aaaa..."), self-overlapping ("aaab", "ababa:") or
    random."""
    u = r.random()
    n = int(r.integers(1, 9)) if u < 0.45 else int(r.integers(9, 41)) if u < 0.97 else int(r.integers(41, 256))
    kind = r.random()
    if kind < 0.35:
        unit = _bytes(r, alpha, int(r.integers(1, 4)))
        return (unit * n)[:n]
    if kind < 0.65 and n >= 2:
        unit = _bytes(r, alpha, int(r.integers(1, 3)))
        body = (unit * n)[:n - 1]
        other = [c for c in alpha if c != body[-1]]
        return body + bytes([other[int(r.integers(0, len(other)))]])
    return _bytes(r, alpha, n)


def near_miss(r, lit, alpha):
    """A prefix of lit, or lit with its last byte changed (empty for a 1-byte literal's prefix)."""
    if len(lit) >= 2 and r.random() < 0.5:
        return lit[:int(r.integers(1, len(lit)))]
    other = [c for c in alpha if c != lit[-1]]
    return lit[:-1] + bytes([other[int(r.integers(0, len(other)))]])


def fuzz_formats(r, n, long=False):
    """Random chains over a tiny alphabet so that literals recur inside captured text."""
    alpha = b"ab =:"
    out = []
    for _ in range(n):
        k = int(r.integers(1, 5))
        if long:
            lits = [long_literal(r, alpha) for _ in range(k + 1)]
        else:
            lits = [bytes(alpha[int(i)] for i in r.integers(0, len(alpha), int(r.integers(1, 4)))) for _ in range(k + 1)]
        if r.random() < 0.4:
            lits[0] = b""
        ends = r.random() < 0.5
        out.append((lits, ends))
    return out


def fuzz_text(r, lits, ends, near_miss_p=0.0):
    alpha = b"ab =:xy"
    if r.random() < 0.25:                                        # arbitrary text, mostly non-matching
        return bytes(alpha[int(i)] for i in r.integers(0, len(alpha), int(r.integers(0, 24))))
    t = b""
    for i, lit in enumerate(lits):
        if near_miss_p and i and lit and r.random() < near_miss_p:
            t += near_miss(r, lit, b"ab =:")
        t += lit
        if i < len(lits) - 1 or ends:
            t += bytes(alpha[int(j)] for j in r.integers(0, len(alpha), int(r.integers(0, 9))))
    if r.random() < 0.15:
        t = t[:int(r.integers(0, len(t) + 1))]
    return t


NORMS = [(True, True, True), (True, False, False), (False, True, False), (False, False, True), (True, False, True)]
ALL_NORMS = [(bool(f & 1), bool(f & 2), bool(f & 4)) for f in range(8)]


def norm_fuzz_template(r, long=False):
    """A template over an alphabet with spaces, punctuation and capitals, whose literals keep at least one
    letter (so that normalisation never empties the text between two wildcards)."""
    alpha = b"aB =:c-"
    k = int(r.integers(1, 4))
    lits = []
    for _ in range(k + 1):
        raw = long_literal(r, alpha) if long else bytes(alpha[int(i)] for i in r.integers(0, len(alpha), int(r.integers(1, 4))))
        at = int(r.integers(0, len(raw) + 1))
        lits.append(raw[:at] + (b"a", b"B", b"c")[int(r.integers(0, 3))] + raw[at:])
        if long and len(lits[-1]) > 255:
            lits[-1] = lits[-1][:255]
    if r.random() < 0.3:
        lits[0] = b""
    ends = r.random() < 0.5
    if not ends and r.random() < 0.3:
        lits[-1] = b"'"                                          # punctuation only: vanishes under remove_punctuation
    return lits, ends


def norm_fuzz_text(r, lits, ends, near_miss_p=0.0):
    alpha = b"aB =:c-xY\t.A"
    t = b""
    for i, lit in enumerate(lits):
        if near_miss_p and i and lit and r.random() < near_miss_p:
            t += near_miss(r, lit, b"aB =:c-")
        t += lit if r.random() < 0.8 else lit.swapcase().replace(b" ", b"  ")
        if i < len(lits) - 1 or ends:
            t += bytes(alpha[int(j)] for j in r.integers(0, len(alpha), int(r.integers(0, 9))))
    if r.random() < 0.2:
        t = bytes(alpha[int(i)] for i in r.integers(0, len(alpha), int(r.integers(0, 24))))
    return t


# ------------------------------------------------------------------------------------------ whole configurations
# header formats: Content running to the end; Content in front of an end-anchored "]"; Content first, h behind " @"
HEADERS = [b"<h>|<Content>", b"<h> [<Content>]", b"<Content> @<h>"]


def header_line(fmt_i, h, content):
    return (h + b"|" + content, h + b" [" + content + b"]", content + b" @" + h)[fmt_i]


def _words(lits):
    return sum((len(l) + 3) // 4 for l in lits)


def template_set(r, k, norm):
    """k templates as (literals, ends, shadowed) -- shadowed: an earlier template of its family shares its prefix and
    fails late (one more literal, or a different final literal) -- plus possibly a template of 32 captures that ends
    with a literal.  Kept inside the device's 512 literals and 4096 bytes of literal text."""
    out, n_lits, words = [], 4, 4
    if r.random() < 0.5:
        big = [b""] + [b"k%02dq" % i for i in range(32)]         # distinct literals: the regex oracle stays linear
        out.append((big, False, False))
        n_lits, words = n_lits + 33, words + _words(big)
    while len(out) < k:
        lits, ends = norm_fuzz_template(r, long=True) if norm else fuzz_formats(r, 1, long=True)[0]
        fam = []
        if r.random() < 0.6 and lits[-1] != b"'":              # ("'" is a final literal R-norm may empty)
            extra = long_literal(r, b"ab =:")[:254] + b"c"
            fam.append((lits + [extra], ends))                   # one literal more: fails at its very end
        if r.random() < 0.6 and len(lits) > 1:
            last = lits[-1]
            alt = last[:-1] + (b"B" if last[-1:] != b"B" else b"c")
            fam.append((lits[:-1] + [alt], ends))                # diverges in the last literal
        fam.append((lits, ends))
        for j, (l, e) in enumerate(fam):
            if len(out) >= k:
                break
            if n_lits + len(l) > 512 or words + _words(l) > 1024:
                return out
            out.append((l, e, j > 0))
            n_lits, words = n_lits + len(l), words + _words(l)
    return out


def template_text(lits, ends):
    return b"<*>".join(lits) + (b"<*>" if ends else b"")


def n_captures(lits, ends, norm_flags):
    """Wildcards of the template as the device compiles it (a final literal R-norm empties turns into the end)."""
    from detectmateservice_b200.logformat import normalise
    if not ends and len(lits) > 1 and norm_flags and normalise(lits[-1], norm_flags) == b"":
        return len(lits) - 1
    return len(lits) - (0 if ends else 1)


def monitor_config(r, caps, content_monitor, n_train):
    """Global and event-scoped header monitors (EventID -1 included), per-event variable monitors at indices 0, 31,
    the last capture, one past the capture count and >= 32."""
    glob = {"g": {"header_variables": [{"pos": "h"}] + ([{"pos": "Content"}] if content_monitor else [])}}
    events = {-1: {"unmatched": {"header_variables": [{"pos": "h"}]}}}
    n = len(glob["g"]["header_variables"]) + 1
    order = [int(t) for t in r.permutation(len(caps))]
    if 32 in caps:
        order.insert(0, caps.index(32))
    for t in order:
        if t in events:
            continue
        pos = sorted({0, 31, max(caps[t] - 1, 0), caps[t], 32 + int(r.integers(0, 9))})
        if n + len(pos) + 1 > 32:
            break
        events[t] = {"v": {"variables": [{"pos": p} for p in pos]}, "hh": {"header_variables": [{"pos": "h"}]}}
        n += len(pos) + 1
        if len(events) >= 5:
            break
    return {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": n_train,
                                               "global": glob, "events": events}}}


def format_case(seed, norm, n_records=400, n_templates=None):
    """One configuration and one message: (log_format, templates, cfg, lines, n_train, shadowed templates)."""
    from detectmateservice_b200.logformat import norm_flags
    r = np.random.Generator(np.random.PCG64(seed))
    flags = norm_flags(*norm)
    k = n_templates or int(r.choice([2, 3, 5, 8, 16, 63]))
    ts = template_set(r, k, bool(flags))
    fmt_i = int(r.integers(0, len(HEADERS)))
    caps = [n_captures(l, e, flags) for l, e, _ in ts]
    n_train = int(r.integers(n_records // 5, n_records // 2)) | 1
    cfg = monitor_config(r, caps, r.random() < 0.3, n_train)
    hvals = [b"h%d" % i for i in range(4)]
    lines = []
    while len(lines) < n_records:
        h = hvals[int(r.integers(0, 4))] if r.random() < 0.97 else b"new%d" % int(r.integers(0, 99))
        u = r.random()
        if u < 0.03:
            lines.append(b"")                                    # empty record
        elif u < 0.06:
            lines.append(b"no header " + _bytes(r, b"ab =:", int(r.integers(0, 12))))
        elif u < 0.08:
            lines.append(header_line(fmt_i, h, b" -.:\t" + (b"" if r.random() < 0.5 else b"!?")))   # normalises to nothing
        elif u < 0.10:
            lines.append(header_line(fmt_i, h, b"\ra\x7fb\x80\xff" + _bytes(r, b"ab =:", int(r.integers(0, 5))) + b"\r"))
        elif u < 0.104:                                          # a run of 0-3 byte Contents
            for _ in range(int(r.integers(10, 60))):
                lines.append(header_line(fmt_i, h, _bytes(r, b"ab =:", int(r.integers(0, 4)))))
        else:
            t = int(r.integers(0, len(ts))) if r.random() < 0.7 else len(ts) - 1 - int(r.integers(0, min(3, len(ts))))
            lits, ends, _ = ts[t]
            c = norm_fuzz_text(r, lits, ends, 0.5) if flags else fuzz_text(r, lits, ends, 0.5)
            lines.append(header_line(fmt_i, h, c.replace(b"\n", b"")))
    lines = lines[:n_records]
    return {"log_format": HEADERS[fmt_i], "templates": [template_text(l, e) for l, e, _ in ts], "cfg": cfg,
            "lines": lines, "n_train": n_train, "shadowed": [s for _, _, s in ts], "norm": norm}
