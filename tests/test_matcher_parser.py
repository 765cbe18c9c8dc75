"""The MatcherParser stage (B200MatcherParser, rule R-parse in DESIGN.md), CPU tier.

- The host path, which is the specification, against an independent oracle: every ParserSchema decoded with
  protobuf's runtime and compared field by field with what oracle.rfmt (Python's `re`) and protobuf's LogSchema give.
- The configuration: the reference's parser_config.yaml loads, and every refusal raises.
- The kernels of dm_kernels_parse.cuh on the CPU emulator (tests/emu) behind a stand-in for DeviceDetector: the component's device path must return the host path's bytes.
"""
import ctypes as C
import os
import random

import numpy as np
import pytest
import yaml

from detectmateservice_b200 import wire
from detectmateservice_b200.detector import parser_format_strings
from detectmateservice_b200.parser import B200MatcherParser
from lsgen import Gen as LogGen, protobuf_text
from oracle.rfmt import FormatParser
from oracle.schemas import ParserSchema

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
NGINX = '<IP> - - [<Time>] "<Method> <URL> <Protocol>" <Status> <Bytes> "<Referer>" "<UserAgent>"'
AUDIT = "type=<Type> msg=audit(<Time>): <Content>"
NOW = 1773848383


def nginx_line(url, ip="172.18.0.1"):
    return ('%s - - [18/Mar/2026:15:39:43 +0000] "GET %s HTTP/1.1" 404 162 "-" "curl/8.5.0"' % (ip, url)).encode()


def parser(log_format, templates=(), norm=(False, False, False), **params):
    """A B200MatcherParser configured as the reference's parser_config.yaml configures MatcherParser."""
    p = dict(params)
    p.update({"remove_spaces": norm[0], "remove_punctuation": norm[1], "lowercase": norm[2]})
    if templates:
        p["templates"] = [t if isinstance(t, str) else t.decode("utf-8", "surrogateescape") for t in templates]
    cfg = {"parsers": {"MatcherParser": {"method_type": "matcher_parser", "auto_config": False,
                                         "log_format": log_format, "time_format": None, "params": p}}}
    comp = B200MatcherParser(config=cfg)
    comp.clock = lambda: NOW
    return comp


def log_records(texts, seed, mutate=0.1):
    """LogSchema records of the texts (lsgen: shuffled, repeated and unknown fields; some malformed or unusable)."""
    return LogGen(seed, mutate=mutate).records(texts)


# ------------------------------------------------------------------------------------------ the oracle
def oracle_fields(comp, records, first_id):
    """What each record must become, by protobuf's LogSchema and the regex matcher: a list of dicts (None for a record
    that gives no output)."""
    lf = comp.logformat
    fp = FormatParser(lf.source, lf.template_sources, lf.content_name, bool(lf.flags & 1), bool(lf.flags & 2),
                      bool(lf.flags & 4))
    out, j = [], first_id
    for rec in records:
        text, log_id = protobuf_text(rec)
        if text is None:
            out.append(None)
            continue
        p = fp.parse_line(text)
        d = {"__version__": "1.0.0", "parserType": comp.method_type, "parserID": comp.parser_id, "EventID": -1,
             "template": "", "variables": [], "logFormatVariables": {}, "parsedLogID": str(j), "logID": log_id,
             "log": text.decode("utf-8"), "receivedTimestamp": NOW, "parsedTimestamp": NOW}
        if p is not None:
            d["EventID"] = p["EventID"]
            if p["EventID"] >= 0:
                d["template"] = lf.template_sources[p["EventID"]].decode("utf-8")
            d["variables"] = [v.decode("utf-8") for v in p["variables"]]
            d["logFormatVariables"] = {k: v.decode("utf-8") for k, v in p["logFormatVariables"].items()}
        out.append(d)
        j += 1
    return out


def decoded(blob):
    """Each ParserSchema of a varint-delimited reply as protobuf's runtime reads it, as a dict."""
    out = []
    for m in wire.split_delimited(blob or b""):
        x = ParserSchema()
        x.ParseFromString(m)
        out.append({"__version__": x.__version__, "parserType": x.parserType, "parserID": x.parserID,
                    "EventID": x.EventID, "template": x.template, "variables": list(x.variables),
                    "logFormatVariables": dict(x.logFormatVariables), "parsedLogID": x.parsedLogID, "logID": x.logID,
                    "log": x.log, "receivedTimestamp": x.receivedTimestamp, "parsedTimestamp": x.parsedTimestamp})
    return out


def check_against_oracle(comp, records, first_id=0):
    reply = comp._parse_host(wire.frame_delimited(records), delimited=True)
    want = [d for d in oracle_fields(comp, records, first_id) if d is not None]
    assert decoded(reply) == want
    return reply


# ------------------------------------------------------------------------------------------ generated cases
def fmt_case(seed, norm, n_records=400, n_templates=None, mutate=0.1):
    """(component, LogSchema records) from fmtgen's configurations, plus empty captures and non-ASCII text."""
    import fmtgen
    c = fmtgen.format_case(seed, norm, n_records=n_records, n_templates=n_templates)
    comp = parser(c["log_format"].decode(), c["templates"], norm)
    lines = list(c["lines"])
    fmt_i = fmtgen.HEADERS.index(c["log_format"])
    r = random.Random(seed)
    for _ in range(n_records // 20):                             # non-ASCII Content, empty header captures
        lines.insert(r.randrange(len(lines) + 1), fmtgen.header_line(fmt_i, r.choice([b"", "hôte".encode()]),
                                                                      "naïve café – 日本 %d".encode() % r.randrange(9)))
    return comp, log_records(lines, seed, mutate)


def audit_case(seed, norm=(True, True, True), n_records=400):
    lines = open(os.path.join(GOLDEN, "audit_sample.log"), "rb").read().split(b"\n")
    lines = [ln for ln in lines if ln][:n_records]
    comp = parser(AUDIT, norm=norm, path_templates=os.path.join(GOLDEN, "audit_templates.txt"))
    return comp, log_records(lines, seed)


def nginx_case(seed, n_records=400):
    r = random.Random(seed)
    lines = [nginx_line("/p%d" % r.randrange(50), "10.0.%d.%d" % (r.randrange(4), r.randrange(256))) for _ in range(n_records)]
    lines += [b"not an access-log line", b"", nginx_line("/caf\xc3\xa9"), nginx_line("")]
    return parser(NGINX), log_records(lines, seed)


def wide_case(seed, n_records=300):
    """A log_format of 32 captures (Content the last), with as many of fmtgen's templates as the literal budget leaves."""
    import fmtgen
    c = fmtgen.format_case(seed, (False, False, False), n_records=n_records, n_templates=63)
    fmt = "|".join("<c%02d>" % i for i in range(31)) + "|<Content>"
    ts = list(c["templates"])
    while True:
        try:
            comp = parser(fmt, ts)
            break
        except ValueError:
            ts.pop()
    r = random.Random(seed)
    lines = []
    for ln in c["lines"]:
        content = ln.split(b"|", 1)[-1] if b"|" in ln else ln
        lines.append(b"|".join(b"v%d" % r.randrange(3) if r.random() < 0.9 else b"" for _ in range(31)) + b"|" + content)
    return comp, log_records(lines, seed)


CASES = [("fmt", s, n) for s, n in ((1, (False, False, False)), (2, (True, False, False)), (3, (False, True, False)),
                                    (4, (False, False, True)), (5, (True, True, True)))]
CASES += [("fmt63", 10, (True, True, True)), ("fmt63", 11, (False, False, False))]
CASES += [("audit", 6, (True, True, True)), ("audit", 7, (False, False, False)), ("nginx", 8, None), ("wide", 9, None)]


def make_case(kind, seed, norm, n_records=400):
    if kind == "fmt":
        return fmt_case(seed, norm, n_records)
    if kind == "fmt63":
        return fmt_case(seed, norm, n_records, n_templates=63)
    if kind == "audit":
        return audit_case(seed, norm, n_records)
    if kind == "nginx":
        return nginx_case(seed, n_records)
    return wide_case(seed, n_records)


# ------------------------------------------------------------------------------------------ host path
def test_docs_nginx_lines_pinned():
    """The docs' three requests: three ParserSchemas whose logFormatVariables["URL"] are the paths."""
    comp = parser(NGINX)
    recs = [wire.encode_log_schema({"__version__": "1.0.0", "logID": "id-%d" % i, "log": nginx_line(u).decode() + "\n"})
            for i, u in enumerate(("/hello", "/world", "/foobar"))]
    got = decoded(check_against_oracle(comp, recs))
    assert [d["logFormatVariables"]["URL"] for d in got] == ["/hello", "/world", "/foobar"]
    assert [d["parsedLogID"] for d in got] == ["0", "1", "2"]
    assert [d["logID"] for d in got] == ["id-0", "id-1", "id-2"]
    assert all(d["EventID"] == -1 and d["parserID"] == "MatcherParser" and d["parserType"] == "matcher_parser" for d in got)


@pytest.mark.parametrize("kind,seed,norm", CASES)
def test_host_path_against_oracle(kind, seed, norm):
    comp, recs = make_case(kind, seed, norm)
    check_against_oracle(comp, recs, first_id=0)


def test_host_path_bare_record_and_numbering():
    comp = parser(NGINX, start_id=-2)
    one = wire.encode_log_schema({"logID": "a", "log": nginx_line("/x").decode()})
    got = decoded(wire.frame_delimited([comp._parse_host(one, delimited=False)]))
    assert got[0]["parsedLogID"] == "-2" and got[0]["logFormatVariables"]["URL"] == "/x"
    with pytest.raises(wire.WireError):
        comp._parse_host(one[:-3], delimited=False)                  # malformed: raises, takes no parsedLogID
    assert decoded(comp._parse_host(wire.frame_delimited([one]), delimited=True))[0]["parsedLogID"] == "-1"
    assert comp._parse_host(b"", delimited=True) is None


# ------------------------------------------------------------------------------------------ configuration
def _reference_config(tmp_path):
    """The reference's container/config/parser_config.yaml verbatim, with its template file path pointed at an empty
    file here (the reference ships that file empty)."""
    cfg = yaml.safe_load(open(os.path.join(GOLDEN, "parser_config.yaml")))
    empty = tmp_path / "templates.txt"
    empty.write_bytes(b"")
    cfg["parsers"]["MatcherParser"]["params"]["path_templates"] = str(empty)
    return cfg


def test_reference_parser_config_loads(tmp_path):
    comp = B200MatcherParser(config=_reference_config(tmp_path))
    assert comp.logformat.source == NGINX and comp.logformat.templates == []
    assert comp.method_type == "matcher_parser" and comp.parser_id == "MatcherParser" and comp.input_format == "log_schema_batch"
    named = B200MatcherParser(name="accesslogparser", config=_reference_config(tmp_path))
    assert named.parser_id == "accesslogparser"


@pytest.mark.parametrize("change,match", [
    ({"auto_config": True}, "auto_config"),
    ({"time_format": "%d/%b/%Y:%H:%M:%S %z"}, "time_format"),
    ({"log_format": None}, "log_format"),
    ({"params": {"path_templates": "BAD"}}, "UTF-8"),
    ({"params": {"input_format": "raw_lines"}}, "input_format"),
])
def test_config_refusals(tmp_path, change, match):
    cfg = _reference_config(tmp_path)
    entry = cfg["parsers"]["MatcherParser"]
    for k, v in change.items():
        if k == "params":
            for pk, pv in v.items():
                if pv == "BAD":
                    bad = tmp_path / "bad.txt"
                    bad.write_bytes(b"ok <*>\nnot \xff UTF-8 <*>\n")
                    pv = str(bad)
                entry["params"][pk] = pv
        else:
            entry[k] = v
    with pytest.raises(ValueError, match=match):
        B200MatcherParser(config=cfg)


# ------------------------------------------------------------------------------------------ the kernels on the emulator
@pytest.fixture(scope="module")
def emu():
    import emu_harness
    return emu_harness.lib()


class EmuParseDevice:
    """Stands in for DeviceDetector.parse_logs: the dm_parse_logs sequence on the CPU emulator (tests only), on a handle
    set up as the component sets up its own (no monitors, its log_format, its parser format)."""

    def __init__(self, L, comp):
        import emu_harness
        lf = comp.logformat
        self.L = L
        self.det = emu_harness.EmuDetector([], table_log2=10)
        self.h = self.det.h
        self.det.set_monitors(None, 0)
        ts = list(lf.template_sources)
        self.det.set_format(lf.source, ts, lf.flags, lf.content_name.encode())
        strs, order = parser_format_strings("1.0.0", comp.method_type, comp.parser_id, ts, lf.header.names)
        why = L.emu_set_parser_format(self.h, len(strs), b"".join(strs), (C.c_uint32 * len(strs))(*[len(s) for s in strs]),
                                      (C.c_uint32 * max(1, len(order)))(*order))
        assert why is None, why

    def close(self):
        self.det.close()

    def parse_logs(self, buf, delimited, first_parsed_id, now):
        buf = bytes(buf)
        cap = 4 * len(buf) + 4096
        while True:
            out = np.zeros(cap, np.uint8)
            out_len, n_rec, n_emit = C.c_uint64(), C.c_uint64(), C.c_uint64()
            rc = self.L.emu_parse_logs(self.h, buf, len(buf), int(delimited), first_parsed_id, now, out.ctypes.data, cap,
                                       C.byref(out_len), C.byref(n_rec), C.byref(n_emit))
            if rc != -4:
                break
            cap = out_len.value
        if rc == -1:
            raise wire.WireError("framing")
        assert rc == 0, rc
        return out[:out_len.value].tobytes(), n_rec.value, n_emit.value, n_rec.value - n_emit.value


def device_and_host(emu, comp_dev, comp_host, msg, delimited):
    """(device reply, host reply) of one message; the device path is the component's own, on the emulator."""
    return comp_dev._parse_device(msg, delimited), comp_host._parse_host(msg, delimited)


@pytest.mark.parametrize("kind,seed,norm", CASES)
def test_emulated_kernels_match_host_path(emu, kind, seed, norm):
    comp_host, recs = make_case(kind, seed, norm)
    comp_dev, _ = make_case(kind, seed, norm)
    comp_dev._det = EmuParseDevice(emu, comp_dev)
    try:
        # two messages, so that parsedLogID carries over from one to the next
        half = len(recs) // 3
        for part in (recs[:half], recs[half:]):
            dev, host = device_and_host(emu, comp_dev, comp_host, wire.frame_delimited(part), True)
            assert dev == host
            assert comp_dev.n_parsed == comp_host.n_parsed and comp_dev.last_n_malformed == comp_host.last_n_malformed
    finally:
        comp_dev._det.close()


def test_emulated_kernels_edges(emu):
    """An empty batch, bare records (usable, unusable, malformed, empty), a batch of only malformed records, and a
    negative start_id."""
    comp_host, comp_dev = parser(NGINX, start_id=-3), parser(NGINX, start_id=-3)
    comp_dev._det = EmuParseDevice(emu, comp_dev)
    try:
        assert comp_dev._parse_device(b"", True) is None and comp_host._parse_host(b"", True) is None
        good = wire.encode_log_schema({"logID": "é", "log": nginx_line("/a").decode() + "\n"})
        for bare in (good, b"", wire.encode_log_schema({"log": "no match"})):
            assert comp_dev._parse_device(bare, False) == comp_host._parse_host(bare, False)
        for bad in (good[:-2], wire.encode_log_schema({"log": "two\nlines"})):
            with pytest.raises(wire.WireError):
                comp_dev._parse_device(bad, False)
            with pytest.raises(wire.WireError):
                comp_host._parse_host(bad, False)
            assert comp_dev._parse_device(wire.frame_delimited([bad, bad]), True) is None
            assert comp_host._parse_host(wire.frame_delimited([bad, bad]), True) is None
        assert comp_dev.n_parsed == comp_host.n_parsed == 3
    finally:
        comp_dev._det.close()
