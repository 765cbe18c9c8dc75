"""LogSchema input (DESIGN.md R-log), CPU tier: the host codec against protobuf's runtime, the device unwrap kernels
(walk, scan, compact, copy) on the CPU emulator against the protobuf-decode / filter / join oracle, and the
component's routing with a device stand-in."""
import random
import struct

import numpy as np
import pytest

from detectmateservice_b200 import wire
from lsgen import Gen, protobuf_text, unwrap
from oracle.schemas import LogSchema
from pbgen import BAD_UTF8, frame, ld, tag, varint

NAMES = ("__version__", "logID", "log", "logSource", "hostname")


def _texts(r, n):
    pool = [b"type=USER_ACCT msg=audit(1642723741.072:375): res=success", b"", b"k=v", "é=ü 😀".encode(),
            b"type=LOGIN res=1\r", b"trailing\n", b"x" * 300]
    return [r.choice(pool) + (b" n=%d" % r.randint(0, 5) if r.random() < 0.5 else b"") for _ in range(n)]


def _ours(rec):
    try:
        d = wire.decode_log_schema(rec)
    except wire.WireError:
        return None
    return d


# ------------------------------------------------------------------------------------------ host codec
def test_decode_log_schema_matches_protobuf_on_fuzzed_records():
    r = random.Random(7)
    g = Gen(seed=7, mutate=0.35)
    n_ok = n_bad = n_unusable = 0
    for rec in g.records(_texts(r, 3000)):
        m = LogSchema()
        try:
            m.ParseFromString(rec)
            pb_ok = True
        except Exception:
            pb_ok = False
        text, _ = protobuf_text(rec)
        d = _ours(rec)
        if not pb_ok or (d is None):
            # a group is the one record protobuf keeps and R-log refuses
            assert d is None and text is None, rec
            n_bad += 1
            continue
        assert {k: d[k] for k in NAMES} == {k: getattr(m, k) for k in NAMES}, rec
        try:
            line = wire.log_schema_line(d)
        except wire.WireError:
            line = None
            n_unusable += 1
        assert line == text
        n_ok += 1
    assert n_ok > 2000 and n_bad > 100 and n_unusable > 10


def test_decode_log_schema_edges():
    body = ld(2, b"id7") + ld(3, b"first") + ld(1, b"1.0.0") + ld(3, b"second\n")
    d = wire.decode_log_schema(body)
    assert d["log"] == "second\n" and d["logID"] == "id7" and wire.log_schema_line(d) == b"second"
    assert wire.decode_log_schema(b"") == {k: "" for k in NAMES}
    # overlong tag (5 bytes) and length (10 bytes) are accepted, a 6-byte tag is not
    assert wire.decode_log_schema(tag(3, 2, 5) + varint(2, 10) + b"ok")["log"] == "ok"
    with pytest.raises(wire.WireError):
        wire.decode_log_schema(tag(3, 2, 6) + varint(2) + b"ok")
    # unknown and mistyped fields are skipped unless strict; groups are refused
    for extra in (tag(3, 0) + varint(9), ld(9, b"\xff"), tag(6, 5) + b"abcd", tag(4, 1) + b"\0" * 8):
        assert wire.decode_log_schema(ld(3, b"t") + extra)["log"] == "t"
        with pytest.raises(wire.WireError):
            wire.decode_log_schema(ld(3, b"t") + extra, strict=True)
    with pytest.raises(wire.WireError):
        wire.decode_log_schema(ld(3, b"t") + tag(9, 3) + tag(9, 4))
    # bad UTF-8 in each string field
    for f in range(1, 6):
        for _name, bad in BAD_UTF8:
            rec = ld(f, b"a" + bad)
            with pytest.raises(wire.WireError):
                wire.decode_log_schema(rec)
            assert protobuf_text(rec) == (None, None)
    # newlines: one trailing '\n' is dropped, "\r\n" keeps its '\r', an inner '\n' is unusable
    assert wire.log_schema_line({"log": "a\r\n"}) == b"a\r"
    assert wire.log_schema_line({"log": "\n"}) == b""
    for t in ("a\nb", "a\n\n", "\n\n"):
        with pytest.raises(wire.WireError):
            wire.log_schema_line({"log": t})


def test_encode_log_schema_roundtrip_through_protobuf():
    rec = {"__version__": "1.0.0", "logID": "42", "log": "type=X é", "logSource": "/var/log/x", "hostname": "h"}
    m = LogSchema()
    m.ParseFromString(wire.encode_log_schema(rec))
    assert {k: getattr(m, k) for k in NAMES} == rec
    assert wire.decode_log_schema(m.SerializeToString()) == rec


# ------------------------------------------------------------------------------------------ emulator
def _emu_lib():
    import emu_harness
    return emu_harness.lib()


def _emu_unwrap(lib, msg, delimited, n_train, walk_ctas=2, copy_ctas=2):
    n_max = max(1, len(msg))
    cap = ((len(msg) + 1 + 64 + 15) // 16) * 16
    out = np.zeros(cap, np.uint8)
    rec_line = np.zeros(n_max + 1, np.uint32)
    line_rec = np.zeros(n_max + 1, np.uint32)
    line_dst = np.zeros(n_max + 2, np.uint32)
    hdr = np.zeros(4, np.uint64)
    n = lib.emu_logs_unwrap(msg, len(msg), int(delimited), n_train, walk_ctas, copy_ctas, out.ctypes.data, cap,
                            rec_line.ctypes.data, line_rec.ctypes.data, line_dst.ctypes.data, hdr.ctypes.data)
    assert n >= 0
    return n, out, rec_line[:n], line_rec, line_dst, [int(x) for x in hdr]


def _check_unwrap(lib, records, delimited, n_train, **kw):
    msg = frame(records) if delimited else records[0]
    n, out, rec_line, line_rec, line_dst, (total, n_lines, ntr, bound) = _emu_unwrap(lib, msg, delimited, n_train, **kw)
    want, idx, _ids = unwrap(records)
    assert n == len(records)
    assert (total, n_lines) == (len(want), len(idx))
    assert bytes(out[:total]) == want                                   # byte for byte
    assert n == 0 or not out[total:total + 64].any()                    # the zeroed slack (no launch for no records)
    assert line_rec[:n_lines].tolist() == idx
    assert line_dst[n_lines] == total
    want_line = np.full(n, 0xFFFFFFFF, np.uint32)
    want_line[idx] = np.arange(len(idx), dtype=np.uint32)
    assert rec_line.tolist() == want_line.tolist()
    assert ntr == min(n_train, n_lines)
    if n_train == 0:
        assert bound == 0
    elif n_train > n_lines:
        assert bound == n
    else:
        assert bound == idx[n_train - 1] + 1
    return n_lines


def test_emu_unwrap_kernels_fuzzed_batches():
    lib = _emu_lib()
    r = random.Random(11)
    g = Gen(seed=11, mutate=0.2)
    recs = g.records(_texts(r, 1100))                                   # 5 tiles over 2 walk CTAs
    usable = _check_unwrap(lib, recs, True, 0)
    assert 800 < usable < 1100
    for n_train in (1, 5, 600, usable, usable + 1, 5000):
        _check_unwrap(lib, recs, True, n_train)
    _check_unwrap(lib, recs[:300], True, 17, walk_ctas=1, copy_ctas=3)


def test_emu_unwrap_kernels_edges():
    lib = _emu_lib()
    g = Gen(seed=12, mutate=0.0, fuzz=0.0)
    # an empty batch, a batch of malformed records only, a bare record, a bare empty record
    assert _check_unwrap(lib, [], True, 3) == 0
    bad = [b"\x02\x01z", ld(3, b"\xff"), ld(3, b"a\nb"), tag(5, 3) + tag(5, 4)]
    assert _check_unwrap(lib, bad, True, 2) == 0
    rec = g.record(b"type=A res=1", "7")[0]
    assert _check_unwrap(lib, [rec], False, 1) == 1
    assert _check_unwrap(lib, [b""], False, 0) == 1                     # compacts to a single '\n'
    assert _check_unwrap(lib, [bad[0]], False, 0) == 0
    # empty texts next to each other, long texts crossing many 16-byte stores, odd lengths
    texts = [b"", b"", b"a", b"L" * 1000, b"", b"b" * 17, b"c" * 15, b"d" * 16, b"e" * 33]
    _check_unwrap(lib, [g.record(t, str(i))[0] for i, t in enumerate(texts)], True, 4)
    # one long record among short ones
    _check_unwrap(lib, [g.record(t, str(i))[0] for i, t in enumerate([b"x=1", b"y" * 70000, b"z=2"])], True, 1)


# ------------------------------------------------------------------------------------------ component routing
class StandIn:
    """Device stand-in: a usable record whose text holds b"EVIL" (or b"/foobar") is anomalous in monitor 0 once
    training is over (mask bit 0, or the first combination's bit); malformed records are judged by protobuf's runtime."""

    def __init__(self, mask=1):
        self.mask = mask
        self.calls = []
        self.last_n_anomalies = 0
        self._anoms = []

    def process_logs(self, buf, n_train_records=0, delimited=True):
        self.calls.append(("process_logs", n_train_records, delimited))
        frames = wire.split_delimited(buf) if delimited else [bytes(buf)]
        flags = np.zeros(len(frames), np.uint8)
        scores = np.zeros(len(frames), np.float32)
        self._anoms, n_bad, seen = [], 0, 0
        for i, fr in enumerate(frames):
            text, _ = protobuf_text(fr)
            if text is None:
                n_bad += 1
                continue
            seen += 1
            if seen > n_train_records and (b"EVIL" in text or b"/foobar" in text):
                flags[i], scores[i] = 1, 1.0
                self._anoms.append((i, self.mask, 0))
        self.last_n_anomalies = len(self._anoms)
        return flags, scores, n_bad

    def anomalies(self):
        return list(self._anoms)

    def process_values(self, *a, **k):
        self.calls.append(("process_values",))
        return np.zeros(1, np.uint8), np.zeros(1, np.float32), np.zeros(1, np.uint32)

    def process_records(self, buf, n_train_records=0):
        self.calls.append(("process_records",))
        n = len(wire.split_delimited(buf))
        return np.zeros(n, np.uint8), np.zeros(n, np.float32), np.zeros(n, np.uint32)

    def process_lines(self, buf, n_train_lines=0, copy=True):
        self.calls.append(("process_lines",))
        n = bytes(buf).count(b"\n") + (0 if bytes(buf).endswith(b"\n") else 1)
        self.last_n_anomalies = 0
        return np.zeros(n, np.uint8), np.zeros(n, np.float32)


NGINX = '<IP> - - [<Time>] "<Method> <URL> <Protocol>" <Status> <Bytes> "<Referer>" "<UserAgent>"'


def _comp(params, cls="B200NewValueDetector", training=2, combo=False):
    from detectmateservice_b200 import component
    inst = {"header_variables": [{"pos": "URL"}]} if "log_format" in params else {"header_variables": [{"pos": "type"}]}
    if combo:
        inst = {"header_variables": [{"pos": "type"}, {"pos": "res"}]} if "log_format" not in params else \
            {"header_variables": [{"pos": "URL"}, {"pos": "Method"}]}
    cfg = {"detectors": {"D": {"method_type": "new_value_detector", "data_use_training": training, "auto_config": False,
                               "params": params, "global": {"g": inst}}}}
    c = getattr(component, cls)(name="D", config=cfg)
    c.clock = lambda: 1773848383
    c._det = StandIn(mask=1 << len(c.monitors) if combo else 1)
    return c


def _ls(text, log_id, source=True):
    rec = {"__version__": "1.0.0", "logID": log_id, "log": text}
    if source:
        rec["logSource"] = "/var/log/x.log"
    return wire.encode_log_schema(rec)


def nginx_line(url):
    return '172.18.0.1 - - [18/Mar/2026:15:39:43 +0000] "GET %s HTTP/1.1" 404 162 "-" "curl/8.5.0"' % url


@pytest.mark.parametrize("with_format", [False, True])
@pytest.mark.parametrize("cls", ["B200NewValueDetector", "B200NewValueComboDetector"])
def test_component_bare_log_schema(with_format, cls):
    params = {"input_format": "log_schema"}
    if with_format:
        params["log_format"] = NGINX
    combo = cls.endswith("ComboDetector")
    c = _comp(params, cls, combo=combo)
    good = (lambda u: nginx_line(u)) if with_format else (lambda u: "type=%s res=ok" % u)
    assert c.process(_ls(good("/hello" if with_format else "A"), "r1")) is None
    assert c.process(_ls(good("/world" if with_format else "B") + "\n", "r2")) is None
    with pytest.raises(wire.WireError):
        c.process(b"\x02\x01z")                                          # malformed: raises, no training slot
    with pytest.raises(wire.WireError):
        c.process(_ls("two\nlines", "r3"))                               # unusable: the same
    assert c.n_seen == 2
    out = c.process(_ls(good("/foobar" if with_format else "EVIL"), "the-third"))
    a = wire.decode_detector_schema(out)                                # one bare DetectorSchema
    assert a["logIDs"] == ["the-third"] and a["alertID"] == "10"
    if combo:
        key = "Global - (URL, Method)" if with_format else "Global - (type, res)"
        val = "Unknown value combination: ('/foobar', 'GET')" if with_format else "Unknown value combination: ('EVIL', 'ok')"
        assert a["alertsObtain"] == {key: val}
    elif with_format:
        assert a["alertsObtain"] == {"Global - URL": "Unknown value: '/foobar'"}
        assert a["extractedTimestamps"] == [1773848383]
    else:
        assert a["alertsObtain"] == {"Global - type": "Unknown value: 'EVIL'"}
    assert [x[0] for x in c._det.calls] == ["process_logs"] * 5
    assert [x[2] for x in c._det.calls] == [False] * 5


@pytest.mark.parametrize("with_format", [False, True])
def test_component_log_schema_batch_and_training_slots(with_format):
    params = {"input_format": "log_schema_batch"}
    if with_format:
        params["log_format"] = NGINX
    c = _comp(params, training=3)
    t = (lambda u: nginx_line(u)) if with_format else (lambda u: "type=%s" % u)
    evil = "/foobar" if with_format else "EVIL"
    recs = [_ls(t("a"), "0"), b"\x02\x01z", _ls(t(evil), "2"), _ls("x\ny", "3"), _ls(t("b"), "4"), _ls(t(evil), "5"),
            _ls(t(evil), "6", source=False)]
    out = c.process(frame(recs))
    # training takes 3 usable records (0, 2, 4); 5 and 6 alert
    assert c._det.calls[-1] == ("process_logs", 3, True)
    assert c.n_seen == 5 and c.last_n_malformed == 2
    alerts = [wire.decode_detector_schema(b) for b in wire.split_delimited(out)]
    assert [a["logIDs"] for a in alerts] == [["5"], ["6"]]
    assert [a["alertID"] for a in alerts] == ["10", "11"]
    # training over: nothing left to train; an empty batch and a batch of malformed records only
    assert c.process(frame([b"\x02\x01z"])) is None and c.n_seen == 5
    assert c._det.calls[-1] == ("process_logs", 0, True)
    # compact output: every record, malformed ones with flag 0
    c.output_format = "compact"
    blob = c.process(frame([_ls(t(evil), "7"), b"\xff", _ls(t("c"), "8")]))
    (n,) = struct.unpack_from("<I", blob)
    from detectmateservice_b200.component import decode_compact
    f, s = decode_compact(blob)
    assert n == 3 and f.tolist() == [1, 0, 0] and s.tolist() == [1.0, 0.0, 0.0]


def test_component_log_schema_refuses_oversized_batch():
    c = _comp({"input_format": "log_schema_batch", "max_batch_bytes": 64})
    with pytest.raises(ValueError):
        c.process(frame([_ls("type=A " + "x" * 80, "1")]))
    assert c._det.calls == []


def test_component_auto_unchanged_on_log_schema():
    """`auto` never picks the LogSchema path: a LogSchema without logSource reads as a ParserSchema, one with it as
    raw text, exactly as before this input format existed."""
    for params in ({}, {"log_format": NGINX}):
        c = _comp(params)
        c.process(_ls("type=A", "1", source=False))
        c.process(_ls("type=A", "1", source=True))
        assert "process_logs" not in [x[0] for x in c._det.calls]
    c = _comp({})
    c.process(_ls("type=A", "1", source=False))
    c.process(_ls("type=A", "1", source=True))
    assert [x[0] for x in c._det.calls] == ["process_values", "process_lines"]
    with pytest.raises(ValueError):
        _comp({"input_format": "logschema"})
