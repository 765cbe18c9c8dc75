"""DetectorSchema alerts of LogSchema and ParserSchema batches encoded on the device (DESIGN.md R-alert, R-log and the
record contract), CPU tier: the whole dm_process_logs sequence (unwrap, line path, scatter) or dm_process_records, then
the encoder kernels of dm_kernels_alerts.cuh, run on the CPU emulator behind a stand-in for DeviceDetector.  Every
reply must come out byte for byte as the component's host encoder writes it for the same emulated detection."""
import ctypes as C
import os
import random

import numpy as np
import pytest

from detectmateservice_b200 import wire
from detectmateservice_b200.synth import MONITORED_KEYS, AuditSynth
from lsgen import Gen as LogGen
from pbgen import Gen as RecGen, frame, ld, tag, varint
from test_emu_alerts import AUDIT, NOW, EmuDevice

VARIANTS = {"stream": 0, "chain": 1, "lanes": 2, "format": 3}


@pytest.fixture(scope="module")
def lib():
    import emu_harness
    return emu_harness.lib()


class EmuBatchDevice(EmuDevice):
    """Stands in for DeviceDetector on LogSchema and ParserSchema batches: detection and the alert encoder on the CPU
    emulator (tests only).  The handle has the component's monitors, combinations and log_format, as the real one."""

    def __init__(self, lib, comp, variant, capacity, anomaly_cap=None):
        import emu_harness
        from test_format_combos import _monitor_array
        self.lib, self.capacity = lib, capacity
        self.variant = "format" if comp.logformat is not None else variant
        self.det = emu_harness.EmuDetector([bytes(m.key) for m in comp.monitors], table_log2=14, variant=self.variant)
        self.h = self.det.h
        self.det.set_monitors(_monitor_array(comp.monitors), len(comp.monitors))
        if comp.logformat is not None:
            lf = comp.logformat
            self.det.set_format(lf.source, lf.template_sources, lf.flags, lf.content_name.encode())
        combos = getattr(comp, "combos", None) or ()
        self.det.set_combos(combos, (1 << len(comp.monitors)) - 1 if combos else 0)
        if anomaly_cap is not None:
            lib.emu_set_anomaly_cap(self.h, anomaly_cap)
        self.last_n_anomalies = 0
        self.encoded = self.declined = 0

    def process_logs(self, buf, n_train_records=0, delimited=True):
        buf = bytes(buf)
        cap = len(buf) + 2
        flags, scores = np.zeros(cap, np.uint8), np.zeros(cap, np.float32)
        n, bad, an = C.c_uint64(), C.c_uint64(), C.c_uint64()
        rc = self.lib.emu_process_logs(self.h, VARIANTS[self.variant], buf, len(buf), int(delimited), n_train_records,
                                       flags.ctypes.data, scores.ctypes.data, cap, C.byref(n), C.byref(bad), C.byref(an))
        if rc == -1:
            raise wire.WireError("framing")
        assert rc == 0, rc
        self.last_n_anomalies = an.value
        return flags[:n.value], scores[:n.value], bad.value

    def process_records(self, buf, n_train_records=0):
        buf = bytes(buf)
        cap = len(buf) + 2
        flags, scores, masks = np.zeros(cap, np.uint8), np.zeros(cap, np.float32), np.zeros(cap, np.uint32)
        rc, n, an = self.det.process_records(buf, n_train_records, flags, scores, masks, cap)
        assert rc == 0, rc
        self.last_n_anomalies = an
        return flags[:n], scores[:n], masks[:n]

    def stats(self):
        return self.det.stats()


class HostOnly:
    """The same emulated detection without the encoder: the component words the alerts on the host."""

    def __init__(self, dev):
        self.dev = dev

    def process_logs(self, buf, n_train_records=0, delimited=True):
        r = self.dev.process_logs(buf, n_train_records, delimited)
        self.last_n_anomalies = self.dev.last_n_anomalies
        return r

    def process_records(self, buf, n_train_records=0):
        r = self.dev.process_records(buf, n_train_records)
        self.last_n_anomalies = self.dev.last_n_anomalies
        return r

    def anomalies(self):
        return self.dev.anomalies()

    def stats(self):
        return self.dev.stats()


def _pair(lib, cfg, combo=False, variant="stream", capacity=1 << 20, anomaly_cap=None):
    """Two components of one config: device-encoded alerts, and the host encoder on the same emulated detection."""
    from detectmateservice_b200.component import B200NewValueComboDetector, B200NewValueDetector
    comps = []
    for host in (False, True):
        c = (B200NewValueComboDetector if combo else B200NewValueDetector)(config=cfg)
        dev = EmuBatchDevice(lib, c, "lanes" if combo else variant, capacity, anomaly_cap)
        c._det = HostOnly(dev) if host else dev
        c.DEVICE_ALERTS_MIN = 1                                      # every batch with alerts goes to the encoder
        c.clock = lambda: NOW
        comps.append(c)
    return comps


def _run(dev_c, host_c, messages):
    for msg in messages:
        got = dev_c.process(msg)
        want = host_c.process(msg)
        assert got == want
        assert dev_c.n_alerts == host_c.n_alerts and dev_c.n_seen == host_c.n_seen
    return dev_c._det


def _cfg(n_train, fmt="log_schema_batch", cls="B200NewValueDetector", **params):
    return {"detectors": {cls: {"method_type": "new_value_detector", "data_use_training": n_train, "auto_config": False,
                                "params": dict(params, input_format=fmt)}}}


# ------------------------------------------------------------------------------------------------ LogSchema
def _ls_records(lines, seed, first_id=0):
    """LogSchema records of the texts: lsgen's encodings and mutations (malformed and unusable records mixed in), and
    every seventh one with an absent, repeated or non-ASCII logID."""
    g = LogGen(seed, mutate=0.08)
    recs = g.records(lines, first_id)
    for i in range(0, len(recs), 7):
        t = lines[i]
        recs[i] = [ld(3, t), ld(2, b"first") + ld(3, t) + ld(2, b"last"), ld(2, ("ïd-☃-%d" % i).encode()) + ld(3, t),
                   tag(2, 0) + varint(5) + ld(3, t)][(i // 7) % 4]
    return recs


def _audit_lines(g, n, inject):
    return g.batch(n, inject=inject)[0].rstrip(b"\n").split(b"\n")


@pytest.mark.parametrize("variant", ["stream", "lanes"])
def test_log_schema_key_value(lib, variant):
    g = AuditSynth(seed=21, anomaly_rate=1e-1)
    cfg = _cfg(400)
    cfg["detectors"]["B200NewValueDetector"]["global"] = {"g": {"header_variables": [{"pos": k} for k in MONITORED_KEYS]}}
    dev_c, host_c = _pair(lib, cfg, variant=variant)
    train = frame(_ls_records(_audit_lines(g, 400, False), 1))
    msgs = [frame(_ls_records(_audit_lines(g, 700, True), s, 1000 * s)) for s in (2, 3)]
    dev = _run(dev_c, host_c, [train] + msgs)
    assert dev.encoded == 2 and dev.declined == 0 and dev_c.n_alerts > 60


@pytest.mark.parametrize("combo", [False, True])
def test_log_schema_bare_record(lib, combo):
    cfg = {"detectors": {"D": {"method_type": "new_value_detector", "data_use_training": 2, "auto_config": False,
                               "params": {"input_format": "log_schema"},
                               "global": {"g": {"header_variables": [{"pos": "type"}, {"pos": "res"}]}}}}}
    dev_c, host_c = _pair(lib, cfg, combo=combo)
    recs = [ld(2, b"r1") + ld(3, b"type=A res=ok msg=audit(12.5:1)"), ld(3, b"type=B res=ok\n"),
            ld(2, "ïd".encode()) + ld(3, b"type=C res=no msg=audit(1700000000.25:3)"), ld(3, b"type=D res=x"),
            ld(2, b"a") + ld(3, b"type=E") + ld(2, b"")]
    dev = _run(dev_c, host_c, recs)
    assert dev.encoded == dev_c.n_alerts >= 2 and dev.declined == 0


@pytest.mark.parametrize("norm", [False, True])
def test_log_schema_log_format(lib, golden_dir, norm):
    """log_format mode with the audit templates, R-norm off and all three switches on; events and global monitors."""
    from test_format_combos import AUDIT_TAIL
    params = {"log_format": AUDIT, "path_templates": os.path.join(golden_dir, "audit_templates.txt")}
    if norm:
        params.update(remove_spaces=True, remove_punctuation=True, lowercase=True)
    cfg = _cfg(250, **params)
    cfg["detectors"]["B200NewValueDetector"].update({
        "global": {"g": {"header_variables": [{"pos": "type"}, {"pos": "Content"}]}},
        "events": {0: {"pam": {"variables": [{"pos": 5, "name": "acct"}, {"pos": 6, "name": "exe"},
                                             {"pos": 10, "name": "res"}]}},
                   2: {"login": {"variables": [{"pos": 3, "name": "auid"}, {"pos": 7, "name": "res"}]}}}})
    lines = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read().rstrip(b"\n").split(b"\n")
    tail = (AUDIT_TAIL + b"\ntype=NEW msg=audit(18/Mar/2026:1): a").split(b"\n")
    dev_c, host_c = _pair(lib, cfg)
    dev = _run(dev_c, host_c, [frame(_ls_records(lines[:250], 5)), frame(_ls_records(lines[250:] + tail, 6, 250))])
    assert dev.encoded == 1 and dev.declined == 0 and dev_c.n_alerts > 5


def test_log_schema_combinations(lib, golden_dir):
    from test_format_combos import AUDIT_COMBO_CFG, AUDIT_TAIL
    cfg = {"detectors": {"NewValueComboDetector": dict(AUDIT_COMBO_CFG["detectors"]["NewValueComboDetector"], params={
        "input_format": "log_schema_batch", "log_format": AUDIT,
        "path_templates": os.path.join(golden_dir, "audit_templates.txt")})}}
    lines = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read().rstrip(b"\n").split(b"\n")
    dev_c, host_c = _pair(lib, cfg, combo=True)
    dev = _run(dev_c, host_c, [frame(_ls_records(lines[:250], 7)),
                               frame(_ls_records(lines[250:] + AUDIT_TAIL.split(b"\n"), 8))])
    assert dev.encoded == 1 and dev_c.n_alerts >= 3
    # key=value combinations (lanes kernel)
    cfg = {"detectors": {"NewValueComboDetector": {
        "method_type": "new_value_combo_detector", "data_use_training": 3, "auto_config": False,
        "params": {"input_format": "log_schema_batch"},
        "global": {"c1": {"header_variables": [{"pos": "type"}, {"pos": "acct"}]},
                   "c2": {"header_variables": [{"pos": "res"}, {"pos": "type"}]}}}}}
    dev_c, host_c = _pair(lib, cfg, combo=True)
    train = frame([ld(3, b"type=A acct=x res=ok")] * 3)
    msg = frame([ld(2, b"1") + ld(3, b"type=A acct=y res=ok"), ld(3, b"type=B acct=x res=ok msg=audit(5.5:1)"),
                 b"\xff", ld(2, b"3") + ld(3, b"type=A acct=x res=no"), ld(3, b"type=\xc3\xa9 acct=\"q r\" res=ok")])
    dev = _run(dev_c, host_c, [train, msg])
    assert dev.encoded == 1 and dev_c.n_alerts == 3


# ------------------------------------------------------------------------------------------------ ParserSchema
def _pcfg(n_train, cls="B200NewValueDetector", **params):
    """Global and event-scoped header and variable monitors."""
    cfg = _cfg(n_train, "parser_schema_batch", cls, **params)
    cfg["detectors"][cls].update({
        "global": {"g": {"header_variables": [{"pos": "user"}, {"pos": "clé"}], "variables": [{"pos": 0, "name": "v0"}]}},
        "events": {4: {"e": {"header_variables": [{"pos": "level"}], "variables": [{"pos": 2, "name": "v2"}]}},
                   -7: {"n": {"header_variables": [{"pos": "k"}]}}}})
    return cfg


def _prec(r, i, novel, time=None):
    """One ParserSchema record written field by field: duplicate map keys, map entries with a foreign field, an absent,
    repeated or non-ASCII logID, a Time entry."""
    vals = ["a", "b", "é"] + (["new%d" % i] if novel else [])
    items = [tag(4, 0) + varint(r.choice([4, -7, 0]))] if r.random() < 0.8 else []
    items += [ld(6, r.choice(vals).encode()) for _ in range(r.randint(0, 4))]
    for key in ("user", "clé", "level", "k"):
        if r.random() < 0.8:
            items.append(ld(10, ld(1, key.encode()) + ld(2, r.choice(vals).encode())))
        if r.random() < 0.15:                                       # a duplicate key: the last entry wins
            items.append(ld(10, ld(1, key.encode()) + ld(2, r.choice(vals).encode())))
        if r.random() < 0.1:                                        # a foreign field: protobuf drops the entry
            items.append(ld(10, ld(1, key.encode()) + ld(2, b"dropped%d" % i) + ld(3, b"q")))
    lid = r.random()
    if lid < 0.6:
        items.append(ld(8, b"log-%d" % i))
    elif lid < 0.7:
        items.append(ld(8, b"x") + ld(9, b"text") + ld(8, b"y-%d" % i))
    elif lid < 0.8:
        items.append(ld(8, ("ïd-☃-%d" % i).encode()))
    elif lid < 0.85:
        items.append(tag(8, 0) + varint(3))                         # not a string: protobuf skips it
    if time is not None:
        items.append(ld(10, ld(1, b"Time") + ld(2, time.encode())))
    r.shuffle(items)
    return b"".join(items)


GOOD_TIMES = [None, "1700000000.5", "17", "", "18/Mar/2026:11:43:30 +0000", "0000000001.000001", "abc x"]


@pytest.mark.parametrize("combo", [False, True])
def test_parser_schema_batches(lib, combo):
    r = random.Random(41 + combo)
    dev_c, host_c = _pair(lib, _pcfg(300, "NewValueComboDetector" if combo else "B200NewValueDetector"), combo=combo)
    train = frame([_prec(r, i, False, r.choice(GOOD_TIMES)) for i in range(300)])
    pb = RecGen(seed=3 + combo, novel=0.2, mutate=0.25)
    msgs = []
    for m in range(3):
        recs = [_prec(r, i, r.random() < 0.2, r.choice(GOOD_TIMES)) for i in range(600)]
        for j in range(0, 600, 5):                                   # pbgen records, malformed ones among them
            rec, _tags = pb.record()
            recs[j] = rec.replace(b"\x04Time", b"\x04Tim_")           # (their Time values are mostly not numbers)
        msgs.append(frame(recs))
    dev = _run(dev_c, host_c, [train] + msgs)
    assert dev.encoded == 3 and dev.declined == 0 and dev_c.n_alerts > 100


def test_parser_schema_pbgen_batches_equal_or_declined(lib):
    """pbgen's records as they come (Time entries of every kind): each batch is encoded or declined, the reply the same."""
    dev_c, host_c = _pair(lib, _pcfg(0))
    pb = RecGen(seed=8, novel=0.5, mutate=0.25)
    dev = _run(dev_c, host_c, [frame(pb.records(40)[0]) for _ in range(12)])
    assert dev.encoded + dev.declined == 12 and dev.encoded > 0


def test_parser_schema_bare_record_combo(lib):
    """The combo detector's single ParserSchema goes through the batch path and splits the encoded reply itself."""
    dev_c, host_c = _pair(lib, _pcfg(1, "NewValueComboDetector"), combo=True)
    from detectmateservice_b200.wire import encode_parser_schema
    base = {"EventID": 4, "variables": ["a", "b", "c"], "logFormatVariables": {"user": "u", "clé": "c", "level": "l"}}
    new = dict(base, logID="lid-1", logFormatVariables={"user": "NEW", "clé": "c", "level": "l", "Time": "99.5"})
    dev_c.input_format = host_c.input_format = "parser_schema"
    dev = _run(dev_c, host_c, [encode_parser_schema(base), encode_parser_schema(new)])
    assert dev.encoded == 1 and dev_c.n_alerts == 1


def _time_batch(r, times):
    return frame([ld(6, b"v%d" % (1000 + i)) + ld(8, b"id") + ld(10, ld(1, b"Time") + ld(2, t.encode()))
                  for i, t in enumerate(times)])


def test_parser_schema_time_strings(lib):
    """Fuzzed Time strings: each batch equal to the host's bytes or declined; the named cases as the rule says."""
    cfg = _cfg(1, "parser_schema_batch")
    cfg["detectors"]["B200NewValueDetector"]["global"] = {"g": {"variables": [{"pos": 0, "name": "v"}]}}
    dev_c, host_c = _pair(lib, cfg)
    _run(dev_c, host_c, [frame([ld(6, b"seed")])])
    dev = dev_c._det
    for t, outcome in [("１７００", "declined"), ("\xa017", "declined"), ("18/Mar/2026:11:43:30 +0000", NOW),
                       ("1700000000.5", 1700000000), ("", NOW), ("17 ", "declined"), ("é1", "declined"),
                       ("éx", NOW)]:
        enc0, dec0 = dev.encoded, dev.declined
        out = dev_c.process(_time_batch(None, [t]))
        assert out == host_c.process(_time_batch(None, [t]))
        if outcome == "declined":
            assert dev.declined == dec0 + 1, t
        else:
            assert dev.encoded == enc0 + 1, t
            assert wire.decode_detector_schema(wire.split_delimited(out)[0])["extractedTimestamps"] == [outcome], t
    r = random.Random(6)
    alphabet = "0123456789.eE+-_ xinf:\xa0１٣é "
    for _ in range(40):
        times = ["".join(r.choice(alphabet) for _ in range(r.randint(0, 10))) for _ in range(3)]
        try:
            want = host_c.process(_time_batch(r, times))
        except OverflowError:                                       # int(float("inf")): the host fails the message
            with pytest.raises(OverflowError):
                dev_c.process(_time_batch(r, times))
            continue
        assert dev_c.process(_time_batch(r, times)) == want
    assert dev.encoded > 5 and dev.declined > 10


def test_time_of_a_str_is_exact_where_it_accepts(lib):
    """emu_alert_time_str: every str it converts gives int(float(s)), every clock is a ValueError of float(s)."""
    r = random.Random(12)
    ts = C.c_longlong()
    alphabet = "0123456789.eE+-_ xinf:\t\xa0 １٣éÿ€😀"
    cases = ["".join(r.choice(alphabet) for _ in range(r.randint(0, 10))) for _ in range(40000)]
    cases += ["１７００", "\xa017", "18/Mar/2026:11:43:30 +0000", "1700000000.5", "", "é", "1é", "é x"]
    accepted = 0
    for s in cases:
        b = s.encode()
        if not lib.emu_alert_time_str(b, len(b), NOW, C.byref(ts)):
            continue
        accepted += 1
        try:
            want = int(float(s))
        except ValueError:
            want = NOW
        assert ts.value == want, s
    assert accepted > 10000


def test_more_anomalous_records_than_the_encoder_holds(lib):
    """A ParserSchema batch with more anomalous records than the per-record arrays (the anomaly list's capacity)
    declines as a whole; the host words it."""
    cfg = _cfg(1, "parser_schema_batch")
    cfg["detectors"]["B200NewValueDetector"]["global"] = {"g": {"variables": [{"pos": 0, "name": "v"}]}}
    dev_c, host_c = _pair(lib, cfg, anomaly_cap=50)
    batch = lambda n, b: frame([ld(6, b"%s%d" % (b, i)) + ld(8, b"%d" % i) for i in range(n)])
    dev = _run(dev_c, host_c, [batch(1, b"t"), batch(50, b"a"), batch(51, b"b")])
    assert dev.encoded == 1 and dev.declined == 1 and dev_c.n_alerts == 101


@pytest.mark.parametrize("fmt", ["log_schema_batch", "parser_schema_batch"])
def test_small_output_buffer_declines(lib, fmt):
    cfg = _cfg(1, fmt)
    cfg["detectors"]["B200NewValueDetector"]["global"] = {"g": {"header_variables": [{"pos": "type"}]}}
    dev_c, host_c = _pair(lib, cfg, capacity=600)
    if fmt == "log_schema_batch":
        batch = lambda n, b: frame([ld(2, b"id%d" % i) + ld(3, b"type=%s%d" % (b, i)) for i in range(n)])
    else:
        batch = lambda n, b: frame([ld(10, ld(1, b"type") + ld(2, b"%s%d" % (b, i))) for i in range(n)])
    dev = _run(dev_c, host_c, [batch(1, b"t"), batch(2, b"a"), batch(40, b"b")])
    assert dev.encoded == 1 and dev.declined == 1 and dev_c.n_alerts == 42

