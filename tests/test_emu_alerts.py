"""DetectorSchema alerts encoded on the device (DESIGN.md R-alert), CPU tier: the encoder kernels of
dm_kernels_alerts.cuh run on the CPU emulator after the emulated detect kernels (stream, stream with the chained re-check,
lanes), behind an emulator-backed stand-in for DeviceDetector.  Every message must come out byte for byte as the
component's host encoder writes it for the same batch."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from detectmateservice_b200 import wire
from detectmateservice_b200.synth import MONITORED_KEYS, AuditSynth

NOW = 1773848383


def _emu_lib():
    import emu_harness
    src = os.path.join(emu_harness.EMU, "emu_alerts.cpp")
    so = os.path.join(emu_harness.EMU, "_build", "libemu_alerts.so")
    deps = [src, os.path.join(emu_harness.EMU, "emu_tile.cpp"), os.path.join(emu_harness.EMU, "emu_format_combo.cpp"), os.path.join(emu_harness.EMU, "cuda_emu.h")] + [
        os.path.join(emu_harness.CSRC, f) for f in os.listdir(emu_harness.CSRC)] + [
        os.path.join(emu_harness.ROOT, "include", "dmdetect.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        # (-Bsymbolic: the library binds to its own emulator runtime, whatever else the process has loaded)
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-DDM_EMU", "-I" + emu_harness.EMU, "-I" + emu_harness.CSRC,
                               "-shared", "-fPIC", "-pthread", "-Wl,-Bsymbolic", "-o", so, src])
    lib = C.CDLL(so)
    fn = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64,
          C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    for name in ("emu_process_stream", "emu_process_stream_chain", "emu_process_lanes", "emu_process_format_combo"):
        getattr(lib, name).argtypes = fn
    lib.emu_create.restype = C.c_void_p
    lib.emu_create.argtypes = [C.c_uint32, C.c_char_p, C.POINTER(C.c_uint32), C.c_uint32, C.c_uint64, C.c_uint64]
    lib.emu_destroy.argtypes = [C.c_void_p]
    lib.emu_set_combos.argtypes = [C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_uint32]
    lib.emu_get_anomalies.restype = C.c_uint32
    lib.emu_get_anomalies.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    lib.emu_set_alert_format.restype = C.c_char_p
    lib.emu_set_alert_format.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                         C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                         C.c_uint32]
    lib.emu_set_format.restype = C.c_char_p
    lib.emu_set_format.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_char_p),
                                   C.c_uint32]
    lib.emu_encode_alerts.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int64, C.c_int64,
                                      C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int)]
    lib.emu_utf8_replace.restype = C.c_uint32
    lib.emu_utf8_replace.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p]
    lib.emu_alert_time.argtypes = [C.c_char_p, C.c_uint32, C.c_longlong, C.POINTER(C.c_longlong)]
    return lib


@pytest.fixture(scope="module")
def lib():
    return _emu_lib()


class _Anomaly(C.Structure):
    _fields_ = [("line", C.c_uint32), ("mask", C.c_uint32), ("offset", C.c_uint64)]


class EmuDevice:
    """Stands in for DeviceDetector: detection and the alert encoder on the CPU emulator (tests only)."""

    def __init__(self, lib, keys, variant="stream", combos=(), capacity=1 << 20, comp=None):
        self.lib, self.variant, self.capacity = lib, variant, capacity
        if variant == "format":                                      # the component's log_format, templates, R-norm
            from test_format_combos import _monitor_array
            lf = comp.logformat
            ts = [t if isinstance(t, bytes) else t.encode() for t in lf.template_sources]
            err = lib.emu_set_format(_monitor_array(comp.monitors), len(comp.monitors), lf.source.encode(),
                                     lf.content_name.encode(), len(ts), (C.c_char_p * max(1, len(ts)))(*ts), lf.flags)
            assert err is None, err
        self.keys = [bytes(k) for k in keys]
        lens = (C.c_uint32 * max(1, len(self.keys)))(*[len(k) for k in self.keys])
        self.h = lib.emu_create(len(self.keys), b"".join(self.keys), lens, 14, 64, 1 << 20)
        off, flat = [0], []
        for members in combos:
            flat.extend(members)
            off.append(len(flat))
        lib.emu_set_combos(len(combos), (C.c_uint32 * len(off))(*off), (C.c_uint32 * max(1, len(flat)))(*flat),
                           (1 << len(self.keys)) - 1 if combos else 0)
        self.last_n_anomalies = 0
        self.encoded = self.declined = 0

    def close(self):
        if self.h:
            self.lib.emu_destroy(self.h)
            self.h = None

    def process_lines(self, buf, n_train_lines=0, copy=True):
        self._msg = bytes(buf)
        cap = self._msg.count(b"\n") + 2
        flags, scores = np.zeros(cap, np.uint8), np.zeros(cap, np.float32)
        n, na, err = C.c_uint64(), C.c_uint64(), C.c_uint32()
        fn = {"stream": self.lib.emu_process_stream, "chain": self.lib.emu_process_stream_chain,
              "lanes": self.lib.emu_process_lanes, "format": self.lib.emu_process_format_combo}[self.variant]
        assert fn(self.h, self._msg, len(self._msg), n_train_lines, flags.ctypes.data, scores.ctypes.data, cap,
                  C.byref(n), C.byref(na), C.byref(err)) == 0 and err.value == 0
        self._scores = scores
        self.last_n_anomalies = na.value
        return flags[:n.value], scores[:n.value]

    def anomalies(self):
        arr = (_Anomaly * 65536)()
        k = self.lib.emu_get_anomalies(self.h, arr, 65536)
        return [(arr[i].line, arr[i].mask, arr[i].offset) for i in range(k)]

    def set_alert_format(self, version, detector_id, detector_type, description, alert_keys, combos=(), capacity=0,
                         time_capture=None):
        strs = [s.encode() for s in (version, detector_id, detector_type, description)] + [k.encode() for k, _ in alert_keys]
        off, flat = [0], []
        for _k, bits in alert_keys:
            flat.extend(bits)
            off.append(len(flat))
        c_off, c_mem = [0], []
        for members in combos:
            c_mem.extend(members)
            c_off.append(len(c_mem))
        u32 = lambda v: (C.c_uint32 * max(1, len(v)))(*v)
        why = self.lib.emu_set_alert_format(self.h, len(strs), b"".join(strs), u32([len(s) for s in strs]), u32(off),
                                            u32(flat), len(combos), u32(c_off), u32(c_mem),
                                            0xFFFFFFFF if time_capture is None else time_capture)
        assert why is None, why

    def encode_alerts(self, first_log_id, first_alert_id, now):
        out = np.zeros(self.capacity + 1, np.uint8)
        ln, n, dec = C.c_uint64(), C.c_uint64(), C.c_int()
        assert self.lib.emu_encode_alerts(self.h, int(self.variant == "format"), self._msg, len(self._msg), self._scores.ctypes.data, first_log_id,
                                          first_alert_id, now, out.ctypes.data, self.capacity, C.byref(ln), C.byref(n),
                                          C.byref(dec)) == 0
        if dec.value:
            self.declined += 1
            return None
        self.encoded += 1
        return out[:ln.value].tobytes(), n.value


class HostOnly:
    """The same emulated detection without the encoder: the component words the alerts on the host."""

    def __init__(self, dev):
        self.dev = dev

    def process_lines(self, buf, n_train_lines=0, copy=True):
        f, s = self.dev.process_lines(buf, n_train_lines, copy)
        self.last_n_anomalies = self.dev.last_n_anomalies
        return f, s

    def anomalies(self):
        return self.dev.anomalies()

    def close(self):
        self.dev.close()


def _pair(lib, cfg, variant="stream", combo=False, capacity=1 << 20):
    """Two components of one config: device-encoded alerts, and the host encoder on the same emulated detection."""
    from detectmateservice_b200.component import B200NewValueComboDetector, B200NewValueDetector
    cls = B200NewValueComboDetector if combo else B200NewValueDetector
    comps = []
    for host in (False, True):
        c = cls(config=cfg)
        combos = c.combos if combo else ()
        v = variant if c.logformat is not None or not combo else "lanes"
        dev = EmuDevice(lib, [m.key for m in c.monitors], "format" if c.logformat is not None else v, combos, capacity, c)
        c._det = HostOnly(dev) if host else dev
        c.DEVICE_ALERTS_MIN = 1                                      # every batch with alerts goes to the encoder
        c.clock = lambda: NOW
        comps.append(c)
    return comps


def _run(dev_c, host_c, messages):
    """Both components over the same messages; the device stand-in, which counts the messages it encoded / declined."""
    for msg in messages:
        got = dev_c.process(msg)
        want = host_c.process(msg)
        assert got == want
        assert dev_c.n_alerts == host_c.n_alerts and dev_c.n_seen == host_c.n_seen
    return dev_c._det


def _cfg(keys, n_train, **params):
    return {"detectors": {"B200NewValueDetector": {
        "method_type": "new_value_detector", "data_use_training": n_train, "auto_config": False, "params": params,
        "global": {"g": {"header_variables": [{"pos": k} for k in keys]}}}}}


@pytest.mark.parametrize("variant", ["stream", "chain", "lanes"])
def test_audit_sample_golden(lib, golden_dir, variant):
    import json
    exp = json.load(open(os.path.join(golden_dir, "audit_sample.expected.json")))
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read()
    dev_c, host_c = _pair(lib, _cfg(exp["keys"], exp["n_train"]), variant)
    half = buf.index(b"\n", len(buf) // 2) + 1
    dev = _run(dev_c, host_c, [buf[:half], buf[half:], b"type=NEVER_SEEN msg=audit(1642723741.072:1): pid=1\n"])
    assert dev.encoded >= 2 and dev.declined == 0
    assert sum(1 for f in exp["flags"] if f) + 1 == dev_c.n_alerts


@pytest.mark.parametrize("variant", ["stream", "chain", "lanes"])
def test_audit_synth_burst(lib, variant):
    g = AuditSynth(seed=11, anomaly_rate=1e-1)
    train, _ = g.batch(2048, inject=False)
    msgs = [g.batch(3000, inject=True)[0] for _ in range(2)]
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 2048, start_id=-5), variant)
    dev = _run(dev_c, host_c, [train] + msgs)
    assert dev.encoded == 2 and dev.declined == 0 and dev_c.n_alerts > 300


def test_varlen_lookalikes_duplicates_and_values(lib):
    """Quoted look-alikes, duplicate keys (the first true field wins), keys after a single quote, empty values,
    records without the field, '\\r', a record without its final '\\n', values of ill-formed UTF-8."""
    keys = ["type", "acct", "exe", "res"]
    train = b"".join(b"type=A acct=u%d exe=/bin/x res=ok msg=audit(1.5:1)\n" % i for i in range(4))
    recs = [b'type=NEW acct="x type=Q" type=DUP exe=/bin/x res=ok',
            b'x="a type=HIDDEN" type=A acct=u1 res=ok',
            b"'type=QUOTE' acct=new1 res=ok msg=audit(1700000000.123:9):",
            b'type=A acct= res=ok msg=audit(12345678)',
            b'type=A exe="/usr/bin/a b" res=fail\r',
            b"type=\xff\xfe\xc3 acct=\xe2\x82 res=\xed\xa0\x80\xf0\x9f\x98\x80 msg=audit(0:1)",
            b"type=A acct=u0 msg=\"audit(9.9:1)\" res=\xc0\xaf"]
    msg = b"\n".join(recs)                                            # (no final '\n': the last record still counts)
    for variant in ("stream", "chain", "lanes"):
        dev_c, host_c = _pair(lib, _cfg(keys, 4), variant)
        dev = _run(dev_c, host_c, [train, msg])
        assert dev.encoded == 1 and dev_c.n_alerts == 6


def test_non_ascii_labels_and_colliding_alert_keys(lib):
    """Alert keys sort by their UTF-8 bytes; two monitors with one alert key: the last one flagged wins."""
    cfg = {"detectors": {"B200NewValueDetector": {
        "method_type": "new_value_detector", "data_use_training": 2, "auto_config": False, "params": {"detector_id": "Dé"},
        "global": {"a": {"header_variables": [{"pos": "zé"}, {"pos": "type"}, {"pos": "Ω"}, {"pos": "acct"}]},
                   "b": {"header_variables": [{"pos": "type"}, {"pos": "b"}]}}}}}
    from detectmateservice_b200.component import B200NewValueDetector
    assert [m.alert_key for m in B200NewValueDetector(config=cfg).monitors].count("Global - type") == 2
    train = "zé=1 type=T Ω=w acct=a b=1\nzé=1 type=T Ω=w acct=a b=1\n".encode()
    msg = "zé=2 type=T Ω=w acct=a b=1\nzé=1 type=X Ω=v acct=b b=2\nb=3 type=Y\nΩ=ω\n".encode()
    for variant in ("stream", "lanes"):
        dev_c, host_c = _pair(lib, cfg, variant)
        dev = _run(dev_c, host_c, [train, msg])
        assert dev.encoded == 1 and dev_c.n_alerts == 4


def test_fuzzed_values_utf8(lib):
    r = random.Random(5)
    pool = [b"\x80", b"\xc2", b"\xc3\xa9", b"\xe0\x80", b"\xe0\xa0\x80", b"\xed\x9f\xbf", b"\xed\xa0\x80", b"\xef\xbf",
            b"\xf0\x90\x80", b"\xf0\x9f\x98\x80", b"\xf4\x8f\xbf\xbf", b"\xf4\x90", b"\xf5", b"\xff", b"a", b"'", b'"']
    keys = ["type", "acct"]
    train = b"type=T acct=a\n" * 2
    lines = []
    for i in range(400):
        v1 = b"".join(r.choice(pool) for _ in range(r.randint(0, 6))).replace(b" ", b"")
        v2 = b"".join(r.choice(pool) for _ in range(r.randint(0, 4)))
        lines.append(b"type=" + v1 + b" acct=" + v2 + b"%d" % i)
    msg = b"\n".join(lines) + b"\n"
    dev_c, host_c = _pair(lib, _cfg(keys, 2), "stream")
    dev = _run(dev_c, host_c, [train, msg])
    assert dev.encoded == 1 and dev_c.n_alerts == 400


def test_utf8_replace_matches_python_codec(lib):
    r = random.Random(9)
    out = np.zeros(3 * 64 + 3, np.uint8)
    cases = [bytes([a, b]) for a in range(0x80, 0x100) for b in (0x7F, 0x80, 0x9F, 0xA0, 0xBF, 0xC0)]
    cases += [bytes(r.randrange(256) if r.random() < 0.5 else r.choice(b"\x80\xbf\xc2\xe0\xed\xf0\xf4\xa0\x90\x8f")
                    for _ in range(r.randint(0, 64))) for _ in range(20000)]
    for s in cases:
        n = lib.emu_utf8_replace(s, len(s), out.ctypes.data)
        assert out[:n].tobytes() == s.decode("utf-8", "replace").encode("utf-8"), s


def _py_time(s: bytes):
    try:
        return int(float(s))
    except (ValueError, OverflowError):
        return None                                                  # (inf, nan: the device must have declined)


def test_time_grammar_is_exact_where_it_accepts(lib):
    """Every string the device converts gives int(float(s)); the grammar [0-9]{1,10}(\\.[0-9]{0,6})? is all accepted."""
    r = random.Random(3)
    ts = C.c_longlong()
    digits = "0123456789"
    grammar = ["9999999999.999999", "0", "0.", "1642723741.072", "0000000000.000000", "4294967295.5", "1.999999"]
    grammar += ["".join(r.choice(digits) for _ in range(r.randint(1, 10))) + (
        "." + "".join(r.choice(digits) for _ in range(r.randint(0, 6))) if r.random() < 0.7 else "") for _ in range(50000)]
    for s in grammar:
        assert lib.emu_alert_time(s.encode(), len(s), NOW, C.byref(ts)) == 1, s
        assert ts.value == int(float(s)), s
    other = ["", ".5", "1e3", "1_0", " 1", "1 ", "inf", "nan", "-1", "+1", "12345678901", "1.2345678", "1.9999999",
             "99999999999.5", "0x10", "1..2", "١"]
    alphabet = "0123456789.eE+-_ xi"
    other += ["".join(r.choice(alphabet) for _ in range(r.randint(0, 14))) for _ in range(50000)]
    other += ["18/Mar/2026:11:43:30 +0000", "1642723741.072:375", "12:00", "\x00", "1\xff"]
    other += [bytes(r.randrange(256) for _ in range(r.randint(0, 8))).decode("latin-1") for _ in range(20000)]
    n_now = 0
    for s in other:
        b = s.encode("latin-1") if max(map(ord, s), default=0) < 256 else s.encode()
        if lib.emu_alert_time(b, len(b), NOW, C.byref(ts)):
            want = _py_time(b)
            if want is None:                                         # float() raises ValueError: the host takes the clock
                with pytest.raises(ValueError):
                    float(b)
                n_now += 1
                assert ts.value == NOW, s
            else:
                assert ts.value == want, s
    assert n_now > 10000


def test_fuzzed_time_strings_equal_or_declined(lib):
    """Per message: device bytes equal to the host's, or declined and then the host's bytes (the component falls back)."""
    r = random.Random(4)
    alphabet = "0123456789.eE+-_ xinf:"
    dev_c, host_c = _pair(lib, _cfg(["type"], 1), "stream")
    _run(dev_c, host_c, [b"type=T\n"])
    n_dec = 0
    for i in range(60):
        t = "".join(r.choice(alphabet) for _ in range(r.randint(0, 12))) if r.random() < 0.5 else "%d.%03d" % (
            r.randrange(10 ** 10), r.randrange(1000))
        msg = ("type=N%d msg=audit(%s:1)\n" % (i, t)).encode()
        try:
            want = host_c.process(msg)
        except OverflowError:                                        # int(float("inf")): the host fails the message
            with pytest.raises(OverflowError):
                dev_c.process(msg)
            continue
        assert dev_c.process(msg) == want
        n_dec = dev_c._det.declined
    assert 0 < n_dec < dev_c._det.declined + dev_c._det.encoded


def test_combinations_key_value(lib):
    cfg = {"detectors": {"B200NewValueComboDetector": {
        "method_type": "new_value_combo_detector", "data_use_training": 3, "auto_config": False, "params": {},
        "global": {"c1": {"header_variables": [{"pos": "type"}, {"pos": "acct"}]},
                   "c2": {"header_variables": [{"pos": "exe"}]},
                   "c3": {"header_variables": [{"pos": "res"}, {"pos": "type"}]}}}}}
    train = b"type=A acct=x exe=/a res=ok\n" * 3
    msg = (b"type=A acct=y exe=/a res=ok\ntype=B acct=x exe=/b res=ok\ntype=A acct=x exe=/a res=no\n"
           b"acct=x exe=/a\ntype=\xff acct=\"q r\" exe=/a res=ok msg=audit(77.1:2)\n")
    dev_c, host_c = _pair(lib, cfg, combo=True)
    dev = _run(dev_c, host_c, [train, msg, b"type=Z acct=x exe=/a res=ok\n"])
    assert dev.encoded == 2 and dev_c.n_alerts == 4


def test_chunked_message_and_small_output_buffer(lib):
    g = AuditSynth(seed=12, anomaly_rate=5e-2)
    train, _ = g.batch(512, inject=False)
    big, _ = g.batch(4000, inject=True)
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 512, max_batch_bytes=200_000))
    dev = _run(dev_c, host_c, [train, big])
    assert len(big) > 200_000 and dev.encoded >= 4 and dev.declined == 0
    # an output buffer too small for a batch: declined, the host words it, the bytes are the same
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 512), capacity=2000)
    dev = _run(dev_c, host_c, [train, big, g.batch(200, inject=False)[0] + b"type=ONLY1 res=x\n"])
    assert dev.declined == 1 and dev.encoded == 1


def test_few_alerts_stay_on_the_host(lib):
    """Below DEVICE_ALERTS_MIN anomalous records the host encoder is cheaper; from it on the device encodes."""
    from detectmateservice_b200.component import B200NewValueDetector
    dev_c, host_c = _pair(lib, _cfg(["type"], 1))
    del dev_c.DEVICE_ALERTS_MIN, host_c.DEVICE_ALERTS_MIN              # the class default
    k = B200NewValueDetector.DEVICE_ALERTS_MIN
    few = b"".join(b"type=F%d\n" % i for i in range(k - 1))
    many = b"".join(b"type=M%d\n" % i for i in range(k))
    dev = _run(dev_c, host_c, [b"type=T\n", few])
    assert dev.encoded == 0 and dev_c.n_alerts == k - 1
    _run(dev_c, host_c, [many])
    assert dev.encoded == 1 and dev_c.n_alerts == 2 * k - 1


AUDIT = "type=<type> msg=audit(<Time>): <Content>"


@pytest.mark.parametrize("norm", [False, True])
def test_log_format_with_templates(lib, golden_dir, norm):
    """log_format mode: header captures verbatim, template variables sliced from the Content (R-norm off, and all three
    switches on), Time from the <Time> capture; events and global monitors, a colliding alert key."""
    from test_format_combos import AUDIT_TAIL
    params = {"log_format": AUDIT, "path_templates": os.path.join(golden_dir, "audit_templates.txt")}
    if norm:
        params.update(remove_spaces=True, remove_punctuation=True, lowercase=True)
    cfg = {"detectors": {"B200NewValueDetector": {
        "method_type": "new_value_detector", "data_use_training": 250, "auto_config": False, "params": params,
        "global": {"g": {"header_variables": [{"pos": "type"}, {"pos": "Content"}]}},
        "events": {0: {"pam": {"variables": [{"pos": 5, "name": "acct"}, {"pos": 6, "name": "exe"},
                                             {"pos": 10, "name": "res"}]}},
                   2: {"login": {"variables": [{"pos": 3, "name": "auid"}, {"pos": 7, "name": "res"}]}}}}}}
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read()
    cut = 0
    for _ in range(250):
        cut = buf.index(b"\n", cut) + 1
    odd = (b"type=\xff\xfeX msg=audit(1642723741.5:1): pid=1 uid=0 auid=4294967295 ses=1 msg='op=\xc3 acct=\"r\xe2\x82\" "
           b"exe=\"/x\" hostname=? addr=? terminal=cron res=success'\n"
           b"type=NEW msg=audit(18/Mar/2026:1): a\n")
    dev_c, host_c = _pair(lib, cfg)
    dev = _run(dev_c, host_c, [buf[:cut], buf[cut:] + AUDIT_TAIL + b"\n" + odd])
    assert dev.encoded == 1 and dev.declined == 0 and dev_c.n_alerts > 5


def test_log_format_combinations_and_declined_time(lib, golden_dir):
    from test_format_combos import AUDIT_COMBO_CFG, AUDIT_TAIL
    cfg = {"detectors": {"NewValueComboDetector": dict(AUDIT_COMBO_CFG["detectors"]["NewValueComboDetector"], params={
        "log_format": AUDIT, "path_templates": os.path.join(golden_dir, "audit_templates.txt"),
        "remove_spaces": True, "remove_punctuation": True, "lowercase": True})}}
    buf = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read()
    cut = 0
    for _ in range(250):
        cut = buf.index(b"\n", cut) + 1
    dev_c, host_c = _pair(lib, cfg, combo=True)
    dev = _run(dev_c, host_c, [buf[:cut], buf[cut:] + AUDIT_TAIL + b"\n",
                               b"type=ZZ msg=audit(1e3): x\n"])             # a Time the device cannot convert
    assert dev.encoded == 1 and dev.declined == 1 and dev_c.n_alerts > 3
