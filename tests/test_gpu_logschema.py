"""LogSchema input on the H100 (DESIGN.md R-log): dm_process_logs against the rule's oracle -- decode with protobuf's
runtime, drop the malformed and unusable records, run the raw-line oracle on the joined texts, scatter back -- in
key=value mode (both stream re-check choices and the lanes kernel), in log_format mode (templates, every R-norm switch)
and with combinations in both; against dm_process_lines on the joined text; at its edges; and behind the unmodified
reference service."""
import os
import random
import time

import numpy as np
import pytest

from detectmateservice_b200 import wire
from lsgen import Gen, batch, unwrap
from oracle.nvcd import NewValueComboDetectorOracle
from oracle.nvd import NewValueDetectorOracle
from oracle.rfmt import FormatParser
from pbgen import frame

pytestmark = pytest.mark.gpu

AUDIT = "type=<type> msg=audit(<Time>): <Content>"
NGINX = '<IP> - - [<Time>] "<Method> <URL> <Protocol>" <Status> <Bytes> "<Referer>" "<UserAgent>"'
KV_KEYS = ["type", "exe", "terminal", "acct", "res"]


def _cfg(training, glob, events=None, combo=False):
    return {"detectors": {"D": {"method_type": "new_value_combo_detector" if combo else "new_value_detector",
                                "data_use_training": training, "auto_config": False, "global": glob,
                                "events": events or {}}}}


KV_CFG = lambda training: _cfg(training, {"g": {"header_variables": [{"pos": k} for k in KV_KEYS]}})
KV_COMBO_CFG = lambda training: _cfg(training, {"a": {"header_variables": [{"pos": "type"}, {"pos": "res"}]},
                                                "b": {"header_variables": [{"pos": "exe"}, {"pos": "acct"}, {"pos": "terminal"}]}},
                                     combo=True)
AUDIT_EVENTS = {0: {"pam": {"variables": [{"pos": 4, "name": "op"}, {"pos": 6, "name": "exe"}],
                            "header_variables": [{"pos": "type"}]}},
                2: {"login": {"variables": [{"pos": 3, "name": "auid"}, {"pos": 7, "name": "res"}]}}}
FMT_CFG = lambda training: _cfg(training, {"g": {"header_variables": [{"pos": "type"}]}}, AUDIT_EVENTS)
FMT_COMBO_CFG = lambda training: _cfg(training, {"g": {"header_variables": [{"pos": "type"}, {"pos": "Time"}]}},
                                      {0: {"pam": {"variables": [{"pos": 4}, {"pos": 6}]}}},
                                      combo=True)


def _audit_lines(golden_dir, n, seed):
    """audit_sample.log lines, cycled, with some values changed so that detection finds new ones."""
    base = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read().split(b"\n")
    base = [b for b in base if b]
    r = random.Random(seed)
    out = []
    for i in range(n):
        ln = base[i % len(base)]
        if r.random() < 0.02:
            ln = ln.replace(b"res=success", b"res=odd%d" % r.randint(0, 3)).replace(b"type=", b"type=X", 1 if r.random() < 0.3 else 0)
        out.append(ln)
    return out


def _synth_lines(n, seed):
    from detectmateservice_b200.synth import AuditSynth
    msg, _ = AuditSynth(seed=seed).batch(n, inject=True)
    return msg.split(b"\n")[:n]


def _templates(golden_dir):
    from detectmateservice_b200.logformat import load_templates
    return load_templates(os.path.join(golden_dir, "audit_templates.txt"))


class RuleOracle:
    """R-log on top of a raw-line oracle step (text -> (flag, score, alerts))."""

    def __init__(self, step):
        self.step = step

    def batch(self, records):
        _joined, idx, ids = unwrap(records)
        texts = [t for t in _joined.split(b"\n")][:len(idx)]
        alerts = []
        for j, t in enumerate(texts):
            f, s, a = self.step(t)
            if f:
                alerts.append((ids[idx[j]], a, s))
        return alerts, len(records) - len(idx)


def _format_step(orc, parser):
    def step(line):
        rec = parser.parse_line(line)
        step.mismatch += rec is None                            # (a bad_record of the line path)
        return orc.step(rec if rec is not None else {"EventID": None, "variables": [], "logFormatVariables": {}})
    step.mismatch = 0
    return step


def _component(cls, cfg, params):
    from detectmateservice_b200 import component
    det = dict(cfg["detectors"]["D"])
    det["params"] = dict(params, input_format="log_schema_batch", max_batch_bytes=8 << 20)
    c = getattr(component, cls)(name="D", config={"detectors": {"D": det}})
    c.clock = lambda: 1773848383
    return c


def _run(comp, oracle, lines, seed, per_msg=1500):
    """Feeds the lines as fuzzed LogSchema batches (malformed records among them); alerts, logIDs, scores and
    bad_records must equal the oracle's."""
    g = Gen(seed=seed, mutate=0.06)
    r = random.Random(seed)
    got, want, bad = [], [], 0
    for lo in range(0, len(lines), per_msg):
        recs = g.records(lines[lo:lo + per_msg], id_base=lo)
        out = comp.process(batch(recs, r))
        got += [wire.decode_detector_schema(b) for b in wire.split_delimited(out)] if out else []
        w, nb = oracle.batch(recs)
        want += w
        bad += nb
    assert [(a["logIDs"], a["alertsObtain"], a["score"]) for a in got] == [([i], al, s) for i, al, s in want]
    st = comp.stats()
    assert st["bad_records"] - getattr(oracle.step, "mismatch", 0) == bad > 0 and st["lines"] == len(lines) and st["anomalies"] == len(want) > 0
    comp.close()


@pytest.mark.parametrize("variant", [("stream", "thread"), ("stream", "chain"), ("lanes", "auto")])
def test_gpu_logschema_key_value_vs_oracle(monkeypatch, variant):
    monkeypatch.setenv("DM_KERNEL", variant[0])
    monkeypatch.setenv("DM_STREAM_RECHECK", variant[1])
    lines = _synth_lines(9000, seed=31)
    orc = NewValueDetectorOracle(config=KV_CFG(4000), name="D", clock=lambda: 1773848383)
    _run(_component("B200NewValueDetector", KV_CFG(4000), {}), RuleOracle(orc.step_line), lines, seed=31)


@pytest.mark.parametrize("norm", [(False, False, False), (True, False, False), (False, True, False), (False, False, True),
                                  (True, True, True)])
def test_gpu_logschema_log_format_vs_oracle(golden_dir, norm):
    tm = _templates(golden_dir)
    lines = _audit_lines(golden_dir, 3000, seed=32)
    parser = FormatParser(AUDIT, tm, remove_spaces=norm[0], remove_punctuation=norm[1], lowercase=norm[2])
    orc = NewValueDetectorOracle(config=FMT_CFG(800), name="D", clock=lambda: 1773848383)
    params = {"log_format": AUDIT, "templates": [t.decode() for t in tm], "remove_spaces": norm[0],
              "remove_punctuation": norm[1], "lowercase": norm[2]}
    _run(_component("B200NewValueDetector", FMT_CFG(800), params), RuleOracle(_format_step(orc, parser)), lines, seed=32,
         per_msg=700)


def test_gpu_logschema_combos_key_value_vs_oracle():
    lines = _synth_lines(6000, seed=33)
    orc = NewValueComboDetectorOracle(config=KV_COMBO_CFG(3000), name="D", clock=lambda: 1773848383)
    _run(_component("B200NewValueComboDetector", KV_COMBO_CFG(3000), {}), RuleOracle(orc.step_line), lines, seed=33)


@pytest.mark.parametrize("norm", [(False, False, False), (True, True, True)])
def test_gpu_logschema_combos_log_format_vs_oracle(golden_dir, norm):
    tm = _templates(golden_dir)
    lines = _audit_lines(golden_dir, 2000, seed=34)
    parser = FormatParser(AUDIT, tm, remove_spaces=norm[0], remove_punctuation=norm[1], lowercase=norm[2])
    orc = NewValueComboDetectorOracle(config=FMT_COMBO_CFG(700), name="D", clock=lambda: 1773848383)
    params = {"log_format": AUDIT, "templates": [t.decode() for t in tm], "remove_spaces": norm[0],
              "remove_punctuation": norm[1], "lowercase": norm[2]}
    _run(_component("B200NewValueComboDetector", FMT_COMBO_CFG(700), params), RuleOracle(_format_step(orc, parser)),
         lines, seed=34, per_msg=500)


# ------------------------------------------------------------------------------------------ device level
def _det(max_batch_bytes=8 << 20, **kw):
    from detectmateservice_b200.detector import DeviceDetector
    return DeviceDetector([k.encode() for k in KV_KEYS], device=0, max_batch_bytes=max_batch_bytes, table_log2_slots=18, **kw)


def _payload_offsets(msg):
    from detectmateservice_b200.wire import _read_varint
    offs, pos = [], 0
    while pos < len(msg):
        ln, pos = _read_varint(msg, pos)
        offs.append(pos)
        pos += ln
    return offs


def _check_against_lines(records, n_train, max_batch_bytes=8 << 20, delimited=True):
    """dm_process_logs on the records == dm_process_lines on the joined usable texts, scattered back; statistics as
    the rule says."""
    msg = frame(records) if delimited else records[0]
    joined, idx, _ = unwrap(records)
    a, b = _det(max_batch_bytes), _det(max_batch_bytes)
    try:
        f, s, n_bad = a.process_logs(msg, n_train, delimited)
        anoms = a.anomalies()
        st = a.stats()
        ntl = min(n_train, len(idx))
        lf, ls = b.process_lines(joined, ntl) if idx else (np.zeros(0, np.uint8), np.zeros(0, np.float32))
        lan = b.anomalies() if idx and b.last_n_anomalies else []
        n = len(records)
        assert f.size == n and n_bad == n - len(idx)
        wf = np.zeros(n, np.uint8); ws = np.zeros(n, np.float32)
        wf[idx] = lf; ws[idx] = ls
        assert (f == wf).all() and (s == ws).all()
        offs = _payload_offsets(msg) if delimited else [0]
        assert anoms == [(idx[ln], mask, offs[idx[ln]]) for ln, mask, _o in lan]
        bound = 0 if ntl == 0 else (n if n_train > len(idx) else idx[ntl - 1] + 1)
        assert (st["lines"], st["train_lines"], st["detect_lines"], st["bytes"], st["bad_records"]) == (
            n, ntl, n - bound, len(msg), n - len(idx))
        return f, s
    finally:
        a.close(); b.close()


def test_gpu_logschema_clean_batches_equal_process_lines():
    lines = _synth_lines(20000, seed=35)
    g = Gen(seed=35, mutate=0.0)
    recs = g.records(lines)
    _check_against_lines(recs, 9000)
    _check_against_lines(recs[:5000], 0)


def test_gpu_logschema_edges_training_bound():
    lines = _synth_lines(3000, seed=36)
    g = Gen(seed=36, mutate=0.15)
    recs = g.records(lines)
    _joined, idx, _ = unwrap(recs)
    bad = [i for i in range(len(recs)) if i not in set(idx)]
    assert len(bad) > 100
    b0 = bad[3]
    # n_train ending just before, on (the record past it is malformed) and past a malformed record, and past the end
    before = idx.index(b0 - 1) + 1 if (b0 - 1) in idx else 1
    for n_train in (0, 1, before, before + 1, len(idx) - 1, len(idx), len(idx) + 1, len(recs) + 50):
        _check_against_lines(recs, n_train)


def test_gpu_logschema_edges_sizes():
    # empty batch; malformed records only; a bare record; a bare empty record
    with _det() as d:
        st0 = d.stats()
        f, s, nb = d.process_logs(b"", 5, True)
        assert f.size == 0 and nb == 0 and d.stats()["lines"] == st0["lines"]
        f, s, nb = d.process_logs(frame([b"\x02\x01z", b"\x1a\x01\xff", b"\x1a\x03a\nb"]), 5, True)
        assert f.tolist() == [0, 0, 0] and nb == 3 and d.stats()["bad_records"] == 3 and d.stats()["train_lines"] == 0
        assert d.anomalies() == []
    g = Gen(seed=37, mutate=0.0, fuzz=0.0)
    _check_against_lines([g.record(b"type=A res=1", "1")[0]], 1, delimited=False)
    _check_against_lines([g.record(b"type=A res=1", "1")[0]], 0, delimited=False)
    _check_against_lines([b""], 0, delimited=False)
    # 64k records of the config-2 shape; more records than the walk grid has threads (4 CTAs per SM x 256)
    lines = _synth_lines(65536, seed=38)
    _check_against_lines(Gen(seed=38, mutate=0.02).records(lines), 30000, max_batch_bytes=24 << 20)
    short = [b"type=T%d res=%d" % (i % 7, i % 13) for i in range(200000)]
    _check_against_lines(Gen(seed=39, mutate=0.01, fuzz=0.2).records(short), 100000, max_batch_bytes=16 << 20)
    # one record with an 8 MiB log between short ones
    big = b"type=BIG exe=" + b"e" * (8 << 20) + b" res=x"
    recs = [g.record(t, str(i))[0] for i, t in enumerate([b"type=A res=1", big, b"type=B res=2", big[:100]])]
    _check_against_lines(recs, 1, max_batch_bytes=24 << 20)


# ------------------------------------------------------------------------------------------ reference service
def _reference_src():
    from oracle.ref_engine import reference_path
    return reference_path()


@pytest.mark.skipif(_reference_src() is None, reason="the reference service is not in oracle/_ref (make -C oracle ref)")
def test_reference_service_reader_to_fused_detector(tmp_path, ipc_dir, monkeypatch):
    """reader -> fused parser + detector: the unmodified reference Service loads the component with input_format
    log_schema and the docs' nginx log_format, and is fed one LogSchema per message over its socket."""
    import yaml
    from detectmateservice_b200.compat import install_shims
    monkeypatch.syspath_prepend(_reference_src())
    install_shims()
    import pynng
    from service.core import Service
    from service.settings import ServiceSettings

    cfg_file = tmp_path / "detector_config.yaml"
    cfg_file.write_text(yaml.safe_dump({"detectors": {"B200NewValueDetector": {
        "method_type": "new_value_detector", "data_use_training": 2, "auto_config": False,
        "params": {"input_format": "log_schema", "log_format": NGINX},
        "global": {"global_instance": {"header_variables": [{"pos": "URL"}]}}}}}))
    addr = f"ipc://{ipc_dir}/fused.ipc"
    settings = ServiceSettings(component_type="detectmateservice_b200.component.B200NewValueDetector",
                               component_name="b200-fused", engine_addr=addr, config_file=cfg_file,
                               log_dir=tmp_path / "logs", log_to_file=False, log_to_console=False,
                               http_port=18233, engine_autostart=False)
    svc = Service(settings=settings)
    svc.start()
    try:
        with pynng.Pair0(dial=addr, recv_timeout=2000) as c:
            time.sleep(0.2)
            for i, url in enumerate(("/hello", "/world", "/foobar")):
                line = '172.18.0.1 - - [18/Mar/2026:15:39:43 +0000] "GET %s HTTP/1.1" 404 162 "-" "curl/8.5.0"\n' % url
                c.send(wire.encode_log_schema({"__version__": "1.0.0", "logID": "reader-%d" % i, "log": line,
                                               "logSource": "/var/log/nginx/access.log", "hostname": "web"}))
                if i < 2:
                    c.recv_timeout = 500
                    with pytest.raises(pynng.Timeout):
                        c.recv()
                else:
                    c.recv_timeout = 5000
                    alert = wire.decode_detector_schema(c.recv())
                    assert alert["alertsObtain"] == {"Global - URL": "Unknown value: '/foobar'"}
                    assert alert["logIDs"] == ["reader-2"]
    finally:
        svc.stop()
    assert svc.library_component.det.stats()["lines"] == 3
    svc.library_component.close()
