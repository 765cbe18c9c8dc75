"""DetectorSchema alerts of LogSchema and ParserSchema batches encoded on the device (DESIGN.md R-alert) through the
real library: every reply must come out byte for byte as the component's host encoder writes it for the same batch, for
both components, in key=value and log_format mode, and the handle must encode whichever kind of batch came last.
Needs an H100."""
import os

import pytest

from detectmateservice_b200 import wire
from detectmateservice_b200.synth import MONITORED_KEYS, AuditSynth
from test_gpu_alerts import NOW, _pair, _run

pytestmark = pytest.mark.gpu

AUDIT = "type=<type> msg=audit(<Time>): <Content>"


def _lines(seed, n, rate):
    return AuditSynth(seed=seed, anomaly_rate=rate).batch(n, inject=rate > 0)[0].rstrip(b"\n").split(b"\n")


def _logs(lines, base=0):
    return wire.frame_delimited([wire.encode_log_schema({"__version__": "1.0.0", "logID": "id-%d" % (base + i),
                                                         "log": ln.decode(), "logSource": "/var/log/audit/audit.log"})
                                 for i, ln in enumerate(lines)])


def _records(lines, keys, base=0):
    recs = []
    for i, ln in enumerate(lines):
        f = dict(t.split("=", 1) for t in ln.decode().split(" ") if "=" in t)
        lfv = {k: f[k] for k in keys if k in f}
        if f.get("msg", "").startswith("audit("):
            lfv["Time"] = f["msg"][6:].split(":")[0]
        rec = {"EventID": i % 3, "variables": [f.get("type", ""), f.get("res", "")], "logFormatVariables": lfv}
        if i % 11:
            rec["logID"] = "id-%d" % (base + i)
        recs.append(wire.encode_parser_schema(rec))
    return wire.frame_delimited(recs)


def _cfg(fmt, n_train, cls="B200NewValueDetector", scope=None, **params):
    return {"detectors": {cls: {"method_type": "new_value_detector", "data_use_training": n_train, "auto_config": False,
                                "params": dict(params, input_format=fmt),
                                "global": scope or {"g": {"header_variables": [{"pos": k} for k in MONITORED_KEYS]}}}}}


@pytest.mark.parametrize("fmt", ["log_schema_batch", "parser_schema_batch"])
def test_64k_batches_at_ten_percent(fmt):
    make = _logs if fmt == "log_schema_batch" else (lambda ls, base=0: _records(ls, MONITORED_KEYS, base))
    dev_c, host_c = _pair(_cfg(fmt, 65536), overlap=False)
    dev = _run(dev_c, host_c, [make(_lines(41, 65536, 0)), make(_lines(42, 65536, 1e-1), 1 << 20)])
    assert dev.encoded == 1 and dev.declined == 0 and dev_c.n_alerts > 5000
    dev_c.close()
    host_c.close()


@pytest.mark.parametrize("fmt", ["log_schema_batch", "parser_schema_batch"])
def test_combinations(fmt):
    scope = {"c1": {"header_variables": [{"pos": "type"}, {"pos": "acct"}]}, "c2": {"header_variables": [{"pos": "exe"}]},
             "c3": {"header_variables": [{"pos": "res"}, {"pos": "type"}]}}
    if fmt == "parser_schema_batch":
        scope["c4"] = {"header_variables": [{"pos": "acct"}], "variables": [{"pos": 1, "name": "res"}]}
    make = _logs if fmt == "log_schema_batch" else (lambda ls, base=0: _records(ls, ["type", "acct", "exe", "res"], base))
    dev_c, host_c = _pair(_cfg(fmt, 8192, "B200NewValueComboDetector", scope), combo=True, overlap=False)
    dev = _run(dev_c, host_c, [make(_lines(43, 8192, 0)), make(_lines(44, 20000, 5e-2))])
    assert dev.encoded == 1 and dev.declined == 0 and dev_c.n_alerts > 100
    dev_c.close()
    host_c.close()


@pytest.mark.parametrize("combo", [False, True])
def test_log_schema_log_format(golden_dir, combo):
    from test_format_combos import AUDIT_COMBO_CFG, AUDIT_TAIL
    params = {"input_format": "log_schema_batch", "log_format": AUDIT,
              "path_templates": os.path.join(golden_dir, "audit_templates.txt"),
              "remove_spaces": True, "remove_punctuation": True, "lowercase": True}
    if combo:
        cfg = {"detectors": {"NewValueComboDetector": dict(AUDIT_COMBO_CFG["detectors"]["NewValueComboDetector"],
                                                           params=params)}}
    else:
        cfg = _cfg("log_schema_batch", 250, scope={"g": {"header_variables": [{"pos": "type"}, {"pos": "Content"}]}},
                   **{k: v for k, v in params.items() if k != "input_format"})
        cfg["detectors"]["B200NewValueDetector"]["events"] = {
            0: {"pam": {"variables": [{"pos": 5, "name": "acct"}, {"pos": 6, "name": "exe"}, {"pos": 10, "name": "res"}]}}}
    lines = open(os.path.join(golden_dir, "audit_sample.log"), "rb").read().rstrip(b"\n").split(b"\n")
    dev_c, host_c = _pair(cfg, combo=combo, overlap=False)
    dev = _run(dev_c, host_c, [_logs(lines[:250]), _logs(lines[250:] + AUDIT_TAIL.split(b"\n"), 250)])
    assert dev.encoded == 1 and dev.declined == 0 and dev_c.n_alerts > 3
    dev_c.close()
    host_c.close()


def test_last_batch_switches_between_inputs():
    """Raw lines after a LogSchema batch, LogSchema after raw lines, ParserSchema in between: each encode words the
    batch that came last."""
    dev_c, host_c = _pair(_cfg("raw_lines", 4096), overlap=True)
    train = _lines(45, 4096, 0)
    _run(dev_c, host_c, [b"\n".join(train) + b"\n"])
    steps = [("log_schema_batch", _logs(_lines(46, 3000, 1e-1))), ("raw_lines", b"\n".join(_lines(47, 3000, 1e-1)) + b"\n"),
             ("log_schema_batch", _logs(_lines(48, 3000, 1e-1), 9000)),
             ("parser_schema_batch", _records(_lines(49, 3000, 1e-1), MONITORED_KEYS)),
             ("raw_lines", b"\n".join(_lines(50, 3000, 1e-1)) + b"\n")]
    for fmt, msg in steps:
        dev_c.input_format = host_c.input_format = fmt
        _run(dev_c, host_c, [msg])
    assert dev_c._det.encoded == 5 and dev_c._det.declined == 0
    dev_c.close()
    host_c.close()
