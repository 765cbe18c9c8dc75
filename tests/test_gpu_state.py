"""Learnt state across restarts on the H100 (params.state_path, DESIGN.md R-state): the device export of the known set,
and components restarted from their state file replying byte for byte what one uninterrupted component replies."""
import json
import os
import random

import numpy as np
import pytest

from detectmateservice_b200 import state as S
from detectmateservice_b200 import wire
from oracle import fingerprint
from oracle.native import NativeOracle

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CLOCK = 1773848383
AUDIT = "type=<type> msg=audit(<Time>): <Content>"


# ---------------------------------------------------------------------------------------------- the device export
def test_export_of_a_2_24_slot_table_at_half_load():
    from detectmateservice_b200.detector import DeviceDetector
    rng = np.random.default_rng(24)
    keys = np.unique(rng.integers(1, 2**64 - 1, size=(1 << 23) + 4096, dtype=np.uint64, endpoint=True))
    keys = keys[keys != 0][: 1 << 23]
    rng.shuffle(keys)
    with DeviceDetector([b"a"], max_batch_bytes=1 << 20, table_log2_slots=24) as det:
        det.import_known(keys)
        got = det.export_known()
        assert got.dtype == np.uint64 and np.array_equal(got, np.sort(keys))
        assert det.stats()["known_keys"] == keys.size
        det.reset()
        assert det.export_known().size == 0
        det.import_known(keys[:1])
        assert det.export_known().tolist() == [int(keys[0])]


def test_export_after_training_equals_the_oracle():
    from detectmateservice_b200.detector import DeviceDetector
    from detectmateservice_b200.synth import AuditSynth, MONITORED_KEYS
    g = AuditSynth(seed=77)
    keys = [k.encode() for k in MONITORED_KEYS]
    o = NativeOracle(keys)
    with DeviceDetector(keys, max_batch_bytes=32 << 20, table_log2_slots=22) as det:
        for _ in range(3):
            msg, _ = g.batch(65536, inject=True)
            det.process_lines(msg, 65536)
            o.process(msg, 65536)
        want = sorted(fingerprint.table_key(i, v) for i in range(len(keys)) for v in o.known_values(i))
        assert det.export_known().tolist() == want


# ---------------------------------------------------------------------------------------------- restart parity
def _audit_lines():
    lines = open(os.path.join(GOLDEN, "audit_sample.log"), "rb").read().splitlines()
    r = random.Random(5)
    novel = []
    for i in range(60):                                     # detection lines with values training never saw
        ln = r.choice(lines[200:])
        for old, new in ((b'acct="root"', b'acct="u%d"' % i), (b"res=success", b"res=fail%d" % (i % 7)),
                         (b"type=USER_ACCT", b"type=USER_X%d" % (i % 5))):
            if r.random() < 0.5:
                ln = ln.replace(old, new)
        novel.append(ln)
    return lines[:240], lines[240:] + novel


def _chunks(items, n):
    k = (len(items) + n - 1) // n
    return [items[i:i + k] for i in range(0, len(items), k)]


def _raw_case():
    train, detect = _audit_lines()
    msgs = lambda ls: [b"".join(l + b"\n" for l in c) for c in _chunks(ls, 2)]
    cfg = {"global": {"t": {"header_variables": [{"pos": "type"}]},
                      "u": {"header_variables": [{"pos": "acct"}, {"pos": "res"}]}}}
    return cfg, {}, msgs(train), msgs(detect), len(train)


def _format_case():
    train, detect = _audit_lines()
    msgs = lambda ls: [b"".join(l + b"\n" for l in c) for c in _chunks(ls, 2)]
    cfg = {"global": {"type": {"header_variables": [{"pos": "type"}]}},
           "events": {0: {"pam": {"variables": [{"pos": 5, "name": "acct"}, {"pos": 10, "name": "res"}]}},
                      2: {"login": {"variables": [{"pos": 3, "name": "auid"}, {"pos": 7, "name": "res"}]}}}}
    params = {"log_format": AUDIT, "path_templates": os.path.join(GOLDEN, "audit_templates.txt"),
              "remove_spaces": True, "remove_punctuation": True, "lowercase": True}
    return cfg, params, msgs(train), msgs(detect), len(train)


def _parser_schema_case():
    r = random.Random(9)
    vocab = [["v%d_%d" % (p, j) for j in range(6)] for p in range(4)]

    def rec(i, novel):
        eid = r.randrange(2)
        variables = [r.choice(vocab[p]) for p in range(4)]
        typ = r.choice(["A", "B", "C"])
        if novel and r.random() < 0.4:
            variables[r.randrange(4)] = "new%d" % r.randrange(30)
        if novel and r.random() < 0.1:
            typ = "T%d" % r.randrange(5)
        return wire.encode_parser_schema({"EventID": eid, "logID": "id%d" % i, "variables": variables,
                                          "logFormatVariables": {"type": typ, "Time": str(1642723741 + i)}})
    train = [rec(i, False) for i in range(300)]
    detect = [rec(300 + i, True) for i in range(400)]
    cfg = {"global": {"t": {"header_variables": [{"pos": "type"}]}},
           "events": {0: {"e0": {"header_variables": [{"pos": "type"}], "variables": [{"pos": 1, "name": "x"}]}},
                      1: {"e1": {"variables": [{"pos": 0, "name": "y"}, {"pos": 3, "name": "z"}]}}}}
    msgs = lambda rs: [wire.frame_delimited(c) for c in _chunks(rs, 2)]
    return cfg, {"input_format": "parser_schema_batch"}, msgs(train), msgs(detect), len(train)


def _log_schema_case():
    train, detect = _audit_lines()
    recs = lambda ls, base: [wire.encode_log_schema({"logID": "L%d" % (base + i), "log": l.decode()})
                             for i, l in enumerate(ls)]
    msgs = lambda rs: [wire.frame_delimited(c) for c in _chunks(rs, 2)]
    cfg = {"global": {"t": {"header_variables": [{"pos": "type"}]},
                      "u": {"header_variables": [{"pos": "acct"}, {"pos": "res"}]}}}
    return cfg, {"input_format": "log_schema_batch"}, msgs(recs(train, 0)), msgs(recs(detect, 1000)), len(train)


CASES = {"raw": _raw_case, "format": _format_case, "parser_schema": _parser_schema_case, "log_schema": _log_schema_case}
CLASSES = {"B200NewValueDetector": "new_value_detector", "B200NewValueComboDetector": "new_value_combo_detector"}


def _config(cls, case_cfg, params, training, state_path=None, **extra):
    p = dict(params, max_batch_bytes=4 << 20, table_log2_slots=16, **extra)
    if state_path is not None:
        p["state_path"] = str(state_path)
    name = cls[4:]
    return {"detectors": {name: dict(case_cfg, method_type=CLASSES[cls], data_use_training=training, params=p)}}


def _comp(cls, cfg):
    from detectmateservice_b200 import component
    c = getattr(component, cls)(config=cfg)
    c.clock = lambda: CLOCK
    return c


def _run(c, msgs):
    return [c.process(m) for m in msgs]


@pytest.mark.parametrize("cls", list(CLASSES))
@pytest.mark.parametrize("case", list(CASES))
def test_restart_replies_byte_for_byte(tmp_path, case, cls):
    case_cfg, params, train, detect, n_train = CASES[case]()
    path = tmp_path / "state.bin"
    a = _comp(cls, _config(cls, case_cfg, params, n_train))
    assert _run(a, train) == [None] * len(train)
    want = _run(a, detect)
    assert any(w is not None for w in want) and a.n_alerts > 0

    b = _comp(cls, _config(cls, case_cfg, params, n_train, path))
    _run(b, train)
    saved = S.read_state(str(path))                          # written by the message that ended training
    assert saved[0]["n_seen"] == n_train and saved[0]["component"] == cls
    b.close()

    c = _comp(cls, _config(cls, case_cfg, params, n_train, path))
    assert c.n_seen == n_train
    got = _run(c, detect)
    assert got == want
    assert (c.n_seen, c.n_alerts) == (a.n_seen, a.n_alerts)
    assert np.array_equal(c.det.export_known(), a.det.export_known())
    assert c.det.stats()["known_keys"] == a.det.stats()["known_keys"]
    c.close()
    assert S.read_state(str(path))[0]["n_alerts"] == a.n_alerts     # close() saved the alerts counted since
    a.close()


@pytest.mark.parametrize("cls", list(CLASSES))
def test_restart_in_the_middle_of_training(tmp_path, cls):
    case_cfg, params, train, detect, n_train = _format_case()
    path = tmp_path / "state.bin"
    a = _comp(cls, _config(cls, case_cfg, params, n_train))
    _run(a, train)
    want = _run(a, detect)
    b = _comp(cls, _config(cls, case_cfg, params, n_train, path))
    _run(b, train[:1])
    b.close()
    c = _comp(cls, _config(cls, case_cfg, params, n_train, path))
    assert 0 < c.n_seen < n_train
    assert _run(c, train[1:]) == [None] * (len(train) - 1)
    assert np.array_equal(c.det.export_known(), a.det.export_known())
    assert _run(c, detect) == want
    a.close()
    c.close()


def test_changed_monitors_train_from_scratch_and_geometry_does_not(tmp_path):
    cls = "B200NewValueDetector"
    case_cfg, params, train, detect, n_train = _raw_case()
    path = tmp_path / "state.bin"
    b = _comp(cls, _config(cls, case_cfg, params, n_train, path))
    _run(b, train)
    b.close()
    # geometry: a larger table and batch load the state
    a = _comp(cls, _config(cls, case_cfg, params, n_train))
    _run(a, train)
    want = _run(a, detect)
    geo = _config(cls, case_cfg, params, n_train, path)
    geo["detectors"]["NewValueDetector"]["params"].update(table_log2_slots=18, max_batch_bytes=8 << 20)
    c = _comp(cls, geo)
    assert c.n_seen == n_train
    assert _run(c, detect) == want
    c.close()
    # other monitors: training starts again, and the file is replaced when that window ends
    other = {"global": {"t": {"header_variables": [{"pos": "type"}, {"pos": "exe"}]}}}
    d = _comp(cls, _config(cls, other, params, n_train, path))
    assert d.n_seen == 0
    before = open(path, "rb").read()
    _run(d, train[:1])
    assert open(path, "rb").read() == before
    _run(d, train[1:])
    hdr, keys = S.read_state(str(path))
    assert hdr["n_seen"] == n_train and hdr["key_signature"]["monitors"][1][2] == "exe"
    assert np.array_equal(keys, d.det.export_known())
    d.close()
    a.close()


# ---------------------------------------------------------------------------------------------- the reference service
def _reference_src():
    from oracle.ref_engine import reference_path
    return reference_path()


@pytest.mark.skipif(_reference_src() is None, reason="the reference service is not in oracle/_ref (make -C oracle ref)")
def test_reference_service_restarts_with_its_state(tmp_path, ipc_dir, monkeypatch):
    """The unmodified reference Service on the component-loader route: the first service trains and shuts down; a
    second one with the same configuration alerts on the detection record with no training record sent."""
    import time
    import yaml
    from detectmateservice_b200.compat import install_shims
    monkeypatch.syspath_prepend(_reference_src())
    install_shims()
    import pynng
    from service.core import Service
    from service.settings import ServiceSettings

    g = json.load(open(os.path.join(GOLDEN, "docs_golden.json")))
    det_cfg = dict(g["config"]["detectors"]["NewValueDetector"])
    det_cfg["params"] = dict(det_cfg.get("params") or {}, state_path=str(tmp_path / "state.bin"))
    cfg_file = tmp_path / "detector_config.yaml"
    cfg_file.write_text(yaml.safe_dump({"detectors": {"B200NewValueDetector": det_cfg}}))
    recs = [wire.encode_parser_schema({"EventID": 0, "logID": f"id{i}", "logFormatVariables": {"URL": u}})
            for i, u in enumerate(g["urls"])]
    n_train = int(det_cfg["data_use_training"])

    def service(i):
        addr = f"ipc://{ipc_dir}/svc{i}.ipc"
        settings = ServiceSettings(component_type="detectmateservice_b200.component.B200NewValueDetector",
                                   component_name=f"b200-state-{i}", engine_addr=addr, config_file=cfg_file,
                                   log_dir=tmp_path / "logs", log_to_file=False, log_to_console=False,
                                   http_port=18241 + i, engine_autostart=False)
        return Service(settings=settings), addr

    svc, addr = service(0)
    svc.start()
    try:
        with pynng.Pair0(dial=addr, recv_timeout=500) as c:
            time.sleep(0.2)
            for r in recs[:n_train]:
                c.send(r)
                with pytest.raises(pynng.Timeout):
                    c.recv()
    finally:
        svc.stop()
    assert S.read_state(str(tmp_path / "state.bin"))[0]["n_seen"] == n_train
    svc.library_component.close()

    svc, addr = service(1)
    assert svc.library_component.n_seen == n_train
    svc.start()
    try:
        with pynng.Pair0(dial=addr, recv_timeout=5000) as c:
            time.sleep(0.2)
            c.send(recs[n_train])
            alert = wire.decode_detector_schema(c.recv())
            assert alert["alertsObtain"] == g["expected"]["alertsObtain"] and alert["alertID"] == "10"
    finally:
        svc.stop()
    svc.library_component.close()
