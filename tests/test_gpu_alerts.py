"""DetectorSchema alerts encoded on the device (DESIGN.md R-alert) through the real library: every message must come out
byte for byte as the component's host encoder writes it for the same batch, on every key=value kernel, with overlapping
launches, for both components.  Needs an H100."""
import os
import time

import pytest

from detectmateservice_b200 import wire
from detectmateservice_b200.synth import MONITORED_KEYS, AuditSynth

pytestmark = pytest.mark.gpu

NOW = 1773848383


class HostReference:
    """The real handle without its encoder: the component words the alerts on the host."""

    def __init__(self, det):
        self._d = det

    def __getattr__(self, name):
        if name in ("encode_alerts", "set_alert_format"):
            raise AttributeError(name)
        return getattr(self._d, name)


class Counting:
    """The real handle, counting the batches its encoder wrote and declined."""

    def __init__(self, det):
        self._d = det
        self.encoded = self.declined = 0

    def __getattr__(self, name):
        return getattr(self._d, name)

    def encode_alerts(self, *a):
        r = self._d.encode_alerts(*a)
        if r is None:
            self.declined += 1
        else:
            self.encoded += 1
        return r


def _pair(cfg, combo=False, overlap=True):
    from detectmateservice_b200.component import B200NewValueComboDetector, B200NewValueDetector
    cls = B200NewValueComboDetector if combo else B200NewValueDetector
    out = []
    for encoder in (True, False):
        c = cls(config=cfg)
        c.clock = lambda: NOW
        det = c.det
        if overlap:
            det.set_overlap(True)
        c._det = Counting(det) if encoder else HostReference(det)
        c.DEVICE_ALERTS_MIN = 1                                      # every batch with alerts goes to the encoder
        out.append(c)
    return out


def _run(dev_c, host_c, messages):
    for msg in messages:
        got, want = dev_c.process(msg), host_c.process(msg)
        assert got == want
        assert dev_c.n_alerts == host_c.n_alerts
    return dev_c._det


def _cfg(keys, n_train, **params):
    return {"detectors": {"B200NewValueDetector": {
        "method_type": "new_value_detector", "data_use_training": n_train, "auto_config": False, "params": params,
        "global": {"g": {"header_variables": [{"pos": k} for k in keys]}}}}}


LOOKALIKES = (b'type=NEW acct="x type=Q" type=DUP exe=/bin/x res=ok\n'
              b'x="a type=HIDDEN" type=A acct=u1 res=ok\n'
              b"'type=QUOTE' acct=new1 res=ok msg=audit(1700000000.123:9):\n"
              b"type=\xff\xfe\xc3 acct=\xe2\x82 res=\xed\xa0\x80\xf0\x9f\x98\x80 msg=audit(0:1)\n"
              b"type=A acct=u0 msg=audit(1e5:1) res=\xc0\xaf\n")


@pytest.mark.parametrize("kernel,recheck", [("stream", "thread"), ("stream", "chain"), ("lanes", None)])
def test_device_alerts_equal_host_alerts(monkeypatch, kernel, recheck):
    monkeypatch.setenv("DM_KERNEL", kernel)
    if recheck:
        monkeypatch.setenv("DM_STREAM_RECHECK", recheck)
    g = AuditSynth(seed=21, anomaly_rate=1e-1)
    train, _ = g.batch(8192, inject=False)
    # consecutive overlapped messages, each with its own anomalies, then one record alone, then look-alikes and a
    # Time string outside the device's grammar (declined: the host words that message)
    msgs = [train] + [g.batch(n, inject=True)[0] for n in (20000, 7000, 65536)]
    msgs += [b"type=ONLY msg=audit(1642723741.072:1): res=x\n", LOOKALIKES]
    dev_c, host_c = _pair(_cfg(MONITORED_KEYS, 8192, start_id=-3))
    dev = _run(dev_c, host_c, msgs)
    assert dev.encoded == 4 and dev.declined == 1 and dev_c.n_alerts > 9000
    dev_c.close()
    host_c.close()


def test_device_alerts_combinations():
    cfg = {"detectors": {"B200NewValueComboDetector": {
        "method_type": "new_value_combo_detector", "data_use_training": 4096, "auto_config": False, "params": {},
        "global": {"c1": {"header_variables": [{"pos": "type"}, {"pos": "acct"}]},
                   "c2": {"header_variables": [{"pos": "exe"}]},
                   "c3": {"header_variables": [{"pos": "res"}, {"pos": "type"}]}}}}}
    g = AuditSynth(seed=22, anomaly_rate=5e-2)
    msgs = [g.batch(4096, inject=False)[0]] + [g.batch(10000, inject=True)[0] for _ in range(2)]
    dev_c, host_c = _pair(cfg, combo=True)
    dev = _run(dev_c, host_c, msgs)
    assert dev.encoded == 2 and dev.declined == 0 and dev_c.n_alerts > 100
    dev_c.close()
    host_c.close()


def test_device_alerts_chunked_and_small_buffer():
    g = AuditSynth(seed=23, anomaly_rate=1e-1)
    train, _ = g.batch(4096, inject=False)
    big, _ = g.batch(40000, inject=True)
    dev_c, host_c = _pair(_cfg(MONITORED_KEYS, 4096, max_batch_bytes=1 << 20), overlap=False)
    dev = _run(dev_c, host_c, [train, big])
    assert len(big) > (3 << 20) and dev.encoded >= 4 and dev.declined == 0
    # an output buffer smaller than one batch's alerts: declined, and the host's bytes
    dev._d.set_alert_format("1.0.0", dev_c.detector_id, dev_c.method_type, dev_c._description(), dev_c._alert_keys(),
                            capacity=4096)
    out = dev_c.process(g.batch(20000, inject=True)[0])
    assert dev.declined >= 1 and len(out) > 4096
    dev_c.close()
    host_c.close()


def test_device_alerts_refused_after_other_inputs():
    from detectmateservice_b200 import _lib
    c = _pair(_cfg(["type"], 1), overlap=False)[0]
    c.process(b"type=A\n")
    det = c._det._d
    c.process(b"type=B\n")
    det.process_values([[(0, b"zz")]])
    with pytest.raises(_lib.DmError):
        det.encode_alerts(0, 0, NOW)
    c.close()


def test_device_resident_overlapped_batches_encode_their_own_alerts():
    """Device-resident messages enqueued back to back with overlap on: after each enqueue the encoder words that batch
    (the next dm_process_lines is enqueued only after dm_encode_alerts returned), equal to the host path's bytes."""
    import numpy as np
    import torch
    g = AuditSynth(seed=31, anomaly_rate=1e-1)
    train, _ = g.batch(4096, inject=False)
    msgs = [g.batch(n, inject=True)[0] for n in (9000, 3000, 12000)]
    dev_c, host_c = _pair(_cfg(MONITORED_KEYS, 4096), overlap=False)
    for c in (dev_c, host_c):
        c.process(train)
    det = dev_c._det._d
    det.set_overlap(True)
    det.set_alert_format("1.0.0", dev_c.detector_id, dev_c.method_type, dev_c._description(), dev_c._alert_keys())
    bufs = []
    for m in msgs:
        t = torch.zeros(len(m) + 64, dtype=torch.uint8, device="cuda")
        t[:len(m)] = torch.from_numpy(np.frombuffer(m, np.uint8).copy()).cuda()
        bufs.append(t)
    torch.cuda.synchronize()
    base, n_alerts = dev_c.n_seen, dev_c.n_alerts
    for m, t in zip(msgs, bufs):
        det.enqueue_device(t.data_ptr(), len(m))
        blob, count = det.encode_alerts(base, dev_c.start_id + n_alerts, NOW)
        want = host_c.process(m)
        assert blob == want and count == len(wire.split_delimited(want))
        base += m.count(b"\n")
        n_alerts += count
    dev_c.close()
    host_c.close()


AUDIT = "type=<type> msg=audit(<Time>): <Content>"


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("combo", [False, True])
def test_device_alerts_log_format(golden_dir, norm, combo):
    """log_format mode with the reference's audit templates (R-norm off / all three switches on), single monitors and
    combinations: header captures verbatim, template variables from the (normalised) Content, Time from <Time>."""
    params = {"log_format": AUDIT, "path_templates": os.path.join(golden_dir, "audit_templates.txt")}
    if norm:
        params.update(remove_spaces=True, remove_punctuation=True, lowercase=True)
    name = "NewValueComboDetector" if combo else "B200NewValueDetector"
    cfg = {"detectors": {name: {
        "method_type": "new_value_combo_detector" if combo else "new_value_detector", "data_use_training": 4096,
        "auto_config": False, "params": params,
        "global": {"g": {"header_variables": [{"pos": "type"}]}},
        "events": {0: {"pam": {"variables": [{"pos": 5, "name": "acct"}, {"pos": 6, "name": "exe"},
                                             {"pos": 10, "name": "res"}]}}}}}}
    g = AuditSynth(seed=24, anomaly_rate=1e-1)
    msgs = [g.batch(4096, inject=False)[0]] + [g.batch(n, inject=True)[0] for n in (20000, 5000)]
    msgs.append(b"type=NEWTYPE msg=audit(1e3): x\n")                 # a Time the device cannot convert: declined
    dev_c, host_c = _pair(cfg, combo=combo)
    dev = _run(dev_c, host_c, msgs)
    assert dev.encoded == 2 and dev.declined == 1 and dev_c.n_alerts > 50
    dev_c.close()
    host_c.close()


def _reference_src():
    from oracle.ref_engine import reference_path
    return reference_path()


@pytest.mark.skipif(_reference_src() is None, reason="the reference service is not in oracle/_ref (make -C oracle ref)")
def test_reference_service_nginx_alerts_from_the_device(tmp_path, ipc_dir, monkeypatch):
    """The docs' nginx example through the unmodified reference Service, raw lines in, its alert encoded on the device."""
    import yaml
    from detectmateservice_b200.compat import install_shims
    from detectmateservice_b200.component import B200NewValueDetector
    monkeypatch.syspath_prepend(_reference_src())
    monkeypatch.setattr(B200NewValueDetector, "DEVICE_ALERTS_MIN", 1)
    install_shims()
    import pynng
    from service.core import Service
    from service.settings import ServiceSettings
    nginx = '<IP> - - [<Time>] "<Method> <URL> <Protocol>" <Status> <Bytes> "<Referer>" "<UserAgent>"'
    cfg_file = tmp_path / "detector_config.yaml"
    cfg_file.write_text(yaml.safe_dump({"detectors": {"B200NewValueDetector": {
        "method_type": "new_value_detector", "data_use_training": 2, "auto_config": False,
        "params": {"input_format": "raw_lines", "log_format": nginx},
        "global": {"global_instance": {"header_variables": [{"pos": "URL"}]}}}}}))
    addr = f"ipc://{ipc_dir}/nginx.ipc"
    settings = ServiceSettings(component_type="detectmateservice_b200.component.B200NewValueDetector",
                               component_name="b200-nginx", engine_addr=addr, config_file=cfg_file,
                               log_dir=tmp_path / "logs", log_to_file=False, log_to_console=False,
                               http_port=18234, engine_autostart=False)
    svc = Service(settings=settings)
    svc.start()
    encoded = []
    try:
        comp = svc.library_component
        comp.clock = lambda: NOW
        real = comp.det
        comp._det = Counting(real)
        encoded.append(comp._det)
        with pynng.Pair0(dial=addr, recv_timeout=2000) as c:
            time.sleep(0.2)
            for i, url in enumerate(("/hello", "/world", "/foobar")):
                line = '172.18.0.1 - - [18/Mar/2026:15:39:43 +0000] "GET %s HTTP/1.1" 404 162 "-" "curl/8.5.0"\n' % url
                c.send(line.encode())
                if i < 2:
                    c.recv_timeout = 500
                    with pytest.raises(pynng.Timeout):
                        c.recv()
                else:
                    c.recv_timeout = 5000
                    alert = wire.decode_detector_schema(c.recv())
                    assert alert["alertsObtain"] == {"Global - URL": "Unknown value: '/foobar'"}
                    assert alert["logIDs"] == ["2"] and alert["extractedTimestamps"] == [NOW]
    finally:
        svc.stop()
    assert encoded[0].encoded == 1 and encoded[0].declined == 0
    svc.library_component.close()
