"""DetectorSchema alerts of pipelined raw-line messages (component._detect_pipelined) encoded on the device through the
real library: dm_collect makes each piece's slot the last batch and dm_encode_alerts words it before the slot is
submitted again.  Every reply must equal the host encoder's for the same message, and every piece at or above
DEVICE_ALERTS_MIN must have gone to the device encoder, so a silent host fallback cannot pass.  Needs an H100."""
import numpy as np
import pytest

from detectmateservice_b200.synth import MONITORED_KEYS, AuditSynth
from test_gpu_alerts import LOOKALIKES, NOW, Counting, HostReference, _cfg, _run

pytestmark = pytest.mark.gpu

PIECE = 4 << 20


class PipeCounting(Counting):
    """Counting, also recording the anomalous records of every collected piece."""

    def __init__(self, det):
        super().__init__(det)
        self.pieces = []

    def collect(self, slot=0):
        r = self._d.collect(slot)
        self.pieces.append(self._d.last_n_anomalies)
        return r


def _pair(cfg, piece=PIECE):
    from detectmateservice_b200.component import B200NewValueDetector
    out = []
    for encoder in (True, False):
        c = B200NewValueDetector(config=cfg)
        c.clock = lambda: NOW
        c._det = PipeCounting(c.det) if encoder else HostReference(c.det)
        if piece:
            c.PIPE_MIN_BYTES = c.PIPE_PIECE_BYTES = piece
        out.append(c)
    return out


def _close(*comps):
    for c in comps:
        c.close()


def _encoded_all_it_could(dev, k):
    """Every piece with at least k anomalous records went to the encoder, and no other."""
    assert dev.encoded + dev.declined == sum(1 for a in dev.pieces if a >= k)


@pytest.fixture(scope="module")
def messages():
    """Training records, then per record shape detection messages of ~20 MiB at rates 1e-3, 1e-2 and 1e-1, quoted
    look-alikes spread through the last."""
    g = AuditSynth(seed=51)
    out = {"train": g.batch(8192, inject=False)[0]}
    for shape in ("config2", "varlen"):
        msgs = []
        for rate in (1e-3, 1e-2, 1e-1):
            g.anomaly_rate = rate
            m = g.batch(80000, inject=True)[0] if shape == "config2" else g.batch_varlen(60000, inject=True)[0]
            msgs.append(m)
        lines = msgs[-1].split(b"\n")
        for i in range(1, 9):
            j = i * len(lines) // 9
            lines[j:j] = LOOKALIKES.replace(b"msg=audit(1e5:1) ", b"").rstrip(b"\n").split(b"\n")
        msgs[-1] = b"\n".join(lines)
        out[shape] = msgs
    return out


@pytest.mark.parametrize("shape", ["config2", "varlen"])
@pytest.mark.parametrize("recheck", ["thread", "chain", "auto"])
def test_pipelined_alerts_equal_host_alerts(monkeypatch, messages, recheck, shape):
    monkeypatch.setenv("DM_STREAM_RECHECK", recheck)
    dev_c, host_c = _pair(_cfg(MONITORED_KEYS, 8192, start_id=-3, max_batch_bytes=32 << 20))
    _run(dev_c, host_c, [messages["train"]])
    dev = _run(dev_c, host_c, messages[shape])
    assert all(len(m) >= 2 * PIECE for m in messages[shape]) and len(dev.pieces) >= 12
    _encoded_all_it_could(dev, dev_c.DEVICE_ALERTS_MIN)
    assert dev.declined == 0 and dev.encoded >= 8 and dev_c.n_seen == host_c.n_seen
    _close(dev_c, host_c)


def test_declined_piece_and_small_output_buffer(messages):
    """A Time string outside the device's grammar declines its piece alone; an output buffer too small for one dense
    piece declines that piece alone.  The host words both, and the reply is the host encoder's."""
    g = AuditSynth(seed=52, anomaly_rate=1e-3)
    sparse = [g.batch(16384, inject=True)[0] for _ in range(5)]           # 4 MiB each
    odd = b"".join(b"type=NOVEL_T%d acct=x msg=audit(1e5:1) res=ok\n" % i for i in range(20))
    msg = sparse[0] + sparse[1][:1 << 20] + odd + sparse[1][1 << 20:] + sparse[2]
    dev_c, host_c = _pair(_cfg(MONITORED_KEYS, 8192, max_batch_bytes=32 << 20))
    _run(dev_c, host_c, [messages["train"]])
    dev = _run(dev_c, host_c, [msg])
    _encoded_all_it_could(dev, dev_c.DEVICE_ALERTS_MIN)
    assert dev.declined == 1 and dev.encoded >= 1
    g.anomaly_rate = 0.5
    dense = g.batch(16384, inject=True)[0]
    dev.set_alert_format("1.0.0", dev_c.detector_id, dev_c.method_type, dev_c._description(), dev_c._alert_keys(),
                         capacity=64 << 10)
    dev.pieces, dev.encoded, dev.declined = [], 0, 0
    dev = _run(dev_c, host_c, [sparse[3] + dense + sparse[4]])
    _encoded_all_it_could(dev, dev_c.DEVICE_ALERTS_MIN)
    assert dev.declined == 1 and dev.encoded >= 1
    _close(dev_c, host_c)


def test_real_defaults():
    """The component's own constants: a 28 MiB message is cut into two pieces, both encoded on the device."""
    g = AuditSynth(seed=53, anomaly_rate=1e-2)
    train, _ = g.batch(8192, inject=False)
    msg, _ = g.batch(28 << 12, inject=True)                                # 28 MiB
    dev_c, host_c = _pair(_cfg(MONITORED_KEYS, 8192), piece=0)
    assert dev_c.max_batch_bytes == 64 << 20 and len(msg) >= dev_c.PIPE_MIN_BYTES == 24 << 20
    dev = _run(dev_c, host_c, [train, msg])
    assert len(dev.pieces) == 2 and dev.encoded == 2 and dev.declined == 0
    _close(dev_c, host_c)


def test_message_above_max_batch_bytes(messages):
    """Cut into max_batch_bytes chunks first, each of them pipelined; numbering runs on across chunks and pieces."""
    msg = b"".join(messages["config2"][:2])                                   # ~40 MiB
    dev_c, host_c = _pair(_cfg(MONITORED_KEYS, 8192, max_batch_bytes=16 << 20))
    dev = _run(dev_c, host_c, [messages["train"], msg])
    assert len(msg) > 32 << 20 and len(dev.pieces) >= 8
    _encoded_all_it_could(dev, dev_c.DEVICE_ALERTS_MIN)
    assert dev.encoded >= 5
    _close(dev_c, host_c)


def test_each_batch_words_its_own_alerts(messages):
    """A pipelined message, then a plain one: each reply is its own batch's.  encode_alerts then words the plain batch
    again; right after a submit it is refused; after the collect it words the collected slot."""
    from detectmateservice_b200 import _lib, wire
    dev_c, host_c = _pair(_cfg(MONITORED_KEYS, 8192, max_batch_bytes=32 << 20))
    plain = b"type=PLAIN%d res=x\n" % 1 + b"type=PLAIN2 res=y\n"
    dev = _run(dev_c, host_c, [messages["train"], messages["config2"][1], plain])
    assert dev.encoded >= 4
    det = dev._d
    blob, count = det.encode_alerts(0, 0, NOW)
    assert count == 2 and [wire.decode_detector_schema(b)["logIDs"] for b in wire.split_delimited(blob)] == [["0"], ["1"]]
    piece = np.frombuffer(messages["config2"][2][:1 << 20], np.uint8)
    det.submit(piece, 0, 0)
    with pytest.raises(_lib.DmError):
        det.encode_alerts(0, 0, NOW)
    det.collect(0)
    blob, count = det.encode_alerts(0, 0, NOW)
    assert count == det.last_n_anomalies == len(det.collect_anomalies(0)) > 0
    assert len(wire.split_delimited(blob)) == count
    _close(dev_c, host_c)
