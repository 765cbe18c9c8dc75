"""DetectorSchema alerts of pipelined raw-line messages (component._detect_pipelined), CPU tier: a stand-in for the
library's two-slot path on the CPU emulator, whose collect() runs the piece's emulated stream kernel and makes it the
last batch, which encode_alerts() then words with the encoder kernels.  Every reply, n_alerts and n_seen must equal
those of the same component with the host encoder on the same emulated detection."""
import pytest

from detectmateservice_b200.synth import MONITORED_KEYS, AuditSynth
from test_emu_alerts import NOW, EmuDevice, _cfg, _run

PIECE = 16 << 10                                                     # messages of 48 KiB and more are pipelined


@pytest.fixture(scope="module")
def lib():
    import emu_harness
    return emu_harness.lib()


class EmuPipelined(EmuDevice):
    """EmuDevice with submit / collect / collect_anomalies.  As in the library, submit() leaves no last batch (the
    encoder then refuses), collect() makes the slot's batch the last one, and a slot is collected before it is
    submitted again.  Records each collected piece's anomalous records and the anomaly lists the component fetched."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self._slots = [None, None]
        self._last_slot = None                                       # the slot collected last, while it is the last batch
        self._has_batch = False
        self.collected, self.fetched = [], 0
        self.piece_encoded = self.piece_declined = 0                 # encoder calls on collected pieces

    def process_lines(self, buf, n_train_lines=0, copy=True):
        out = super().process_lines(buf, n_train_lines, copy)
        self._has_batch, self._last_slot = True, None
        return out

    def submit(self, buf, n_train_lines=0, slot=0):
        assert self._slots[slot] is None, "slot submitted twice without a collect"
        self._slots[slot] = (bytes(buf), n_train_lines)
        self._has_batch = False

    def collect(self, slot=0):
        buf, n_train = self._slots[slot]
        self._slots[slot] = None
        f, s = self.process_lines(buf, n_train)
        self._last_slot = slot
        self.collected.append(self.last_n_anomalies)
        return f, s

    def collect_anomalies(self, slot=0, cap=1 << 20):
        assert slot == self._last_slot, "the emulated handle keeps the anomaly list of the slot collected last only"
        self.fetched += 1
        return self.det.anomalies()

    def encode_alerts(self, first_log_id, first_alert_id, now):
        if not self._has_batch:
            raise RuntimeError("no last batch")                      # dm_encode_alerts: DM_ERR_STATE
        r = super().encode_alerts(first_log_id, first_alert_id, now)
        if self._last_slot is not None:
            self.piece_encoded += r is not None
            self.piece_declined += r is None
        return r


class HostPipelined:
    """The same emulated detection without the encoder: the component words every piece on the host."""

    def __init__(self, dev):
        self._d = dev

    def __getattr__(self, name):
        if name in ("encode_alerts", "set_alert_format"):
            raise AttributeError(name)
        return getattr(self._d, name)


def _pair(lib, cfg, alerts_min=None, piece=PIECE, capacity=1 << 20, variant="stream"):
    from detectmateservice_b200.component import B200NewValueDetector
    comps = []
    for host in (False, True):
        c = B200NewValueDetector(config=cfg)
        dev = EmuPipelined(lib, [m.key for m in c.monitors], variant, capacity=capacity)
        c._det = HostPipelined(dev) if host else dev
        c.PIPE_PIECE_BYTES, c.PIPE_MIN_BYTES = piece, 3 * piece
        if alerts_min is not None:
            c.DEVICE_ALERTS_MIN = alerts_min
        c.clock = lambda: NOW
        comps.append(c)
    return comps


def _check_split(dev, alerts_min):
    """Every piece at or above the threshold went to the encoder; the host fetched the anomaly lists of the others and of
    those the encoder declined, and no more."""
    big = sum(1 for a in dev.collected if a >= alerts_min)
    small = sum(1 for a in dev.collected if 0 < a < alerts_min)
    assert dev.piece_encoded + dev.piece_declined == big
    assert dev.fetched == small + dev.piece_declined


@pytest.mark.parametrize("rate", [1e-3, 1e-2, 1e-1, 3e-1])
@pytest.mark.parametrize("variant", ["stream", "chain"])
def test_anomaly_rates(lib, rate, variant):
    g = AuditSynth(seed=41, anomaly_rate=rate)
    train, _ = g.batch(1024, inject=False)
    msgs = [g.batch(n, inject=True)[0] for n in (300, 420)]         # 75 and 105 KiB: 5 and 6 pieces
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 1024, start_id=-7), alerts_min=1, variant=variant)
    dev = _run(dev_c, host_c, [train] + msgs)
    assert len(dev.collected) == 11
    _check_split(dev, 1)
    assert dev.declined == 0 and dev.fetched == 0
    if rate >= 1e-2:
        assert dev.encoded >= 3 and dev_c.n_alerts > 3


def test_pieces_on_both_sides_of_the_threshold(lib):
    """The threshold applies per piece: in one message some pieces go to the device and some stay on the host, and the
    alert numbers run on across them."""
    from detectmateservice_b200.component import B200NewValueDetector
    k = B200NewValueDetector.DEVICE_ALERTS_MIN
    g = AuditSynth(seed=42, anomaly_rate=1e-1)
    train, _ = g.batch(1024, inject=False)
    msgs = [g.batch(384, inject=True)[0] for _ in range(3)]
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 1024))
    dev = _run(dev_c, host_c, [train] + msgs)
    _check_split(dev, k)
    assert dev.encoded >= 2 and 0 < sum(1 for a in dev.collected if 0 < a < k)


def test_declined_piece_amid_encoded_ones(lib):
    """A Time string outside the device's grammar declines its piece, which the host words; the pieces around it stay on
    the device."""
    g = AuditSynth(seed=43, anomaly_rate=1e-1)
    train, _ = g.batch(1024, inject=False)
    body = g.batch(384, inject=True)[0].split(b"\n")
    body[160:160] = [b"type=NOVEL_D%d acct=x msg=audit(1e5:1) res=ok" % i for i in range(3)]     # amid the third piece
    msg = b"\n".join(body)
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 1024), alerts_min=1)
    dev = _run(dev_c, host_c, [train, msg])
    _check_split(dev, 1)
    assert dev.declined == 1 and dev.encoded >= 4


def test_lookalikes_and_duplicate_keys(lib):
    """Quoted look-alikes, duplicate keys (the first true field wins), a key after a single quote, values of ill-formed
    UTF-8, '\\r', records without the field -- across piece boundaries."""
    keys = ["type", "acct", "exe", "res"]
    train = b"".join(b"type=A acct=u%d exe=/bin/x res=ok msg=audit(1.5:1)\n" % (i % 4) for i in range(64))
    recs = []
    for i in range(1500):
        recs.append([b'type=NEW%d acct="x type=Q" type=DUP exe=/bin/x res=ok' % i,
                     b'x="a type=HIDDEN%d" type=A acct=u1 res=ok' % i,
                     b"'type=QUOTE' acct=new%d res=ok msg=audit(1700000000.123:9):" % i,
                     b"type=\xff\xfe\xc3 acct=\xe2\x82%d res=\xed\xa0\x80\xf0\x9f\x98\x80 msg=audit(0:1)" % i,
                     b'type=A exe="/usr/bin/a b%d" res=fail\r' % i,
                     b"type=A acct=u0 res=ok pad=" + b"y" * (i % 97)][i % 6])
    msg = b"\n".join(recs) + b"\n"
    assert len(msg) > 3 * PIECE
    dev_c, host_c = _pair(lib, _cfg(keys, 64), alerts_min=1)
    dev = _run(dev_c, host_c, [train, msg])
    _check_split(dev, 1)
    assert dev.encoded >= 3 and dev.declined == 0 and dev_c.n_alerts == 1000


def test_message_larger_than_max_batch_bytes(lib):
    """The chunked path: each chunk of max_batch_bytes is pipelined on its own, numbering carried over."""
    g = AuditSynth(seed=44, anomaly_rate=5e-2)
    train, _ = g.batch(1024, inject=False)
    big, _ = g.batch(1000, inject=True)                              # 250 KB: chunks of at most 100 KB
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 1024, max_batch_bytes=100_000), alerts_min=1)
    dev = _run(dev_c, host_c, [train, big, big])
    _check_split(dev, 1)
    assert len(dev.collected) >= 10 and dev.encoded >= 8


def test_training_message_then_pipelined_ones(lib):
    """A message that trains goes through one call, even when large; the pipelined messages after it are numbered from
    where it ended."""
    g = AuditSynth(seed=45, anomaly_rate=1e-1)
    first = g.batch(512, inject=False)[0] + g.batch(256, inject=True)[0]      # trains on its first 512 records
    msgs = [g.batch(256, inject=True)[0] for _ in range(2)]
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 512, start_id=100), alerts_min=1)
    dev = _run(dev_c, host_c, [first] + msgs)
    assert len(dev.collected) == 8 and dev.piece_encoded >= 7 and dev.encoded == dev.piece_encoded + 1
    _check_split(dev, 1)
    assert dev_c.n_seen == 512 + 256 * 3


def test_one_record_message_is_bare(lib):
    """A pipelined message of one record replies with its DetectorSchema alone, as a one-record message always does."""
    from detectmateservice_b200 import wire
    train = b"type=A acct=u msg=audit(7.5:1)\n"
    rec = b"type=LONE acct=u msg=audit(1642723741.5:3) pad=" + b"z" * 3000 + b"\n"
    dev_c, host_c = _pair(lib, _cfg(["type", "acct"], 1), alerts_min=1, piece=512)
    dev = _run(dev_c, host_c, [train, rec])
    assert dev.encoded == 1
    out = dev_c.process(b"type=LONE2 acct=u2 pad=" + b"w" * 3000)               # (no final '\n')
    assert out == host_c.process(b"type=LONE2 acct=u2 pad=" + b"w" * 3000)
    alert = wire.decode_detector_schema(out)
    assert alert["logIDs"] == ["2"] and alert["extractedTimestamps"] == [NOW] and dev.encoded == 2


def test_small_output_buffer_declines_one_piece(lib):
    """A piece whose alerts do not fit the output buffer is declined and worded on the host; the sparse pieces around it
    still fit."""
    g = AuditSynth(seed=46, anomaly_rate=3e-2)
    train, _ = g.batch(1024, inject=False)
    g_dense = AuditSynth(seed=46, anomaly_rate=1.0)
    msg = g.batch(160, inject=True)[0] + g_dense.batch(48, inject=True)[0] + g.batch(176, inject=True)[0]
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 1024), alerts_min=1, capacity=6000)
    dev = _run(dev_c, host_c, [train, msg])
    _check_split(dev, 1)
    assert dev.declined >= 1 and dev.encoded >= 1


def test_compact_output_is_unchanged(lib):
    g = AuditSynth(seed=47, anomaly_rate=1e-1)
    train, _ = g.batch(1024, inject=False)
    msg, _ = g.batch(384, inject=True)
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 1024, output_format="compact"), alerts_min=1)
    dev = _run(dev_c, host_c, [train, msg])
    assert len(dev.collected) == 6 and dev.encoded == dev.declined == dev.fetched == 0


def test_failed_piece_leaves_no_slot_in_flight(lib):
    """An error while a piece is encoded fails the message, leaves no slot in flight and counts nothing: the next
    message runs and numbers as if the failed one had not come."""
    g = AuditSynth(seed=48, anomaly_rate=1e-1)
    train, _ = g.batch(1024, inject=False)
    msg, _ = g.batch(384, inject=True)
    dev_c, host_c = _pair(lib, _cfg(MONITORED_KEYS, 1024), alerts_min=1)
    dev = _run(dev_c, host_c, [train])

    def fail(*a):
        raise RuntimeError("encoder failed")
    dev.encode_alerts = fail
    with pytest.raises(RuntimeError):
        dev_c.process(msg)
    assert dev._slots == [None, None] and dev_c.n_alerts == 0
    del dev.encode_alerts
    _run(dev_c, host_c, [msg])
    assert dev.piece_encoded == 6
