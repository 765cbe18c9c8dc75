"""Buffers a handle allocates on first use and grows when a batch needs more (csrc/dm_buf.h), on the H100.

Each test runs the same calls on two handles with the same known set: on `grown` every buffer is already large enough,
because an earlier call of the same kind was large; on `fresh` the buffers grow in the middle of the sequence and the
calls after the growth are smaller again.  Every output must be byte for byte the same.  Detection only (no training),
so the known sets stay equal.  Needs an H100."""
import numpy as np
import pytest

from detectmateservice_b200 import _lib, wire
from detectmateservice_b200.synth import MONITORED_KEYS, AuditSynth

pytestmark = pytest.mark.gpu

KEYS = [k.encode() for k in MONITORED_KEYS]
SMALL, LARGE = 100, 20000          # LARGE is past the first allocation of every batch-sized buffer (4096 records)


def _lines(seed, n, rate=2e-2):
    return AuditSynth(seed=seed, anomaly_rate=rate).batch(n, inject=True)[0].rstrip(b"\n").split(b"\n")


def _logs(lines):
    return wire.frame_delimited([wire.encode_log_schema({"__version__": "1.0.0", "logID": "id-%d" % i, "log": ln.decode(),
                                                         "logSource": "/var/log/audit/audit.log"})
                                 for i, ln in enumerate(lines)])


def _records(lines):
    recs = []
    for i, ln in enumerate(lines):
        f = dict(t.split("=", 1) for t in ln.decode().split(" ") if "=" in t)
        recs.append(wire.encode_parser_schema({"EventID": 0, "logID": "id-%d" % i,
                                               "logFormatVariables": {k: f[k] for k in MONITORED_KEYS if k in f}}))
    return wire.frame_delimited(recs)


@pytest.fixture(scope="module")
def seed_keys():
    from detectmateservice_b200.detector import DeviceDetector
    with DeviceDetector(KEYS, max_batch_bytes=16 << 20, table_log2_slots=20) as t:
        msg = b"\n".join(_lines(1, 20000, 0)) + b"\n"
        t.process_lines(msg, 20000)
        return t.export_known()


def _handle(seed_keys, table_log2=20, alerts_cap=0):
    from detectmateservice_b200.detector import DeviceDetector
    d = DeviceDetector(KEYS, max_batch_bytes=16 << 20, table_log2_slots=table_log2)
    d.set_monitors([{"event_id": None, "source": "header", "pos": k} for k in MONITORED_KEYS])
    if seed_keys is not None:
        d.import_known(seed_keys)
    if alerts_cap:
        d.set_alert_format("1.0.0", "det", "new_value_detector", "growth", [(k, [i]) for i, k in enumerate(MONITORED_KEYS)],
                           capacity=alerts_cap)
    return d


def _alerts(d):
    return d.encode_alerts(first_log_id=7, first_alert_id=11, now=1773848383)


def _outputs(d, call, batch):
    out = call(d, batch)
    return [np.asarray(x).tobytes() if isinstance(x, np.ndarray) else x for x in out] + [d.anomalies(), _alerts(d)]


@pytest.mark.parametrize("kind", ["parser_schema", "log_schema"])
def test_batches_small_large_small(seed_keys, kind):
    make, call = {"parser_schema": (_records, lambda d, b: d.process_records(b)),
                  "log_schema": (_logs, lambda d, b: d.process_logs(b))}[kind]
    batches = [make(_lines(10 + i, n)) for i, n in enumerate((SMALL, LARGE, SMALL, LARGE // 2, SMALL))]
    fresh, grown = _handle(seed_keys, alerts_cap=4 << 20), _handle(seed_keys, alerts_cap=4 << 20)
    _outputs(grown, call, make(_lines(9, LARGE)))
    try:
        n_alerts = 0
        for b in batches:
            want = _outputs(grown, call, b)
            assert _outputs(fresh, call, b) == want
            assert want[-1] is not None                            # (encoded on the device, not declined)
            n_alerts += want[-1][1]
        assert n_alerts > 0
    finally:
        fresh.close()
        grown.close()


def test_alert_capacity_changes_between_encodes(seed_keys):
    fresh, grown = _handle(seed_keys, alerts_cap=1 << 20), _handle(seed_keys, alerts_cap=8 << 20)
    try:
        for i, cap in enumerate((8 << 20, 2 << 20, 1 << 20)):
            msg = b"\n".join(_lines(20 + i, LARGE // 4)) + b"\n"
            fresh.set_alert_format("1.0.0", "det", "new_value_detector", "growth",
                                   [(k, [j]) for j, k in enumerate(MONITORED_KEYS)], capacity=cap)
            got = [x.tobytes() for x in fresh.process_lines(msg)] + [_alerts(fresh)]
            want = [x.tobytes() for x in grown.process_lines(msg)] + [_alerts(grown)]
            assert got == want and want[-1] is not None and want[-1][1] > 0
    finally:
        fresh.close()
        grown.close()


def test_exports_around_a_growth_of_the_known_set():
    """2^10 slots: the export scratch first holds the load limit's 512 keys; an import past the limit (reported as
    DM_ERR_TABLE_FULL, the keys kept) makes the next export grow it."""
    rng = np.random.default_rng(3)
    keys = np.unique(rng.integers(1, 2**63, size=900, dtype=np.uint64))[:700]
    fresh, grown = _handle(None, table_log2=10), _handle(None, table_log2=10)
    try:
        with pytest.raises(_lib.DmError) as e:
            grown.import_known(keys)
        assert e.value.code == _lib.DM_ERR_TABLE_FULL
        assert grown.export_known().size == keys.size
        grown.reset()
        for h in (fresh, grown):
            h.import_known(keys[:300])
        first = [h.export_known().tobytes() for h in (fresh, grown)]
        for h in (fresh, grown):
            with pytest.raises(_lib.DmError):
                h.import_known(keys[300:])
        second = [h.export_known() for h in (fresh, grown)]
        assert first[0] == first[1] == np.sort(keys[:300]).tobytes()
        assert second[0].tobytes() == second[1].tobytes() == np.sort(keys).tobytes()
    finally:
        fresh.close()
        grown.close()


def test_pipelined_slots_after_process_lines(seed_keys):
    msgs = [b"\n".join(_lines(30 + i, n)) + b"\n" for i, n in enumerate((SMALL, LARGE, SMALL, LARGE))]
    fresh, grown = _handle(seed_keys, alerts_cap=4 << 20), _handle(seed_keys, alerts_cap=4 << 20)
    try:
        grown.submit(msgs[1], slot=0)
        grown.collect(0)
        grown.submit(msgs[1], slot=1)
        grown.collect(1)
        got, want = ([x.tobytes() for x in h.process_lines(msgs[0])] + [_alerts(h)] for h in (fresh, grown))
        assert got == want
        for i, m in enumerate(msgs):
            out = []
            for h in (fresh, grown):
                h.submit(m, slot=i % 2)
                f, s = h.collect(i % 2)
                out.append([f.tobytes(), s.tobytes(), h.collect_anomalies(i % 2), _alerts(h)])
            assert out[0] == out[1] and out[1][-1] is not None
    finally:
        fresh.close()
        grown.close()
