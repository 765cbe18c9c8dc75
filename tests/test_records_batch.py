"""Record mode on the device (batches of length-delimited ParserSchema records):
the kernel source on the CPU emulator (CPU tier) and the real library (GPU tier), both
against the per-record Python oracle (oracle/nvd.py), which decodes with protobuf's own
runtime -- an independent codec from the kernel's hand-written field walk."""

import numpy as np
import pytest

from detectmateservice_b200 import wire
from oracle.nvd import NewValueDetectorOracle
from oracle import schemas as oschemas

CFG = {"detectors": {"NewValueDetector": {
    "method_type": "new_value_detector", "data_use_training": 300, "auto_config": False, "params": {},
    "global": {"g": {"header_variables": [{"pos": "level"}, {"pos": "type"}]}},
    "events": {1: {"t": {"params": {}, "variables": [{"pos": 0, "name": "var1"}], "header_variables": [{"pos": "user"}]}},
               2: {"t": {"variables": [{"pos": 1}]}},
               -7: {"neg": {"header_variables": [{"pos": "level"}]}}}}}}


def make_records(n, seed=3):
    r = np.random.Generator(np.random.PCG64(seed))
    recs = []
    for i in range(n):
        late = i > n // 2
        lfv = {"level": ["INFO", "WARN", "ERR", "DBG", ""][int(r.integers(0, 5 if late else 2))],
               "user": "u%d" % r.integers(0, 9 if late else 4), "Time": str(1634567890 + i)}
        if r.random() < 0.7:
            lfv["type"] = ["A", "BB", "a value with spaces", "é-utf8"][int(r.integers(0, 4 if late else 2))]
        rec = {"EventID": [1, 2, 3, -7][int(r.integers(0, 4))], "logID": str(i), "parserType": "p", "parserID": "x" * int(r.integers(0, 200)),
               "variables": ["v%d" % r.integers(0, 8 if late else 3) for _ in range(int(r.integers(0, 4)))],
               "logFormatVariables": lfv, "receivedTimestamp": 1634567890 + i, "log": "raw " * int(r.integers(0, 40))}
        if r.random() < 0.1:
            del rec["EventID"]
        recs.append(rec)
    return recs


def oracle_run(recs, n_train_cfg=300):
    orc = NewValueDetectorOracle(config=CFG, clock=lambda: 1773848383)
    flags, scores, masks = [], [], []
    for rec in recs:
        out = orc.process(wire.encode_parser_schema(rec))
        if out is None:
            flags.append(0); scores.append(0.0); masks.append(0)
            continue
        m = oschemas.DetectorSchema()
        m.ParseFromString(out)
        keys = [mon.alert_key for mon in orc.monitors]
        mask = 0
        # two monitors may share an alert key text only if configured twice; here they are distinct
        for i, k in enumerate(keys):
            if k in m.alertsObtain:
                mask |= 1 << i
        flags.append(1); scores.append(float(m.score)); masks.append(mask)
    return flags, scores, masks, orc


def monitors_of(cfg):
    from detectmateservice_b200.component import parse_monitors, select_component_config
    return parse_monitors(select_component_config(cfg, "NewValueDetector"))


def test_emu_record_batch_kernel():
    import emu_harness
    from detectmateservice_b200 import _lib
    recs = make_records(900)
    want_f, want_s, want_m, orc = oracle_run(recs)
    mons = monitors_of(CFG)
    assert [m.alert_key for m in mons] == [m.alert_key for m in orc.monitors]
    det = emu_harness.EmuDetector([m.key for m in mons], table_log2=12)
    arr = (_lib.Monitor * len(mons))()
    for i, m in enumerate(mons):
        arr[i].event_id = m.event_id if m.event_id is not None else 0
        arr[i].has_event = 0 if m.event_id is None else 1
        if m.source == "header":
            kb = m.pos.encode()
            arr[i].source, arr[i].key_len = 0, len(kb)
            for j, c in enumerate(kb):
                arr[i].key[j] = c
        else:
            arr[i].source, arr[i].var_index = 1, m.pos
    det.set_monitors(arr, len(mons))
    got_f, got_s, got_m = [], [], []
    seen = 0
    for lo in range(0, len(recs), 250):                         # several messages; training spans two of them
        batch = wire.frame_delimited([wire.encode_parser_schema(r) for r in recs[lo:lo + 250]])
        n_train = max(0, min(250, 300 - seen))
        f = np.full(300, 9, np.uint8); s = np.full(300, -1, np.float32); m = np.zeros(300, np.uint32)
        rc, k, n_an = det.process_records(batch, n_train, f, s, m, 300)
        assert rc == 0
        seen += k
        got_f += f[:k].tolist(); got_s += s[:k].tolist(); got_m += m[:k].tolist()
        assert n_an == int(f[:k].sum())
    assert got_f == want_f and got_s == want_s and got_m == want_m
    assert sum(want_f) > 50


def test_emu_frame_split_matches_split_delimited():
    """The framing split libdmdetect and the emulator share (dm_frame_split) against wire.split_delimited on pbgen
    batches: length prefixes padded up to 10 bytes are taken, an 11-byte one is refused, as are a prefix the message
    cuts short and a record that runs past the end; each error at the byte libdmdetect's message names."""
    import ctypes as C
    import random
    import emu_harness
    from pbgen import Gen, frame, varint
    lib = emu_harness.lib()

    def split(buf):
        off, ln, at = np.zeros(len(buf) + 1, np.uint32), np.zeros(len(buf) + 1, np.uint32), C.c_uint64()
        n = lib.emu_frame_split(buf, len(buf), off.ctypes.data, ln.ctypes.data, len(buf) + 1, C.byref(at))
        if n < 0:
            return n, at.value
        return [buf[o:o + k] for o, k in zip(off[:n].tolist(), ln[:n].tolist())]

    recs, _ = Gen(seed=5).records(300)
    r = random.Random(5)
    for overlong_p in (0.0, 0.5, 1.0):
        buf = frame(recs, r, overlong_p)
        assert split(buf) == wire.split_delimited(buf) == recs
    assert split(b"") == wire.split_delimited(b"") == []
    head = frame(recs[:3])
    ten = head + varint(3, 10) + b"abc"
    assert split(ten) == wire.split_delimited(ten) == recs[:3] + [b"abc"]
    bad = {head + varint(3, 11) + b"abc": (-1, len(head) + 10),        # 11-byte prefix
           head + b"\x83": (-1, len(head) + 1),                      # prefix cut short by the end of the message
           head + b"\x83\x80": (-1, len(head) + 2),
           head + varint(4) + b"abc": (-2, len(head) + 1),            # record runs past the end
           varint(1 << 40, 10): (-2, 10)}
    for buf, want in bad.items():
        with pytest.raises(wire.WireError):
            wire.split_delimited(buf)
        assert split(buf) == want, buf


@pytest.mark.gpu
def test_gpu_record_batch_through_component():
    from detectmateservice_b200.component import B200NewValueDetector, decode_compact
    recs = make_records(3000, seed=5)
    want_f, want_s, want_m, orc = oracle_run(recs)
    comp = B200NewValueDetector(name="NewValueDetector", config=CFG)
    comp.clock = lambda: 1773848383
    orc2 = NewValueDetectorOracle(config=CFG, clock=lambda: 1773848383)
    got_alerts, want_alerts = [], []
    for lo in range(0, len(recs), 700):
        blobs = [wire.encode_parser_schema(r) for r in recs[lo:lo + 700]]
        out = comp.process(wire.frame_delimited(blobs))
        if out:
            got_alerts += [wire.decode_detector_schema(b) for b in wire.split_delimited(out)]
        for b in blobs:
            w = orc2.process(b)
            if w is not None:
                m = oschemas.DetectorSchema()
                m.ParseFromString(w)
                want_alerts.append(m)
    assert len(got_alerts) == len(want_alerts) == sum(want_f)
    for a, b in zip(got_alerts, want_alerts):
        assert a["alertsObtain"] == dict(b.alertsObtain) and a["score"] == b.score
        assert a["alertID"] == b.alertID and a["logIDs"] == list(b.logIDs)
        assert a["extractedTimestamps"] == list(b.extractedTimestamps)
    st = comp.stats()
    assert st["lines"] == 3000 and st["train_lines"] == 300 and st["anomalies"] == sum(want_f)
    assert st["score_sum"] == int(sum(want_s))
    # compact output + a malformed record in the middle of a batch is counted, not scored
    comp2 = B200NewValueDetector(name="NewValueDetector", config={"detectors": {"NewValueDetector": dict(
        CFG["detectors"]["NewValueDetector"], params={"output_format": "compact", "input_format": "parser_schema_batch"})}})
    blobs = [wire.encode_parser_schema(r) for r in recs[:400]]
    f, s = decode_compact(comp2.process(wire.frame_delimited(blobs)))
    assert f.tolist() == want_f[:400] and s.tolist() == want_s[:400]
    bad = wire.frame_delimited([blobs[0], b"\x52\x7f\x01", blobs[1]])          # map entry running past its end
    f, s = decode_compact(comp2.process(bad))
    assert f.size == 3 and f[1] == 0
    comp.close(); comp2.close()
