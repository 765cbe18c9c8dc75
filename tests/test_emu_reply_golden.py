"""Every reply of both detector components, pinned to recorded bytes, CPU tier.

The other emulator tests compare a device-encoded component with a host-encoded one, so a mistake in the reply code
both sides share passes them.  Here one component per input shape -- raw lines (key=value and log_format, chunked),
ParserSchema batches and bare records, LogSchema batches and bare records, pipelined raw lines, compact output -- gets a
sequence of messages whose anomaly counts sit below and at the class default DEVICE_ALERTS_MIN, on the CPU emulator's
detection and alert encoder.  Every reply, n_alerts and n_seen must equal tests/golden/component_replies.json.xz,
which scripts/make_reply_golden.py writes."""
import json
import lzma
import os

import pytest

from detectmateservice_b200 import wire
from pbgen import frame, ld
from test_emu_alerts import AUDIT, NOW, EmuDevice
from test_emu_pipelined_alerts import EmuPipelined
from test_emu_record_alerts import EmuBatchDevice
from test_format_combos import AUDIT_COMBO_CFG

FIXTURE = "component_replies.json.xz"
PIECE = 1024                              # pipelined pieces of 17 records of 64 bytes


@pytest.fixture(scope="module")
def lib():
    import emu_harness
    return emu_harness.lib()


class EmuValuesDevice(EmuBatchDevice):
    """EmuBatchDevice with dm_process_values (B200NewValueDetector's bare ParserSchema record), which the emulator does
    not have: per-monitor known sets, a monitor's bit set for a value not learnt, the score its bit count."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.known = {}

    def process_values(self, records, n_train_records=0, record_bytes=0):
        import numpy as np
        flags, scores, masks = [], [], []
        for r, vals in enumerate(records):
            m = 0
            for f, v in vals:
                if r < n_train_records:
                    self.known.setdefault(f, set()).add(v)
                elif v not in self.known.get(f, ()):
                    m |= 1 << f
            flags.append(1 if m else 0)
            scores.append(float(bin(m).count("1")))
            masks.append(m)
        self.last_n_anomalies = sum(flags)
        return np.array(flags, np.uint8), np.array(scores, np.float32), np.array(masks, np.uint32)


# ------------------------------------------------------------------------------------------------ messages
def _kv_known(i):
    return b"type=A acct=u%d res=ok msg=audit(1700000000.%d:1)" % (i % 4, i)


def _kv_novel(j, declined=False):
    """Four kinds of anomalous key=value record: a new acct, a new type without a Time, new acct and res, a quoted value
    after a look-alike field; declined: a Time outside the device's grammar, so the device declines the batch."""
    if declined:
        return b"type=A acct=d%d res=ok msg=audit(1e5:5)" % j
    return [b"type=A acct=n%d res=ok msg=audit(1700000%d.5:2)" % (j, j),
            b"type=T%d acct=u1 res=ok" % j,
            b"type=A acct=m%d res=bad%d msg=audit(12.25:3)" % (j, j),
            b'type=A x="acct=FAKE" acct="q %d" res=ok msg=audit(99:4)' % j][j % 4]


def _kv_msg(n_novel, n_known, first=0, declined=False):
    """n_novel anomalous records spread over n_known known ones, '\\n'-terminated; declined: the last one declines."""
    recs = [_kv_known(i) for i in range(n_known)]
    for j in range(n_novel):
        recs.insert(j * (n_known + n_novel) // n_novel, _kv_novel(first + j, declined and j == n_novel - 1))
    return b"".join(r + b"\n" for r in recs)


def _kv_fixed(rec):
    return rec + b" pad=" + b"p" * (58 - len(rec)) + b"\n"         # 64 bytes


def _pipelined_msg(counts, first):
    """One record block of 17 fixed-size records per piece, counts[k] of them anomalous; the last block takes 20."""
    recs, j = [], first
    for k, c in enumerate(counts):
        n = 20 if k == len(counts) - 1 else 17
        block = [_kv_fixed(_kv_known(i)) for i in range(n - c)]
        for t in range(c):
            block.insert(2 * t, _kv_fixed(_kv_novel(j)))
            j += 1
        recs += block
    return b"".join(recs)


def _audit_lines(golden_dir):
    return open(os.path.join(golden_dir, "audit_sample.log"), "rb").read().rstrip(b"\n").split(b"\n")


def _lf_msg(lines, n_novel, first):
    """Known audit records with n_novel copies of the first one (USER_ACCT, template 0) carrying a new acct."""
    recs = lines[1:13]
    for j in range(n_novel):
        recs.insert(2 * j, lines[0].replace(b'acct="root"', b'acct="x%d"' % (first + j)))
    return recs


def _ls(recs, first_id=0):
    """LogSchema records of the texts; every fifth one without a logID."""
    return [(b"" if i % 5 == 4 else ld(2, b"log-%d" % (first_id + i))) + ld(3, t) for i, t in enumerate(recs)]


def _ps(i, user, time=None):
    lfv = {"user": user, "level": "l%d" % (i % 2)}
    if time is not None:
        lfv["Time"] = time
    return wire.encode_parser_schema({"EventID": 4, "logID": "rec-%d" % i, "variables": ["a", "b%d" % (i % 3), "c"],
                                      "logFormatVariables": lfv})


def _ps_msg(n_novel, n_known, first):
    recs = [_ps(i, "u%d" % (i % 3), "1700000000.5" if i % 2 else None) for i in range(n_known)]
    for j in range(n_novel):
        recs.insert(3 * j, _ps(1000 + first + j, "new%d" % (first + j), ["17", "", "18/Mar/2026:1", None][j % 4]))
    return recs


# ------------------------------------------------------------------------------------------------ configs
def _kv_cfg(combo, n_train, **params):
    scope = ({"c1": {"header_variables": [{"pos": "type"}, {"pos": "acct"}]}, "c2": {"header_variables": [{"pos": "res"}]}}
             if combo else {"g": {"header_variables": [{"pos": k} for k in ("type", "acct", "res")]}})
    return {"method_type": "new_value_detector", "data_use_training": n_train, "auto_config": False, "params": params,
            "global": scope}


def _lf_cfg(combo, golden_dir, **params):
    params = dict(params, log_format=AUDIT, path_templates=os.path.join(golden_dir, "audit_templates.txt"))
    if combo:
        return dict(AUDIT_COMBO_CFG["detectors"]["NewValueComboDetector"], params=params)
    return {"method_type": "new_value_detector", "data_use_training": 250, "auto_config": False, "params": params,
            "global": {"g": {"header_variables": [{"pos": "type"}, {"pos": "Content"}]}},
            "events": {0: {"pam": {"variables": [{"pos": 5, "name": "acct"}, {"pos": 10, "name": "res"}]}}}}


def _ps_cfg(n_train, **params):
    return {"method_type": "new_value_detector", "data_use_training": n_train, "auto_config": False, "params": params,
            "global": {"g": {"header_variables": [{"pos": "user"}], "variables": [{"pos": 0, "name": "v0"}]}},
            "events": {4: {"e": {"header_variables": [{"pos": "level"}], "variables": [{"pos": 1, "name": "v1"}]}}}}


def _class_scenarios(lib, golden_dir, combo):
    """(name, make_component, messages) per input shape for one detector class."""
    from detectmateservice_b200.component import B200NewValueComboDetector, B200NewValueDetector
    cls = B200NewValueComboDetector if combo else B200NewValueDetector
    kind = "combo" if combo else "value"
    variant = "lanes" if combo else "stream"                     # key=value combinations run on the lanes kernel

    def make(cfg, dev, pipelined=False):
        def new():
            c = cls(config={"detectors": {cls.__name__: cfg}})
            c._det = dev(c)
            c.clock = lambda: NOW
            if pipelined:
                c.PIPE_PIECE_BYTES, c.PIPE_MIN_BYTES = PIECE, 3 * PIECE
            return c
        return new

    kv_dev = lambda c: EmuDevice(lib, [m.key for m in c.monitors], variant, getattr(c, "combos", ()), comp=c)
    lf_dev = lambda c: EmuDevice(lib, [m.key for m in c.monitors], "format", getattr(c, "combos", ()), comp=c)
    pipe_dev = lambda c: EmuPipelined(lib, [m.key for m in c.monitors], variant, getattr(c, "combos", ()))
    batch_dev = lambda c: EmuValuesDevice(lib, c, variant, 1 << 20)
    lines = _audit_lines(golden_dir)
    kv_train = b"".join(_kv_known(i) + b"\n" for i in range(16))
    kv_msgs = [kv_train, _kv_msg(0, 12), _kv_msg(7, 13, 0), _kv_msg(8, 12, 10), _kv_msg(9, 11, 20, declined=True),
               _kv_msg(1, 0, 40), _kv_msg(0, 1), _kv_msg(20, 80, 50)]          # the last one is cut into 3 pieces
    lf_msgs = [b"".join(t + b"\n" for t in lines[:250])] + [
        b"".join(t + b"\n" for t in _lf_msg(lines, k, 10 * k)) for k in (0, 7, 8)] + [
        lines[0].replace(b'acct="root"', b'acct="lone"') + b"\n"]
    pipe_msgs = [kv_train, _pipelined_msg([7, 8, 0, 9], 0), _pipelined_msg([0, 1, 12, 7], 100)]
    ps_msgs = [frame([_ps(i, "u%d" % (i % 3)) for i in range(12)])] + [
        frame(_ps_msg(k, 10, 10 * k)) for k in (0, 7, 8)] + [frame(_ps_msg(1, 0, 90))]
    bare_ps = [_ps(i, "u%d" % (i % 3)) for i in range(3)] + _ps_msg(3, 2, 40)
    ls_msgs = [frame(_ls([_kv_known(i) for i in range(16)]))] + [
        frame(_ls(_kv_msg(k, 12, 10 * k).rstrip(b"\n").split(b"\n"), 100 * k)) for k in (0, 7, 8)] + [
        frame(_ls(_kv_msg(8, 4, 90).rstrip(b"\n").split(b"\n")) + [b"\xff"])]        # with a malformed record
    ls_lf_msgs = [frame(_ls(lines[:250]))] + [frame(_ls(_lf_msg(lines, k, 10 * k), 1000 * k)) for k in (0, 7, 8)]
    bare_ls = [_ls([_kv_known(i)], i)[0] for i in range(16)] + _ls(
        [_kv_novel(1), _kv_known(3), _kv_novel(2), _kv_novel(3, declined=True)], 50) + [
        b"\xff\x01", _ls([_kv_novel(5)], 60)[0]]                            # a malformed record raises WireError
    return [
        ("raw_lines_kv_" + kind, make(_kv_cfg(combo, 16, max_batch_bytes=2048), kv_dev), kv_msgs),
        ("raw_lines_compact_" + kind, make(_kv_cfg(combo, 16, max_batch_bytes=2048, output_format="compact"), kv_dev),
         kv_msgs),
        ("raw_lines_log_format_" + kind, make(_lf_cfg(combo, golden_dir), lf_dev), lf_msgs),
        ("pipelined_" + kind, make(_kv_cfg(combo, 16), pipe_dev, pipelined=True), pipe_msgs),   # (combo: one call)
        ("parser_schema_batch_" + kind, make(_ps_cfg(12, input_format="parser_schema_batch"), batch_dev), ps_msgs),
        ("parser_schema_batch_compact_" + kind,
         make(_ps_cfg(12, input_format="parser_schema_batch", output_format="compact"), batch_dev), ps_msgs),
        ("parser_schema_" + kind, make(_ps_cfg(3, input_format="parser_schema"), batch_dev), bare_ps),
        ("parser_schema_compact_" + kind,
         make(_ps_cfg(3, input_format="parser_schema", output_format="compact"), batch_dev), bare_ps),
        ("log_schema_batch_kv_" + kind, make(_kv_cfg(combo, 16, input_format="log_schema_batch"), batch_dev), ls_msgs),
        ("log_schema_batch_compact_" + kind,
         make(_kv_cfg(combo, 16, input_format="log_schema_batch", output_format="compact"), batch_dev), ls_msgs),
        ("log_schema_batch_log_format_" + kind,
         make(_lf_cfg(combo, golden_dir, input_format="log_schema_batch"), batch_dev), ls_lf_msgs),
        ("log_schema_" + kind, make(_kv_cfg(combo, 16, input_format="log_schema"), batch_dev), bare_ls),
    ]


def scenarios(lib, golden_dir):
    return _class_scenarios(lib, golden_dir, False) + _class_scenarios(lib, golden_dir, True)


def run_scenario(make, messages):
    """One component over the messages: per message its reply (hex, or None) or the name of the error it raised, with
    n_alerts and n_seen after it."""
    comp = make()
    got = []
    for msg in messages:
        try:
            out = comp.process(msg)
            entry = {"reply": None if out is None else out.hex()}
        except wire.WireError as e:
            entry = {"error": type(e).__name__}
        entry.update(n_alerts=comp.n_alerts, n_seen=comp.n_seen)
        got.append(entry)
    comp._det.close()
    return got


def record(lib, golden_dir):
    return {name: run_scenario(make, msgs) for name, make, msgs in scenarios(lib, golden_dir)}


def test_replies_match_the_recorded_bytes(lib, golden_dir):
    from detectmateservice_b200.component import B200NewValueDetector
    assert B200NewValueDetector.DEVICE_ALERTS_MIN == 8             # the messages' 7, 8 and 9 anomalies straddle it
    with lzma.open(os.path.join(golden_dir, FIXTURE), "rt") as f:
        want = json.load(f)
    cases = scenarios(lib, golden_dir)
    assert sorted(name for name, _m, _msgs in cases) == sorted(want)
    for name, make, msgs in cases:
        got = run_scenario(make, msgs)
        assert len(got) == len(want[name]), name
        for i, (g, w) in enumerate(zip(got, want[name])):
            assert g == w, (name, i)
