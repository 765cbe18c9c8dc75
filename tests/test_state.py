"""The detector state file (detectmateservice_b200/state.py) and the component's save points (params.state_path), on a
device stand-in: no GPU needed."""
import hashlib
import logging
import os
import threading

import numpy as np
import pytest

from detectmateservice_b200 import state as S
from detectmateservice_b200._lib import DM_ERR_TABLE_FULL, DmError

HEADER = {"component": "B200NewValueDetector", "key_signature": {"monitors": []}, "key_probe": 5, "n_seen": 3,
          "n_alerts": 1}


# ---------------------------------------------------------------------------------------------- the file format
def test_round_trip(tmp_path):
    keys = np.array([1, 7, 2**63, 2**64 - 1], dtype=np.uint64)
    p = str(tmp_path / "s.bin")
    S.write_state(p, HEADER, keys)
    hdr, got = S.read_state(p)
    assert hdr == dict(HEADER, n_keys=4)
    assert got.dtype == np.uint64 and np.array_equal(got, keys)
    blob = open(p, "rb").read()
    assert blob[:8] == b"DMSTATE\0" and blob[-8:] == b"\xff" * 8
    assert not os.path.exists(p + ".tmp")
    S.write_state(p, HEADER, np.zeros(0, np.uint64))
    assert S.read_state(p)[1].size == 0


def _blob(keys=(1, 2, 3), **hdr):
    return S.encode_state(dict(HEADER, **hdr), np.array(keys, dtype=np.uint64))


def _with_keys(raw_keys):
    """A valid blob whose key bytes are replaced by raw_keys (same count)."""
    b = _blob(keys=range(1, len(raw_keys) + 1))
    return b[:len(b) - 8 * len(raw_keys)] + np.array(raw_keys, dtype="<u8").tobytes()


@pytest.mark.parametrize("cut", [0, 5, 15, 16, 40, -9, -1])
def test_truncated(cut):
    b = _blob()
    with pytest.raises(ValueError, match="truncated|key bytes|JSON"):
        S.decode_state(b[:cut] if cut >= 0 else b[:len(b) + cut])


@pytest.mark.parametrize("blob,match", [
    (b"DMSTATF\0" + _blob()[8:], "magic"),
    (_blob()[:8] + (2).to_bytes(4, "little") + _blob()[12:], "version"),
    (_with_keys([3, 2, 5]), "ascending"),
    (_with_keys([1, 1, 5]), "ascending"),
    (_with_keys([0, 2, 5]), "zero key"),
    (_blob() + b"\0" * 8, "counts 3 keys"),
    (_blob(keys=(1, 2)).replace(b'"n_keys":2', b'"n_keys":3'), "counts 3 keys"),
    (_blob(keys=(1, 2), n_seen=30).replace(b'"n_seen":30', b'"n_seen":-3'), "n_seen"),
], ids=["magic", "version", "unsorted", "duplicate", "zero", "extra-key", "count", "negative"])
def test_corrupt(blob, match):
    with pytest.raises(ValueError, match=match):
        S.decode_state(blob)


def test_failed_replace_leaves_the_old_file(tmp_path, monkeypatch):
    p = str(tmp_path / "s.bin")
    S.write_state(p, HEADER, np.array([4, 9], dtype=np.uint64))
    before = open(p, "rb").read()

    def boom(src, dst):
        raise OSError("disk gone")
    monkeypatch.setattr(S.os, "replace", boom)
    with pytest.raises(OSError, match="disk gone"):
        S.write_state(p, dict(HEADER, n_seen=99), np.array([1, 2, 3], dtype=np.uint64))
    assert open(p, "rb").read() == before
    assert not os.path.exists(p + ".tmp")


# ---------------------------------------------------------------------------------------------- the component
def _key(line):
    return int.from_bytes(hashlib.sha1(line).digest()[:8], "little") | 1


class StateDevice:
    """DeviceDetector stand-in: a record's key is its line's hash; compact output only.  full: training raises
    DM_ERR_TABLE_FULL after learning, as the library does."""
    made = []

    def __init__(self, keys, device=0, max_batch_bytes=0, table_log2_slots=20):
        self.known, self.full, self.closed, self.gate = set(), False, False, None
        self.imported, self.geometry = [], (device, max_batch_bytes, table_log2_slots)
        self.last_n_anomalies = 0
        StateDevice.made.append(self)

    def set_monitors(self, mons):
        pass

    def set_format(self, *a):
        pass

    def set_combos(self, combos, member_only_mask=0):
        self.combos = combos

    def process_lines(self, buf, n_train_lines=0, copy=True):
        if self.gate is not None:
            self.gate.wait(10)
        lines = bytes(buf).split(b"\n")[:-1]
        flags = np.zeros(len(lines), np.uint8)
        for i, ln in enumerate(lines):
            if i < n_train_lines:
                self.known.add(_key(ln))
            elif _key(ln) not in self.known:
                flags[i] = 1
        if n_train_lines and self.full:
            raise DmError(DM_ERR_TABLE_FULL, "known-set table over its load limit")
        self.last_n_anomalies = int(flags.sum())
        return flags, flags.astype(np.float32)

    def export_known(self):
        return np.array(sorted(self.known), dtype=np.uint64)

    def import_known(self, keys):
        self.imported.append(np.array(keys))
        self.known.update(int(k) for k in keys)

    def reset(self):
        self.known.clear()

    def close(self):
        self.closed = True


@pytest.fixture
def fake(monkeypatch):
    from detectmateservice_b200 import detector
    monkeypatch.setattr(detector, "DeviceDetector", StateDevice)
    StateDevice.made = []
    return StateDevice


def _cfg(path, training=4, keys=("type", "res"), **params):
    p = {"output_format": "compact", "input_format": "raw_lines", **params}
    if path is not None:
        p["state_path"] = str(path)
    return {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": training,
                                               "global": {"g": {"header_variables": [{"pos": k} for k in keys]}},
                                               "params": p}}}


def _comp(cfg, cls="B200NewValueDetector"):
    from detectmateservice_b200 import component
    return getattr(component, cls)(config=cfg)


def _lines(*vals):
    return b"".join(b"type=%s res=ok\n" % v for v in vals)


def _flags(reply):
    from detectmateservice_b200.component import decode_compact
    return decode_compact(reply)[0].tolist()


def _saved(path):
    hdr, keys = S.read_state(str(path))
    return hdr["n_seen"], hdr["n_alerts"], set(keys.tolist())


def test_training_end_saves_and_a_restart_continues(tmp_path, fake):
    p = tmp_path / "state.bin"
    a = _comp(_cfg(p))
    a.process(_lines(b"A", b"B"))
    assert not p.exists()                                    # nothing mid-training
    a.process(_lines(b"C", b"D", b"E"))                     # ends the window (4 of 5 records train)
    n_seen, n_alerts, keys = _saved(p)
    assert n_seen == 5 and keys == {_key(b"type=%s res=ok" % v) for v in (b"A", b"B", b"C", b"D")}
    mtime = os.stat(p).st_mtime_ns
    assert _flags(a.process(_lines(b"A", b"Z"))) == [0, 1]  # detection: no save
    assert os.stat(p).st_mtime_ns == mtime and _saved(p)[0] == 5
    a.n_alerts = 7
    a.close()                                                # close() saves
    assert _saved(p)[:2] == (7, 7)
    c = _comp(_cfg(p))
    assert (c.n_seen, c.n_alerts) == (7, 7)                  # counters at construction
    assert _flags(c.process(_lines(b"A", b"Z", b"E"))) == [0, 1, 1]   # keys imported with the handle, before the message
    assert len(fake.made[-1].imported) == 1 and c.n_seen == 10


def test_dropped_training_message_still_saves(tmp_path, fake):
    p = tmp_path / "state.bin"
    a = _comp(_cfg(p, training=3))
    a.det.full = True
    with pytest.raises(DmError):
        a.process(_lines(b"A", b"B", b"C"))
    assert a.n_seen == 3 and _saved(p)[0] == 3


def test_exit_handler_saves_while_a_handle_is_live(tmp_path, fake):
    p = tmp_path / "state.bin"
    a = _comp(_cfg(p, training=10))
    a.process(_lines(b"A"))
    assert not p.exists() and a._finalizer is not None and a._finalizer.alive
    a._finalizer()                                           # what interpreter exit runs
    assert _saved(p)[0] == 1
    b = _comp(_cfg(tmp_path / "other.bin", training=10))
    b.process(_lines(b"A"))
    fin = b._finalizer
    b.close()
    assert not fin.alive                                     # close() saved and detached it


def test_reset_import_and_reconfigure_save(tmp_path, fake):
    p = tmp_path / "state.bin"
    a = _comp(_cfg(p, training=10))
    a.process(_lines(b"A", b"B"))
    a.reset_state()
    assert _saved(p) == (0, 0, set())
    a.import_state({"known": [5, 3], "n_seen": 12, "n_alerts": 2})
    assert _saved(p) == (12, 2, {3, 5})
    assert a.reconfigure(_cfg(p, training=20, start_id=50)) is False
    assert _saved(p)[0] == 12


def test_rebuilding_reconfigure_writes_nothing_until_training_ends(tmp_path, fake):
    p = tmp_path / "state.bin"
    a = _comp(_cfg(p, training=2))
    a.process(_lines(b"A", b"B"))
    old = open(p, "rb").read()
    assert a.reconfigure(_cfg(p, training=2, keys=("type",))) is True
    a.process(_lines(b"C"))
    a.close()
    assert open(p, "rb").read() == old                       # the old configuration still finds its state
    b = _comp(_cfg(p, training=2, keys=("type",)))           # mismatch: from scratch
    assert b.n_seen == 0
    assert b.reconfigure(_cfg(p, training=2, keys=("type", "res"))) is True
    b.process(_lines(b"D", b"E"))                            # the new window ends: now it saves
    n_seen, _, keys = _saved(p)
    assert n_seen == 2 and keys == {_key(b"type=D res=ok"), _key(b"type=E res=ok")}


def test_mismatch_is_ignored_with_a_warning_and_replaced(tmp_path, fake, caplog):
    p = tmp_path / "state.bin"
    a = _comp(_cfg(p, training=1))
    a.process(_lines(b"A"))
    a.close()
    with caplog.at_level(logging.WARNING, logger="detectmateservice_b200.component"):
        b = _comp(_cfg(p, training=1, keys=("type",)))
    assert "key_signature" in caplog.text and b.n_seen == 0
    b.process(_lines(b"B"))
    assert fake.made[-1].imported == []
    hdr, keys = S.read_state(str(p))
    assert hdr["key_signature"]["monitors"] == [[None, "header", "type", b"type".hex()]]
    assert keys.tolist() == [_key(b"type=B res=ok")]
    # geometry is not part of the signature: a larger table or batch still loads the state
    c = _comp(_cfg(p, training=1, keys=("type",), table_log2_slots=22, max_batch_bytes=1 << 20))
    assert c.n_seen == 1
    c.process(_lines(b"B"))
    assert fake.made[-1].geometry[1:] == (1 << 20, 22) and len(fake.made[-1].imported) == 1


def test_other_component_class_or_probe_is_a_mismatch(tmp_path, fake, monkeypatch):
    p = tmp_path / "state.bin"
    a = _comp(_cfg(p, training=1))
    a.process(_lines(b"A"))
    a.close()
    assert _comp(_cfg(p, training=1), cls="B200NewValueComboDetector").n_seen == 0
    monkeypatch.setattr(S, "probe_key", lambda: 12345)
    assert _comp(_cfg(p, training=1)).n_seen == 0


def test_corrupt_file_fails_construction(tmp_path, fake):
    p = tmp_path / "state.bin"
    p.write_bytes(b"DMSTATE\0" + b"\1\0\0\0")
    with pytest.raises(ValueError, match="truncated"):
        _comp(_cfg(p))


def test_no_state_path_writes_nothing(tmp_path, fake, monkeypatch):
    monkeypatch.chdir(tmp_path)
    a = _comp(_cfg(None, training=2))
    a.process(_lines(b"A", b"B", b"C"))
    a.reset_state()
    a.import_state({"known": [1], "n_seen": 1})
    a.reconfigure(_cfg(None, training=3))
    a.process(_lines(b"A"))
    a.close()
    assert a._finalizer is None
    assert os.listdir(tmp_path) == []


def test_save_off_the_engine_thread_waits_for_process(tmp_path, fake):
    p = tmp_path / "state.bin"
    a = _comp(_cfg(p, training=10))
    a.process(_lines(b"A"))
    gate = threading.Event()
    a.det.gate = gate
    t = threading.Thread(target=a.process, args=(_lines(b"B"),))
    t.start()
    saver = threading.Thread(target=a.save_state)
    saver.start()
    saver.join(0.3)
    assert saver.is_alive() and not p.exists()              # process() is running: the save waits
    gate.set()
    t.join(5)
    saver.join(5)
    assert _saved(p)[0] == 2


def test_service_stop_saves(tmp_path, fake, monkeypatch):
    from oracle.ref_engine import reference_path
    if reference_path() is None:
        pytest.skip("the reference service is not in oracle/_ref (make -C oracle ref)")
    monkeypatch.syspath_prepend(reference_path())
    from detectmateservice_b200 import service as svc
    a = _comp(_cfg(tmp_path / "state.bin", training=10))
    a.process(_lines(b"A"))
    cls = svc.b200_detector_service()
    stub = cls.__new__(cls)
    stub.detector = a
    stub._running = False                                    # Service.stop returns at once for a stopped engine
    stub.stop()
    assert _saved(tmp_path / "state.bin")[0] == 1
