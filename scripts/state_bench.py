"""Time the known-set export (dm_export_known) and a full state save and load (params.state_path) at 2^20, 2^24 and
2^27 table slots, each table filled to its 1/2 load limit with random keys.

    python scripts/state_bench.py [--parent-lib PATH] [--sizes 20,24,27] [--reps 5]

export: DeviceDetector.export_known() -- the count query, then the sorted keys into host memory.  With --parent-lib
(a libdmdetect.so built from another commit, e.g. one whose export copies the table to the host and sorts it there)
the same two calls on that library's handle run alternately with this build's, in the same process, on the same keys.
save: export + state.write_state (file in a temporary directory, fsynced); load: state.read_state + import_known into
a reset handle.  Prints one JSON line: per size the median and range in ms, with the card's name and power limit.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from detectmateservice_b200 import _lib, state  # noqa: E402
from detectmateservice_b200.detector import DeviceDetector  # noqa: E402


class ParentHandle:
    """A handle of another libdmdetect build: create, import, export only."""

    def __init__(self, path, log2):
        self.lib = C.CDLL(path)
        for name in ("dm_create", "dm_import_known", "dm_export_known", "dm_destroy"):
            fn = getattr(self.lib, name)
            fn.restype, fn.argtypes = _lib.SYMBOLS[name]
        self.lib.dm_last_error.restype = C.c_char_p
        h = C.c_void_p()
        self._check(self.lib.dm_create(0, 1, b"a", (C.c_uint32 * 1)(1), 1 << 20, 0, log2, C.byref(h)))
        self.h = h

    def _check(self, rc):
        if rc:
            raise RuntimeError(self.lib.dm_last_error().decode())

    def import_known(self, keys):
        self._check(self.lib.dm_import_known(self.h, keys.ctypes.data_as(C.POINTER(C.c_uint64)), keys.size))

    def export_known(self):
        n = C.c_uint64()
        self._check(self.lib.dm_export_known(self.h, None, 0, C.byref(n)))
        out = np.zeros(max(1, n.value), dtype=np.uint64)
        self._check(self.lib.dm_export_known(self.h, out.ctypes.data_as(C.POINTER(C.c_uint64)), n.value, C.byref(n)))
        return out[:n.value]

    def close(self):
        self.lib.dm_destroy(self.h)


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def summary(ms):
    return {"median_ms": round(float(np.median(ms)), 3), "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3),
            "n": len(ms)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in q.split(",")]
        return name, limit
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--sizes", default="20,24,27")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    name, limit = card()
    result = {"gpu": name, "power_limit": limit, "sizes": {}}
    tmp = tempfile.mkdtemp(prefix="dmstate")
    path = os.path.join(tmp, "state.bin")
    rng = np.random.default_rng(2027)
    for log2 in (int(s) for s in args.sizes.split(",")):
        n = 1 << (log2 - 1)
        keys = np.unique(rng.integers(1, 2**64 - 1, size=n + (n >> 6) + 64, dtype=np.uint64, endpoint=True))[:n]
        rng.shuffle(keys)
        want = np.sort(keys)
        det = DeviceDetector([b"a"], max_batch_bytes=1 << 20, table_log2_slots=log2)
        det.import_known(keys)
        other = DeviceDetector([b"a"], max_batch_bytes=1 << 20, table_log2_slots=log2)
        parent = None
        if args.parent_lib:
            parent = ParentHandle(args.parent_lib, log2)
            parent.import_known(keys)
        reps = args.reps if log2 < 27 else max(3, args.reps // 2)
        dev, par, save, load = [], [], [], []
        assert np.array_equal(det.export_known(), want)          # (also allocates the export scratch)
        if parent:
            assert np.array_equal(parent.export_known(), want)
        header = {"component": "bench", "key_signature": {}, "key_probe": state.probe_key(), "n_seen": n, "n_alerts": 0}
        for _ in range(reps):
            ms, got = timed(det.export_known)
            dev.append(ms)
            if parent:
                ms, _ = timed(parent.export_known)
                par.append(ms)
            ms, _ = timed(lambda: state.write_state(path, header, det.export_known()))
            save.append(ms)
            other.reset()

            def _load():
                _hdr, k = state.read_state(path)
                other.import_known(k)
            ms, _ = timed(_load)
            load.append(ms)
        assert np.array_equal(got, want) and np.array_equal(other.export_known(), want)
        row = {"keys": n, "device_export": summary(dev), "save": summary(save), "load": summary(load)}
        if parent:
            row["parent_export"] = summary(par)
        result["sizes"][f"2^{log2}"] = row
        det.close()
        other.close()
        if parent:
            parent.close()
        print(json.dumps({f"2^{log2}": row}), file=sys.stderr, flush=True)
    os.unlink(path)
    os.rmdir(tmp)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
