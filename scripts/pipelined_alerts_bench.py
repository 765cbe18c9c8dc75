"""What the default output (`output_format: alerts`) costs on messages large enough for the two-slot pipeline:
B200NewValueDetector.process() of 32 MiB and 48 MiB raw-line messages (config-2 records of 256 B, handed over as a
memoryview of pinned memory, as the service's receive frames are), with the default PIPE_MIN_BYTES / PIPE_PIECE_BYTES
and max_batch_bytes 64 MiB, after a clean training message.  Workloads: no anomalies (the training records again),
anomaly rates 1e-3, 1e-2 and 1e-1, and the training records with k = 1, 8, 32 of them given a new type.  Two arms, run
alternately call by call: `host` (the host encoder, forced by hiding the device encoder from the component) and
`device` (dm_encode_alerts on every piece with alerts).  Per workload one JSON line: median and range of the wall time
of process() per arm, in ms.  The card's name and power limit are printed first.

    python scripts/pipelined_alerts_bench.py [--calls 11] [--sizes 32,48]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from alerts_bench import HostEncoder  # noqa: E402
from logschema_bench import card  # noqa: E402


def pinned(msg: bytes):
    """A memoryview of a pinned copy of msg."""
    import numpy as np
    import torch
    t = torch.empty(len(msg), dtype=torch.uint8, pin_memory=True)
    t.numpy()[:] = np.frombuffer(msg, dtype=np.uint8)
    return memoryview(t.numpy())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=11)
    ap.add_argument("--sizes", default="32,48", help="message sizes in MiB")
    args = ap.parse_args()
    from detectmateservice_b200 import wire
    from detectmateservice_b200.component import B200NewValueDetector
    from detectmateservice_b200.synth import LINE_BYTES, MONITORED_KEYS, AuditSynth

    print(json.dumps(card()), flush=True)
    sizes = [int(s) for s in args.sizes.split(",")]
    n_train = (max(sizes) << 20) // LINE_BYTES
    train = AuditSynth(seed=7).batch(n_train, inject=False)[0]
    cfg = {"detectors": {"B200NewValueDetector": {
        "method_type": "new_value_detector", "data_use_training": n_train, "auto_config": False,
        "params": {"input_format": "raw_lines", "max_batch_bytes": 64 << 20},
        "global": {"g": {"header_variables": [{"pos": k} for k in MONITORED_KEYS]}}}}}
    arms = {"host": B200NewValueDetector(config=cfg), "device": B200NewValueDetector(config=cfg)}
    for name, c in arms.items():
        c.clock = lambda: 1773848383
        c.process(pinned(train))
        if name == "host":
            c._det = HostEncoder(c.det)
        else:
            c.DEVICE_ALERTS_MIN = 1
    for mib in sizes:
        n = (mib << 20) // LINE_BYTES
        clean = train[:n * LINE_BYTES]
        workloads = [("none", clean)]
        for rate in (1e-3, 1e-2, 1e-1):
            workloads.append(("rate=%g" % rate, AuditSynth(seed=8, anomaly_rate=rate).batch(n, inject=True)[0]))
        for k in (1, 8, 32):                               # the clean records, k of them with a new type
            lines = clean.split(b"\n")
            for i in range(k):
                j = i * (n // k)
                lines[j] = lines[j].replace(b"type=", b"type=NEW%d" % i, 1)[:LINE_BYTES - 1]
            workloads.append(("new_types=%d" % k, b"\n".join(lines)))
        for label, raw in workloads:
            msg = pinned(raw)
            assert len(msg) >= B200NewValueDetector.PIPE_MIN_BYTES
            for c in arms.values():                        # (the same alertIDs in both arms)
                c.n_alerts = 0
            outs = {name: c.process(msg) for name, c in arms.items()}
            assert outs["host"] == outs["device"]
            times = {name: [] for name in arms}
            for _ in range(args.calls):
                for name, c in arms.items():
                    t0 = time.perf_counter()
                    c.process(msg)
                    times[name].append((time.perf_counter() - t0) * 1e3)
            n_alerts = len(wire.split_delimited(outs["device"])) if outs["device"] else 0
            print(json.dumps({"mib": mib, "workload": label, "records": n, "alerts": n_alerts,
                              "process_ms": {a: {"median": round(statistics.median(t), 3), "min": round(min(t), 3),
                                                 "max": round(max(t), 3)} for a, t in times.items()}}), flush=True)
    for c in arms.values():
        c.close()


if __name__ == "__main__":
    main()
