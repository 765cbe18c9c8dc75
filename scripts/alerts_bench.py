"""What the default output (`output_format: alerts`) costs per raw-line message: B200NewValueDetector.process() on 64k
synthetic audit records of 256 B (config 2), after a clean training message, at anomaly rates 1e-3, 1e-2 and 1e-1, plus
messages whose only anomalies are k records, k = 1, 4, 8, 16, 32 (where the component's DEVICE_ALERTS_MIN is chosen).  Three arms, run alternately call by call on a memoryview of a pinned
copy of the message: `compact` (no alerts), `host` (the host encoder, forced here by hiding the device encoder from the
component) and `device` (dm_encode_alerts, forced here for every message with alerts).  Per workload one JSON line: median and range of the wall time of
process() per arm, in ms, and the summed device time of the encoder kernels (dm_k_alert_*) per call, from a separate
torch.profiler run.  The card's name and power limit are printed first.

    python scripts/alerts_bench.py [--calls 21]
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

from logschema_bench import card, kernel_us  # noqa: E402


class HostEncoder:
    """The component's handle with the device encoder hidden: the component words alerts on the host."""

    def __init__(self, det):
        self._d = det

    def __getattr__(self, name):
        if name in ("encode_alerts", "set_alert_format"):
            raise AttributeError(name)
        return getattr(self._d, name)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=65536)
    ap.add_argument("--calls", type=int, default=21)
    args = ap.parse_args()
    import torch
    from detectmateservice_b200 import wire
    from detectmateservice_b200.component import B200NewValueDetector
    from detectmateservice_b200.synth import MONITORED_KEYS, AuditSynth

    print(json.dumps(card()), flush=True)
    cfg = lambda fmt: {"detectors": {"B200NewValueDetector": {
        "method_type": "new_value_detector", "data_use_training": args.records, "auto_config": False,
        "params": {"output_format": fmt, "max_batch_bytes": 32 << 20},
        "global": {"g": {"header_variables": [{"pos": k} for k in MONITORED_KEYS]}}}}}
    g0 = AuditSynth(seed=7)
    train, _ = g0.batch(args.records, inject=False)
    arms = {"compact": B200NewValueDetector(config=cfg("compact")), "host": B200NewValueDetector(config=cfg("alerts")),
            "device": B200NewValueDetector(config=cfg("alerts"))}
    for name, c in arms.items():
        c.clock = lambda: 1773848383
        c.process(train)
        if name == "host":
            c._det = HostEncoder(c.det)
        if name == "device":
            c.DEVICE_ALERTS_MIN = 1
    workloads = []
    for rate in (1e-3, 1e-2, 1e-1):
        msg, _ = AuditSynth(seed=8, anomaly_rate=rate).batch(args.records, inject=True)
        workloads.append(("rate=%g" % rate, msg))
    lines = train.split(b"\n")
    for k in (1, 4, 8, 16, 32):                            # a clean message whose first k records have a new type
        msg = lines[:]
        for i in range(k):
            msg[i * 997] = b"type=NEW%d" % i
        workloads.append(("alerts=%d" % k, b"\n".join(msg)))
    for label, msg in workloads:
        pin = torch.empty(len(msg), dtype=torch.uint8, pin_memory=True)
        pin.numpy()[:] = memoryview(msg)
        mv = memoryview(pin.numpy())
        for c in arms.values():                            # (the same logIDs and alertIDs in both alert arms)
            c.n_seen, c.n_alerts = args.records, 0
        outs = {name: c.process(mv) for name, c in arms.items()}
        assert outs["host"] == outs["device"]
        times = {name: [] for name in arms}
        for _ in range(args.calls):
            for name, c in arms.items():
                t0 = time.perf_counter()
                c.process(mv)
                times[name].append((time.perf_counter() - t0) * 1e3)
        ku = kernel_us(lambda: arms["device"].process(mv), args.calls)
        enc = {k: round(v, 2) for k, v in ku.items() if k.startswith("dm_k_alert")}
        n_alerts = len(wire.split_delimited(outs["device"])) if outs["device"] else 0
        print(json.dumps({"workload": label, "records": args.records, "alerts": n_alerts,
                          "process_ms": {n: {"median": round(statistics.median(t), 3), "min": round(min(t), 3),
                                             "max": round(max(t), 3)} for n, t in times.items()},
                          "encoder_kernels_us": round(sum(enc.values()), 2), "encoder_by_kernel_us": enc,
                          "detect_kernels_us": round(sum(v for k, v in ku.items() if not k.startswith("dm_k_alert")), 2)}),
              flush=True)
    for c in arms.values():
        c.close()


if __name__ == "__main__":
    main()
