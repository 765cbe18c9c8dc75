"""What the default output (`output_format: alerts`) costs per LogSchema and ParserSchema batch: B200NewValueDetector
.process() of 64k-record `log_schema_batch` and `parser_schema_batch` messages (synthetic audit records of 256 B; the
LogSchema record wraps the line, the ParserSchema record carries the monitored fields and the audit Time in
logFormatVariables), after a clean training message, at anomaly rates 1e-3, 1e-2 and 1e-1, plus clean messages whose
only anomalies are k records, k = 1, 4, 8, 16, 32.  Two arms, run alternately call by call: `host` (the host encoder,
forced by hiding the device encoder from the component) and `device` (dm_encode_alerts, forced for every message with
alerts).  Per workload one JSON line: median and range of the wall time of process() per arm, in ms, and the summed
device time of the encoder kernels (dm_k_alert_*) per call, from a separate torch.profiler run.  The card's name and
power limit are printed first.

    python scripts/record_alerts_bench.py [--records 65536] [--calls 21]
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
from logschema_bench import card, kernel_us  # noqa: E402


def log_batch(lines):
    from detectmateservice_b200 import wire
    return wire.frame_delimited([wire.encode_log_schema({"__version__": "1.0.0", "logID": "id-%d" % i, "log": ln.decode(),
                                                         "logSource": "/var/log/audit/audit.log"})
                                 for i, ln in enumerate(lines)])


def parser_batch(lines, keys):
    """One ParserSchema per audit line: its monitored key=value fields and its audit Time in logFormatVariables."""
    from detectmateservice_b200 import wire
    recs = []
    for i, ln in enumerate(lines):
        f = dict(t.split("=", 1) for t in ln.decode().split(" ") if "=" in t)
        lfv = {k: f[k] for k in keys if k in f}
        m = f.get("msg", "")
        if m.startswith("audit("):
            lfv["Time"] = m[6:].split(":")[0]
        recs.append(wire.encode_parser_schema({"EventID": 1, "logID": "id-%d" % i, "logFormatVariables": lfv}))
    return wire.frame_delimited(recs)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=65536)
    ap.add_argument("--calls", type=int, default=21)
    args = ap.parse_args()
    from detectmateservice_b200 import wire
    from detectmateservice_b200.component import B200NewValueDetector
    from detectmateservice_b200.synth import MONITORED_KEYS, AuditSynth

    print(json.dumps(card()), flush=True)
    g0 = AuditSynth(seed=7)
    train_lines = g0.batch(args.records, inject=False)[0].rstrip(b"\n").split(b"\n")
    inputs = {"log_schema_batch": lambda lines: log_batch(lines),
              "parser_schema_batch": lambda lines: parser_batch(lines, MONITORED_KEYS)}
    for fmt, make in inputs.items():
        cfg = {"detectors": {"B200NewValueDetector": {
            "method_type": "new_value_detector", "data_use_training": args.records, "auto_config": False,
            "params": {"input_format": fmt, "max_batch_bytes": 64 << 20},
            "global": {"g": {"header_variables": [{"pos": k} for k in MONITORED_KEYS]}}}}}
        arms = {"host": B200NewValueDetector(config=cfg), "device": B200NewValueDetector(config=cfg)}
        train = make(train_lines)
        for name, c in arms.items():
            c.clock = lambda: 1773848383
            c.process(train)
            if name == "host":
                c._det = HostEncoder(c.det)
            else:
                c.DEVICE_ALERTS_MIN = 1
        workloads = []
        for rate in (1e-3, 1e-2, 1e-1):
            lines = AuditSynth(seed=8, anomaly_rate=rate).batch(args.records, inject=True)[0].rstrip(b"\n").split(b"\n")
            workloads.append(("rate=%g" % rate, make(lines)))
        for k in (1, 4, 8, 16, 32):                        # a clean message whose k records have a new type
            lines = train_lines[:]
            for i in range(k):
                lines[i * 997] = lines[i * 997].replace(b"type=", b"type=NEW%d" % i, 1)
            workloads.append(("alerts=%d" % k, make(lines)))
        for label, msg in workloads:
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
            ku = kernel_us(lambda: arms["device"].process(msg), args.calls)
            enc = {k: round(v, 2) for k, v in ku.items() if k.startswith("dm_k_alert")}
            n_alerts = len(wire.split_delimited(outs["device"])) if outs["device"] else 0
            print(json.dumps({"input": fmt, "workload": label, "records": args.records, "alerts": n_alerts,
                              "process_ms": {n: {"median": round(statistics.median(t), 3), "min": round(min(t), 3),
                                                 "max": round(max(t), 3)} for n, t in times.items()},
                              "encoder_kernels_us": round(sum(enc.values()), 2), "encoder_by_kernel_us": enc}),
                  flush=True)
        for c in arms.values():
            c.close()


if __name__ == "__main__":
    main()
