"""Device time of LogSchema input (dm_process_logs) against raw lines (dm_process_lines) on one batch of the
config-2 shape: 64k synthetic audit records of 256 B, each wrapped in a LogSchema (logID, log, logSource) and framed
as one varint-length-delimited batch.  Detection only (the table is trained first), in key=value mode and in
log_format mode (the audit log_format and templates of tests/golden).

Per mode it prints one JSON line:
  unwrap_us     summed device time of the four unwrap kernels (walk, scan, compact, copy) per call
  scatter_us    device time of the kernel that maps the results back to record order
  detect_us     device time of the line kernels inside dm_process_logs
  logs_kernels_us / lines_kernels_us   every kernel of one dm_process_logs / dm_process_lines call
  logs_call_us / lines_call_us         host wall time of one whole synchronous call (median)
Kernel times come from torch.profiler (CUPTI); the card's name and power limit are printed first, as they are part of
every number.

    python scripts/logschema_bench.py [--records 65536] [--iters 20]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

UNWRAP = ("dm_k_logs_walk", "dm_k_logs_scan", "dm_k_logs_compact", "dm_k_logs_copy")
AUDIT = "type=<type> msg=audit(<Time>): <Content>"


def card() -> dict:
    import torch
    out = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,power.max_limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        out["power_limit"] = q
    except Exception as e:                                    # (no nvidia-smi: the number goes out without it)
        out["power_limit"] = "unknown (%s)" % type(e).__name__
    return out


def kernel_us(fn, iters: int) -> dict:
    """Summed device time per call of every kernel fn launches, by kernel name (torch.profiler / CUPTI)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        name = e.name[5:] if e.name.startswith("void ") else e.name       # (templated kernels: "void dm_k_x<...>(...)")
        if str(getattr(e, "device_type", "")).endswith("CUDA") and name.startswith("dm_k"):
            dt = getattr(e, "device_time", None)
            if dt is None:
                dt = e.cuda_time
            name = name.split("(")[0].split("<")[0]
            out[name] = out.get(name, 0.0) + dt / iters
    return out


def wall_us(fn, iters: int) -> float:
    fn()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e6)
    return statistics.median(ts)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from detectmateservice_b200 import wire
    from detectmateservice_b200.detector import DeviceDetector
    from detectmateservice_b200.logformat import load_templates
    from detectmateservice_b200.synth import MONITORED_KEYS, AuditSynth

    print(json.dumps(card()), flush=True)
    g = AuditSynth(seed=2024)
    train, _ = g.batch(args.records, inject=False)
    msg, _ = g.batch(args.records, inject=True)
    lines = msg.split(b"\n")[:args.records]
    recs = [wire.encode_log_schema({"__version__": "1.0.0", "logID": str(i), "log": ln.decode(),
                                    "logSource": "/var/log/audit/audit.log"}) for i, ln in enumerate(lines)]
    batch = wire.frame_delimited(recs)
    templates = load_templates(os.path.join(ROOT, "tests", "golden", "audit_templates.txt"))
    keys = [k.encode() for k in MONITORED_KEYS]
    for mode in ("key_value", "log_format"):
        det = DeviceDetector(keys, device=0, max_batch_bytes=32 << 20, table_log2_slots=20)
        if mode == "log_format":
            det.set_monitors([{"event_id": None, "source": "header", "pos": "type"}] +
                             [{"event_id": 0, "source": "variable", "pos": i} for i in (4, 6, 9, 10)])
            det.set_format(AUDIT, templates)
        det.process_lines(train, args.records)
        logs = lambda: det.process_logs(batch, 0, True)
        plain = lambda: det.process_lines(msg, 0)
        f_logs, s_logs, _ = logs()
        f_lines, s_lines = plain()
        assert (f_logs == f_lines).all() and (s_logs == s_lines).all()
        kl = kernel_us(logs, args.iters)
        kp = kernel_us(plain, args.iters)
        unwrap = sum(v for k, v in kl.items() if k in UNWRAP)
        scatter = kl.get("dm_k_logs_scatter", 0.0)
        out = {"mode": mode, "records": args.records, "batch_bytes": len(batch), "text_bytes": len(msg),
               "unwrap_us": round(unwrap, 2), "unwrap_by_kernel_us": {k: round(kl.get(k, 0.0), 2) for k in UNWRAP},
               "scatter_us": round(scatter, 2),
               "detect_us": round(sum(kl.values()) - unwrap - scatter, 2),
               "logs_kernels_us": round(sum(kl.values()), 2), "lines_kernels_us": round(sum(kp.values()), 2),
               "lines_kernels": {k: round(v, 2) for k, v in kp.items()},
               "logs_call_us": round(wall_us(logs, args.iters), 1), "lines_call_us": round(wall_us(plain, args.iters), 1),
               "anomalies": int(f_logs.sum())}
        print(json.dumps(out), flush=True)
        det.close()


if __name__ == "__main__":
    main()
