"""What the MatcherParser stage costs: B200MatcherParser.process() of 64k-record `log_schema_batch` messages, parsed on
the device (dm_parse_logs) against the host path (the specification, one record at a time in Python), in two shapes:
the audit lines of tests/golden/audit_sample.log with `type=<Type> msg=audit(<Time>): <Content>`, the templates of
tests/golden/audit_templates.txt and all three R-norm switches; and nginx access-log lines with the docs' log_format.
The two arms run alternately call by call.  Per shape one JSON line: median and range of the wall time per arm in ms,
the output bytes, and the device time per call of each kernel and of the output's device-to-host copy from a separate
torch.profiler run.  Then bare records (one LogSchema per message), host against device, which is what the component's
choice of the host for bare records rests on.  The card's name and power limit are printed first.

    python scripts/parser_bench.py [--records 65536] [--calls 11] [--host-calls 3] [--bare 2000]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from logschema_bench import card  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
NGINX = '<IP> - - [<Time>] "<Method> <URL> <Protocol>" <Status> <Bytes> "<Referer>" "<UserAgent>"'


def component(log_format, norm=False, path_templates=None):
    from detectmateservice_b200.parser import B200MatcherParser
    params = {"remove_spaces": norm, "remove_punctuation": norm, "lowercase": norm}
    if path_templates:
        params["path_templates"] = path_templates
    return B200MatcherParser(config={"parsers": {"MatcherParser": {"log_format": log_format, "time_format": None,
                                                                   "params": params}}})


def shapes(n):
    r = random.Random(1)
    audit = [ln.decode() for ln in open(os.path.join(GOLDEN, "audit_sample.log"), "rb").read().split(b"\n") if ln]
    nginx = ['10.%d.%d.%d - - [18/Mar/2026:15:39:%02d +0000] "GET /p%d HTTP/1.1" %d %d "-" "curl/8.5.0"'
             % (r.randrange(9), r.randrange(256), r.randrange(256), r.randrange(60), r.randrange(5000),
                r.choice((200, 404)), r.randrange(9999)) for _ in range(n)]
    return {"audit": (component("type=<Type> msg=audit(<Time>): <Content>", True,
                                os.path.join(GOLDEN, "audit_templates.txt")), [audit[i % len(audit)] for i in range(n)]),
            "nginx": (component(NGINX), nginx)}


def log_records(lines):
    from detectmateservice_b200 import wire
    return [wire.encode_log_schema({"__version__": "1.0.0", "logID": "id-%d" % i, "log": ln + "\n",
                                    "logSource": "/var/log/x.log"}) for i, ln in enumerate(lines)]


def kernel_times(fn, iters):
    """Device time per call of every dm_k kernel fn launches (template arguments kept) and of its device-to-host copies."""
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
        if not str(getattr(e, "device_type", "")).endswith("CUDA"):
            continue
        name = e.name[5:] if e.name.startswith("void ") else e.name
        if "DtoH" in name or "Device -> Pageable" in name or "Device -> Pinned" in name:
            name = "memcpy DtoH"
        elif not name.startswith("dm_k"):
            continue
        name = name.split("(")[0]
        dt = getattr(e, "device_time", None)
        out[name] = round(out.get(name, 0.0) + (dt if dt is not None else e.cuda_time) / iters, 1)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=65536)
    ap.add_argument("--calls", type=int, default=11)
    ap.add_argument("--host-calls", type=int, default=3)
    ap.add_argument("--bare", type=int, default=2000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("parser_bench.py measures the device path: no CUDA device")
    from detectmateservice_b200 import wire
    print(json.dumps(card()), flush=True)
    for name, (comp, lines) in shapes(args.records).items():
        recs = log_records(lines)
        msg = wire.frame_delimited(recs)
        comp.clock = lambda: 1773848383
        dev = comp._parse_device(msg, True)
        comp.n_parsed = 0                                        # (the same parsedLogIDs for the host's reply)
        assert dev == comp._parse_host(msg, True), "device and host replies differ"
        t = {"device": [], "host": []}
        for i in range(max(args.calls, args.host_calls)):
            for arm in ("device", "host"):
                if arm == "host" and i >= args.host_calls:
                    continue
                t0 = time.perf_counter()
                comp._parse_device(msg, True) if arm == "device" else comp._parse_host(msg, True)
                t[arm].append((time.perf_counter() - t0) * 1e3)
        row = {"shape": name, "records": len(recs), "in_bytes": len(msg), "out_bytes": len(dev)}
        for arm, v in t.items():
            row[arm + "_ms"] = {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3),
                                "calls": len(v)}
        row["kernel_us"] = kernel_times(lambda: comp._parse_device(msg, True), 10)
        print(json.dumps(row), flush=True)
        # bare records: one LogSchema per message, host against device, alternately
        bt = {"device": [], "host": []}
        for rec in recs[:args.bare]:
            for arm in ("device", "host"):
                t0 = time.perf_counter()
                comp._parse_device(rec, False) if arm == "device" else comp._parse_host(rec, False)
                bt[arm].append((time.perf_counter() - t0) * 1e6)
        print(json.dumps({"shape": name, "bare_records": len(bt["host"]),
                          **{arm + "_us": {"median": round(statistics.median(v), 1), "min": round(min(v), 1),
                                           "max": round(max(v), 1)} for arm, v in bt.items()}}), flush=True)
        comp.close()


if __name__ == "__main__":
    main()
