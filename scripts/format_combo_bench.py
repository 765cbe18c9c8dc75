#!/usr/bin/env python
"""log_format + template mode with single-value monitors against the same fields as NewValueComboDetector
combinations, on the workload of scripts/format_bench.py (64k x 256 B audit records per message, one template),
device-resident, CUDA events on the launching stream.

  arms      single   global `type` + event-scoped acct, exe, terminal, res (format_bench.py's configuration)
            combo    the same fields as combinations: (type), (acct, exe, terminal, res), (acct, exe); every
                     monitor member-only
  --runs N  every arm runs N times in its own process, arms alternating (`--parent-lib PATH` adds the single arm on
            another build of libdmdetect.so, loaded through DM_LIB_PATH, so that two builds can be compared)

Prints one JSON line per run and a summary: median and range of ms per message, and whether the flags and scores
of the last message agree between builds."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

AUDIT = "type=<type> msg=audit(<Time>): <Content>"
TMPL = "pid=<*> uid=<*> auid=<*> ses=<*> msg='op=<*> acct=<*> exe=<*> hostname=<*> addr=<*> terminal=<*> res=<*>' pad=<*>"
PAM = [{"pos": 5, "name": "acct"}, {"pos": 6, "name": "exe"}, {"pos": 9, "name": "terminal"}, {"pos": 10, "name": "res"}]
LINES = 65536


def configs():
    single = {"detectors": {"NewValueDetector": {"method_type": "new_value_detector", "data_use_training": LINES,
              "global": {"g": {"header_variables": [{"pos": "type"}]}}, "events": {0: {"pam": {"variables": PAM}}}}}}
    combo = {"detectors": {"NewValueComboDetector": {"method_type": "new_value_combo_detector", "data_use_training": LINES,
             "global": {"g": {"header_variables": [{"pos": "type"}]}},
             "events": {0: {"pam": {"variables": PAM}, "pair": {"variables": PAM[:2]}}}}}}
    return single, combo


def child(arm, steps, warmup, n_msgs):
    import torch
    from detectmateservice_b200.component import parse_combos, parse_monitors, select_component_config
    from detectmateservice_b200.detector import DeviceDetector
    from detectmateservice_b200.synth import AuditSynth
    single, combo = configs()
    if arm == "combo":
        mons, combos = parse_combos(select_component_config(combo, "NewValueComboDetector"))
    else:
        mons, combos = parse_monitors(select_component_config(single, "NewValueDetector")), []
    g = AuditSynth(seed=7)
    msgs = [g.batch(LINES, inject=(i > 0))[0] for i in range(n_msgs)]
    dev = torch.device("cuda:0")
    bufs = []
    for m in msgs:
        t = torch.zeros(len(m) + 64, dtype=torch.uint8, device=dev)
        t[:len(m)] = torch.frombuffer(bytearray(m), dtype=torch.uint8).to(dev)
        bufs.append(t)
    flags = torch.zeros(LINES, dtype=torch.uint8, device=dev)
    scores = torch.zeros(LINES, dtype=torch.float32, device=dev)
    det = DeviceDetector([m.key for m in mons], max_batch_bytes=32 << 20)
    det.set_monitors([{"event_id": m.event_id, "source": m.source, "pos": m.pos} for m in mons])
    det.set_format(AUDIT, [TMPL])
    if combos:
        det.set_combos(combos, member_only_mask=(1 << len(mons)) - 1)
    st = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(st):
        det.enqueue_device(bufs[0].data_ptr(), len(msgs[0]), LINES, flags.data_ptr(), scores.data_ptr(), LINES, st.cuda_stream)
        for i in range(warmup):
            j = 1 + i % (n_msgs - 1)
            det.enqueue_device(bufs[j].data_ptr(), len(msgs[j]), 0, flags.data_ptr(), scores.data_ptr(), LINES, st.cuda_stream)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        st.synchronize()
        e0.record(st)
        for i in range(steps):
            j = 1 + i % (n_msgs - 1)
            det.enqueue_device(bufs[j].data_ptr(), len(msgs[j]), 0, flags.data_ptr(), scores.data_ptr(), LINES, st.cuda_stream)
        e1.record(st)
        st.synchronize()
    det.sync()
    ms = e0.elapsed_time(e1) / steps
    digest = hashlib.sha256(flags.cpu().numpy().tobytes() + scores.cpu().numpy().tobytes()).hexdigest()[:16]
    det.close()
    print(json.dumps({"arm": arm, "ms_per_message": round(ms, 4), "lines_per_s": round(LINES / ms * 1e3, 1),
                      "anomalies_last_message": int(flags.sum().item()), "outputs_sha256": digest}))


def gpu_label():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--messages", type=int, default=8)
    ap.add_argument("--parent-lib", default=None, help="another libdmdetect.so to run the single arm on")
    ap.add_argument("--child", choices=["single", "combo"], default=None)
    a = ap.parse_args()
    if a.child:
        child(a.child, a.steps, a.warmup, a.messages)
        return
    arms = [("single", "single", None), ("combo", "combo", None)]
    if a.parent_lib:
        arms.append(("single@parent", "single", os.path.abspath(a.parent_lib)))
    res = {label: [] for label, _, _ in arms}
    for _ in range(a.runs):
        for label, arm, lib in arms:
            env = dict(os.environ)
            env.pop("DM_LIB_PATH", None)
            if lib:
                env["DM_LIB_PATH"] = lib
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", arm, "--steps", str(a.steps),
                                  "--warmup", str(a.warmup), "--messages", str(a.messages)],
                                 capture_output=True, text=True, env=env, check=True).stdout.strip().splitlines()[-1]
            r = dict(json.loads(out), label=label)
            print(json.dumps(r), flush=True)
            res[label].append(r)
    summary = {"workload": "64k x 256 B audit records per message, log_format + 1 template, device-resident",
               "gpu": gpu_label(), "runs": a.runs}
    for label, rs in res.items():
        ms = [r["ms_per_message"] for r in rs]
        summary[label] = {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms),
                          "outputs_sha256": sorted({r["outputs_sha256"] for r in rs})}
    if a.parent_lib:
        summary["single_outputs_identical_across_builds"] = (
            summary["single"]["outputs_sha256"] == summary["single@parent"]["outputs_sha256"])
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
