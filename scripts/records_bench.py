#!/usr/bin/env python
"""Throughput of record mode (SURVEY.md section 8 row f2): one message of length-delimited ParserSchema
records through dm_process_records -- host framing scan, H2D, the decode + detect kernel
(dm_kernels_records.cuh), flags/scores/masks back.  Two figures per message size: the whole call on the
host clock (what a caller sees) and the detect kernel alone from the library's own CUDA-event marks
(dm_profile_enable), with its HBM roofline fraction: algorithmic bytes = the record bytes, read once.
Not the headline metric; quoted in DESIGN.md."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from detectmateservice_b200 import wire
from detectmateservice_b200.component import parse_monitors, select_component_config
from detectmateservice_b200.detector import DeviceDetector

CFG = {"detectors": {"NewValueDetector": {
    "method_type": "new_value_detector", "data_use_training": 0,
    "global": {"g": {"header_variables": [{"pos": "type"}, {"pos": "res"}]}},
    "events": {0: {"pam": {"variables": [{"pos": 4, "name": "op"}, {"pos": 6, "name": "exe"}, {"pos": 9, "name": "terminal"}]}},
               2: {"login": {"variables": [{"pos": 3, "name": "auid"}]}}}}}}


def make_message(n, seed, novel):
    """n ParserSchema records shaped like the MatcherParser output for audit lines (~330 B each)."""
    r = np.random.Generator(np.random.PCG64(seed))
    types = ["USER_ACCT", "CRED_ACQ", "LOGIN", "USER_START", "SERVICE_START"]
    parts = []
    for i in range(n):
        t = types[int(r.integers(0, len(types)))]
        exe = "/usr/sbin/cron" if not (novel and r.random() < 1e-3) else "/tmp/x%d" % i
        var = ["%d" % r.integers(100, 30000), "0", "4294967295", "4294967295", "PAM:accounting", '"root"', exe, "?", "?", "cron", "success"]
        rec = {"EventID": int(r.integers(0, 3)), "logID": str(i), "parserType": "matcher_parser", "parserID": "MatcherParser",
               "variables": var, "logFormatVariables": {"type": t, "Time": "1642723741.%03d:%d" % (i % 1000, i), "res": "success"},
               "receivedTimestamp": 1642723741, "parsedTimestamp": 1642723742,
               "log": "type=%s msg=audit(1642723741.072:%d): pid=%s uid=0 auid=4294967295 ses=4294967295 msg='op=PAM:accounting'" % (t, i, var[0])}
        b = wire.encode_parser_schema(rec)
        ln = bytearray()
        wire._write_varint(ln, len(b))
        parts.append(bytes(ln) + b)
    return b"".join(parts)


def main():
    import torch
    mons = parse_monitors(select_component_config(CFG, "NewValueDetector"))
    out = {"workload": "length-delimited ParserSchema records (~330 B), dm_process_records, host buffers", "sizes": {}}
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = float(peaks.get("hbm_gbs") or 3350.0)          # else the H100 SXM data sheet's HBM3 3.35 TB/s, as bench.py
    for n in (16384, 65536, 262144):
        train = make_message(n, 1, False)
        msgs = [make_message(n, 2 + i, True) for i in range(3)]
        det = DeviceDetector([m.key for m in mons], max_batch_bytes=max(len(m) for m in msgs + [train]) + 4096, max_lines=n + 16)
        det.set_monitors([{"event_id": m.event_id, "source": m.source, "pos": m.pos} for m in mons])
        det.process_records(train, n_train_records=n)
        for m in msgs:
            det.process_records(m)                                # warm-up
        det.profile_enable(True)
        reps = 12
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        anom = 0
        for i in range(reps):
            f, s, k = det.process_records(msgs[i % len(msgs)])
            anom += int(f.sum())
        dt = (time.perf_counter() - t0) / reps
        kms, n_timed, _ = det.profile_read()
        kms /= max(1, n_timed)
        nbytes = sum(len(m) for m in msgs) / len(msgs)
        out["sizes"][str(n)] = {"message_bytes": int(nbytes), "call_ms": round(dt * 1e3, 3), "records_per_s_call": round(n / dt, 1),
                                "kernel_ms": round(kms, 4), "records_per_s_kernel": round(n / kms * 1e3, 1),
                                "kernel_GBps": round(nbytes / kms / 1e6, 1), "roofline_frac": round(nbytes / kms / 1e6 / peak, 4),
                                "anomalies_per_message": anom / reps}
        det.close()
    out["hbm_peak_GBps"] = peak
    print(json.dumps(out))


if __name__ == "__main__":
    main()
