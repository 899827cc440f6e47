"""Where the time of a read sketch goes after the seeding kernel: bench.py's flagship workload (synth.reads(6_666_667,
150), k=31, c=200, device-resident ASCII input) and, with --pairs, 1 Gbp of read pairs (two synth.reads draws).

Two runs per workload, the second only with --trace:
  timed   host clock around the call, which ends in a device synchronisation (warm-up calls first; median and min-max of
          the rest), and the library's per-kernel CUDA-event timers (syl_ctx_kernel_time) for k_seed and k_group_dedup.
  trace   torch.profiler with CUDA activities around --trace calls.  Per call: every kernel, copy and memset that runs
          after the last k_seed launch ends, the span from that end to the last device activity, and the span from it
          to the call's return on the host (profiling stretches the host-side part of that span).
Prints one JSON document with the card's name and power limit; SYLPH_B200_LIB selects another build of the library.

    python scripts/time_sample_post.py [--pairs] [--reps 10] [--warmup 3] [--trace 5] [--out results.json]
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def workload(paired):
    from sylph_b200 import synth
    if not paired:
        b, o = synth.reads(6_666_667, 150, device="cuda")
        return lambda ctx: ctx.sketch_sequences(b, o, k=31, c=200)
    b1, o1 = synth.reads(3_333_333, 150, seed=synth.SEED_READS, device="cuda")
    b2, o2 = synth.reads(3_333_333, 150, seed=synth.SEED_READS + 1000, device="cuda")
    return lambda ctx: ctx.sketch_pair_sequences(b1, o1, b2, o2, k=31, c=200)


def timed(ctx, call, reps, warmup):
    import torch
    for _ in range(warmup):
        call(ctx).free()
    torch.cuda.synchronize()
    ctx.enable_timing(True)
    ctx.kernel_time("seed")
    ctx.kernel_time("group_dedup")
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        s = call(ctx)
        ts.append((time.perf_counter() - t0) * 1e3)
        n, ndup = len(s), s.num_dup_removed
        s.free()
    seed_ms, seed_n = ctx.kernel_time("seed")
    grp_ms, grp_n = ctx.kernel_time("group_dedup")
    ctx.enable_timing(False)
    return {"call_ms_median": float(np.median(ts)), "call_ms_min": min(ts), "call_ms_max": max(ts),
            "k_seed_ms_per_call": seed_ms / reps, "k_seed_launches_per_call": seed_n / reps,
            "k_group_dedup_ms_per_call": grp_ms / reps, "sketch_entries": n, "num_dup_removed": ndup}


def traced(ctx, call, calls):
    """per call: the device activities after the last k_seed ends and the spans from that end"""
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    call(ctx).free()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(calls):
            with record_function("sketch_call_%d" % i):
                s = call(ctx)
            s.free()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            tr = json.load(f)
    ev = tr["traceEvents"] if isinstance(tr, dict) else tr
    calls_w = sorted((e["ts"], e["ts"] + e["dur"]) for e in ev
                     if e.get("ph") == "X" and str(e.get("name", "")).startswith("sketch_call_") and
                     e.get("cat") == "user_annotation")
    dev = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    per_name = collections.defaultdict(list)
    spans_dev, spans_ret, busy = [], [], []
    for c0, c1 in calls_w:
        mine = sorted((e for e in dev if c0 <= e["ts"] <= c1), key=lambda e: e["ts"])
        seeds = [e for e in mine if e["name"].startswith("void syl::k_seed") or "k_seed<" in e["name"]]
        if not seeds:
            continue
        t_seed = max(e["ts"] + e["dur"] for e in seeds)
        post = [e for e in mine if e["ts"] >= t_seed - 1e-3 and e not in seeds]
        t_last = max([e["ts"] + e["dur"] for e in post], default=t_seed)
        spans_dev.append(t_last - t_seed)
        spans_ret.append(c1 - t_seed)
        busy.append(sum(e["dur"] for e in post))
        names = collections.Counter()
        for e in post:
            nm = e["name"].split("(")[0].replace("void ", "")
            names[nm] += 1
            per_name[nm].append(e["dur"])
    n = max(len(spans_dev), 1)
    table = sorted(({"name": k, "us_per_call": sum(v) / n, "launches_per_call": len(v) / n} for k, v in per_name.items()),
                   key=lambda r: -r["us_per_call"])
    return {"calls": len(spans_dev),
            "seed_end_to_last_device_activity_us": float(np.median(spans_dev)) if spans_dev else None,
            "seed_end_to_return_us": float(np.median(spans_ret)) if spans_ret else None,
            "post_pass_device_busy_us": float(np.median(busy)) if busy else None,
            "post_pass": table}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", action="store_true", help="also the 1 Gbp read-pair sketch")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--trace", type=int, default=0, help="calls under torch.profiler (0: no trace run)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import sylph_b200
    from sylph_b200 import _lib
    _lib.lib()
    name, power = card()
    res = {"card": name, "power_limit": power, "library": os.environ.get("SYLPH_B200_LIB", "in-tree"),
           "sample_parts": os.environ.get("SYL_SAMPLE_PARTS", "auto"), "runs": []}
    for paired in ([False, True] if a.pairs else [False]):
        call = workload(paired)
        ctx = sylph_b200.Context(0)
        row = {"workload": "1 Gbp of 150 bp %s, k=31, c=200, device ASCII" % ("read pairs" if paired else "reads")}
        row.update(timed(ctx, call, a.reps, a.warmup))
        if a.trace:
            row["trace"] = traced(ctx, call, a.trace)
        res["runs"].append(row)
        ctx.close()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
