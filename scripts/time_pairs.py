"""Time the read-pair sketch: this build's default post-pass (pair dedup inside k_group_dedup) against the generic
sorted one (SYL_SAMPLE_POSTPASS=sort, read per call), alternated in one process on one GPU.

  python scripts/time_pairs.py --out DIR [--steps 10] [--warmup 3] [--mates 3333333]

Workloads (synthetic, sylph_b200.synth; 2 x 3 333 333 mates of 150 bp = 1 Gbp):
  pairs        two synth.reads draws (2 % of each draw's reads repeat another read of the draw; the pairs do not)
  pairs+dup    the same with 2 % of the pairs replaced by a copy of an earlier pair, so the pair dedup has work
each device-resident and from pinned host ASCII.  Per call: milliseconds from a host clock around the call (it ends
in a synchronise), and in a second pass with the library's kernel timers on, the seeding kernels and k_group_dedup.
Also printed: the card and its power limit, the H2D bytes and chunks of a host call, the share of the slotted events
the group kernel hands to the generic path (from the post-pass's SYL_DEBUG_TIMING report, in a child process), and
the sketches of the two paths are asserted identical.  Fails without a GPU.  Writes DIR/time_pairs.json.

On a build whose library reads SYL_SAMPLE_POSTPASS once per process, or sends every pair sample through the sorted
post-pass, both columns time the same path: that is how the numbers before the group path were taken.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sylph_b200  # noqa: E402
from sylph_b200 import synth  # noqa: E402

PATHS = {"group": None, "sort": "sort"}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip()


def pinned(t):
    p = torch.empty(t.numel(), dtype=t.dtype, pin_memory=True)
    p.copy_(t)
    return p


def workloads(n_mates):
    """name -> (bases1, off1, bases2, off2) on the device"""
    b1, o1 = synth.reads(n_mates, seed=synth.SEED_READS, device="cuda")
    b2, o2 = synth.reads(n_mates, seed=synth.SEED_READS + 1000, device="cuda")
    out = {"pairs": (b1, o1, b2, o2)}
    g = torch.Generator(device="cpu").manual_seed(5)
    dst = torch.randperm(n_mates, generator=g)[:n_mates // 50]
    dst = dst[dst > 0]
    src = (torch.rand(dst.numel(), generator=g, dtype=torch.float64) * dst.to(torch.float64)).to(torch.int64)
    d1, d2 = b1.clone().view(n_mates, -1), b2.clone().view(n_mates, -1)
    d1[dst.cuda()] = b1.view(n_mates, -1)[src.cuda()]
    d2[dst.cuda()] = b2.view(n_mates, -1)[src.cuda()]
    out["pairs+dup"] = (d1.view(-1), o1, d2.view(-1), o2)
    return out


def call(ctx, args, path, c):
    if PATHS[path]:
        os.environ["SYL_SAMPLE_POSTPASS"] = PATHS[path]
    else:
        os.environ.pop("SYL_SAMPLE_POSTPASS", None)
    return ctx.sketch_pair_sequences(*args, c=c)


def time_workload(ctx, args, steps, warmup, c):
    out = {p: {"ms": [], "seed_ms": [], "group_dedup_ms": []} for p in PATHS}
    ref = None
    for p in PATHS:
        for _ in range(warmup):
            s = call(ctx, args, p, c)
            got = s.download() + (s.num_dup_removed,)
            s.free()
            assert ref is None or (np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1]) and ref[2] == got[2]), p
            ref = got
    out["sketch"] = {"kmers": int(len(ref[0])), "num_dup_removed": int(ref[2])}
    for timing in (False, True):
        ctx.enable_timing(timing)
        for _ in range(steps):
            for p in PATHS:
                torch.cuda.synchronize()
                ctx.kernel_time("seed", reset=True)
                ctx.kernel_time("group_dedup", reset=True)
                t0 = time.perf_counter()
                s = call(ctx, args, p, c)
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1e3
                s.free()
                if timing:
                    out[p]["seed_ms"].append(ctx.kernel_time("seed", reset=True)[0])
                    out[p]["group_dedup_ms"].append(ctx.kernel_time("group_dedup", reset=True)[0])
                else:
                    out[p]["ms"].append(ms)
    ctx.enable_timing(False)
    return out


def probe(n_mates, c):
    """child process: one device-resident call per workload with the post-pass's report on stderr"""
    ctx = sylph_b200.Context(0)
    for name, args in workloads(n_mates).items():
        print("@@ " + name, file=sys.stderr, flush=True)
        call(ctx, args, "group", c).free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mates", type=int, default=3333333)
    ap.add_argument("-c", type=int, default=200)
    ap.add_argument("--probe", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_pairs.py needs a GPU")
    if a.probe:
        return probe(a.mates, a.c)
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info(), "steps": a.steps, "warmup": a.warmup, "mates": a.mates, "c": a.c, "workloads": {}}
    print("GPU (name, power limit, max SM clock):", res["gpu"])
    ctx = sylph_b200.Context(0)
    med = lambda v: float(np.median(v)) if v else float("nan")
    for name, dev in workloads(a.mates).items():
        host = tuple(pinned(t).numpy() if i % 2 == 0 else pinned(t).numpy().view(np.uint64) for i, t in enumerate(dev))
        for where, args in (("device", dev), ("pinned host ASCII", host)):
            r = time_workload(ctx, args, a.steps, a.warmup, a.c)
            if where != "device":
                r["h2d_bytes"], r["chunks_packed"], r["chunks_ascii"] = ctx.ingest_stats()
            res["workloads"]["%s, %s" % (name, where)] = r
            for p in PATHS:
                print("%-10s %-18s %-5s call %7.2f ms (min %7.2f, max %7.2f; %d calls)  seed %6.2f ms  k_group_dedup %5.2f ms"
                      % (name, where, p, med(r[p]["ms"]), min(r[p]["ms"]), max(r[p]["ms"]), len(r[p]["ms"]),
                         med(r[p]["seed_ms"]), med(r[p]["group_dedup_ms"])))
            if where != "device":
                print("%-10s %-18s H2D %.1f MB, %d chunks packed, %d ASCII" % (name, where, r["h2d_bytes"] / 1e6,
                                                                               r["chunks_packed"], r["chunks_ascii"]))
        del host
    env = dict(os.environ, SYL_DEBUG_TIMING="1")
    env.pop("SYL_SAMPLE_POSTPASS", None)
    pr = subprocess.run([sys.executable, os.path.abspath(__file__), "--probe", "--out", a.out, "--mates", str(a.mates), "-c", str(a.c)],
                        env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    for block in pr.stderr.split("@@ ")[1:]:
        name, body = block.split("\n", 1)
        m = re.findall(r"events handed to the generic path (\d+) \(([0-9.]+) % of the slotted events\)", body)
        res["workloads"].setdefault(name + ", device", {})["generic_path"] = m[-1] if m else None
        print("%-10s events handed to the generic path: %s" % (name, "%s (%s %% of the slotted events)" % m[-1] if m else
                                                               "no group post-pass ran"))
    with open(os.path.join(a.out, "time_pairs.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
