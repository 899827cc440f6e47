"""Cost of sketching a sample in hash-range parts: 1 Gbp of 150 bp reads and of 150 bp read pairs, from device memory
and from pinned host memory (ASCII), at P = 1, 2, 4 and 8 (SYL_SAMPLE_PARTS).  Per configuration: call time (host
clock around the call, which ends in a device synchronisation; warm-up calls first, median and min-max of the rest),
k_seed and k_group_dedup time summed over the call (syl_ctx_kernel_time), peak device bytes of the block cache plus the
staging rings, and whether the sketch equals the one-pass sketch.  Prints one JSON document with the card's name and
power limit.

    python scripts/time_sample_parts.py [--reps 5] [--warmup 2] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
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


def inputs(n_bases, paired, seed=1):
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    mates = 2 if paired else 1
    n = n_bases // (150 * mates)
    off = np.arange(n + 1, dtype=np.uint64) * 150
    return [(acgt[rng.integers(0, 4, n * 150, dtype=np.uint8)], off) for _ in range(mates)]


def place(data, mem):
    import torch
    out = []
    for b, o in data:
        tb, to = torch.from_numpy(b), torch.from_numpy(o.view(np.int64))
        out.append((tb.cuda(), to.cuda()) if mem == "device" else (tb.pin_memory(), to.pin_memory()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--gbp", type=float, default=1.0)
    ap.add_argument("--c", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import sylph_b200
    name, power = card()
    rows = []
    for paired in (False, True):
        host = inputs(int(a.gbp * 1e9), paired)
        for mem in ("device", "pinned"):
            data = place(host, mem)
            ctx = sylph_b200.Context(0)
            ctx.enable_timing(True)
            ref = None
            for P in (1, 2, 4, 8):
                os.environ["SYL_SAMPLE_PARTS"] = str(P)

                def call():
                    if paired:
                        (b1, o1), (b2, o2) = data
                        return ctx.sketch_pair_sequences(b1, o1, b2, o2, c=a.c)
                    (b, o), = data
                    return ctx.sketch_sequences(b, o, c=a.c)
                for _ in range(a.warmup):
                    call().free()
                ctx.kernel_time("seed")
                ctx.kernel_time("group_dedup")
                ts, seed_ms, grp_ms, peaks = [], [], [], []
                for _ in range(a.reps):
                    ctx.device_bytes(reset_peak=True)
                    t0 = time.perf_counter()
                    s = call()
                    ts.append((time.perf_counter() - t0) * 1e3)
                    peaks.append(ctx.device_bytes()[1] + ctx.ingest_ring_bytes()[0])
                    seed_ms.append(ctx.kernel_time("seed")[0])
                    grp_ms.append(ctx.kernel_time("group_dedup")[0])
                    h, cnt = s.download()
                    if ref is None:
                        ref = (h.copy(), cnt.copy(), s.num_dup_removed)
                    same = bool(np.array_equal(h, ref[0]) and np.array_equal(cnt, ref[1]) and s.num_dup_removed == ref[2])
                    s.free()
                rows.append(dict(input="pairs" if paired else "reads", mem=mem, parts=P, actual_parts=ctx.sample_parts(),
                                 call_ms_median=float(np.median(ts)), call_ms_min=min(ts), call_ms_max=max(ts),
                                 k_seed_ms_median=float(np.median(seed_ms)), group_dedup_ms_median=float(np.median(grp_ms)),
                                 peak_device_plus_ring_bytes=int(max(peaks)), equal_to_one_pass=same))
                print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
            os.environ.pop("SYL_SAMPLE_PARTS", None)
            ctx.close()
            del data
    doc = dict(card=name, power_limit=power, gbp=a.gbp, c=a.c, reps=a.reps, warmup=a.warmup, rows=rows)
    js = json.dumps(doc, indent=1)
    print(js)
    if a.out:
        with open(a.out, "w") as f:
            f.write(js)


if __name__ == "__main__":
    main()
