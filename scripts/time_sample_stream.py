"""Time query and profile of many samples streamed from host memory (syl_*_host_samples) against the same samples as
resident device handles (syl_sample_upload + syl_query / syl_profile, in the driver's batches of 2^22 pairs).

Workload: --samples synthetic samples (synth.reads with one seed each, sketched on the device and downloaded) against
--genomes synthetic 4 Mbp genomes, on one index and on shards cut at a quarter of the entries (4-5 shards).  Each
round runs the resident call, the streamed call from pageable arrays and from pinned arrays, one after the other; rows
of every streamed call must equal the resident rows.  Reports per variant the best and median ms per sample over the
rounds, the H2D bytes of the streamed calls, the ctx's device-memory peak plus the staging ring bytes, and the card's
name and power limit.  Prints JSON lines.

    python scripts/time_sample_stream.py [--samples 256] [--genomes 10000] [--reads 200000] [--rounds 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.db_scale import gpu_info  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(a[f], b[f]) for f in a.dtype.names)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=256)
    ap.add_argument("--genomes", type=int, default=10000)
    ap.add_argument("--reads", type=int, default=200_000, help="150 bp reads per sample")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    import sylph_b200
    from sylph_b200 import synth
    from sylph_b200.api import contain_params
    emit(card=gpu_info())
    ctx = sylph_b200.Context(0)
    t0 = time.time()
    g = synth.sketch_db_range(ctx, 0, args.genomes)
    d = g.download()
    g.free()
    db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200)
    N = int(d["kmer_off"][-1] + d["tracked_off"][-1])
    sh = ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200, max_entries=N // 4 + 1)
    emit(db_genomes=args.genomes, db_entries=N, shards=len(sh), db_s=round(time.time() - t0, 1))
    hs, cs, mrl = [], [], []
    for i in range(args.samples):
        bases, off = synth.reads(args.reads, seed=1000 + i, device="cuda")
        s = ctx.sketch_sequences(bases, off)
        h, c = s.download()
        hs.append(h.copy())
        cs.append(c.copy())
        mrl.append(s.mean_read_length)
        s.free()
    del bases, off
    off = np.concatenate([[0], np.cumsum([len(h) for h in hs])]).astype(np.uint64)
    H, C = np.concatenate(hs), np.concatenate(cs)
    mrl = np.array(mrl)
    pins = [torch.empty(a.nbytes, dtype=torch.uint8, pin_memory=True) for a in (H, C)]
    PH, PC = pins[0].numpy().view(np.uint64), pins[1].numpy().view(np.uint32)
    PH[:], PC[:] = H, C
    handles = []
    for h, c, m in zip(hs, cs, mrl):
        x = ctx.upload_sample(h, c, c=200)
        x.mean_read_length = float(m)
        handles.append(x)
    emit(samples=args.samples, kmers=int(off[-1]), sample_bytes=12 * int(off[-1]))
    per_call = max(1, (1 << 22) // args.genomes)
    for kind, target in (("one_index", db), ("shards", sh)):
        for cmd in ("query", "profile"):
            p = contain_params(pseudotax=cmd == "profile")

            def resident():
                if kind == "shards":
                    return target.profile(handles, p) if cmd == "profile" else target.query(handles, p)
                fn = ctx.profile if cmd == "profile" else ctx.query
                parts = []
                for s0 in range(0, len(handles), per_call):
                    r = fn(target, handles[s0:s0 + per_call], p)
                    r["sample"] += s0
                    parts.append(r)
                return np.concatenate(parts)

            def streamed(h, c):
                fn = ctx.profile_host_samples if cmd == "profile" else ctx.query_host_samples
                return fn(target, h, c, off, 200, mrl, p)

            variants = {"resident": resident, "pageable": lambda: streamed(H, C), "pinned": lambda: streamed(PH, PC)}
            times = {v: [] for v in variants}
            stats = {}
            want = resident()   # warm-up
            for v in ("pageable", "pinned"):
                assert same(variants[v](), want), (kind, cmd, v)
            for _ in range(args.rounds):
                for v, fn in variants.items():
                    h2d0 = ctx.ingest_stats()[0]
                    held, _ = ctx.device_bytes(reset_peak=True)
                    t = time.perf_counter()
                    rows = fn()
                    times[v].append((time.perf_counter() - t) * 1e3 / args.samples)
                    assert same(rows, want), (kind, cmd, v)
                    stats[v] = dict(h2d_bytes=ctx.ingest_stats()[0] - h2d0 if v != "resident" else 0,
                                    peak_device_bytes=ctx.device_bytes()[1], ring_device_bytes=ctx.ingest_ring_bytes()[0])
            for v in variants:
                emit(db=kind, cmd=cmd, variant=v, ms_per_sample_best=round(min(times[v]), 4),
                     ms_per_sample_median=round(float(np.median(times[v])), 4), rows=len(want), **stats[v])
    for x in handles:
        x.free()
    sh.free()
    db.free()
    ctx.close()


if __name__ == "__main__":
    main()
