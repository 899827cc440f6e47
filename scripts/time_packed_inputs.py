"""Time genome and read-pair sketching on ASCII against 2-bit packed input, on one GPU.

  python scripts/time_packed_inputs.py --out DIR [--steps 10] [--warmup 3] [--genomes 250] [--mates 3333333]

Workloads (synthetic, sylph_b200.synth):
  genomes  250 x 4 Mbp (synth.db_chunk), one contig each      syl_sketch_genomes / syl_sketch_genomes_packed2
  pairs    2 x 3.33 M mates of 150 bp, two synth.reads draws   syl_sketch_read_pairs / syl_sketch_read_pairs_packed2
each from device memory and from pinned host memory.  The words are packed once with pack2, outside the timed region.
Per step the ASCII and the packed call alternate.  Reported per call: milliseconds (CUDA events on the ctx stream around
the call, which ends in a synchronise), and in a second pass with the library's kernel timers on, the seeding kernel
and the genome post-pass.  h2d_bytes is what a host-memory call copies: the bases or words plus the offset arrays, one
copy each.  Packed and ASCII results are compared at the timed sizes.  Writes DIR/time_packed_inputs.json.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sylph_b200  # noqa: E402
from sylph_b200 import synth  # noqa: E402
from sylph_b200.api import pack2  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip()


def pinned(a):
    t = torch.empty(a.size, dtype={np.uint8: torch.uint8, np.uint32: torch.int32, np.uint64: torch.int64}[a.dtype.type],
                    pin_memory=True)
    t.numpy().view(a.dtype)[:] = a
    return t.numpy().view(a.dtype)


def timed(ctx, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return r, e0.elapsed_time(e1)


def run(ctx, variants, steps, warmup):
    """variants: name -> zero-argument call.  Alternates the variants every step; returns per-variant lists."""
    for _ in range(warmup):
        for fn in variants.values():
            fn().free()
    out = {n: {"ms": [], "seed_ms": [], "genome_post_ms": []} for n in variants}
    for _ in range(steps):
        for n, fn in variants.items():
            r, ms = timed(ctx, fn)
            r.free()
            out[n]["ms"].append(ms)
    ctx.enable_timing(True)
    ctx.kernel_time("seed", reset=True)
    ctx.kernel_time("genome_post", reset=True)
    for _ in range(steps):
        for n, fn in variants.items():
            fn().free()
            out[n]["seed_ms"].append(ctx.kernel_time("seed", reset=True)[0])
            out[n]["genome_post_ms"].append(ctx.kernel_time("genome_post", reset=True)[0])
    ctx.enable_timing(False)
    return out


def summary(v):
    a = np.array(v)
    return {"min": float(a.min()), "median": float(np.median(a)), "max": float(a.max())}


def same_genomes(a, b):
    da, db = a.download(), b.download()
    return all(np.array_equal(da[k], db[k]) for k in ("kmers", "kmer_off", "tracked", "tracked_off", "gn_size"))


def same_sample(a, b):
    (ha, ca), (hb, cb) = a.download(), b.download()
    return (np.array_equal(ha, hb) and np.array_equal(ca, cb) and a.num_dup_removed == b.num_dup_removed
            and a.mean_read_length == b.mean_read_length)


def genomes(ctx, n_genomes, steps, warmup):
    L = 4_000_000
    bases, off = synth.db_chunk(0, n_genomes, L, device="cuda")
    goff = torch.arange(n_genomes + 1, dtype=torch.int64, device="cuda")
    n = bases.numel()
    h_bases = bases.cpu().numpy()
    h_words = pack2(h_bases)
    d_words = torch.from_numpy(h_words.view(np.int32)).cuda()
    h_off, h_goff = off.cpu().numpy().view(np.uint64), goff.cpu().numpy().view(np.uint64)
    p_bases, p_words, p_off, p_goff = pinned(h_bases), pinned(h_words), pinned(h_off), pinned(h_goff)
    del h_bases
    res = {"bases": n, "h2d_bytes": {"ascii": n + 8 * (h_off.size + h_goff.size),
                                     "packed": 4 * h_words.size + 8 * (h_off.size + h_goff.size)}}
    modes = {
        "device": {"ascii": lambda: ctx.sketch_genomes(bases, off, goff),
                   "packed": lambda: ctx.sketch_genomes(d_words, off, goff, packed_bases=n)},
        "pinned_host": {"ascii": lambda: ctx.sketch_genomes(p_bases, p_off, p_goff),
                        "packed": lambda: ctx.sketch_genomes(p_words, p_off, p_goff, packed_bases=n)},
    }
    for mode, variants in modes.items():
        a, p = variants["ascii"](), variants["packed"]()
        assert same_genomes(a, p), "genomes %s: packed != ASCII" % mode
        res.setdefault("total_kmers", int(a.download()["kmers"].size))
        a.free()
        p.free()
        r = run(ctx, variants, steps, warmup)
        res[mode] = {n_: {k: summary(v) for k, v in x.items()} for n_, x in r.items()}
    return res


def pairs(ctx, n_mates, steps, warmup):
    b1, o1 = synth.reads(n_mates, device="cuda", seed=synth.SEED_READS)
    b2, o2 = synth.reads(n_mates, device="cuda", seed=synth.SEED_READS + 0x100)
    h1, h2 = b1.cpu().numpy(), b2.cpu().numpy()
    w1, w2 = pack2(h1), pack2(h2)
    d1, d2 = torch.from_numpy(w1.view(np.int32)).cuda(), torch.from_numpy(w2.view(np.int32)).cuda()
    ho1, ho2 = o1.cpu().numpy().view(np.uint64), o2.cpu().numpy().view(np.uint64)
    p1, p2, pw1, pw2, po1, po2 = pinned(h1), pinned(h2), pinned(w1), pinned(w2), pinned(ho1), pinned(ho2)
    n = h1.size + h2.size
    del h1, h2
    res = {"bases": n, "pairs": n_mates, "h2d_bytes": {"ascii": n + 8 * (ho1.size + ho2.size),
                                                        "packed": 4 * (w1.size + w2.size) + 8 * (ho1.size + ho2.size)}}
    modes = {
        "device": {"ascii": lambda: ctx.sketch_pair_sequences(b1, o1, b2, o2),
                   "packed": lambda: ctx.sketch_pair_sequences(d1, o1, d2, o2, packed=True)},
        "pinned_host": {"ascii": lambda: ctx.sketch_pair_sequences(p1, po1, p2, po2),
                        "packed": lambda: ctx.sketch_pair_sequences(pw1, po1, pw2, po2, packed=True)},
    }
    for mode, variants in modes.items():
        a, p = variants["ascii"](), variants["packed"]()
        assert same_sample(a, p), "pairs %s: packed != ASCII" % mode
        res.setdefault("sketch_size", len(a))
        res.setdefault("num_dup_removed", a.num_dup_removed)
        a.free()
        p.free()
        r = run(ctx, variants, steps, warmup)
        res[mode] = {n_: {k: summary(v) for k, v in x.items()} for n_, x in r.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--genomes", type=int, default=250)
    ap.add_argument("--mates", type=int, default=3_333_333)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    os.makedirs(a.out, exist_ok=True)
    ctx = sylph_b200.Context(0, stream=torch.cuda.current_stream().cuda_stream)
    res = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(0), "steps": a.steps, "warmup": a.warmup}
    res["genomes"] = genomes(ctx, a.genomes, a.steps, a.warmup)
    torch.cuda.empty_cache()
    res["pairs"] = pairs(ctx, a.mates, a.steps, a.warmup)
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out, "time_packed_inputs.json"), "w") as f:
        json.dump(res, f, indent=1)
    for w in ("genomes", "pairs"):
        for mode in ("device", "pinned_host"):
            for fmt in ("ascii", "packed"):
                x = res[w][mode][fmt]
                print("%-8s %-12s %-7s call %7.2f ms [%.2f-%.2f]  seed %6.3f ms  genome_post %6.3f ms  h2d %d B"
                      % (w, mode, fmt, x["ms"]["median"], x["ms"]["min"], x["ms"]["max"], x["seed_ms"]["median"],
                         x["genome_post_ms"]["median"], res[w]["h2d_bytes"][fmt]))
    print(res["gpu"])


if __name__ == "__main__":
    main()
