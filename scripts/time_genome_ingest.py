"""Genome sketches from host memory: 1 Gbp per call (250 genomes of 4 Mbp, synth.db_chunk) and one large call, from
pinned ASCII, pageable ASCII and host 2-bit words, with this tree's library and, alternating with it in separate
processes, another build (--other-lib, e.g. the parent commit's).  Per configuration: call time (host clock around the
call, which ends in a device synchronisation; warm-up calls first, median and min-max of the rest), k_seed and genome
post-pass time summed over the call (syl_ctx_kernel_time), H2D bytes (syl_ctx_ingest_stats; counted by the chunked
feeder only), the device peak of a fresh ctx (block cache plus staging rings) and a digest of the result, which must
agree between the two libraries.  Prints one JSON document with the card's name and power limit.

    python scripts/time_genome_ingest.py [--other-lib PATH] [--rounds 2] [--reps 5] [--large-gbp 8] [--out F]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GLEN = 4_000_000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def batch(n_genomes):
    """pinned ASCII of genomes [0, n_genomes) of GLEN bases, one contig each"""
    import torch
    from sylph_b200 import synth
    buf = torch.empty(n_genomes * GLEN, dtype=torch.uint8).pin_memory()
    for g0 in range(0, n_genomes, 100):
        g1 = min(n_genomes, g0 + 100)
        b, _ = synth.db_chunk(g0, g1, GLEN, device="cuda")
        buf[g0 * GLEN:g1 * GLEN].copy_(b.cpu())
    return buf


def worker(a):
    """one process, one library: every workload and source, printed as JSON lines"""
    import sylph_b200
    from sylph_b200.api import pack2
    for label, n_genomes, reps, warmup in (("1gbp", 250, a.reps, a.warmup), ("large", int(a.large_gbp * 1e9) // GLEN, 2, 1)):
        if n_genomes == 0:
            continue
        pinned = batch(n_genomes)
        coff = np.arange(n_genomes + 1, dtype=np.uint64) * GLEN
        goff = np.arange(n_genomes + 1, dtype=np.uint64)
        sources = {"pinned-ascii": pinned, "pageable-ascii": np.array(pinned.numpy()), "host-words": pack2(pinned.numpy())}
        for src, b in sources.items():
            kw = {"packed_bases": len(pinned)} if src == "host-words" else {}
            ctx = sylph_b200.Context(0)
            ctx.enable_timing(True)
            times, digest = [], None
            for r in range(warmup + reps):
                ctx.kernel_time("seed", reset=True)
                ctx.kernel_time("genome_post", reset=True)
                t0 = time.perf_counter()
                g = ctx.sketch_genomes(b, coff, goff, **kw)
                t1 = time.perf_counter()
                if r >= warmup:
                    times.append((t1 - t0) * 1e3)
                if digest is None:
                    d = g.download()
                    h = hashlib.sha256()
                    for key in ("kmers", "kmer_off", "tracked", "tracked_off", "gn_size"):
                        h.update(np.ascontiguousarray(d[key]).tobytes())
                    digest = h.hexdigest()[:16]
                g.free()
            seed_ms = ctx.kernel_time("seed")[0]
            post_ms = ctx.kernel_time("genome_post")[0]
            h2d = ctx.ingest_stats()[0]
            peak = ctx.device_bytes()[1] + ctx.ingest_ring_bytes()[0]
            ctx.close()
            print(json.dumps(dict(workload=label, gbp=len(pinned) / 1e9, source=src, ms_median=float(np.median(times)),
                                  ms_min=min(times), ms_max=max(times), reps=len(times), k_seed_ms=seed_ms,
                                  genome_post_ms=post_ms, h2d_bytes=h2d, device_peak_bytes=peak, digest=digest)), flush=True)
        del pinned, sources


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other-lib", default=None, help="another build of the library to alternate with")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--large-gbp", type=float, default=8.0)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a)
        return
    name, power = card()
    libs = {"this": None}
    if a.other_lib:
        libs["other"] = os.path.abspath(a.other_lib)
    rows = []
    for rnd in range(a.rounds):
        for tag, lib in libs.items():
            env = dict(os.environ)
            env.pop("SYLPH_B200_LIB", None)
            if lib:
                env["SYLPH_B200_LIB"] = lib
            args = [sys.executable, os.path.abspath(__file__), "--worker", "--reps", str(a.reps), "--warmup", str(a.warmup),
                    "--large-gbp", str(a.large_gbp)]
            out = subprocess.run(args, env=env, stdout=subprocess.PIPE, text=True, check=True, cwd=ROOT).stdout
            for line in out.splitlines():
                if line.startswith("{"):
                    r = json.loads(line)
                    r.update(lib=tag, round=rnd)
                    rows.append(r)
                    print(json.dumps(r), file=sys.stderr, flush=True)
    doc = dict(card=name, power_limit=power, rows=rows)
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
