"""Time query and profile calls on a host-memory database (syl_db_shards) with pass 1 by the scan formulation
(SYL_DB_SCAN=1: the genome k-mers streamed past the samples' lookup tables) against the index build (SYL_DB_SCAN=0).

The database is generated as scripts/time_db_shards.py does (GTDB-shaped by default: 113 104 genomes, 2.30e9 entries;
scaled down with a note when the host's MemAvailable cannot hold it).  Samples are unions of 64 genomes' k-mers with
Poisson(6) counts.  For each sample count, call kind and host memory kind (pageable numpy arrays, or pinned copies), the
two paths run alternated in one process for --rounds rounds.  Reported per call: wall time, the scan / stats / boot
kernel times, the H2D bytes and chunks of the scan (from the library's SYL_DEBUG_TIMING line), the ctx's device-memory
peak, whether the rows equal the first run's, and the card's name and power limit.  Prints JSON lines.

    python scripts/time_db_scan.py [--entries 2.3e9] [--samples 1,2,4,8,16,32,64] [--kinds query,profile]
                                   [--memory pageable,pinned] [--rounds 2]
"""
import argparse
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["SYL_DEBUG_TIMING"] = "1"   # read once per process by the library

from scripts.db_scale import gpu_info, mem_available  # noqa: E402
from scripts.time_db_shards import emit, fit, gen_db, make_samples, same, with_stderr  # noqa: E402

SCAN_RE = re.compile(r"\[db scan\] samples \d+ chunks (\d+) genome k-mers \d+: H2D (\d+) bytes")


def pinned(d):
    import torch
    out, keep = {}, []
    for k, a in d.items():
        t = torch.empty(a.nbytes, dtype=torch.uint8, pin_memory=True)
        out[k] = t.numpy().view(a.dtype)
        out[k][:] = a
        keep.append(t)
    return out, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=113104)
    ap.add_argument("--mean", type=float, default=17400)
    ap.add_argument("--entries", type=float, default=2.3e9)
    ap.add_argument("--samples", default="1,2,4,8,16,32,64")
    ap.add_argument("--kinds", default="query,profile")
    ap.add_argument("--memory", default="pageable,pinned")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    import numpy as np
    import sylph_b200
    from sylph_b200.api import contain_params

    emit(gpu=gpu_info())
    rng = np.random.default_rng(a.seed)
    G = int(a.genomes * a.entries / 2.3e9) if a.entries < 2.3e9 else a.genomes
    G, entries = fit(G, a.entries, mem_available() / (2 if "pinned" in a.memory else 1), "db")
    d = gen_db(rng, G, a.mean, entries)
    emit(genomes=G, genome_kmers=int(d["kmer_off"][-1]), entries=int(d["kmer_off"][-1] + d["tracked_off"][-1]))
    counts = [int(x) for x in a.samples.split(",")]
    raw = make_samples(rng, d, max(counts))
    ctx = sylph_b200.Context(0)
    ctx.enable_timing(True)
    samples = [ctx.upload_sample(h, c, c=200) for h, c in raw]
    for mem in a.memory.split(","):
        arrays, keep = (d, None) if mem == "pageable" else pinned(d)
        sh = ctx.db_shards(arrays["kmers"], arrays["kmer_off"], arrays["tracked"], arrays["tracked_off"], arrays["gn_size"], c=200)
        for kind in a.kinds.split(","):
            p = contain_params(pseudotax=kind == "profile")
            for ns in counts:
                first = None
                for r in range(a.rounds):
                    for scan in ("1", "0"):
                        os.environ["SYL_DB_SCAN"] = scan
                        for w in ("scan", "stats", "boot", "join"):
                            ctx.kernel_time(w, reset=True)
                        held0 = ctx.device_bytes(reset_peak=True)[0]
                        t = time.perf_counter()
                        fn = sh.profile if kind == "profile" else sh.query
                        rows, err = with_stderr(lambda: fn(samples[:ns], p))
                        wall = time.perf_counter() - t
                        peak = ctx.device_bytes()[1] - held0
                        m = SCAN_RE.search(err)
                        if first is None:
                            first = rows
                        emit(memory=mem, kind=kind, samples=ns, round=r, path="scan" if scan == "1" else "build",
                             wall_s=round(wall, 3), **{w + "_ms": round(ctx.kernel_time(w)[0], 1) for w in ("scan", "stats", "boot", "join")},
                             chunks=int(m.group(1)) if m else 0, h2d_gb=round(int(m.group(2)) / 1e9, 3) if m else 0.,
                             peak_gb=round(peak / 1e9, 3), rows=len(rows), rows_equal=bool(same(rows, first)))
        os.environ.pop("SYL_DB_SCAN", None)
        sh.free()
        keep = None
    ctx.close()


if __name__ == "__main__":
    main()
