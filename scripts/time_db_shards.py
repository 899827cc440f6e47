"""Time `profile` against a GTDB-shaped database swept in shards (syl_db_shards) against the one-index call, and profile
a database past one index's 2^32-2 entries.

The database is generated as scripts/db_scale.py does (--genomes genomes of about --mean k-mers, tracked k-mers up to
--entries in all, below 2^64 / 200; scaled down with a note when the host's MemAvailable cannot hold it).  Samples are
unions of 64 genomes' k-mers with Poisson(6) counts.  For 1 and 16 samples it times the one-index call (build +
profile) and sh.profile with 1, 2, 4 and 8 shards, each once, and reports per call the wall time, the per-shard index
build and pass-1 time and the survivor index (from the library's SYL_DEBUG_TIMING lines), the ctx's device-memory peak,
and whether the rows equal the one-index rows.  --past-limit ENTRIES then generates a database of that many entries
(4.6e9: GTDB at c = 100), profiles one sample with the default shard cap, and checks its rows against the same call at
half that cap.  Prints JSON lines, and the card's name and power limit.

    python scripts/time_db_shards.py [--entries 2.3e9] [--past-limit 4.6e9] [--skip-sweep]
"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["SYL_DEBUG_TIMING"] = "1"   # read once per process by the library

from scripts.db_scale import gpu_info, mem_available  # noqa: E402

SHARD_RE = re.compile(r"\[db shard (\d+)/(\d+)\] genomes \d+\+(\d+) entries (\d+): build ([\d.]+) ms, pass 1 ([\d.]+) ms")
SURV_RE = re.compile(r"\[survivor index\] samples \d+\.\.\d+ genomes (\d+) entries (\d+): gather\+build ([\d.]+) ms, profile ([\d.]+) ms")


def emit(**kw):
    print(json.dumps(kw), flush=True)


def with_stderr(fn):
    """-> (fn(), what the library wrote to fd 2 meanwhile)"""
    with tempfile.TemporaryFile(mode="w+") as tf:
        saved = os.dup(2)
        os.dup2(tf.fileno(), 2)
        try:
            r = fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tf.seek(0)
        return r, tf.read()


def gen_db(rng, G, mean, entries):
    import numpy as np
    nk = np.maximum(rng.normal(mean, mean / 3, G), 100).astype(np.int64)
    share = max(entries - nk.sum(), 0) / nk.sum()
    nt = (nk * share * rng.uniform(0.5, 1.5, G)).astype(np.int64)
    hi = np.uint64((2**64 - 1) // 200)
    koff = np.concatenate([[0], np.cumsum(nk)]).astype(np.uint64)
    toff = np.concatenate([[0], np.cumsum(nt)]).astype(np.uint64)
    kmers = rng.integers(0, hi, int(koff[-1]), dtype=np.uint64)
    tracked = rng.integers(0, hi, int(toff[-1]), dtype=np.uint64)
    return dict(kmers=kmers, kmer_off=koff, tracked=tracked, tracked_off=toff, gn_size=(nk * 200).astype(np.uint64))


def fit(G, entries, avail, what):
    need = entries * 8 * 1.25
    if need > avail * 0.85:
        f = avail * 0.85 / need
        emit(note="%s: host MemAvailable %.1f GB cannot hold %.2e entries; scaled to %.2e" % (what, avail / 1e9, entries, entries * f))
        return max(1000, int(G * f)), entries * f
    return G, entries


def make_samples(rng, d, n):
    """-> n (hashes, counts) of 64 genomes each"""
    import numpy as np
    G = len(d["kmer_off"]) - 1
    out = []
    for _ in range(n):
        pick = np.sort(rng.choice(G, 64, replace=False))
        hs = np.unique(np.concatenate([d["kmers"][int(d["kmer_off"][g]):int(d["kmer_off"][g + 1])] for g in pick]))
        out.append((hs, np.maximum(rng.poisson(6, len(hs)), 1).astype(np.uint32)))
    return out


def same(a, b):
    return len(a) == len(b) and all((a[f] == b[f]).all() for f in a.dtype.names)


def sharded(ctx, d, samples, cap, p):
    sh = ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200, max_entries=cap)
    ctx.device_bytes(reset_peak=True)
    held0 = ctx.device_bytes()[0]
    t = time.perf_counter()
    rows, err = with_stderr(lambda: sh.profile(samples, p))
    wall = time.perf_counter() - t
    peak = ctx.device_bytes()[1] - held0
    shards = [dict(genomes=int(m[2]), entries=int(m[3]), build_ms=float(m[4]), pass1_ms=float(m[5])) for m in SHARD_RE.findall(err)]
    surv = [dict(genomes=int(m[0]), entries=int(m[1]), gather_build_ms=float(m[2]), profile_ms=float(m[3])) for m in SURV_RE.findall(err)]
    n = len(sh)
    sh.free()
    return rows, dict(shards=n, wall_s=round(wall, 3), peak_gb=round(peak / 1e9, 3), per_shard=shards, survivor=surv)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=113104)
    ap.add_argument("--mean", type=float, default=17400)
    ap.add_argument("--entries", type=float, default=2.3e9)
    ap.add_argument("--past-limit", type=float, default=4.6e9)
    ap.add_argument("--skip-sweep", action="store_true")
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    import numpy as np
    import sylph_b200
    from sylph_b200.api import contain_params

    emit(gpu=gpu_info())
    p = contain_params(pseudotax=True)
    ctx = sylph_b200.Context(0)
    if not a.skip_sweep:
        rng = np.random.default_rng(a.seed)
        G, entries = fit(a.genomes, a.entries, mem_available(), "sweep")
        d = gen_db(rng, G, a.mean, entries)
        N = int(d["kmer_off"][-1] + d["tracked_off"][-1])
        emit(genomes=G, entries=N)
        raw = make_samples(rng, d, 16)
        samples = [ctx.upload_sample(h, c, c=200) for h, c in raw]
        for ns in (1, 16):
            one = sylph_b200.Context(0)   # its own ctx: its cached blocks would blur the shards' peak
            smp1 = [one.upload_sample(h, c, c=200) for h, c in raw[:ns]]
            held0 = one.device_bytes()[0]
            t = time.perf_counter()
            db = one.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200)
            build = time.perf_counter() - t
            t = time.perf_counter()
            want = one.profile(db, smp1, p)
            prof = time.perf_counter() - t
            peak = one.device_bytes()[1] - held0
            db.free()
            for x in smp1:
                x.free()
            one.close()
            emit(samples=ns, mode="one index", build_s=round(build, 3), profile_s=round(prof, 3),
                 wall_s=round(build + prof, 3), peak_gb=round(peak / 1e9, 3), rows=len(want), runs=1)
            for k in (1, 2, 4, 8):
                rows, info = sharded(ctx, d, samples[:ns], N // k + 1, p)
                emit(samples=ns, mode="shards", equal_to_one_index=same(rows, want), runs=1, **info)
        for s in samples:
            s.free()
        del d
    if a.past_limit:
        rng = np.random.default_rng(a.seed + 1)
        G, entries = fit(a.genomes, a.past_limit, mem_available(), "past limit")  # c = 100: twice the k-mers per genome
        d = gen_db(rng, G, a.mean * a.past_limit / a.entries, entries)
        N = int(d["kmer_off"][-1] + d["tracked_off"][-1])
        emit(genomes=G, entries=N, over_one_index=N >= 2**32 - 2)
        smp = [ctx.upload_sample(h, c, c=200) for h, c in make_samples(rng, d, 1)]
        rows, info = sharded(ctx, d, smp, 0, p)
        emit(mode="shards, default cap", rows=len(rows), runs=1, **info)
        half = max(x["entries"] for x in info["per_shard"]) // 2 + 1
        rows2, info2 = sharded(ctx, d, smp, half, p)
        emit(mode="shards, half the cap", equal_to_default_cap=same(rows, rows2), runs=1, **info2)
    ctx.close()


if __name__ == "__main__":
    main()
