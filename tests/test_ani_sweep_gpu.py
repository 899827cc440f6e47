"""Every ANI of about 10^4 rows through the real kernels, bit for bit against the correctly rounded oracle.

One sample against 10^4 uploaded genomes built from count multisets (as in tests/contain_scripts.py): |genome_kmers|
from 50 to 2^20, hits from 1 to all of them, counts that reach each lambda status, most of them the ratio-lambda branch
(so the adjusted ANI and both bootstrap ANI percentiles are computed too).  With minimum_ani = 0 every hit genome
prints, in query and profile, in both formulations (per-pair count histograms, CSR), and once through db shards with
pass 1 scanned (SYL_DB_SCAN=1).  This is the device-side counterpart of tests/cpp/crmath_check.cpp's host sweep of
crmath.cuh: the naive ANI's pow and the adjusted ANI's exp / pow as the statistics and bootstrap kernels evaluate them.
The glibc oracle (the reference's arithmetic) must differ from the correctly rounded one in some of these values, so
the comparison is known to see a last-bit difference."""
import os

import numpy as np
import pytest

from tests.contain_compare import compare, cr_params, sort_query_rows

pytestmark = pytest.mark.gpu

K = 31
N_GENOMES = 10000
N_BIG = 24                      # genomes of 2^12 - 2^20 k-mers; the others 50 - 2^12
NTHREADS = os.cpu_count() or 1


def mix64(x):
    """splitmix64's finalizer: a bijection of the 64-bit integers"""
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def sweep_world(seed=0xA11):
    """-> (db arrays, sample hashes, sample counts in a shuffled order)"""
    rng = np.random.default_rng(seed)
    small = np.exp(rng.uniform(np.log(50), np.log(4096), N_GENOMES - N_BIG))
    big = np.exp(rng.uniform(np.log(4096), np.log(2**20), N_BIG - 1))
    glen = np.concatenate([small, big, [2**20]]).astype(np.int64)
    glen = glen[rng.permutation(N_GENOMES)]
    hits = np.minimum(glen, np.maximum(1, (glen * rng.uniform(0, 1, N_GENOMES) ** 0.7).astype(np.int64)))
    kind = rng.choice(3, size=N_GENOMES, p=[0.84, 0.08, 0.08])     # 0 lambda, 1 high, 2 low (a single count value)
    total = int(glen.sum())
    keys = mix64(np.arange(total, dtype=np.uint64) + np.uint64(seed << 32))    # distinct: mix64 is a bijection
    assert not (keys == np.uint64(2**64 - 1)).any()                            # the oracle's empty-slot marker
    off = np.concatenate([[0], np.cumsum(glen)])
    counts = []
    for g in range(N_GENOMES):
        n = int(hits[g])
        if kind[g] == 0:
            c = 1 + rng.poisson(rng.uniform(0.05, 1.5), n)
        elif kind[g] == 1:
            c = 1 + rng.poisson(rng.uniform(3.0, 40.0), n)
        else:
            c = np.full(n, int(rng.integers(1, 3)))
        counts.append(c)
    hit_idx = np.concatenate([np.arange(off[g], off[g] + hits[g]) for g in range(N_GENOMES)])
    sh = keys[hit_idx]
    sc = np.concatenate(counts).astype(np.uint32)
    p = rng.permutation(len(sh))
    tracked = np.zeros(0, np.uint64)
    d = dict(kmers=keys, kmer_off=off.astype(np.uint64), tracked=tracked, tracked_off=np.zeros(N_GENOMES + 1, np.uint64),
             gn_size=(1_000_000 + 137 * np.arange(N_GENOMES)).astype(np.uint64))
    return d, sh[p], sc[p]


@pytest.fixture(scope="module")
def world(ctx):
    from oracle import oracle as O
    d, sh, sc = sweep_world()
    smp = O.Sample(sh, sc)

    def oracle(pseudotax, cr):
        p = cr_params(pseudotax=pseudotax, minimum_ani=0.0) if cr else O.default_params(pseudotax=pseudotax, minimum_ani=0.0)
        return O.contain_sample(p, d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], smp,
                                nthreads=NTHREADS)

    exp = {pt: oracle(pt, True) for pt in (False, True)}
    g = ctx.upload_genomes(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=1)
    db = ctx.build_db(g)
    dsmp = ctx.upload_sample(sh, sc, c=1)
    yield dict(d=d, exp=exp, glibc=oracle(False, False), db=db, smp=dsmp)
    dsmp.free()
    db.free()
    g.free()


def ani_values(rows):
    """(genome, which, value) of every ANI a row carries: naive, final, and the two bootstrap ANI percentiles"""
    out = []
    for e in rows:
        out += [(e.genome, "naive", e.naive_ani), (e.genome, "final", e.final_est_ani)]
        if e.ci_valid:
            out += [(e.genome, "ci_low", e.ci[0]), (e.genome, "ci_high", e.ci[1])]
    return out


def test_sweep_covers_the_ani_shapes(world):
    """about 10^4 rows; most of them ratio-lambda rows, every status present; about 10^4 values of each ANI"""
    exp = world["exp"][False]
    st = np.bincount([e.lambda_status for e in exp], minlength=3)
    assert len(exp) > 9000 and st.min() > 300 and st[2] > 7000, st
    assert sum(e.final_est_ani != e.naive_ani for e in exp) > 7000
    assert sum(e.ci_valid for e in exp) > 6000
    glens = [e.glen for e in exp]
    assert min(glens) < 60 and max(glens) == 2**20


def test_glibc_differs_in_some_ani_values(world):
    """The reference's glibc pow / exp misround about 1 in 1000 calls: some ANI values of the sweep differ by one ulp
    between the glibc oracle and the correctly rounded one (the rows the device must equal), so a device that rounded
    like glibc, or lost a bit anywhere else, would fail the comparisons below."""
    cr = {(g, w): v for g, w, v in ani_values(world["exp"][False])}
    gl = {(g, w): v for g, w, v in ani_values(world["glibc"])}
    assert cr.keys() == gl.keys()
    diff = [key for key in cr if cr[key] != gl[key]]
    by = {w: sum(1 for _, x in diff if x == w) for w in ("naive", "final", "ci_low", "ci_high")}
    print("ANI values: %d; glibc != correctly rounded: %d %s" % (len(cr), len(diff), by))
    assert len(diff) >= 5, by
    for key in diff:
        assert abs(cr[key] - gl[key]) <= 2 * np.spacing(cr[key]), key


@pytest.mark.parametrize("formulation", ["hist", "csr"])
@pytest.mark.parametrize("pseudotax", [False, True])
def test_sweep_rows_equal_the_correctly_rounded_oracle(ctx, world, monkeypatch, formulation, pseudotax):
    from sylph_b200.api import contain_params
    monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)
    if formulation == "csr":
        monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
    p = contain_params(pseudotax=pseudotax, minimum_ani=0.0)
    rows = ctx.profile(world["db"], [world["smp"]], p) if pseudotax else sort_query_rows(ctx.query(world["db"], [world["smp"]], p))
    compare(rows, world["exp"][pseudotax], pseudotax)


def test_sweep_through_scanned_db_shards(ctx, world, monkeypatch):
    """the same sample through db shards with pass 1 scanned past the sample (SYL_DB_SCAN=1): query and profile"""
    from sylph_b200.api import contain_params
    for k in ("SYL_CONTAIN_CSR", "SYL_DB_SHARD_ENTRIES", "SYL_DB_SCAN_CHUNK", "SYL_SAMPLE_BATCH"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("SYL_DB_SCAN", "1")
    d = world["d"]
    sh = ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], k=K, c=1)
    try:
        ctx.enable_timing(True)
        ctx.kernel_time("scan", reset=True)
        for pseudotax in (False, True):
            p = contain_params(pseudotax=pseudotax, minimum_ani=0.0)
            rows = sh.profile([world["smp"]], p) if pseudotax else sort_query_rows(sh.query([world["smp"]], p))
            compare(rows, world["exp"][pseudotax], pseudotax)
        assert ctx.kernel_time("scan")[1] > 0
    finally:
        ctx.enable_timing(False)
        sh.free()
