"""GPU parity: containment query/profile vs the CPU oracle in its correctly rounded mode, every field bit-exact
(tests/contain_compare.py)."""
import os

import numpy as np
import pytest

from tests.contain_compare import compare, cr_params, oracle_rows, sort_query_rows
from tests.util import DATA, flatten, read_fastx

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("contain_mode")]



@pytest.fixture(params=["device-driven", "synchronous"])
def contain_mode(request, monkeypatch):
    """syl_query / syl_profile in both formulations of the staged driver (the library reads SYL_CONTAIN_CSR per call):
    "device-driven" = the per-pair count histograms, one host synchronisation per call (the CSR formulation only where
    a count >= 256 or the size asks for it); "synchronous" = the CSR formulation throughout, which synchronises once
    more to size its value array.  The ids are those of the former device-driven / synchronous paths, so test ids stay
    stable."""
    monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)
    if request.param == "synchronous":
        monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
    return request.param


@pytest.fixture(scope="module")
def ecoli(ctx):
    bufs, coffs, goff = [], [0], [0]
    for name in ("e.coli-EC590.fasta.gz", "e.coli-o157.fasta.gz", "e.coli-K12.fasta.gz"):
        for _, s in read_fastx(os.path.join(DATA, name)):
            bufs.append(s)
            coffs.append(coffs[-1] + len(s))
        goff.append(len(coffs) - 1)
    buf = np.frombuffer(b"".join(bufs), dtype=np.uint8)
    g = ctx.sketch_genomes(buf, np.array(coffs, np.uint64), np.array(goff, np.uint64))
    recs = read_fastx(os.path.join(DATA, "o157_reads.fastq.gz"))
    rb, ro = flatten([s for _, s in recs])
    smp = ctx.sketch_sequences(rb, ro)
    return g, g.download(), smp, smp.download()


def test_config1_query_three_rows(ctx, ecoli):
    g, d, smp, hc = ecoli
    db = ctx.build_db(g)
    rows = sort_query_rows(ctx.query(db, [smp]))
    exp = oracle_rows(d, hc, False)
    assert len(rows) == 3  # tests/integration_test.rs:128-140: header + 3 rows
    compare(rows, exp, False)


def test_config1_profile_one_row_vs_ec590(ctx, ecoli):
    g, d, smp, hc = ecoli
    one = {k: v for k, v in d.items()}
    n0, t0 = int(d["kmer_off"][1]), int(d["tracked_off"][1])
    one = dict(kmers=d["kmers"][:n0], kmer_off=d["kmer_off"][:2], tracked=d["tracked"][:t0],
               tracked_off=d["tracked_off"][:2], gn_size=d["gn_size"][:1])
    g1 = ctx.upload_genomes(one["kmers"], one["kmer_off"], one["tracked"], one["tracked_off"], one["gn_size"])
    db = ctx.build_db(g1)
    rows = ctx.profile(db, [smp])
    assert len(rows) == 1  # tests/integration_test.rs:117-126: header + 1 row
    compare(rows, oracle_rows(one, hc, True), True)


def test_config1_profile_three(ctx, ecoli):
    g, d, smp, hc = ecoli
    db = ctx.build_db(g)
    rows = ctx.profile(db, [smp])
    compare(rows, oracle_rows(d, hc, True), True)


def synth_db_and_sample(ctx, n_genomes, genome_len, n_reads, n_comm, c=200, read_seed=None):
    from sylph_b200 import synth
    bases, off = synth.db_chunk(0, n_genomes, genome_len)
    goff = np.arange(n_genomes + 1, dtype=np.uint64)
    g = ctx.sketch_genomes(bases.numpy(), off.numpy().astype(np.uint64), goff, c=c)
    kw = {} if read_seed is None else {"seed": read_seed}
    rb, ro = synth.reads(n_reads, n_comm=n_comm, genome_len=genome_len, **kw)
    smp = ctx.sketch_sequences(rb.numpy(), ro.numpy().astype(np.uint64), c=c)
    return g, smp


@pytest.mark.parametrize("pseudotax", [False, True])
def test_synthetic_community_with_mutant_genomes(ctx, pseudotax):
    """200 genomes (genomes 99 and 199 are ~97 % mutants of 98 / 198 => shared k-mers, k-mer
    reassignment and derep in profile), community = first 120 genomes, coverage from <0.1x to >20x
    so LOW / lambda / HIGH statuses and the bootstrap all occur."""
    g, smp = synth_db_and_sample(ctx, 200, 120000, 150000, 120, c=20)
    d, hc = g.download(), smp.download()
    db = ctx.build_db(g)
    if pseudotax:
        rows = ctx.profile(db, [smp])
    else:
        rows = sort_query_rows(ctx.query(db, [smp]))
    exp = oracle_rows(d, hc, pseudotax)
    assert len(exp) > 20
    st = {e.lambda_status for e in exp}
    assert 2 in st and 1 in st
    compare(rows, exp, pseudotax)


def test_params_variants_and_multi_sample(ctx):
    from sylph_b200.api import contain_params
    g, s1 = synth_db_and_sample(ctx, 60, 100000, 40000, 30, c=20)
    _, s2 = synth_db_and_sample(ctx, 1, 100000, 20000, 60, c=20, read_seed=0x5EED0011)
    d = g.download()
    db = ctx.build_db(g, genome_base=0)
    for kw in (dict(no_ci=1), dict(no_adj=1), dict(minimum_ani=50.0), dict(min_number_kmers=6000.0),
               dict(min_count_correct=1.0), dict(mean_coverage=1)):
        rows = ctx.query(db, [s1, s2], contain_params(pseudotax=False, **kw))
        for si, s in enumerate((s1, s2)):
            sub = sort_query_rows(rows[rows["sample"] == si])
            compare(sub, oracle_rows(d, s.download(), False, **kw), False)


@pytest.mark.parametrize("pseudotax", [False, True])
def test_several_samples_of_unequal_size_one_call(ctx, pseudotax):
    """Several samples in one call take the tiled (hash range, sample) mapping of the join kernels: samples of
    very different sizes (one of them empty, one a handful of reads) == the oracle, sample by sample."""
    from sylph_b200 import synth
    from sylph_b200.api import contain_params
    g, s_big = synth_db_and_sample(ctx, 200, 120000, 150000, 120, c=20)
    _, s_mid = synth_db_and_sample(ctx, 1, 120000, 30000, 40, c=20, read_seed=0x5EED0011)
    rb, ro = synth.reads(50, n_comm=5, genome_len=120000, seed=0x5EED0012)
    s_tiny = ctx.sketch_sequences(rb.numpy(), ro.numpy().astype(np.uint64), c=20)
    s_empty = ctx.sketch_sequences(np.zeros(0, np.uint8), np.zeros(1, np.uint64), c=20)
    d = g.download()
    db = ctx.build_db(g)
    samples = [s_mid, s_empty, s_big, s_tiny, s_mid]
    P = contain_params(pseudotax=pseudotax)
    rows = ctx.profile(db, samples, P) if pseudotax else ctx.query(db, samples, P)
    n_rows = 0
    for si, smp in enumerate(samples):
        sub = rows[rows["sample"] == si]
        if not pseudotax:
            sub = sort_query_rows(sub)
        exp = oracle_rows(d, smp.download(), pseudotax)
        compare(sub, exp, pseudotax)
        n_rows += len(exp)
    assert n_rows == len(rows) and n_rows > 40


def test_uploaded_sketches_and_zero_counts(ctx):
    """Sketches that come from files: unsorted sample pairs, a zero count (skipped, src/contain.rs:634)."""
    rng = np.random.default_rng(4)
    kmers = np.unique(rng.integers(1, 2**57, size=5000, dtype=np.uint64))[:4000]
    rng.shuffle(kmers)
    koff = np.array([0, 1500, 1500, 4000], dtype=np.uint64)   # genome 1 is empty
    tracked = np.unique(rng.integers(1, 2**57, size=300, dtype=np.uint64))
    toff = np.array([0, 100, 100, len(tracked)], dtype=np.uint64)
    gs = np.array([1000000, 0, 2000000], dtype=np.uint64)
    g = ctx.upload_genomes(kmers, koff, tracked, toff, gs)
    sh = np.concatenate([kmers[:1200], kmers[2000:3900], rng.integers(2**57, 2**58, size=500, dtype=np.uint64)])
    sc = rng.integers(0, 6, size=len(sh)).astype(np.uint32)
    perm = rng.permutation(len(sh))
    smp = ctx.upload_sample(sh[perm], sc[perm])
    db = ctx.build_db(g)
    d = dict(kmers=kmers, kmer_off=koff, tracked=tracked, tracked_off=toff, gn_size=gs)
    compare(sort_query_rows(ctx.query(db, [smp])), oracle_rows(d, (sh, sc), False), False)
    compare(ctx.profile(db, [smp]), oracle_rows(d, (sh, sc), True), True)


def deep_coverage_case(ctx, depth):
    """Three uploaded genomes (genome 0 covered `depth` deep, genome 1 shallow, genome 2 absent) and one sample."""
    rng = np.random.default_rng(1000 + depth)
    kmers = np.unique(rng.integers(1, 2**57, size=9000, dtype=np.uint64))[:8000]
    koff = np.array([0, 3000, 5500, 8000], dtype=np.uint64)
    tracked = np.zeros(0, np.uint64)
    toff = np.zeros(4, np.uint64)
    gs = np.array([600000, 500000, 500000], dtype=np.uint64)
    g = ctx.upload_genomes(kmers, koff, tracked, toff, gs)
    # genome 0 deep, genome 1 shallow (lambda / bootstrap branch), genome 2 absent
    sh = np.concatenate([kmers[:2900], kmers[3000:4200]])
    sc = np.concatenate([rng.poisson(depth, size=2900), rng.poisson(0.7, size=1200)]).astype(np.uint32)
    if depth >= 250:
        sc[:5] = [255, 256, 257, 100000, 255]
    smp = ctx.upload_sample(sh, sc)
    d = dict(kmers=kmers, kmer_off=koff, tracked=tracked, tracked_off=toff, gn_size=gs)
    return g, d, (sh, sc), smp


@pytest.mark.parametrize("depth", [40, 250, 255, 256, 700])
def test_deep_coverage_uploaded_sample(ctx, depth):
    """Coverage around the 256-bin limit of the per-pair count histograms: up to 255 the histogram
    formulation of get_stats answers, from 256 on the call is redone in the CSR formulation
    (contain.hpp COV_BINS); medians >= 30 take the no-cutoff branch (src/contain.rs:664)."""
    g, d, (sh, sc), smp = deep_coverage_case(ctx, depth)
    db = ctx.build_db(g)
    exp = oracle_rows(d, (sh, sc), False)
    assert len(exp) >= 1 and exp[0].median_cov >= 30
    compare(sort_query_rows(ctx.query(db, [smp])), exp, False)
    compare(ctx.profile(db, [smp]), oracle_rows(d, (sh, sc), True), True)


def test_k21_scalar_semantics_end_to_end(ctx):
    """k = 21 with the scalar window set (what sylph computes on non-x86): sketches, query and profile."""
    from oracle import oracle as O
    from sylph_b200 import synth
    from sylph_b200.api import contain_params
    bases, off = synth.db_chunk(0, 30, 80000)
    b, o = bases.numpy(), off.numpy().astype(np.uint64)
    g = ctx.sketch_genomes(b, o, np.arange(31, dtype=np.uint64), k=21, c=15, sem=0)
    rb, ro = synth.reads(40000, n_comm=30, genome_len=80000)
    smp = ctx.sketch_sequences(rb.numpy(), ro.numpy().astype(np.uint64), k=21, c=15, sem=0)
    d, hc = g.download(), smp.download()
    km, tr, _ = O.sketch_genome(b[:80000], np.array([0, 80000], np.uint64), k=21, c=15, sem=0)
    assert np.array_equal(km, d["kmers"][: int(d["kmer_off"][1])]) and np.array_equal(tr, d["tracked"][: int(d["tracked_off"][1])])
    eh, ec, _, _ = O.sketch_reads(rb.numpy(), ro.numpy().astype(np.uint64), k=21, c=15, sem=0)
    assert np.array_equal(hc[0], eh) and np.array_equal(hc[1], ec)
    db = ctx.build_db(g)
    for pt in (False, True):
        rows = ctx.profile(db, [smp], contain_params(k=21, pseudotax=True)) if pt else sort_query_rows(ctx.query(db, [smp], contain_params(k=21)))
        p = cr_params(k=21, pseudotax=pt)
        exp = O.contain_sample(p, d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], O.Sample(*hc))
        assert len(exp) > 5
        compare(rows, exp, pt)


def test_sharded_profile_stages_on_one_gpu(ctx):
    """The three-collective sharded profile (include/sylph_b200.h (5)) with world = 1 (no collectives) must
    equal syl_profile; a row table that is too small is reported and the call is redone with the needed size."""
    from sylph_b200 import dist as D
    from sylph_b200.api import contain_params
    g, s1 = synth_db_and_sample(ctx, 120, 100000, 60000, 100, c=20)
    samples = [s1]
    for si in range(5):
        _, s = synth_db_and_sample(ctx, 1, 100000, 30000, 100, c=20, read_seed=0x5EED0100 + si)
        samples.append(s)
    db = ctx.build_db(g)
    exp = ctx.profile(db, samples, contain_params(pseudotax=True))
    assert len(exp) > 256                     # more rows than the smallest row table holds
    for rpr in (0, 256):
        rows = D.profile_sharded(ctx, g, db, samples, 0, contain_params(pseudotax=True), rows_per_rank=rpr)
        assert len(rows) == len(exp)
        for f in rows.dtype.names:
            assert np.array_equal(rows[f], exp[f]), (rpr, f)


@pytest.mark.parametrize("pseudotax", [False, True])
def test_estimate_unknown_with_read_seq_id(ctx, pseudotax):
    """-u with an explicit --read-seq-id (src/contain.rs:274-279, 377-408): coverage scaled by read identity and the
    read-length / k-mer ratio, sequence abundance by the fraction of the sample the profile explains.  The automatic
    identity estimate is refused (hash-map iteration order)."""
    import sylph_b200
    from oracle import oracle as O
    from sylph_b200.api import contain_params
    g, smp = synth_db_and_sample(ctx, 80, 100000, 60000, 20, c=20)
    d, hc = g.download(), smp.download()
    db = ctx.build_db(g)
    P = contain_params(pseudotax=pseudotax, estimate_unknown=1, read_seq_id=98.0)
    rows = ctx.profile(db, [smp], P) if pseudotax else sort_query_rows(ctx.query(db, [smp], P))
    exp = O.contain_sample(cr_params(pseudotax=pseudotax), d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"],
                           O.Sample(*hc), unknown=O.Unknown(98.0, smp.mean_read_length, 20))
    plain = O.contain_sample(cr_params(pseudotax=pseudotax), d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"],
                             O.Sample(*hc))
    assert len(exp) > 5 and exp[0].final_est_cov > plain[0].final_est_cov
    compare(rows, exp, pseudotax)
    with pytest.raises(sylph_b200.SylphError) as e:
        ctx.query(db, [smp], contain_params(pseudotax=False, estimate_unknown=1))
    assert e.value.code == 5                                          # SYL_ERR_UNSUPPORTED


def test_sharded_profile_deep_coverage_on_one_gpu(ctx, contain_mode):
    """A count >= 256 makes a histogram job of the three-collective sharded profile (world = 1) report
    SYL_ERR_UNSUPPORTED; a job with csr = 1, or any job under SYL_CONTAIN_CSR ("synchronous"), returns syl_profile's
    rows, and so does profile_sharded, which redoes the job with csr = 1.  Field for field."""
    from sylph_b200 import _lib
    from sylph_b200 import dist as D
    from sylph_b200.api import contain_params
    g, _, _, smp = deep_coverage_case(ctx, 700)
    db = ctx.build_db(g)
    P = contain_params(pseudotax=True)
    exp = ctx.profile(db, [smp], P)
    assert len(exp) >= 1
    results = [D.profile_sharded(ctx, g, db, [smp], 0, P)]
    for csr in (False, True):
        job = ctx.profile_shard_begin(db, [smp], P, 1, 0, 0, csr=csr)
        try:
            job.rank()
            job.pass2()
            rows, rc, _ = job.finish()
        finally:
            job.free()
        if csr or contain_mode == "synchronous":
            assert rc == _lib.SYL_OK, csr
            results.append(rows)
        else:
            assert rc == _lib.SYL_ERR_UNSUPPORTED
    for got in results:
        assert len(got) == len(exp)
        for f in got.dtype.names:
            assert np.array_equal(got[f], exp[f]), f


@pytest.mark.parametrize("pseudotax", [False, True])
def test_pass2_tie_goes_to_lowest_genome(ctx, pseudotax):
    """Two genomes with the same statistics share half of their k-mers: their pass-1 ANIs are equal, and in pass 2
    every shared k-mer goes to the lower genome index (the other one counts them as lost).  Both genome orders."""
    rng = np.random.default_rng(77)
    keys = rng.permutation(np.unique(rng.integers(1, 2**57, size=700, dtype=np.uint64)))[:600]
    shared, ea, eb = keys[:200], keys[200:400], keys[400:600]
    c_shared = rng.poisson(2.0, size=200).astype(np.uint32) + 1
    c_own = rng.poisson(2.0, size=200).astype(np.uint32) + 1
    sh = np.concatenate([shared, ea, eb])
    sc = np.concatenate([c_shared, c_own, c_own])                 # the same count multiset for both genomes
    smp = ctx.upload_sample(sh, sc)
    for first, second in ((ea, eb), (eb, ea)):
        kmers = np.concatenate([shared, first, shared, second])
        koff = np.array([0, 400, 800], dtype=np.uint64)
        d = dict(kmers=kmers, kmer_off=koff, tracked=np.zeros(0, np.uint64), tracked_off=np.zeros(3, np.uint64),
                 gn_size=np.array([4000000, 4000000], dtype=np.uint64))
        g = ctx.upload_genomes(d["kmers"], koff, d["tracked"], d["tracked_off"], d["gn_size"])
        db = ctx.build_db(g)
        exp = oracle_rows(d, (sh, sc), pseudotax)
        rows = ctx.profile(db, [smp]) if pseudotax else sort_query_rows(ctx.query(db, [smp]))
        compare(rows, exp, pseudotax)
        if pseudotax:
            assert [(e.genome, e.kmers_lost) for e in sorted(exp, key=lambda e: e.genome)] == [(0, 0), (1, 200)]


def test_more_pairs_than_histograms_hold(ctx):
    """More than 2^23 (sample, genome) pairs in one call: the per-pair count histograms would exceed 8 GB, so the
    call runs in the CSR formulation from the start.  3 samples x 3 M genomes of 3 k-mers each; every genome a
    sample hits yields a row (min_number_kmers = 1).  Rows == the oracle on the genomes that were hit."""
    from sylph_b200.api import contain_params
    rng = np.random.default_rng(23)
    G, K = 3_000_000, 3
    assert 3 * G > 2**23
    kmers = rng.permutation(np.unique(rng.integers(1, 2**57, size=G * K + 100000, dtype=np.uint64)))[: G * K]
    koff = np.arange(0, G * K + 1, K, dtype=np.uint64)
    gs = np.full(G, 1000000, dtype=np.uint64)
    g = ctx.upload_genomes(kmers, koff, np.zeros(0, np.uint64), np.zeros(G + 1, np.uint64), gs)
    db = ctx.build_db(g)
    hit = [np.sort(rng.choice(G, size=40, replace=False)) for _ in range(3)]
    hit[1][:10] = hit[0][:10]                                        # genomes hit by two samples
    samples = []
    for h in hit:
        take = [kmers[K * gi: K * gi + 1 + gi % K] for gi in h]     # 1..3 of the genome's k-mers
        sh = np.concatenate(take + [rng.integers(2**57, 2**58, size=100, dtype=np.uint64)])
        sc = rng.integers(1, 6, size=len(sh)).astype(np.uint32)
        samples.append((sh, sc, ctx.upload_sample(sh, sc)))
    hit_all = np.unique(np.concatenate(hit))
    sub = dict(kmers=np.concatenate([kmers[K * gi: K * gi + K] for gi in hit_all]),
               kmer_off=np.arange(0, K * len(hit_all) + 1, K, dtype=np.uint64),
               tracked=np.zeros(0, np.uint64), tracked_off=np.zeros(len(hit_all) + 1, np.uint64), gn_size=gs[hit_all])
    for pseudotax in (False, True):
        P = contain_params(pseudotax=pseudotax, min_number_kmers=1.0)
        handles = [s for _, _, s in samples]
        rows = ctx.profile(db, handles, P) if pseudotax else ctx.query(db, handles, P)
        assert np.isin(rows["genome"], hit_all).all()
        n_rows = 0
        for si, (sh, sc, _) in enumerate(samples):
            sub_rows = rows[rows["sample"] == si].copy()
            sub_rows["genome"] = np.searchsorted(hit_all, sub_rows["genome"])
            if not pseudotax:
                sub_rows = sort_query_rows(sub_rows)
            exp = oracle_rows(sub, (sh, sc), pseudotax, min_number_kmers=1.0)
            assert len(exp) == 40
            compare(sub_rows, exp, pseudotax)
            n_rows += len(exp)
        assert n_rows == len(rows)
