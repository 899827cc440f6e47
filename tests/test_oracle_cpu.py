"""CPU suite (no GPU): the oracle against everything that pins it.
  * the reference's own pins: hash scalar==AVX2 (tests/unit_test.rs), 1 profile row / 3 query rows
    on config 1 (tests/integration_test.rs:117-140), BYTE_TO_SEQ table (src/types.rs:50-59)
  * an independent pure-Python restatement (oracle/pyref.py) on small random inputs
  * the committed oracle-generated regression fixture tests/golden/config1.json
"""
import json
import os
import re

import numpy as np
import pytest

from oracle import oracle as O
from oracle import pyref as R
from tests.util import DATA, REPO, flatten, read_fastx


def test_hash_kat_and_avx2_equals_scalar():
    # tests/unit_test.rs:6,24: AVX2 hash == scalar hash for this key; value restated in SURVEY §8-a1
    assert O.mm_hash64(19238239812933123) == 0x938A38E0E3559CFF == R.mm_hash64(19238239812933123)
    rng = np.random.default_rng(1)
    for x in rng.integers(0, 2**62, size=200, dtype=np.uint64):
        assert O.mm_hash64(int(x)) == R.mm_hash64(int(x))
    # the unbugged minimap2 hash gives a different value: make sure we did NOT implement that one
    k = 19238239812933123
    key = ((~k) + (k << 21)) & R.MASK64
    assert key != ((~(k + (k << 21))) & R.MASK64)


def test_byte_to_seq_table():
    lib = O.lib()
    exp = [0] * 256
    for ch, v in ((65, 0), (67, 1), (71, 2), (84, 3), (85, 3)):
        exp[ch] = v
        exp[ch + 32] = v
    exp[1], exp[2], exp[3] = 1, 2, 3
    assert [lib.syo_byte_to_seq(i) for i in range(256)] == exp == R.BYTE_TO_SEQ


def rand_seq(rng, n, alphabet=b"ACGTNacgtn"):
    return bytes(rng.choice(list(alphabet), size=n).astype(np.uint8))


@pytest.mark.parametrize("k", [21, 31])
def test_seeding_vs_pyref_and_intrinsics(k):
    rng = np.random.default_rng(k)
    for L in [0, 5, k - 1, k, k + 1, k + 2, k + 3, k + 4, 2 * k - 1, 2 * k, 2 * k + 1, 150, 151, 152, 153, 777]:
        s = rand_seq(rng, L)
        for c in (1, 3, 11):
            pos, h = O.extract_markers_positions(s, k, c, O.SEM_SCALAR)
            assert list(zip(pos.tolist(), h.tolist())) == R.seeds_scalar(s, k, c)
            pos, h = O.extract_markers_positions(s, k, c, O.SEM_AVX2)
            assert sorted(zip(pos.tolist(), h.tolist())) == sorted(R.seeds_avx2(s, k, c, True))
            h = O.extract_markers(s, k, c, O.SEM_AVX2)
            assert sorted(h.tolist()) == sorted(x for _, x in R.seeds_avx2(s, k, c, False))
            hi = O.extract_markers_avx2_intrin(s, k, c)
            assert hi.tolist() == h.tolist()  # same emission order (i-major, lane-minor)


def test_unsupported_k_mirrors_reference_panic():
    with pytest.raises(ValueError):
        O.extract_markers(b"ACGT" * 30, 25, 10, O.SEM_AVX2)
    assert len(O.extract_markers(b"ACGT" * 30, 25, 1, O.SEM_SCALAR)) == 120 - 25 + 1


def test_genome_sketch_vs_pyref():
    rng = np.random.default_rng(5)
    rep = rand_seq(rng, 400, b"ACGT")
    contigs = [rand_seq(rng, 3000, b"ACGT"), b"", rand_seq(rng, 40, b"ACGT"),
               rand_seq(rng, 1000, b"ACGT") + rep + rand_seq(rng, 500, b"ACGT") + rep, rand_seq(rng, 62, b"ACGT")]
    buf, off = flatten(contigs)
    for sem in (O.SEM_AVX2, O.SEM_SCALAR):
        for ms in (30, 3):
            km, tr, gs = O.sketch_genome(buf, off, k=31, c=4, min_spacing=ms, pseudotax=True, sem=sem)
            ek, et, es = R.sketch_genome(contigs, 31, 4, ms, True, sem_avx2=(sem == O.SEM_AVX2))
            assert km.tolist() == ek and tr.tolist() == et and gs == es
    km, tr, _ = O.sketch_genome(buf, off, k=31, c=4, pseudotax=False)
    assert len(tr) == 0


def test_read_sketch_dedup_vs_pyref():
    rng = np.random.default_rng(8)
    genome = rand_seq(rng, 6000, b"ACGT")
    reads = []
    for _ in range(400):
        st = int(rng.integers(0, 5500))
        ln = int(rng.choice([50, 66, 70, 150, 150, 401]))
        reads.append(genome[st:st + ln])
        if rng.random() < 0.4:
            reads.append(genome[st:st + ln])
        if rng.random() < 0.2:
            reads.append(genome[st:st + ln - 2])
    reads += [b"A" * 150] * 3 + [b""]
    buf, off = flatten(reads)
    for no_dedup in (False, True):
        for nthreads in (1, 3):
            h, c, mean, nd = O.sketch_reads(buf, off, k=31, c=7, no_dedup=no_dedup, nthreads=nthreads)
            ec, emean, end = R.sketch_reads(reads, 31, 7, no_dedup=no_dedup)
            assert dict(zip(h.tolist(), c.tolist())) == ec
            assert nd == end and abs(mean - emean) < 1e-12
    assert O.sketch_reads(buf, off, k=31, c=7)[3] > 50


def make_pairs(rng, n, genome, with_short=True):
    """read pairs from one genome: exact duplicate pairs, pairs with the same mate 1 and a shifted mate 2 (no pair key
    in common: each key mixes both mates), mates that overlap (k-mers present in both mates), short mates (< 33 bp: no
    pair key)"""
    r1, r2 = [], []
    G = len(genome)
    for _ in range(n):
        st = int(rng.integers(0, G - 400))
        l1, l2 = int(rng.choice([70, 100, 150])), int(rng.choice([70, 100, 150]))
        gap = int(rng.choice([-60, 0, 40]))
        a, b = genome[st:st + l1], genome[st + l1 + gap:st + l1 + gap + l2]
        if with_short and rng.random() < 0.05:
            b = b[:20]
        r1.append(a)
        r2.append(b)
        if rng.random() < 0.35:
            r1.append(a)
            r2.append(b)
        if rng.random() < 0.15:
            r1.append(a)
            r2.append(genome[st + 17:st + 17 + l2])
    return r1, r2


def test_paired_read_sketch_exact_set_vs_pyref():
    """sketch_pair_sequences with --fpr 0 (src/sketch.rs:771-895): C oracle == pure-Python restatement."""
    rng = np.random.default_rng(21)
    genome = rand_seq(rng, 5000, b"ACGT")
    r1, r2 = make_pairs(rng, 300, genome)
    r1 += [b"A" * 150, b"A" * 150, b""]
    r2 += [b"A" * 150, b"A" * 150, b"ACGT" * 20]
    b1, o1 = flatten(r1)
    b2, o2 = flatten(r2)
    for no_dedup in (False, True):
        h, c, mean, nd = O.sketch_read_pairs(b1, o1, b2, o2, k=31, c=7, no_dedup=no_dedup)
        ec, emean, end = R.sketch_read_pairs(r1, r2, 31, 7, no_dedup=no_dedup)
        assert dict(zip(h.tolist(), c.tolist())) == ec
        assert nd == end and abs(mean - emean) < 1e-12
    assert O.sketch_read_pairs(b1, o1, b2, o2, k=31, c=7)[3] > 100


def test_poisson_cutoffs_and_device_table():
    exp = [11, 15, 18, 21, 24, 26, 28, 31, 33, 35, 37, 39, 41, 43, 45, 46, 48, 50, 52, 53, 55, 57, 58, 60, 62, 63, 65, 67, 68]
    got = [O.poisson_cutoff(m) for m in range(1, 30)]
    assert got == exp
    for m in (1, 2, 7, 15, 23, 29):
        assert R.poisson_cdf(float(m), exp[m - 1]) < 0.9999999999 <= R.poisson_cdf(float(m), exp[m - 1] + 1)
    # the table baked into the CUDA source must be the same list
    src = open(os.path.join(REPO, "sylph_b200", "csrc", "contain.cu")).read()
    m = re.search(r"c_pois_cut\[30\]\s*=\s*\{([^}]*)\}", src)
    dev = [int(x) for x in m.group(1).replace("\n", " ").split(",")]
    assert dev == [0] + exp


def test_poisson_cutoff_table_against_an_independent_regularized_gamma():
    """statrs' Poisson::cdf(x) is the regularized upper incomplete gamma Q(x+1, lambda) (src/contain.rs:664-675 walks it
    up to CUTOFF_PVALUE = 0.9999999999).  The table the kernels use was derived from a direct series; scipy's
    gammaincc (Cephes igamc: a different algorithm) must put every entry on the same side of the threshold, with a
    margin well above double rounding (tightest: m = 7 at 1.7e-13)."""
    from scipy.special import gammaincc
    exp = [11, 15, 18, 21, 24, 26, 28, 31, 33, 35, 37, 39, 41, 43, 45, 46, 48, 50, 52, 53, 55, 57, 58, 60, 62, 63, 65, 67, 68]
    thr = 0.9999999999
    for m, cut in zip(range(1, 30), exp):
        below, above = float(gammaincc(cut + 1, m)), float(gammaincc(cut + 2, m))   # cdf(cut), cdf(cut + 1)
        assert below < thr - 1e-13 and above >= thr + 1e-13, (m, cut, below - thr, above - thr)
        for x in range(m, cut):                                                     # monotone: nothing earlier crosses
            assert float(gammaincc(x + 1, m)) < thr


def test_fastrand_stream_c_vs_pyref():
    rng = R.WyRand(7)
    seq = [rng.usize(17400) for _ in range(50)]
    assert [O.fastrand_usize(7, i + 1, 17400) for i in range(50)] == seq
    assert all(0 <= x < 17400 for x in seq)


def test_get_stats_vs_pyref():
    rng = np.random.default_rng(21)
    for trial, (cov_lambda, present) in enumerate([(0.4, 0.9), (1.2, 0.97), (6.0, 1.0), (0.05, 0.5)]):
        gk = np.unique(rng.integers(1, 2**57, size=3000, dtype=np.uint64))[:2500]
        counts = rng.poisson(cov_lambda, size=len(gk))
        keep = (counts > 0) & (rng.random(len(gk)) < present)
        extra = rng.integers(2**57, 2**58, size=500, dtype=np.uint64)
        sh = np.concatenate([gk[keep], extra])
        sc = np.concatenate([counts[keep], rng.integers(1, 5, size=500)]).astype(np.uint32)
        smp = O.Sample(sh, sc)
        for min_ani in (-1.0, 10.0):
            p = O.default_params(minimum_ani=min_ani)
            r = O.get_stats(p, gk, smp)
            e = R.get_stats(gk.tolist(), dict(zip(sh.tolist(), sc.tolist())), min_ani=0.90 if min_ani < 0 else min_ani / 100)
            assert (r is None) == (e is None)
            if r is None:
                continue
            assert r.contain == e["contain"] and r.glen == e["glen"] and r.median_cov == e["median_cov"]
            assert ["LOW", "HIGH", "LAMBDA"][r.lambda_status] == e["status"]
            for f in ("naive_ani", "final_est_ani", "final_est_cov", "mean_cov"):
                assert abs(getattr(r, f) - e[f]) < 1e-12
            assert bool(r.ci_valid) == (e["ci"] is not None)
            if e["ci"]:
                assert np.allclose(list(r.ci), e["ci"], rtol=0, atol=1e-12)


@pytest.mark.parametrize("pseudotax", [False, True])
def test_contain_sample_vs_pyref(pseudotax):
    """query / profile body (pass 1, winner table, pass 2, derep, abundances, output order) of the C
    oracle against the independent Python restatement, on k-mer sets with close relatives so that
    k-mers are reassigned and a redundant genome is dropped."""
    rng = np.random.default_rng(77 + int(pseudotax))
    pool = np.unique(rng.integers(1, 2**57, size=30000, dtype=np.uint64))
    rng.shuffle(pool)
    base = [pool[0:3000], pool[3000:5500], pool[5500:8000], pool[8000:10000]]
    genomes = [
        dict(kmers=base[0], tracked=pool[20000:20050], gn_size=600000),
        dict(kmers=np.concatenate([base[0][:2700], pool[10000:10300]]), tracked=base[0][2700:2760], gn_size=590000),  # 90 % relative of 0
        dict(kmers=base[1], tracked=pool[20100:20120], gn_size=500000),
        dict(kmers=np.concatenate([base[1][:2490], pool[10300:10310]]), tracked=np.zeros(0, np.uint64), gn_size=500000),  # ~identical to 2
        dict(kmers=base[2], tracked=pool[20200:20230], gn_size=450000),   # low coverage: lambda branch
        dict(kmers=base[3], tracked=np.zeros(0, np.uint64), gn_size=400000),  # absent
        dict(kmers=pool[12000:12040], tracked=np.zeros(0, np.uint64), gn_size=8000),  # fewer than min_number_kmers
        dict(kmers=np.concatenate([pool[13000:15000], base[0][2000:2600]]), tracked=pool[20300:20310], gn_size=520000),  # shares 600 k-mers with 0, survives
    ]
    sample = {}
    for km in base[0]:
        c = int(rng.poisson(6.0))
        if c:
            sample[int(km)] = c
    for km in base[1]:
        c = int(rng.poisson(35.0))  # median >= 30: no Poisson cut-off
        if c:
            sample[int(km)] = c
    for km in base[2]:
        c = int(rng.poisson(0.6))
        if c:
            sample[int(km)] = c
    for km in pool[13000:15000]:
        c = int(rng.poisson(4.0))
        if c:
            sample[int(km)] = c
    for km in pool[10300:10310]:
        sample[int(km)] = 30
    for km in pool[25000:26000]:
        sample[int(km)] = int(rng.integers(1, 4))
    sample[int(base[0][5])] = 0  # a zero count is skipped (src/contain.rs:634-636)
    exp = R.contain_sample([dict(kmers=g["kmers"].tolist(), tracked=g["tracked"].tolist(), gn_size=g["gn_size"]) for g in genomes],
                           sample, pseudotax=pseudotax)
    kmers = np.concatenate([g["kmers"] for g in genomes])
    koff = np.cumsum([0] + [len(g["kmers"]) for g in genomes]).astype(np.uint64)
    tracked = np.concatenate([g["tracked"] for g in genomes]).astype(np.uint64)
    toff = np.cumsum([0] + [len(g["tracked"]) for g in genomes]).astype(np.uint64)
    gs = np.array([g["gn_size"] for g in genomes], dtype=np.uint64)
    sh = np.array(list(sample.keys()), dtype=np.uint64)
    sc = np.array(list(sample.values()), dtype=np.uint32)
    got = O.contain_sample(O.default_params(pseudotax=pseudotax), kmers, koff, tracked, toff, gs, O.Sample(sh, sc))
    assert [r.genome for r in got] == [e["genome"] for e in exp]
    assert len(exp) >= 3
    if pseudotax:
        ids = [e["genome"] for e in exp]
        assert 0 in ids and 7 in ids and 1 not in ids and (2 in ids) != (3 in ids)  # relatives dereplicated
        assert any(e["kmers_lost"] >= 500 for e in exp)
    for r, e in zip(got, exp):
        assert r.contain == e["contain"] and r.glen == e["glen"] and r.median_cov == e["median_cov"]
        assert ["LOW", "HIGH", "LAMBDA"][r.lambda_status] == e["status"]
        assert r.kmers_lost == (e["kmers_lost"] if pseudotax else -1)
        for f in ("naive_ani", "final_est_ani", "final_est_cov", "mean_cov"):
            assert abs(getattr(r, f) - e[f]) < 1e-12, f
        assert bool(r.ci_valid) == (e["ci"] is not None)
        if e["ci"]:
            assert np.allclose(list(r.ci), e["ci"], rtol=0, atol=1e-12)
        if pseudotax:
            assert abs(r.rel_abund - e["rel_abund"]) < 1e-9 and abs(r.seq_abund - e["seq_abund"]) < 1e-9
    # -u / --estimate-unknown with an explicit --read-seq-id (src/contain.rs:274-279, 377-408): coverage scaled by the
    # read identity and the k-mer / read length ratio, sequence abundance by the fraction of reads explained
    unk = (98.5, 142.7, 20000)
    exp_u = R.contain_sample([dict(kmers=g["kmers"].tolist(), tracked=g["tracked"].tolist(), gn_size=g["gn_size"]) for g in genomes],
                             sample, pseudotax=pseudotax, unknown=unk)
    got_u = O.contain_sample(O.default_params(pseudotax=pseudotax), kmers, koff, tracked, toff, gs, O.Sample(sh, sc),
                             unknown=O.Unknown(*unk))
    assert [r.genome for r in got_u] == [e["genome"] for e in exp_u] == [r.genome for r in got]
    for r, e, r0 in zip(got_u, exp_u, got):
        assert abs(r.final_est_cov - e["final_est_cov"]) < 1e-9 * max(1.0, e["final_est_cov"])
        assert r.final_est_cov > r0.final_est_cov and r.final_est_ani == r0.final_est_ani
        if pseudotax:
            assert abs(r.rel_abund - e["rel_abund"]) < 1e-9 and abs(r.seq_abund - e["seq_abund"]) < 1e-9
    if pseudotax:
        assert sum(r.seq_abund for r in got_u) < 99.0 < sum(r.seq_abund for r in got) + 1e-6   # some reads are unexplained


@pytest.fixture(scope="module")
def config1():
    db = []
    for g in ("e.coli-EC590.fasta.gz", "e.coli-o157.fasta.gz", "e.coli-K12.fasta.gz"):
        recs = read_fastx(os.path.join(DATA, g))
        buf, off = flatten([s for _, s in recs])
        db.append(O.sketch_genome(buf, off) + (recs[0][0].decode(), g))
    recs = read_fastx(os.path.join(DATA, "o157_reads.fastq.gz"))
    buf, off = flatten([s for _, s in recs])
    return db, O.sketch_reads(buf, off, nthreads=4)


def run_config1(db, sample, sel, pseudotax):
    h, c = sample[0], sample[1]
    kmers = np.concatenate([db[i][0] for i in sel])
    koff = np.cumsum([0] + [len(db[i][0]) for i in sel]).astype(np.uint64)
    tr = np.concatenate([db[i][1] for i in sel])
    toff = np.cumsum([0] + [len(db[i][1]) for i in sel]).astype(np.uint64)
    gs = np.array([db[i][2] for i in sel], dtype=np.uint64)
    res = O.contain_sample(O.default_params(pseudotax=pseudotax), kmers, koff, tr, toff, gs, O.Sample(h, c))
    return [O.format_row(r, pseudotax, "o157_reads.fastq.gz", db[sel[r.genome]][4], db[sel[r.genome]][3]) for r in res]


def test_reference_pins_row_counts(config1):
    db, sample = config1
    # tests/integration_test.rs:117-126: `profile reads EC590` prints header + exactly 1 row
    assert len(run_config1(db, sample, [0], True)) == 1
    # tests/integration_test.rs:128-140: `query reads EC590 o157 K12` prints header + exactly 3 rows
    assert len(run_config1(db, sample, [0, 1, 2], False)) == 3


def test_golden_regression_fixture(config1):
    import hashlib
    db, sample = config1
    gold = json.load(open(os.path.join(REPO, "tests", "golden", "config1.json")))
    dg = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:32]  # noqa: E731
    for (km, tr, gs, _, _), g in zip(db, gold["genomes"]):
        assert (len(km), len(tr), gs) == (g["n_kmers"], g["n_tracked"], g["gn_size"])
        assert dg(km) == g["kmers_sha"] and dg(tr) == g["tracked_sha"]
    h, c, mean, nd = sample
    r = gold["reads"]
    assert (len(h), int(c.sum()), nd) == (r["n_keys"], r["sum_counts"], r["num_dup_removed"])
    assert dg(h) == r["hash_sha"] and dg(c) == r["count_sha"] and abs(mean - r["mean_read_length"]) < 1e-9
    assert run_config1(db, sample, [0], True) == gold["profile_vs_EC590"]
    assert run_config1(db, sample, [0, 1, 2], False) == gold["query_vs_all"]
    assert run_config1(db, sample, [0, 1, 2], True) == gold["profile_vs_all"]
    recs = read_fastx(os.path.join(DATA, "k12_R1.fq"))
    buf, off = flatten([s for _, s in recs])
    h2, c2, _, nd2 = O.sketch_reads(buf, off, c=20)
    k = gold["k12_R1_c20"]
    assert (len(h2), int(c2.sum()), nd2, dg(h2), dg(c2)) == (k["n_keys"], k["sum_counts"], k["num_dup_removed"], k["hash_sha"], k["count_sha"])
