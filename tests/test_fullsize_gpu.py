"""GPU: the BASELINE.json full-size workloads, bit-exact against the oracle.

  config 2: 1 Gbp of 150 bp reads (6 666 667 reads, 2 % exact duplicates => the order-dependent dedup
            state machine of src/sketch.rs:690-731 runs on ~4 M events) — the oracle sketches the same
            bytes with all host cores in a few seconds; hashes, counts and num_dup_removed must be equal.
  config 3: that sample against 10 000 synthetic 4 Mbp genome sketches — `query` and `profile` rows
            field by field, bit for bit against the correctly rounded oracle (tests/contain_compare.py).
  config 5 shape: a batch of 4 Mbp genomes sketched in ONE call == the oracle's per-genome sketches.
plus the size-independent properties (sortedness, conservation, determinism, host path == device path).
"""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from tests.contain_compare import compare, cr_params, sort_query_rows

pytestmark = pytest.mark.gpu

N_READS = 6_666_667


@pytest.fixture(scope="module")
def gbp(ctx):
    import torch
    from sylph_b200 import synth
    b, o = synth.reads(N_READS, device="cuda")
    torch.cuda.synchronize()
    s = ctx.sketch_sequences(b, o)
    h, c = s.download()
    hb, ho = b.cpu().numpy(), o.cpu().numpy().astype(np.uint64)
    yield dict(b=b, o=o, s=s, h=h, c=c, hb=hb, ho=ho)
    s.free()


def test_one_gbp_bit_exact_vs_oracle(ctx, gbp):
    """src/sketch.rs:917-947 over the whole config-2 sample, dedup ON."""
    from oracle import oracle as O
    cores = os.cpu_count() or 1
    eh, ec, emean, end = O.sketch_reads(gbp["hb"], gbp["ho"], sem=O.SEM_AVX2_INTRIN, nthreads=cores)
    assert len(eh) > 1_000_000 and end > 10_000          # the duplicate reads really exercise the dedup
    assert np.array_equal(gbp["h"], eh)
    assert np.array_equal(gbp["c"], ec)
    assert gbp["s"].num_dup_removed == end
    assert abs(gbp["s"].mean_read_length - emean) <= 1e-9 * emean
    # no_dedup: plain multiplicities
    eh2, ec2, _, nd2 = O.sketch_reads(gbp["hb"], gbp["ho"], no_dedup=True, sem=O.SEM_AVX2_INTRIN, nthreads=cores)
    s2 = ctx.sketch_sequences(gbp["b"], gbp["o"], no_dedup=True)
    h2, c2 = s2.download()
    assert nd2 == 0 and s2.num_dup_removed == 0
    assert np.array_equal(h2, eh2) and np.array_equal(c2, ec2)
    s2.free()


def test_one_gbp_properties(ctx, gbp):
    import torch
    b, o, s1, h1, c1 = gbp["b"], gbp["o"], gbp["s"], gbp["h"], gbp["c"]
    assert np.all(h1[1:] > h1[:-1]) and c1.min() >= 1
    surv = torch.empty(int(b.numel() / 200 * 1.3 + 65536) * 2, dtype=torch.int64, device="cuda")
    n_surv = ctx.extract_markers_batch(b, o, out=surv)
    del surv
    assert int(c1.astype(np.int64).sum()) + s1.num_dup_removed == n_surv
    s2 = ctx.sketch_sequences(b, o)
    h2, c2 = s2.download()
    assert np.array_equal(h1, h2) and np.array_equal(c1, c2) and s1.num_dup_removed == s2.num_dup_removed
    s3 = ctx.sketch_sequences(gbp["hb"], gbp["ho"])   # host buffers: chunked, copies overlapped with seeding
    h3, c3 = s3.download()
    assert np.array_equal(h1, h3) and np.array_equal(c1, c3) and s3.num_dup_removed == s1.num_dup_removed
    s2.free()
    s3.free()


def test_config3_10k_genomes_query_and_profile_vs_oracle(ctx, gbp):
    """src/contain.rs:284-334 for 1 sample x 10 000 genomes: every output field of every row."""
    from oracle import oracle as O
    from sylph_b200 import synth
    cores = os.cpu_count() or 1
    G = 10_000
    genomes = synth.sketch_db_range(ctx, 0, G)
    d = genomes.download()
    assert len(d["kmer_off"]) == G + 1 and int(d["kmer_off"][-1]) > 150_000_000
    db = ctx.build_db(genomes)
    smp = O.Sample(gbp["h"], gbp["c"])
    for pseudotax in (False, True):
        exp = O.contain_sample(cr_params(pseudotax=pseudotax), d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"],
                               d["gn_size"], smp, nthreads=cores)
        rows = ctx.profile(db, [gbp["s"]]) if pseudotax else sort_query_rows(ctx.query(db, [gbp["s"]]))
        assert len(exp) >= 40
        compare(rows, exp, pseudotax)
    # spot-check the db itself: 16 genomes spread over the range == the oracle's sketch of the same bytes
    for g in range(0, G, G // 16):
        gb, _ = synth.db_chunk(g, g + 1, 4_000_000)
        km, tr, gs = O.sketch_genome(gb.numpy(), np.array([0, 4_000_000], np.uint64))
        assert np.array_equal(km, d["kmers"][int(d["kmer_off"][g]):int(d["kmer_off"][g + 1])])
        assert np.array_equal(tr, d["tracked"][int(d["tracked_off"][g]):int(d["tracked_off"][g + 1])])
        assert gs == int(d["gn_size"][g])
    db.free()
    genomes.free()


def test_config5_genome_batch_vs_oracle(ctx):
    """src/sketch.rs:550-622 for a 0.5 Gbp batch (125 x 4 Mbp incl. the mutant genome 99) in one call."""
    from oracle import oracle as O
    from sylph_b200 import synth
    g0, g1, L = 50, 175, 4_000_000
    genomes = synth.sketch_db_range(ctx, g0, g1)
    d = genomes.download()

    def one(g):
        gb, _ = synth.db_chunk(g, g + 1, L)
        return O.sketch_genome(gb.numpy(), np.array([0, L], np.uint64))

    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as ex:
        exp = list(ex.map(one, range(g0, g1)))
    for i, (km, tr, gs) in enumerate(exp):
        assert np.array_equal(km, d["kmers"][int(d["kmer_off"][i]):int(d["kmer_off"][i + 1])]), g0 + i
        assert np.array_equal(tr, d["tracked"][int(d["tracked_off"][i]):int(d["tracked_off"][i + 1])]), g0 + i
        assert gs == int(d["gn_size"][i])
    genomes.free()
