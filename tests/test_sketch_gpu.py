"""GPU parity: sample sketch (a5) and genome sketch (a4) vs the CPU oracle, bit-exact."""
import os

import numpy as np
import pytest

from tests.util import DATA, flatten, read_fastx, seed_mode  # noqa: F401  (seed_mode: fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("seed_mode")]


def check_reads(ctx, buf, off, k=31, c=200, no_dedup=False, sem=1):
    from oracle import oracle as O
    s = ctx.sketch_sequences(buf, off, k=k, c=c, no_dedup=no_dedup, sem=sem)
    h, cnt = s.download()
    eh, ec, mean, nd = O.sketch_reads(buf, off, k=k, c=c, no_dedup=no_dedup, sem=sem)
    assert len(h) == len(eh)
    assert np.array_equal(h, eh)
    assert np.array_equal(cnt, ec)
    assert s.num_dup_removed == nd
    assert abs(s.mean_read_length - mean) <= 1e-6 * max(1.0, mean)
    return len(h), nd


def check_genomes(ctx, buf, coff, goff, k=31, c=200, min_spacing=30, pseudotax=True, individual=False, sem=1):
    from oracle import oracle as O
    g = ctx.sketch_genomes(buf, coff, None if individual else goff, k=k, c=c, min_spacing=min_spacing,
                           pseudotax=pseudotax, individual=individual, sem=sem)
    d = g.download()
    if individual:
        goff = np.arange(len(coff), dtype=np.uint64)
    assert len(g) == len(goff) - 1
    for gi in range(len(goff) - 1):
        c0, c1 = int(goff[gi]), int(goff[gi + 1])
        b0, b1 = int(coff[c0]), int(coff[c1])
        sub_off = (coff[c0:c1 + 1] - coff[c0]).astype(np.uint64)
        km, tr, gs = O.sketch_genome(buf[b0:b1], sub_off, k=k, c=c, min_spacing=min_spacing, pseudotax=pseudotax, sem=sem)
        got_k = d["kmers"][int(d["kmer_off"][gi]):int(d["kmer_off"][gi + 1])]
        got_t = d["tracked"][int(d["tracked_off"][gi]):int(d["tracked_off"][gi + 1])]
        assert np.array_equal(got_k, km), "genome %d kmers" % gi
        assert np.array_equal(got_t, tr), "genome %d tracked" % gi
        assert int(d["gn_size"][gi]) == gs
    return d


def rand_seqs(rng, lengths, alphabet=b"ACGT"):
    return [bytes(rng.choice(list(alphabet), size=int(n)).astype(np.uint8)) for n in lengths]


def check_repeat_and_shared(ctx, rng, k=31, c=200, sem=1):
    """A segment x three times in genome 0 (twice in one contig): all its markers are dropped there.  A segment y
    exactly once in each of genomes 1 and 2: all its markers are kept or tracked in both."""
    from oracle import oracle as O
    x, y, *f = rand_seqs(rng, [20000, 20000, 3000, 3000, 3000, 500, 500, 2000, 2000, 100, 4000, 1000])
    contigs = [f[0] + x + f[1] + x + f[2], f[3] + x + f[4], f[5] + y + f[6], f[7], f[8] + y + f[9]]
    buf, coff = flatten(contigs)
    d = check_genomes(ctx, buf, coff, np.array([0, 2, 3, 5], dtype=np.uint64), k=k, c=c, sem=sem)

    def sketch(g):
        return (set(d["kmers"][int(d["kmer_off"][g]):int(d["kmer_off"][g + 1])].tolist())
                | set(d["tracked"][int(d["tracked_off"][g]):int(d["tracked_off"][g + 1])].tolist()))
    mx, my = (set(O.extract_markers(s, k=k, c=c, sem=sem).tolist()) for s in (x, y))
    assert mx and my
    assert not mx & sketch(0)
    assert my <= sketch(1) and my <= sketch(2)


def test_reads_dedup_k12(ctx):
    recs = read_fastx(os.path.join(DATA, "k12_R1.fq"))
    buf, off = flatten([s for _, s in recs])
    check_reads(ctx, buf, off, c=20)
    check_reads(ctx, buf, off, c=200)


def test_reads_o157_long(ctx):
    recs = read_fastx(os.path.join(DATA, "o157_reads.fastq.gz"))
    buf, off = flatten([s for _, s in recs])
    n, nd = check_reads(ctx, buf, off)
    assert n == 25621


@pytest.mark.parametrize("no_dedup", [False, True])
def test_reads_heavy_duplicates(ctx, no_dedup):
    """Exercise the c<4 state machine: exact duplicate reads, shortened copies (same start, no pair key in common),
    reads > 400 bp (no pair), reads < 66 bp (no pair), homopolymers (p0 == p1).  Matches on one key only and across
    the two key slots are in tests/test_dedup_scripts_gpu.py."""
    rng = np.random.default_rng(123)
    genome = rand_seqs(rng, [150000])[0]
    seqs = []
    for i in range(6000):
        st = int(rng.integers(0, 150000 - 500))
        ln = int(rng.choice([60, 70, 100, 150, 150, 150, 250, 401, 500]))
        s = genome[st:st + ln]
        seqs.append(s)
        if rng.random() < 0.3:
            seqs.append(s)                      # exact duplicate
        if rng.random() < 0.1:
            seqs.append(genome[st:st + ln - 2])  # same start, middle window moved: both keys differ
    seqs += [b"A" * 150, b"A" * 150, b"A" * 150, b"ACGT" * 40, b"ACGT" * 40, b"", b"ACG"]
    order = rng.permutation(len(seqs))
    seqs = [seqs[i] for i in order]
    buf, off = flatten(seqs)
    n, nd = check_reads(ctx, buf, off, c=5, no_dedup=no_dedup)
    if not no_dedup:
        assert nd > 300


def test_reads_synthetic_community(ctx):
    from sylph_b200 import synth
    b, o = synth.reads(60000, n_comm=4, genome_len=200000)
    check_reads(ctx, b.numpy(), o.numpy().astype(np.uint64))
    check_reads(ctx, b.numpy(), o.numpy().astype(np.uint64), k=21, c=50, sem=0)


def test_reads_device_resident_and_empty(ctx):
    import torch
    from sylph_b200 import synth
    b, o = synth.reads(20000, n_comm=2, genome_len=100000)
    s_h = ctx.sketch_sequences(b.numpy(), o.numpy().astype(np.uint64))
    s_d = ctx.sketch_sequences(b.cuda(), o.cuda())
    for x, y in zip(s_h.download(), s_d.download()):
        assert np.array_equal(x, y)
    e = ctx.sketch_sequences(np.zeros(0, np.uint8), np.zeros(1, np.uint64))
    assert len(e) == 0


def test_reads_homopolymers_overflow_the_event_estimate(ctx):
    """mm_hash64(AAA..A) = 0.468 * 2^64 < 2^64 / 2: with c = 2 every window of a poly-A / poly-T read
    survives, so the batch emits far more events than the n_bases / c sizing assumes.  Exercises the
    capacity retry of the event buffer (and the recount of the bucket histogram after it), one k-mer
    with ~10^6 events (generic path for its group) and reads whose pair keys are all identical."""
    from tests.util import flatten
    rng = np.random.default_rng(99)
    seqs = [b"A" * 150] * 5000 + [b"T" * 150] * 4000 + rand_seqs(rng, [150] * 3000) + [b"A" * 60, b"T" * 401, b"C" * 150]
    order = rng.permutation(len(seqs))
    buf, off = flatten([seqs[i] for i in order])
    n, nd = check_reads(ctx, buf, off, k=31, c=2)
    assert n > 1000 and nd > 500000
    check_reads(ctx, buf, off, k=31, c=2, no_dedup=True)


def test_sample_download_into_pinned_buffers(ctx):
    import torch
    from sylph_b200 import synth
    b, o = synth.reads(20000, n_comm=2, genome_len=100000)
    s = ctx.sketch_sequences(b.numpy(), o.numpy().astype(np.uint64))
    h, c = s.download()
    oh = torch.empty(len(s) + 100, dtype=torch.int64, pin_memory=True).numpy().view(np.uint64)
    oc = torch.empty(len(s) + 100, dtype=torch.int32, pin_memory=True).numpy().view(np.uint32)
    h2, c2 = s.download(oh, oc)
    assert np.array_equal(h, h2) and np.array_equal(c, c2) and np.shares_memory(h2, oh)
    with pytest.raises(ValueError):
        s.download(oh[:10], oc)


def test_genomes_ecoli(ctx):
    bufs, coffs, goff = [], [0], [0]
    for name in ("e.coli-EC590.fasta.gz", "e.coli-o157.fasta.gz", "e.coli-K12.fasta.gz"):
        recs = read_fastx(os.path.join(DATA, name))
        for _, s in recs:
            bufs.append(s)
            coffs.append(coffs[-1] + len(s))
        goff.append(len(coffs) - 1)
    buf = np.frombuffer(b"".join(bufs), dtype=np.uint8)
    coff = np.array(coffs, dtype=np.uint64)
    goff = np.array(goff, dtype=np.uint64)
    d = check_genomes(ctx, buf, coff, goff)
    assert [int(x) for x in np.diff(d["kmer_off"])] == [19330, 21899, 19485]
    check_genomes(ctx, buf, coff, goff, pseudotax=False)
    check_genomes(ctx, buf, coff, goff, individual=True)


@pytest.mark.parametrize("k,sem", [(31, 1), (21, 0)])
def test_genomes_multicontig_with_repeats(ctx, k, sem):
    """Many genomes, ragged contigs (incl. < 2k and empty), repeated segments inside a genome
    (must be dropped entirely) and shared segments across genomes (must be kept); c down to 1, where
    every hash below u64::MAX survives."""
    rng = np.random.default_rng(77)
    shared = rand_seqs(rng, [5000])[0]
    contigs, goff = [], [0]
    for g in range(40):
        nc = int(rng.integers(0, 12))
        rep = rand_seqs(rng, [800])[0]
        for ci in range(nc):
            ln = int(rng.choice([0, 10, 40, 61, 62, 63, 500, 3000, 20000]))
            s = rand_seqs(rng, [ln])[0]
            if ln >= 3000 and rng.random() < 0.7:
                s = s[:1000] + rep + s[1800:]       # repeat inside the genome
            if ln >= 20000 and rng.random() < 0.5:
                s = s[:6000] + shared + s[11000:]   # shared across genomes
            contigs.append(s)
        goff.append(len(contigs))
    buf, coff = flatten(contigs)
    check_genomes(ctx, buf, coff, np.array(goff, dtype=np.uint64), k=k, c=11, min_spacing=30, sem=sem)
    check_genomes(ctx, buf, coff, np.array(goff, dtype=np.uint64), k=k, c=3, min_spacing=5, sem=sem)
    check_genomes(ctx, buf, coff, np.array(goff, dtype=np.uint64), k=k, c=2, min_spacing=5, sem=sem)
    d = check_genomes(ctx, buf, coff, np.array(goff, dtype=np.uint64), k=k, c=1, min_spacing=30, sem=sem)
    assert (np.concatenate([d["kmers"], d["tracked"]]) >= np.uint64(1 << 63)).any()   # c = 1: hashes use all 64 bits
    check_repeat_and_shared(ctx, rng, k=k, c=1, sem=sem)


@pytest.mark.parametrize("postpass", ["slots", "sort"])
def test_genomes_c200_slotted_postpass(ctx, monkeypatch, postpass):
    """c >= 96 takes the slotted front half of the post-pass (per-tile slots, no sort, genome.cu); same inputs
    through the sorted front half.  Long contigs (many tiles), repeats inside a genome (dropped), segments shared
    across genomes (kept), genomes with thousands of survivors, empty genomes, --individual-records, no tracked
    k-mers, batches without survivors or without contigs."""
    if postpass == "sort":
        monkeypatch.setenv("SYL_GENOME_POSTPASS", "sort")
    rng = np.random.default_rng(2024)
    shared = rand_seqs(rng, [30000])[0]
    contigs, goff = [], [0]
    for g in range(24):
        nc = (int(rng.integers(0, 5)) if g != 7 else 0) if g != 3 else 3
        rep = rand_seqs(rng, [6000])[0]
        for ci in range(nc):
            ln = int(rng.choice([0, 61, 62, 5000, 70000, 200000, 40000])) if not (g == 3 and ci == 1) else 2500000
            s = rand_seqs(rng, [ln])[0]
            if ln >= 40000 and rng.random() < 0.7:
                s = s[:10000] + rep + s[16000:20000] + rep + s[26000:]   # repeat inside the genome, twice in one contig
            if ln >= 70000 and rng.random() < 0.6:
                s = s[:30000] + shared + s[60000:]                       # shared across genomes
            contigs.append(s)
        goff.append(len(contigs))
    buf, coff = flatten(contigs)
    goff = np.array(goff, dtype=np.uint64)
    d = check_genomes(ctx, buf, coff, goff, c=200)
    assert int(np.diff(d["kmer_off"]).max()) > 6000       # a genome with thousands of survivors
    check_genomes(ctx, buf, coff, goff, c=100, min_spacing=10)
    check_genomes(ctx, buf, coff, goff, c=200, pseudotax=False)
    check_genomes(ctx, buf, coff, goff, c=200, individual=True)
    check_genomes(ctx, buf, coff, goff, k=21, c=128, sem=0)
    check_repeat_and_shared(ctx, rng, c=200)
    # no survivors at all: every contig shorter than k, an empty contig and an empty genome
    buf, coff = flatten([b"ACGT" * 7, b"", b"A" * 30, b"C" * 12])
    d = check_genomes(ctx, buf, coff, np.array([0, 2, 2, 4], dtype=np.uint64), c=200)
    assert d["kmers"].size == 0 and d["tracked"].size == 0 and not d["kmer_off"].any() and not d["tracked_off"].any()
    assert d["gn_size"].tolist() == [28, 0, 42]
    # no contigs at all
    buf, coff = flatten([])
    d = check_genomes(ctx, buf, coff, np.array([0, 0, 0], dtype=np.uint64), c=200)
    assert d["kmers"].size == 0 and not d["kmer_off"].any() and d["gn_size"].tolist() == [0, 0]


def test_genomes_low_complexity_overflows_the_tile_slots(ctx):
    """A tandem repeat whose k-mer survives fills a tile with far more than 512 survivors: the slotted path reports
    the overflow and the call is redone on the generic path (all copies are duplicates and must vanish)."""
    from oracle import oracle as O
    rng = np.random.default_rng(9)
    unit = None
    for _ in range(2000):
        u = rand_seqs(rng, [40])[0]
        if len(O.extract_markers(u * 4, k=31, c=200)) > 0:
            unit = u
            break
    assert unit is not None
    contigs = [unit * 5000, rand_seqs(rng, [150000])[0], unit * 3000 + rand_seqs(rng, [50000])[0]]
    buf, coff = flatten(contigs)
    check_genomes(ctx, buf, coff, np.array([0, 2, 3], dtype=np.uint64), c=200)
