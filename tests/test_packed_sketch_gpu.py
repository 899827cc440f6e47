"""GPU parity of 2-bit packed input for read pairs and genome sketches: packed == ASCII == oracle.
syl_pack2 (host packer, exact BYTE_TO_SEQ) -> syl_sketch_read_pairs_packed2 / syl_sketch_genomes_packed2, from host and
device memory: pair keys read from words at every offset mod 16, the key rule at 33 bp, the last word of a buffer,
every byte value, the seeding kernel's tile edges (32 768 bases), both genome post-passes and the slot overflow."""
import os

import numpy as np
import pytest

from tests.test_oracle_cpu import make_pairs, rand_seq
from tests.test_sketch_gpu import check_genomes
from tests.util import DATA, flatten, read_fastx

pytestmark = pytest.mark.gpu

ALL_BYTES = bytes(range(256))
TILE = 32768   # window starts per CTA tile of the seeding kernel (seed_kernel.cuh SEED_TILE)
GENOME_KEYS = ("kmers", "kmer_off", "tracked", "tracked_off", "gn_size")


def _cuda(a, dt):
    import torch
    return torch.from_numpy(np.array(a).view(dt)).cuda()


def check_pairs_packed(ctx, r1, r2, **kw):
    """ASCII and packed input, host and device memory: all four sketches equal the oracle's, bit for bit."""
    from oracle import oracle as O
    from sylph_b200.api import pack2
    b1, o1 = flatten(r1)
    b2, o2 = flatten(r2)
    eh, ec, emean, end = O.sketch_read_pairs(b1, o1, b2, o2, **kw)
    w1, w2 = pack2(b1), pack2(b2)
    host = {"ascii": (b1, o1, b2, o2, False), "packed": (w1, o1, w2, o2, True)}
    dev = {"ascii": (_cuda(b1, np.uint8), _cuda(o1, np.int64), _cuda(b2, np.uint8), _cuda(o2, np.int64), False),
           "packed": (_cuda(w1, np.int32), _cuda(o1, np.int64), _cuda(w2, np.int32), _cuda(o2, np.int64), True)}
    means = []
    for mem, inputs in (("host", host), ("device", dev)):
        for fmt, (x1, y1, x2, y2, packed) in inputs.items():
            s = ctx.sketch_pair_sequences(x1, y1, x2, y2, packed=packed, **kw)
            h, c = s.download()
            assert np.array_equal(h, eh) and np.array_equal(c, ec), (mem, fmt)
            assert s.num_dup_removed == end, (mem, fmt)
            assert abs(s.mean_read_length - emean) <= 1e-9 * max(1.0, emean), (mem, fmt)
            means.append(s.mean_read_length)
    assert len(set(means)) == 1
    return len(eh), end


def check_genomes_packed(ctx, buf, coff, goff, **kw):
    """ASCII from host memory against the oracle (check_genomes), then ASCII from device memory and packed from host and
    device memory against that result."""
    from sylph_b200.api import pack2
    d = check_genomes(ctx, buf, coff, goff, **kw)
    words = pack2(buf)
    individual = kw.get("individual", False)
    g_host = None if individual else goff
    g_dev = None if individual else _cuda(goff.astype(np.uint64), np.int64)
    runs = [
        ("host packed", words, coff, g_host, {"packed_bases": len(buf)}),
        ("device ascii", _cuda(buf, np.uint8), _cuda(coff.astype(np.uint64), np.int64), g_dev, {}),
        ("device packed", _cuda(words, np.int32), _cuda(coff.astype(np.uint64), np.int64), g_dev, {"packed_bases": len(buf)}),
    ]
    for name, b, o, g, extra in runs:
        got = ctx.sketch_genomes(b, o, g, **kw, **extra).download()
        for key in GENOME_KEYS:
            assert np.array_equal(got[key], d[key]), (name, key)
    return d


# ---- read pairs ----------------------------------------------------------------------------------------------------

def test_pairs_k12_fixture(ctx):
    r1 = [s for _, s in read_fastx(os.path.join(DATA, "k12_R1.fq"))]
    r2 = [s for _, s in read_fastx(os.path.join(DATA, "k12_R2.fq"))]
    n, _ = check_pairs_packed(ctx, r1, r2, c=20)
    assert n == 9916
    check_pairs_packed(ctx, r1, r2, c=200)
    check_pairs_packed(ctx, r1, r2[:-7], c=20)        # unequal files: pairs = records zipped


@pytest.mark.parametrize("no_dedup", [False, True])
def test_pairs_synthetic_with_duplicates(ctx, no_dedup):
    """The duplicate-heavy set of the ASCII pair tests: duplicate pairs, pairs with the same mate 1 only, overlapping
    mates, mates < 33 bp, one k-mer with hundreds of events."""
    rng = np.random.default_rng(31)
    genome = rand_seq(rng, 30000, b"ACGT")
    r1, r2 = make_pairs(rng, 4000, genome)
    hot = genome[1000:1150]
    for i in range(300):
        r1.append(hot)
        r2.append(genome[2000 + (i % 37) * 50:2150 + (i % 37) * 50])
    r1 += [b"A" * 150, b"A" * 150, b"", b"ACGTN" * 30]
    r2 += [b"A" * 150, b"A" * 150, b"ACGT" * 20, b"acgtn" * 30]
    order = rng.permutation(len(r1))
    r1, r2 = [r1[i] for i in order], [r2[i] for i in order]
    _, nd = check_pairs_packed(ctx, r1, r2, c=5, no_dedup=no_dedup)
    assert (nd > 2000) if not no_dedup else (nd == 0)


def test_pairs_mate_starts_walk_every_word_offset(ctx):
    """Mate 1 is 49 bp (start of pair p = 49p = p mod 16), mate 2 is 35 bp (start 3p mod 16): every proto pair is
    repeated at all 16 offsets of a word in both buffers, so a key read with a wrong funnel shift breaks the dedup."""
    rng = np.random.default_rng(40)
    genome = rand_seq(rng, 4000, b"ACGT")
    protos = []
    for _ in range(5):
        st = int(rng.integers(0, 3900))
        protos.append((genome[st:st + 49], genome[st + 20:st + 55]))
    r1 = [protos[p % 5][0] for p in range(160)]
    r2 = [protos[p % 5][1] for p in range(160)]
    o1, o2 = flatten(r1)[1], flatten(r2)[1]
    assert set((o1[:80] % 16).tolist()) == set(range(16)) and set((o2[:80] % 16).tolist()) == set(range(16))
    _, nd = check_pairs_packed(ctx, r1, r2, c=2)
    assert nd > 100
    check_pairs_packed(ctx, r1, r2, k=21, c=2, sem=0)


@pytest.mark.parametrize("k,sem", [(31, 1), (21, 0)])
def test_pairs_key_rule_at_33_bp(ctx, k, sem):
    """Mates of 32, 33 and 34 bp with partners of every length: a pair has keys only when both mates are >= 33 bp."""
    rng = np.random.default_rng(41)
    genome = rand_seq(rng, 6000, b"ACGT")
    r1, r2 = [], []
    for l1 in (32, 33, 34, 100):
        for l2 in (32, 33, 34, 100):
            for _ in range(6):
                st = int(rng.integers(0, 200))         # few distinct starts: many duplicate pairs and shared keys
                r1.append(genome[st:st + l1])
                r2.append(genome[st + 300:st + 300 + l2])
    order = rng.permutation(len(r1))
    r1, r2 = [r1[i] for i in order], [r2[i] for i in order]
    check_pairs_packed(ctx, r1, r2, k=k, c=2, sem=sem)


def test_pairs_last_mates_end_in_the_last_word(ctx):
    """The last pair's mates end the buffers at each of the 16 offsets of the last word (device memory: buffers of
    exactly ceil(n / 16) words), with copies earlier in the sample so that their keys decide the dedup."""
    rng = np.random.default_rng(42)
    genome = rand_seq(rng, 5000, b"ACGT")
    for t in range(16):
        st = int(rng.integers(0, 4000))
        last = (genome[st:st + 33 + t], genome[st + 200:st + 200 + 48 - t])
        r1, r2 = [last[0]], [last[1]]
        for _ in range(30):
            a = int(rng.integers(0, 4800))
            r1.append(genome[a:a + int(rng.integers(20, 160))])
            r2.append(genome[a + 100:a + 100 + int(rng.integers(20, 160))])
        r1.append(genome[:(t * 7) % 16 + 40])          # moves the last pair's start inside its word
        r2.append(genome[:(t * 5) % 16 + 40])
        r1.append(last[0])
        r2.append(last[1])
        _, nd = check_pairs_packed(ctx, r1, r2, c=2)
        assert nd > 0, t


def test_pairs_every_byte_value(ctx):
    rng = np.random.default_rng(43)
    r1, r2 = [], []
    for _ in range(600):
        a = rand_seq(rng, int(rng.integers(0, 200)), ALL_BYTES)
        b = rand_seq(rng, int(rng.integers(0, 200)), ALL_BYTES)
        r1.append(a)
        r2.append(b)
        if rng.random() < 0.3:
            r1.append(a)
            r2.append(b)
    check_pairs_packed(ctx, r1, r2, c=3)
    check_pairs_packed(ctx, r1, r2, k=21, c=3, sem=0)


def test_pairs_across_seeding_tile_edges(ctx):
    """A pair straddles every tile edge 32 768 t of both buffers at offsets 0, 1, k-2, k-1, k, L/2 and L-k, L-1."""
    rng = np.random.default_rng(44)
    k, L = 31, 150
    offsets = [0, 1, k - 2, k - 1, k, L // 2, L - k, L - 1]
    protos = [(rand_seq(rng, L, b"ACGT"), rand_seq(rng, L, b"ACGT")) for _ in range(3)]
    r1, r2, pos = [], [], 0
    for t, d in enumerate(offsets, start=1):
        start = t * TILE - d
        while start - pos > 450:
            ln = int(rng.integers(0, 420))
            dup = rng.random() < 0.03
            a, b = protos[t % 3] if dup else (rand_seq(rng, ln, b"ACGT"), rand_seq(rng, ln, b"ACGT"))
            r1.append(a)
            r2.append(b)
            pos += len(a)
        r1.append(rand_seq(rng, start - pos, b"ACGT"))
        r2.append(rand_seq(rng, start - pos, b"ACGT"))
        r1.append(protos[t % 3][0])
        r2.append(protos[t % 3][1])
        pos = start + L
    r1 += [p[0] for p in protos]
    r2 += [p[1] for p in protos]
    _, nd = check_pairs_packed(ctx, r1, r2, c=7)
    assert nd > 0


def test_pairs_k21_scalar(ctx):
    rng = np.random.default_rng(32)
    genome = rand_seq(rng, 20000, b"ACGT")
    r1, r2 = make_pairs(rng, 1500, genome)
    check_pairs_packed(ctx, r1, r2, k=21, c=9, sem=0)


# ---- genomes -------------------------------------------------------------------------------------------------------

def test_genomes_ecoli(ctx):
    bufs, coffs, goff = [], [0], [0]
    for name in ("e.coli-EC590.fasta.gz", "e.coli-o157.fasta.gz", "e.coli-K12.fasta.gz"):
        for _, s in read_fastx(os.path.join(DATA, name)):
            bufs.append(s)
            coffs.append(coffs[-1] + len(s))
        goff.append(len(coffs) - 1)
    buf = np.frombuffer(b"".join(bufs), dtype=np.uint8)
    coff = np.array(coffs, dtype=np.uint64)
    goff = np.array(goff, dtype=np.uint64)
    d = check_genomes_packed(ctx, buf, coff, goff)
    assert [int(x) for x in np.diff(d["kmer_off"])] == [19330, 21899, 19485]
    check_genomes_packed(ctx, buf, coff, goff, pseudotax=False)
    check_genomes_packed(ctx, buf, coff, goff, individual=True)
    check_genomes_packed(ctx, buf, coff, goff, individual=True, pseudotax=False)


def _contigs_at_tile_edges(rng, k):
    """Genomes whose contig boundaries fall at tile edges 32 768 t + {-k, -1, +1, +k}, with repeats inside a genome
    (dropped), a segment shared across genomes (kept), contigs shorter than 2k, empty contigs and empty genomes."""
    shared = rand_seq(rng, 5000, b"ACGT")
    deltas = [-k, -1, 1, k]
    contigs, goff, pos, t = [], [0], 0, 1
    for g in range(12):
        rep = rand_seq(rng, 800, b"ACGT")
        for ci in range(int(rng.integers(1, 6)) if g != 5 else 0):
            if ci == 1:
                contigs.append(b"")                                # an empty contig
                continue
            if ci == 2:
                ln = int(rng.choice([10, 2 * k - 1, 400]))         # short contigs between the edges
            else:
                ln = t * TILE + deltas[(t - 1) % 4] - pos          # ends at the next tile edge + delta
                t += 1
            s = rand_seq(rng, ln, b"ACGT")
            if ln >= 3000 and rng.random() < 0.7:
                s = s[:1000] + rep + s[1800:]                      # repeat inside the genome
            if ln >= 12000 and rng.random() < 0.5:
                s = s[:6000] + shared + s[11000:]                  # shared across genomes
            contigs.append(s)
            pos += len(s)
        goff.append(len(contigs))
    contigs.append(rand_seq(rng, 2 * k - 3, b"ACGT"))               # a genome shorter than 2k
    goff.append(len(contigs))
    buf, coff = flatten(contigs)
    edges = {int(x) % TILE for x in coff}
    assert {TILE - k, TILE - 1, 1, k} <= edges
    return buf, coff, np.array(goff, dtype=np.uint64)


@pytest.mark.parametrize("postpass", ["slots", "sort"])
@pytest.mark.parametrize("k,sem", [(31, 1), (21, 0)])
def test_genomes_multicontig_at_tile_edges(ctx, monkeypatch, k, sem, postpass):
    """c >= 96 takes the slotted front half of the post-pass unless SYL_GENOME_POSTPASS=sort; c < 96 (down to c = 1,
    where every hash below u64::MAX survives) always takes the sorted one."""
    monkeypatch.delenv("SYL_GENOME_POSTPASS", raising=False)
    if postpass == "sort":
        monkeypatch.setenv("SYL_GENOME_POSTPASS", "sort")
    rng = np.random.default_rng(50 + k)
    buf, coff, goff = _contigs_at_tile_edges(rng, k)
    check_genomes_packed(ctx, buf, coff, goff, k=k, c=200, sem=sem)
    check_genomes_packed(ctx, buf, coff, goff, k=k, c=128, min_spacing=10, sem=sem, individual=True)
    check_genomes_packed(ctx, buf, coff, goff, k=k, c=11, sem=sem)
    check_genomes_packed(ctx, buf, coff, goff, k=k, c=3, min_spacing=5, sem=sem, pseudotax=False)
    check_genomes_packed(ctx, buf, coff, goff, k=k, c=2, min_spacing=5, sem=sem)
    d = check_genomes_packed(ctx, buf, coff, goff, k=k, c=1, sem=sem)
    assert (np.concatenate([d["kmers"], d["tracked"]]) >= np.uint64(1 << 63)).any()   # c = 1: hashes use all 64 bits


def test_genomes_every_byte_value(ctx):
    rng = np.random.default_rng(51)
    contigs = [rand_seq(rng, int(n), ALL_BYTES) for n in rng.integers(0, 40000, size=12)]
    buf, coff = flatten(contigs)
    goff = np.array([0, 3, 3, 8, 12], dtype=np.uint64)
    check_genomes_packed(ctx, buf, coff, goff, c=200)
    check_genomes_packed(ctx, buf, coff, goff, c=5)


def test_genomes_low_complexity_overflows_the_tile_slots(ctx):
    """A tandem repeat whose k-mer survives overflows a tile slot: the slotted path falls back to the sort path, on
    packed input as on ASCII."""
    from oracle import oracle as O
    rng = np.random.default_rng(9)
    unit = None
    for _ in range(2000):
        u = rand_seq(rng, 40, b"ACGT")
        if len(O.extract_markers(u * 4, k=31, c=200)) > 0:
            unit = u
            break
    assert unit is not None
    contigs = [unit * 5000, rand_seq(rng, 150000, b"ACGT"), unit * 3000 + rand_seq(rng, 50000, b"ACGT")]
    buf, coff = flatten(contigs)
    check_genomes_packed(ctx, buf, coff, np.array([0, 2, 3], dtype=np.uint64), c=200)


# ---- arguments -----------------------------------------------------------------------------------------------------

def test_packed_arguments(ctx, monkeypatch):
    """Device word buffers must be 16-byte aligned (SYL_ERR_ARG), host and device word buffers must hold
    ceil(n_bases / 16) words (ValueError before the call)."""
    import torch
    from sylph_b200 import SylphError
    from sylph_b200.api import pack2
    rng = np.random.default_rng(52)
    b, o = flatten([rand_seq(rng, 150, b"ACGT") for _ in range(200)])
    w = pack2(b)
    od = _cuda(o, np.int64)
    wd = _cuda(w, np.int32)
    shifted = _cuda(np.concatenate([np.zeros(1, np.uint32), w]), np.int32)[1:]   # 4 bytes past a 16-byte boundary
    assert shifted.data_ptr() % 16 == 4
    with pytest.raises(SylphError) as e:
        ctx.sketch_pair_sequences(shifted, od, wd, od, packed=True)
    assert e.value.code == 1
    with pytest.raises(SylphError) as e:
        ctx.sketch_pair_sequences(wd, od, shifted, od, packed=True)
    assert e.value.code == 1
    goff = torch.tensor([0, len(o) - 1], dtype=torch.int64, device="cuda")
    for postpass in ("slots", "sort"):
        monkeypatch.setenv("SYL_GENOME_POSTPASS", postpass)
        with pytest.raises(SylphError) as e:
            ctx.sketch_genomes(shifted, od, goff, packed_bases=len(b))
        assert e.value.code == 1
    monkeypatch.delenv("SYL_GENOME_POSTPASS")
    with pytest.raises(ValueError):
        ctx.sketch_pair_sequences(w[:-1], o, w, o, packed=True)
    with pytest.raises(ValueError):
        ctx.sketch_pair_sequences(wd, od, wd[:-1], od, packed=True)
    with pytest.raises(ValueError):
        ctx.sketch_genomes(w[:-1], o, np.array([0, len(o) - 1], dtype=np.uint64), packed_bases=len(b))
    with pytest.raises(ValueError):
        ctx.sketch_genomes(wd[:-1], od, goff, packed_bases=len(b))
    seqs = [bytes(b[int(o[i]):int(o[i + 1])]) for i in range(len(o) - 1)]
    check_pairs_packed(ctx, seqs, seqs, c=5)           # the ctx still works after the refusals
