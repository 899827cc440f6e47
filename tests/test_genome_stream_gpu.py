"""GPU parity: genome batches from host memory through the chunked feeder (chunks of whole genomes, genomes larger than a
chunk staged on their own) against the same batch from device memory, and on small batches against the oracle: every
array of the result equal, for pinned and pageable ASCII and host 2-bit words, under every ingest setting and chunk size.
Also: the device memory of a large host batch stays bounded by the output, the ingest statistics, indexing the result,
and the driver's .syldb."""
import os

import numpy as np
import pytest

from tests.test_driver_gpu import exe, run  # noqa: F401 (exe: the fixture that builds the driver)
from tests.test_sketch_gpu import check_genomes, rand_seqs
from tests.util import DATA, flatten, read_fastx

pytestmark = pytest.mark.gpu

MIB = 1 << 20
ODD = 16 * 4097                     # an odd multiple of 16 bases
KEYS = ("kmers", "kmer_off", "tracked", "tracked_off", "gn_size")
INGEST = {"default": {}, "ascii": {"SYL_HOST_INGEST": "ascii"}, "packed-only": {"SYL_HOST_INGEST": "packed-only"},
          "steal": {"SYL_INGEST_FORCE_STEAL": "1"}}
ENV = ("SYL_HOST_INGEST", "SYL_INGEST_FORCE_STEAL", "SYL_INGEST_CHUNK", "SYL_GENOME_POSTPASS")


def set_env(monkeypatch, ingest="default", chunk=None):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in INGEST[ingest].items():
        monkeypatch.setenv(k, v)
    if chunk:
        monkeypatch.setenv("SYL_INGEST_CHUNK", str(chunk))


def _cuda(a, dt):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(dt)).cuda()


def _pinned(a, dt):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(dt)).pin_memory()


def sketch(ctx, buf, coff, goff, source, **kw):
    from sylph_b200.api import pack2
    g = None if kw.get("individual") else goff
    if source == "device":
        return ctx.sketch_genomes(_cuda(buf, np.uint8), _cuda(coff, np.int64), None if g is None else _cuda(g, np.int64), **kw)
    if source == "pinned":
        return ctx.sketch_genomes(_pinned(buf, np.uint8), _pinned(coff, np.int64), None if g is None else _pinned(g, np.int64), **kw)
    if source == "pageable":
        return ctx.sketch_genomes(buf, coff, g, **kw)
    assert source == "words"
    return ctx.sketch_genomes(pack2(buf), coff, g, packed_bases=len(buf), **kw)


def compare(ctx, buf, coff, goff, sources=("pinned", "pageable", "words"), ref=None, **kw):
    """every host source's result equal to the device-input result (ref: that result, if known) -> the device result"""
    if ref is None:
        g = sketch(ctx, buf, coff, goff, "device", **kw)
        ref = g.download()
        g.free()
    for src in sources:
        g = sketch(ctx, buf, coff, goff, src, **kw)
        got = g.download()
        g.free()
        for key in KEYS:
            assert np.array_equal(got[key], ref[key]), (src, key, kw)
    return ref


def seqs(rng, n):
    return np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes()


def mixed_batch(seed=1):
    """Genomes smaller than, equal to and larger than a chunk of 1 MiB and of ODD bases, several contigs each, a genome
    without contigs, empty contigs and contigs shorter than 2k."""
    rng = np.random.default_rng(seed)
    genomes = [[30000], [ODD], [40000, 25552], [200000, 0, 12], [MIB], [], [700000, 800000], [5000, 20], [ODD + 1],
               [], [3000], [90000, 90000, 90000]]
    contigs, goff = [], [0]
    for lens in genomes:
        contigs += [seqs(rng, n) for n in lens]
        goff.append(len(contigs))
    buf, coff = flatten(contigs)
    return buf, coff, np.array(goff, dtype=np.uint64)


@pytest.fixture(scope="module")
def batch():
    return mixed_batch()


@pytest.mark.parametrize("chunk", [MIB, ODD, None])
@pytest.mark.parametrize("ingest", list(INGEST))
def test_host_batches_equal_device_batches(ctx, monkeypatch, batch, chunk, ingest):
    buf, coff, goff = batch
    set_env(monkeypatch, ingest, chunk)
    for kw in (dict(), dict(pseudotax=False), dict(individual=True), dict(individual=True, pseudotax=False),
               dict(c=50), dict(k=21), dict(sem=0), dict(c=50, k=21, sem=0, individual=True)):
        compare(ctx, buf, coff, goff, **kw)


@pytest.mark.parametrize("chunk", [MIB, ODD, None])
def test_host_batches_equal_the_oracle(ctx, monkeypatch, chunk):
    rng = np.random.default_rng(3)
    contigs = rand_seqs(rng, [40000, 70000, 0, 50, 120000, 66000, 20000, 9000])
    buf, coff = flatten(contigs)
    goff = np.array([0, 1, 4, 4, 5, 8], dtype=np.uint64)
    set_env(monkeypatch, "default", chunk)
    for kw in (dict(), dict(c=50, k=21), dict(individual=True, pseudotax=False, sem=0)):
        d = check_genomes(ctx, buf, coff, goff, **kw)
        compare(ctx, buf, coff, goff, sources=("pinned", "words"), ref=d, **kw)


def test_sorted_front_half_forced(ctx, monkeypatch, batch):
    buf, coff, goff = batch
    set_env(monkeypatch, "default", MIB)
    monkeypatch.setenv("SYL_GENOME_POSTPASS", "sort")
    compare(ctx, buf, coff, goff)
    compare(ctx, buf, coff, goff, c=50)


def test_slot_overflow_in_one_chunk_only(ctx, monkeypatch):
    """A tandem repeat whose k-mer survives overflows the tile slots of its chunk only: that chunk alone is redone on the
    sorted front half."""
    from oracle import oracle as O
    rng = np.random.default_rng(9)
    unit = None
    for _ in range(2000):
        u = rand_seqs(rng, [40])[0]
        if len(O.extract_markers(u * 4, k=31, c=200)) > 0:
            unit = u
            break
    assert unit is not None
    contigs = [seqs(rng, 300000), seqs(rng, 200000), unit * 5000 + seqs(rng, 100000), seqs(rng, 400000), seqs(rng, 5000)]
    buf, coff = flatten(contigs)
    goff = np.array([0, 1, 2, 3, 5], dtype=np.uint64)
    set_env(monkeypatch, "default", 512 * 1024)
    d = check_genomes(ctx, buf, coff, goff, c=200)
    compare(ctx, buf, coff, goff, ref=d)
    compare(ctx, buf, coff, goff, c=200, pseudotax=False)


def test_empty_and_short_genomes(ctx, monkeypatch):
    rng = np.random.default_rng(5)
    set_env(monkeypatch, "default", ODD)
    buf, coff = flatten([])
    d = compare(ctx, buf, coff, np.array([0, 0, 0], dtype=np.uint64))
    assert d["kmers"].size == 0 and not d["kmer_off"].any() and d["gn_size"].tolist() == [0, 0]
    contigs = [b"", seqs(rng, 40), seqs(rng, 61), seqs(rng, 62), b"", seqs(rng, 100000), seqs(rng, 30)]
    buf, coff = flatten(contigs)
    goff = np.array([0, 0, 2, 2, 4, 4, 6, 7, 7], dtype=np.uint64)
    d = check_genomes(ctx, buf, coff, goff)
    compare(ctx, buf, coff, goff, ref=d)
    compare(ctx, buf, coff, goff, individual=True)


def ecoli():
    bufs, coffs, goff = [], [0], [0]
    for name in ("e.coli-EC590.fasta.gz", "e.coli-o157.fasta.gz", "e.coli-K12.fasta.gz"):
        for _, s in read_fastx(os.path.join(DATA, name)):
            bufs.append(s)
            coffs.append(coffs[-1] + len(s))
        goff.append(len(coffs) - 1)
    buf = np.frombuffer(b"".join(bufs), dtype=np.uint8).copy()
    return buf, np.array(coffs, dtype=np.uint64), np.array(goff, dtype=np.uint64)


@pytest.mark.parametrize("chunk", [MIB, None])
def test_golden_ecoli(ctx, monkeypatch, chunk):
    buf, coff, goff = ecoli()
    set_env(monkeypatch, "default", chunk)
    d = check_genomes(ctx, buf, coff, goff)
    assert [int(x) for x in np.diff(d["kmer_off"])] == [19330, 21899, 19485]
    compare(ctx, buf, coff, goff, ref=d)
    compare(ctx, buf, coff, goff, individual=True)


def test_ingest_stats_of_a_packed_call(ctx, monkeypatch, batch):
    buf, coff, goff = batch
    set_env(monkeypatch, "packed-only", MIB)
    ctx.sketch_genomes(buf, coff, goff).free()
    h2d, packed, ascii_ = ctx.ingest_stats()
    n, offs = len(buf), 8 * (len(coff) + len(goff))
    assert packed > 1 and ascii_ >= 1                           # genomes larger than 1 MiB cross as ASCII on their own
    assert h2d < n
    set_env(monkeypatch, "packed-only", None)
    ctx.sketch_genomes(buf, coff, goff).free()
    h2d, packed, ascii_ = ctx.ingest_stats()
    assert (packed, ascii_) == (1, 0)
    assert n / 4 <= h2d <= n / 4 + offs + 64                    # n/4 bytes of words plus the offsets
    rng = np.random.default_rng(2)
    many = [seqs(rng, 500000) for _ in range(8)]
    b2, c2 = flatten(many)
    ctx.sketch_genomes(b2, c2, np.arange(9, dtype=np.uint64)).free()
    h2d, packed, ascii_ = ctx.ingest_stats()
    assert packed == 1 and ascii_ == 0
    set_env(monkeypatch, "packed-only", MIB)
    ctx.sketch_genomes(b2, c2, np.arange(9, dtype=np.uint64)).free()
    h2d, packed, ascii_ = ctx.ingest_stats()
    assert packed == 4 and ascii_ == 0                          # two 0.5 Mbp genomes per 1 MiB chunk
    assert len(b2) / 4 <= h2d <= len(b2) / 4 + 8 * 30 + 64 * 4


def test_handle_is_ready_for_indexing(ctx, monkeypatch, batch):
    buf, coff, goff = batch
    set_env(monkeypatch, "default", ODD)
    gd = sketch(ctx, buf, coff, goff, "device")
    gh = sketch(ctx, buf, coff, goff, "pageable")
    a, b = ctx.build_db(gd).download(), ctx.build_db(gh).download()
    for key in a:
        assert np.array_equal(a[key], b[key]), key


def test_device_memory_of_a_large_host_batch_is_bounded(monkeypatch):
    """2.1 Gbp of host ASCII on a fresh ctx: the device peak (cache plus rings) stays within the final output twice,
    one chunk's working set and the rings, far below the input's own size."""
    import sylph_b200
    import torch
    from sylph_b200 import synth
    set_env(monkeypatch)
    n_genomes, glen = 500, 4_200_000
    buf = torch.empty(n_genomes * glen, dtype=torch.uint8).pin_memory()
    for g0 in range(0, n_genomes, 50):
        b, _ = synth.db_chunk(g0, g0 + 50, glen, device="cuda")
        buf[g0 * glen:(g0 + 50) * glen].copy_(b.cpu())
    coff = np.arange(n_genomes + 1, dtype=np.uint64) * glen
    goff = np.arange(n_genomes + 1, dtype=np.uint64)
    ctx = sylph_b200.Context(0)
    try:
        g = ctx.sketch_genomes(buf, coff, goff)
        peak = ctx.device_bytes()[1] + ctx.ingest_ring_bytes()[0]
        d = g.download()
        out = 8 * (len(d["kmers"]) + len(d["tracked"])) + 3 * 8 * (n_genomes + 1)
        chunk = 32 * MIB
        working = 2 * chunk                                     # tile slots, survivors, post-pass scratch of one chunk
        print("host batch %.2f Gbp: device peak %.1f MB (rings %.1f MB), output %.1f MB" %
              (len(buf) / 1e9, peak / 1e6, ctx.ingest_ring_bytes()[0] / 1e6, out / 1e6))
        assert peak <= 2 * out + working + ctx.ingest_ring_bytes()[0]
        assert peak < len(buf) / 4
        g.free()
    finally:
        ctx.close()


def test_driver_syldb_with_small_chunks(exe, tmp_path):  # noqa: F811
    genomes = [os.path.join(DATA, n) for n in ("e.coli-EC590.fasta.gz", "e.coli-o157.fasta.gz", "e.coli-K12.fasta.gz")]
    run(exe, ["sketch"] + genomes + ["-o", "a"], str(tmp_path))
    run(exe, ["sketch"] + genomes + ["-o", "b"], str(tmp_path), env={"SYL_INGEST_CHUNK": str(ODD)})
    a, b = (open(os.path.join(str(tmp_path), x + ".syldb"), "rb").read() for x in ("a", "b"))
    assert a == b and len(a) > 0
