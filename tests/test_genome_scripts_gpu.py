"""GPU parity on scripted genome batches (tests/genome_scripts.py): the genome post-pass against the CPU oracle, bit
for bit, on inputs built to reach each of its branches -- k_spacing's walks, k_dups' probes, genome and contig
boundaries, the tile slot edge (512 / 513 survivors), the compact-array capacity (N == cap / cap + 1) -- through both
front halves, ASCII and 2-bit input from host and device memory, with and without pseudotax; the launch counts that
show which front half ran; and the FracMinHash threshold edges through every seeding output."""
import numpy as np
import pytest

from tests import genome_scripts as G
from tests.test_packed_sketch_gpu import GENOME_KEYS, _cuda

pytestmark = pytest.mark.gpu

_ORACLE = {}


def _expected(b, ms, pseudotax, individual=False, c=None):
    key = (b.name, b.k, b.c, ms, pseudotax, individual, c)
    if key not in _ORACLE:
        _ORACLE[key] = G.oracle_sketch(b, ms, pseudotax, individual, c)
    return _ORACLE[key]


def _inputs(b, individual):
    from sylph_b200.api import pack2
    words = pack2(b.buf)
    goff = None if individual else b.genome_off
    gdev = None if individual else _cuda(b.genome_off, np.int64)
    odev = _cuda(b.contig_off, np.int64)
    return [("host ascii", b.buf, b.contig_off, goff, {}),
            ("host packed", words, b.contig_off, goff, {"packed_bases": b.n_bases}),
            ("device ascii", _cuda(b.buf, np.uint8), odev, gdev, {}),
            ("device packed", _cuda(words, np.int32), odev, gdev, {"packed_bases": b.n_bases})]


def check_batch(ctx, b, ms, pseudotax, individual=False, c=None):
    """Every input form gives the oracle's CSR exactly."""
    d = _expected(b, ms, pseudotax, individual, c)
    for name, x, o, g, extra in _inputs(b, individual):
        got = ctx.sketch_genomes(x, o, g, k=b.k, c=c or b.c, min_spacing=ms, pseudotax=pseudotax, individual=individual,
                                 **extra).download()
        for key in GENOME_KEYS:
            assert np.array_equal(got[key], d[key]), (b.name, name, ms, pseudotax, individual, c, key)
    return d


@pytest.fixture(params=["slotted", "sort"])
def postpass(request, monkeypatch):
    """slotted: the default (the slotted front half for c >= 96, its fallback when it overflows); sort: the sorted
    front half for every call (SYL_GENOME_POSTPASS=sort, read per call)."""
    monkeypatch.delenv("SYL_GENOME_POSTPASS", raising=False)
    if request.param == "sort":
        monkeypatch.setenv("SYL_GENOME_POSTPASS", "sort")
    return request.param


@pytest.mark.parametrize("name", G.FAMILIES)
def test_family_parity(ctx, postpass, name):
    b = G.batch(name)
    for ms in G.MS[name]:
        for pseudotax in (True, False):
            check_batch(ctx, b, ms, pseudotax)
    if name == "bounds":   # one contig per genome, and c = 96 (slotted) next to the batch's own c = 95 (sorted)
        for pseudotax in (True, False):
            check_batch(ctx, b, 30, pseudotax, individual=True)
            check_batch(ctx, b, 30, pseudotax, c=96)
            check_batch(ctx, b, 30, pseudotax, individual=True, c=96)


@pytest.fixture
def timed_ctx(ctx):
    ctx.enable_timing(True)
    ctx.kernel_time("seed")
    ctx.kernel_time("genome_post")
    yield ctx
    ctx.enable_timing(False)


@pytest.mark.parametrize("name", ["slot512", "slot513", "cap", "cap1", "dups"])
def test_launch_counts(timed_ctx, monkeypatch, name):
    """The seeding and post-pass launches of one call are the classifier's: 1 / 1 without fallback, 2 / 2 after a
    slot or capacity overflow of the slotted front half, 3 / 2 when the sorted front half then also retries with a
    larger buffer; 1 / 1 or 2 / 1 when the sorted front half is forced."""
    ctx = timed_ctx
    b = G.batch(name)
    want = G.classify(b, 30)["launches"]
    d = _expected(b, 30, True)
    for force_sort in (False, True):
        monkeypatch.delenv("SYL_GENOME_POSTPASS", raising=False)
        if force_sort:
            monkeypatch.setenv("SYL_GENOME_POSTPASS", "sort")
        got = ctx.sketch_genomes(b.buf, b.contig_off, b.genome_off, k=b.k, c=b.c, min_spacing=30).download()
        n_seed, n_post = ctx.kernel_time("seed")[1], ctx.kernel_time("genome_post")[1]
        assert (n_seed, n_post) == want[force_sort], (name, force_sort, (n_seed, n_post), want)
        for key in GENOME_KEYS:
            assert np.array_equal(got[key], d[key]), (name, force_sort, key)


EDGES = [(31, W, None) for W in G.EDGE_W] + [(21, W, c) for W in G.EDGE_W for c, _, _ in G.K21_EDGES]


@pytest.mark.parametrize("k,W,c", EDGES)
def test_threshold_edges(ctx, monkeypatch, k, W, c):
    """hash thr - 1 survives and thr does not, at every window offset of a k_seed run of W windows: plain survivors
    (with and without positions), genome sketches (slotted and sorted front half) and read sketches."""
    from oracle import oracle as O
    b = G.edge_batch(k, W, c)
    c = b.c
    kept = sorted({h for e in b.expect for _, h in e})
    n_kept = sum(1 for _, ok, _ in b.labels if ok)
    for with_pos in (True, False):
        sv = ctx.extract_markers_batch(b.buf, b.contig_off, k=k, c=c, with_pos=with_pos)
        got = sorted(zip(sv["rec"].tolist(), sv["pos"].tolist() if with_pos else [0] * len(sv), sv["hash"].tolist()))
        want = sorted((ci, p if with_pos else 0, h) for ci, e in enumerate(b.expect) for p, h in e)
        assert got == want, (with_pos, len(got), len(want))
    for mode in ("slotted", "sort"):
        monkeypatch.delenv("SYL_GENOME_POSTPASS", raising=False)
        if mode == "sort":
            monkeypatch.setenv("SYL_GENOME_POSTPASS", "sort")
        d = check_batch(ctx, b, 30, True, individual=True)
        assert len(d["kmers"]) == n_kept and sorted(set(d["kmers"].tolist())) == kept
    monkeypatch.delenv("SYL_GENOME_POSTPASS", raising=False)
    s = ctx.sketch_sequences(b.buf, b.contig_off, k=k, c=c)
    h, cnt = s.download()
    eh, ec, _, _ = O.sketch_reads(b.buf, b.contig_off, k=k, c=c)
    assert np.array_equal(h, eh) and np.array_equal(cnt, ec)
    assert h.tolist() == kept and cnt.tolist() == [W] * len(kept)   # one read per window offset holds each kept k-mer
