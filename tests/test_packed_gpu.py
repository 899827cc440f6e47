"""GPU parity of the 2-bit packed ingest path (SURVEY §8 f3): packed == ASCII == oracle.
syl_pack2 (host packer, exact BYTE_TO_SEQ) -> syl_seed_batch_packed2 / syl_sketch_reads_packed2, host and
device memory, every byte value, ragged records, the seeding kernel's tile edges (32 768 bases) inside reads and
the chunk ring."""
import numpy as np
import pytest

from tests.test_seed_gpu import oracle_survivors, random_records
from tests.util import flatten

pytestmark = pytest.mark.gpu

ALL_BYTES = bytes(range(256))


def survivors_packed(ctx, buf, off, k, c, sem, with_pos, device):
    from sylph_b200.api import pack2
    words = pack2(buf)
    if device:
        import torch
        w = torch.from_numpy(words.view(np.int32)).cuda()
        o = torch.from_numpy(off.astype(np.int64)).cuda()
        return ctx.extract_markers_batch(w, o, k=k, c=c, sem=sem, with_pos=with_pos, packed_bases=len(buf))
    return ctx.extract_markers_batch(words, off, k=k, c=c, sem=sem, with_pos=with_pos, packed_bases=len(buf))


@pytest.mark.parametrize("k", [31, 21])
@pytest.mark.parametrize("sem", [1, 0])
@pytest.mark.parametrize("device", [False, True])
def test_seeding_packed_equals_oracle_all_byte_values(ctx, k, sem, device):
    rng = np.random.default_rng(3 + k + sem)
    lengths = [0, 1, k - 1, k, k + 1, k + 3, 2 * k - 1, 2 * k, 66, 150, 151, 400, 401, 4095, 4096, 4097, 4096 + 47, 4096 + 48,
               3 * 4096 + 5, 0, 17, 40000] + list(rng.integers(0, 500, size=600))
    buf, off = random_records(rng, lengths, alphabet=ALL_BYTES)
    sv = survivors_packed(ctx, buf, off, k, 5, sem, True, device)
    exp = oracle_survivors(buf, off, k, 5, sem, True)
    got = sorted((int(a), int(b), int(h)) for h, a, b in zip(sv["hash"], sv["rec"], sv["pos"]))
    assert got == sorted(exp) and len(exp) > 1000
    sv2 = ctx.extract_markers_batch(buf, off, k=k, c=5, sem=sem, with_pos=True)      # ASCII path, same survivors
    assert got == sorted((int(a), int(b), int(h)) for h, a, b in zip(sv2["hash"], sv2["rec"], sv2["pos"]))


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("no_dedup", [False, True])
def test_read_sketch_packed_equals_ascii_equals_oracle(ctx, device, no_dedup):
    """Pair keys come from the packed stream (in-tile) or from packed global memory (reads cut by a tile
    edge: k_events_fix<true, false>); duplicates make the dedup state machine depend on them."""
    from oracle import oracle as O
    from sylph_b200.api import pack2
    rng = np.random.default_rng(77)
    genome = bytes(rng.choice(list(b"ACGT"), size=120000).astype(np.uint8))
    seqs = []
    for _ in range(9000):
        st = int(rng.integers(0, 120000 - 450))
        ln = int(rng.choice([60, 66, 70, 100, 149, 150, 150, 151, 250, 400, 401]))
        s = genome[st:st + ln]
        if rng.random() < 0.05:
            s = bytes(rng.choice(list(ALL_BYTES), size=ln).astype(np.uint8))   # arbitrary bytes
        seqs.append(s)
        if rng.random() < 0.3:
            seqs.append(s)
    seqs += [b"", b"A", b"N" * 150, b"acgtn" * 30]
    buf, off = flatten([seqs[i] for i in rng.permutation(len(seqs))])
    eh, ec, _, nd = O.sketch_reads(buf, off, c=5, no_dedup=no_dedup)
    words = pack2(buf)
    if device:
        import torch
        sp = ctx.sketch_sequences(torch.from_numpy(words.view(np.int32)).cuda(), torch.from_numpy(off.astype(np.int64)).cuda(),
                                  c=5, no_dedup=no_dedup, packed_bases=len(buf))
        sa = ctx.sketch_sequences(torch.from_numpy(buf).cuda(), torch.from_numpy(off.astype(np.int64)).cuda(), c=5, no_dedup=no_dedup)
    else:
        sp = ctx.sketch_sequences(words, off, c=5, no_dedup=no_dedup, packed_bases=len(buf))
        sa = ctx.sketch_sequences(buf, off, c=5, no_dedup=no_dedup)
    for s in (sp, sa):
        h, c = s.download()
        assert np.array_equal(h, eh) and np.array_equal(c, ec) and s.num_dup_removed == nd
    if not no_dedup:
        assert nd > 1000


def test_host_ingest_chunk_ring(ctx, monkeypatch):
    """Host ASCII -> worker-pool packer -> pinned ring -> device: chunks far smaller than the input so that every
    staging slot is recycled many times, records larger than a chunk, and 1-thread / many-thread pools agree."""
    from oracle import oracle as O
    rng = np.random.default_rng(5)
    lengths = list(rng.integers(0, 400, size=4000)) + [70000, 150, 150, 33, 0, 0, 9000]
    buf, off = random_records(rng, [lengths[i] for i in rng.permutation(len(lengths))], alphabet=b"ACGTNacgt")
    eh, ec, _, nd = O.sketch_reads(buf, off, c=11)
    for chunk in ("4096", "65536", None):
        if chunk:
            monkeypatch.setenv("SYL_INGEST_CHUNK", chunk)
        else:
            monkeypatch.delenv("SYL_INGEST_CHUNK", raising=False)
        s = ctx.sketch_sequences(buf, off, c=11)
        h, c = s.download()
        assert np.array_equal(h, eh) and np.array_equal(c, ec) and s.num_dup_removed == nd, chunk


def ascii_chunk_plan(off, chunk):
    """Records [r0, r1) per chunk of ASCII-only host ingest: as many as fit in `chunk` bases, at least one."""
    plan, r0 = [], 0
    while r0 < len(off) - 1:
        r1 = max(r0 + 1, int(np.searchsorted(off, off[r0] + np.uint64(chunk), side="right")) - 1)
        plan.append((r0, r1))
        r0 = r1
    return plan


@pytest.mark.parametrize("pinned", [True, False])
def test_host_ingest_ascii_only_chunks(ctx, monkeypatch, pinned):
    """SYL_HOST_INGEST=ascii: every chunk crosses the link as ASCII, front to back through the two-slot ring, from
    pinned or pageable caller memory.  Chunks far smaller than the input (every slot recycled many times), records
    longer than a chunk, empty records, N and lower-case bases, duplicated reads in distant chunks.  The call ships
    exactly the planned chunks: their bases and their offsets (one more than the chunk's records)."""
    import torch
    from oracle import oracle as O
    chunk = 8192
    rng = np.random.default_rng(9)
    lengths = list(rng.integers(0, 400, size=3000)) + [30000, 9000, 0, 0, 0, 150, 33]
    one, one_off = random_records(rng, [lengths[i] for i in rng.permutation(len(lengths))], alphabet=b"ACGTNacgtn")
    # the first third of the reads twice, in distant chunks: order-dependent dedup
    off = np.concatenate([one_off, one_off[-1] + one_off[1:np.searchsorted(one_off, len(one) // 3)]]).astype(np.uint64)
    buf = np.concatenate([one, one])[: int(off[-1])]
    assert (np.diff(off) == 0).any() and np.diff(off).max() > chunk
    eh, ec, _, nd = O.sketch_reads(buf, off, c=11)
    assert nd > 100
    plan = ascii_chunk_plan(off, chunk)
    assert len(plan) > 40
    h2d_exp = sum(int(off[r1] - off[r0]) + 8 * (r1 - r0 + 1) for r0, r1 in plan)
    if pinned:
        hb = torch.empty(len(buf), dtype=torch.uint8, pin_memory=True)
        hb.numpy()[:] = buf
        ho = torch.empty(len(off), dtype=torch.int64, pin_memory=True)
        ho.numpy()[:] = off.astype(np.int64)
        b, o = hb.numpy(), ho.numpy().view(np.uint64)
    else:
        b, o = buf, off
    monkeypatch.setenv("SYL_HOST_INGEST", "ascii")
    monkeypatch.setenv("SYL_INGEST_CHUNK", str(chunk))
    s = ctx.sketch_sequences(b, o, c=11)
    h, c = s.download()
    assert np.array_equal(h, eh) and np.array_equal(c, ec) and s.num_dup_removed == nd
    h2d, n_packed, n_ascii = ctx.ingest_stats()
    assert n_packed == 0 and n_ascii == len(plan) and h2d == h2d_exp


TILE = 32768   # window starts per CTA tile of the seeding kernel (seed_kernel.cuh SEED_TILE)
HALO = 48      # bases staged past the tile


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("L", [66, 150, 400])
def test_tile_edges_inside_reads(ctx, monkeypatch, L, device):
    """Tile edges at chosen offsets of reads of length L: the first and last windows, the pair keys' first 32
    bases and the 32 from the middle, and the edge of the staged halo (the middle window ending exactly at, or
    one base past, tile + HALO).  Short random filler reads put one such read across every tile edge.  The edge
    reads are copies of reads elsewhere in the sample, so deduplication compares keys taken from the staged tile
    with keys filled in from global memory.  ASCII and packed input: survivors with positions and read sketches."""
    import torch
    from oracle import oracle as O
    from sylph_b200.api import pack2
    monkeypatch.delenv("SYL_INGEST_CHUNK", raising=False)   # host input: one chunk, so tile edges sit at multiples of TILE
    k = 31
    h = L // 2
    # h - 16: the middle 32 bases end exactly at TILE + HALO (keys from the tile); h - 17: one base past (from global memory)
    offsets = [0, 1, k - 2, k - 1, k, h - 1, h, h + 31, h + 32, L - k, L - 1, h - 16, h - 17]
    rng = np.random.default_rng(1000 + L)
    bases = list(b"ACGT")
    proto = [bytes(rng.choice(bases, size=L).astype(np.uint8)) for _ in range(3)]
    seqs, pos = [], 0
    for t, d in enumerate(offsets, start=1):
        start = t * TILE - d                      # the edge read covers tile edge t * TILE at its offset d
        while start - pos > 450:
            dup = rng.random() < 0.03
            seqs.append(proto[t % 3] if dup else bytes(rng.choice(bases, size=int(rng.integers(0, 420))).astype(np.uint8)))
            pos += len(seqs[-1])
        seqs.append(bytes(rng.choice(bases, size=start - pos).astype(np.uint8)))
        seqs.append(proto[t % 3])
        pos = start + L
    seqs += proto
    buf, off = flatten(seqs)
    words = pack2(buf)
    if device:
        o = torch.from_numpy(off.astype(np.int64)).cuda()
        inputs = [(torch.from_numpy(buf).cuda(), o, {}), (torch.from_numpy(words.view(np.int32)).cuda(), o, {"packed_bases": len(buf)})]
    else:
        inputs = [(buf, off, {}), (words, off, {"packed_bases": len(buf)})]
    exp = sorted(oracle_survivors(buf, off, k, 7, 1, True))
    eh, ec, _, nd = O.sketch_reads(buf, off, c=7)
    assert nd > 0
    for b, o, kw in inputs:
        sv = ctx.extract_markers_batch(b, o, k=k, c=7, with_pos=True, **kw)
        assert sorted((int(a), int(p), int(x)) for x, a, p in zip(sv["hash"], sv["rec"], sv["pos"])) == exp, kw
        s = ctx.sketch_sequences(b, o, c=7, **kw)
        hh, cc = s.download()
        assert np.array_equal(hh, eh) and np.array_equal(cc, ec) and s.num_dup_removed == nd, kw


def test_host_ingest_mixed_packed_and_ascii_chunks(ctx, monkeypatch):
    """Pinned caller memory: chunks the packers have not started may cross the link as ASCII (taken from the back
    of the sample, out of order — the read indices travel with the chunk).  Forced here to alternate."""
    import torch
    from oracle import oracle as O
    rng = np.random.default_rng(6)
    lengths = list(rng.integers(0, 400, size=6000)) + [150] * 3000 + [70000, 33, 0]
    buf, off = random_records(rng, [lengths[i] for i in rng.permutation(len(lengths))], alphabet=b"ACGTNacgt")
    seqs_dup = np.concatenate([buf, buf[: len(buf) // 3]])   # duplicated reads across distant chunks: order-dependent dedup
    off_dup = np.concatenate([off, off[-1] + off[1:np.searchsorted(off, len(buf) // 3)]]).astype(np.uint64)
    seqs_dup = seqs_dup[: int(off_dup[-1])]
    eh, ec, _, nd = O.sketch_reads(seqs_dup, off_dup, c=11)
    hb = torch.empty(len(seqs_dup), dtype=torch.uint8, pin_memory=True)
    hb.numpy()[:] = seqs_dup
    ho = torch.empty(len(off_dup), dtype=torch.int64, pin_memory=True)
    ho.numpy()[:] = off_dup.astype(np.int64)
    monkeypatch.setenv("SYL_INGEST_CHUNK", "16384")
    for force in (True, False):
        if force:
            monkeypatch.setenv("SYL_INGEST_FORCE_STEAL", "1")
        else:
            monkeypatch.delenv("SYL_INGEST_FORCE_STEAL", raising=False)
        s = ctx.sketch_sequences(hb.numpy(), ho.numpy().view(np.uint64), c=11)
        h, c = s.download()
        assert np.array_equal(h, eh) and np.array_equal(c, ec) and s.num_dup_removed == nd, force
        h2d, n_packed, n_ascii = ctx.ingest_stats()   # what the call moved (bench.py's e2e.h2d_bytes_per_step)
        assert n_packed + n_ascii >= len(seqs_dup) // 16384 // 2 and n_packed > 0   # chunks end on record boundaries; one record is 70 kb
        if force:
            assert n_ascii > 0
        assert len(seqs_dup) // 4 <= h2d <= len(seqs_dup) + 8 * (len(off_dup) + n_packed + n_ascii)
    assert nd > 100
    monkeypatch.setenv("SYL_HOST_INGEST", "ascii")
    s = ctx.sketch_sequences(hb.numpy(), ho.numpy().view(np.uint64), c=11)
    h, c = s.download()
    assert np.array_equal(h, eh) and np.array_equal(c, ec)
    h2d, n_packed, n_ascii = ctx.ingest_stats()
    assert n_packed == 0 and n_ascii >= 1 and h2d >= len(seqs_dup) + 8 * len(off_dup)
