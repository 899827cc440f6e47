"""GPU: read and pair sketches cut into hash-range parts (sylph_b200/csrc/sample_parts.hpp).  With SYL_SAMPLE_PARTS
forcing P parts, every input form gives the one-pass sketch and the oracle's: hashes, counts, num_dup_removed and
mean_read_length.  K-mers next to every part's bounds are counted once.  A budget of a quarter of the one-pass peak
is met by parts, a budget below the floor is refused before anything is allocated, and query / profile rows and the
driver's .sylsp files do not change."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import dedup_scripts as D
from tests import genome_scripts as GS
from tests.test_driver_devices_gpu import _sketch
from tests.test_driver_gpu import d, exe, sk  # noqa: F401 (fixtures)
from tests.test_pairs_stream_gpu import ENV, _cuda, _pinned, check, sketch
from tests.test_sample_retry_gpu import homopolymer_pairs
from tests.test_sketch_gpu import rand_seqs
from tests.util import DATA, flatten, read_fastx

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PARTS = (2, 3, 7, 16)
U64 = 2**64 - 1
FORMS = {"host": ("host", {}), "host-ascii": ("host", {"SYL_HOST_INGEST": "ascii"}),
         "host-tiny-chunks": ("host", {"SYL_INGEST_CHUNK": "4096"}),
         "pinned-steal": ("pinned", {"SYL_INGEST_FORCE_STEAL": "1", "SYL_INGEST_CHUNK": "8192"}),
         "host-packed": ("host-packed", {}), "device": ("device", {}), "device-packed": ("device-packed", {})}


@pytest.fixture(scope="module")
def ctx():
    import sylph_b200
    c = sylph_b200.Context(0)
    yield c
    c.close()


def set_env(monkeypatch, env, parts=None):
    for k in ENV + ("SYL_SAMPLE_PARTS",):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    if parts:
        monkeypatch.setenv("SYL_SAMPLE_PARTS", str(parts))


def sketch_single(ctx, buf, off, source, **kw):
    from sylph_b200.api import pack2
    if source == "host":
        return ctx.sketch_sequences(buf, off, **kw)
    if source == "pinned":
        return ctx.sketch_sequences(_pinned(buf, np.uint8), _pinned(off, np.int64), **kw)
    if source == "device":
        return ctx.sketch_sequences(_cuda(buf, np.uint8), _cuda(off, np.int64), **kw)
    w = pack2(buf)
    if source == "host-packed":
        return ctx.sketch_sequences(w, off, packed_bases=len(buf), **kw)
    return ctx.sketch_sequences(_cuda(w, np.int32), _cuda(off, np.int64), packed_bases=len(buf), **kw)


def result(s):
    h, c = s.download()
    out = (h.copy(), c.copy(), s.num_dup_removed, s.mean_read_length)
    s.free()
    return out


def same(a, b, what):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), what
    assert a[2] == b[2] and a[3] == b[3], (what, a[2:], b[2:])


def dup_reads(seed, n=3000):
    """150 bp reads with exact duplicates (same pair keys) and near duplicates, so dedup removes events"""
    rng = np.random.default_rng(seed)
    base = rand_seqs(rng, [150] * n)
    reads = base + [base[i] for i in rng.integers(0, n, n // 2)] + rand_seqs(rng, [int(x) for x in rng.integers(40, 500, 200)])
    return [reads[i] for i in rng.permutation(len(reads))]


@pytest.mark.parametrize("k,sem", [(31, 1), (21, 0)])
@pytest.mark.parametrize("form", list(FORMS))
def test_single_end_parts_equal_one_pass_and_oracle(ctx, monkeypatch, form, k, sem):
    from oracle import oracle as O
    buf, off = flatten(dup_reads(7 + k))
    source, env = FORMS[form]
    for no_dedup in (False, True):
        kw = dict(k=k, c=10, sem=sem, no_dedup=no_dedup)
        eh, ec, emean, end = O.sketch_reads(buf, off, **kw)
        set_env(monkeypatch, env)
        one = result(sketch_single(ctx, buf, off, source, **kw))
        assert ctx.sample_parts() == 1
        same(one, (eh, ec, end, one[3]), (form, "one pass"))
        assert abs(one[3] - emean) <= 1e-9 * emean
        for P in PARTS:
            set_env(monkeypatch, env, P)
            got = result(sketch_single(ctx, buf, off, source, **kw))
            assert ctx.sample_parts() == P
            same(got, one, (form, P, no_dedup))


@pytest.mark.parametrize("k,sem", [(31, 1), (21, 0)])
@pytest.mark.parametrize("form", list(FORMS))
def test_pairs_parts_equal_one_pass_and_oracle(ctx, monkeypatch, form, k, sem):
    from oracle import oracle as O
    rng = np.random.default_rng(11 + k)
    r1, r2 = dup_reads(3), dup_reads(4)
    r2 = [r2[i] for i in rng.permutation(len(r2))][:len(r1)] + [b"ACGT" * 5]   # a mate too short for keys
    r1 = r1 + [b"T" * 150]
    source, env = FORMS[form]
    for no_dedup in (False, True):
        kw = dict(k=k, c=10, sem=sem, no_dedup=no_dedup)
        flat = flatten(r1) + flatten(r2)
        expect = O.sketch_read_pairs(*flat, **kw)
        set_env(monkeypatch, env)
        check(ctx, r1, r2, source, expect=expect, **kw)
        for P in PARTS:
            set_env(monkeypatch, env, P)
            check(ctx, r1, r2, source, expect=expect, **kw)
            assert ctx.sample_parts() == P


CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, %(root)r)
import sylph_b200
from oracle import oracle as O
from tests.test_sample_parts_gpu import dup_reads
from tests.test_sample_retry_gpu import homopolymer_pairs
from tests.util import flatten
ctx = sylph_b200.Context(0)
buf, off = flatten(dup_reads(5))
eh, ec, _, end = O.sketch_reads(buf, off, c=10)
s = ctx.sketch_sequences(buf, off, c=10)
h, c = s.download()
assert np.array_equal(h, eh) and np.array_equal(c, ec) and s.num_dup_removed == end
assert ctx.sample_parts() == %(parts)d
r1, r2 = homopolymer_pairs()
flat = flatten(r1) + flatten(r2)
eh, ec, _, end = O.sketch_read_pairs(*flat, c=2)
s = ctx.sketch_pair_sequences(*flat, c=2)
h, c = s.download()
assert np.array_equal(h, eh) and np.array_equal(c, ec) and s.num_dup_removed == end
print("ok")
"""


@pytest.mark.parametrize("env", [{"SYL_SAMPLE_POSTPASS": "sort"}, {"SYL_GROUP_CAP": "48"},
                                 {"SYL_GROUP_CAP": "48", "SYL_SAMPLE_POSTPASS": "sort"}])
def test_generic_postpass_small_groups_and_capacity_retry_in_parts(env):
    """the sort post-pass, fallback groups inside a part (SYL_GROUP_CAP is read once per process: a child), and the
    homopolymer pairs of tests/test_sample_retry_gpu.py, whose events overflow inside a part and are redone there"""
    e = dict(os.environ, SYL_SAMPLE_PARTS="7", SYL_DEBUG_TIMING="1", **env)
    r = subprocess.run([sys.executable, "-c", CHILD % dict(root=ROOT, parts=7)], env=e, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr[-3000:]
    assert "part 7/7" in r.stderr and "(attempt 1)" in r.stderr   # a part was redone with the exact capacity


# ---- k-mers at the parts' bounds ---------------------------------------------------------------------------------------
def part_bounds(n_bases, n_records, k, c, P):
    """sample_parts.hpp restated: the one-pass map and the hash bounds of P parts"""
    n_exp = max(n_bases - n_records * (k - 1), 0) // c
    nbk = 32 * (n_exp // 640 + 1)
    thr = U64 // c
    mb = min((nbk << 64) // (thr + 1), U64)
    first = lambda b: 0 if b == 0 else min((((b << 64) + mb - 1) // mb), thr)  # noqa: E731
    P = min(P, nbk)
    cuts = [nbk * p // P for p in range(P + 1)]
    return [(0 if p == 0 else first(cuts[p]), thr if p == P - 1 else first(cuts[p + 1])) for p in range(P)]


def kmer_near(h, k, step, limit):
    """bases of the canonical k-mer whose hash is the first of h, h + step, ... that is one (up to limit)"""
    for i in range(4000):
        x = h + i * step
        if not (limit[0] <= x < limit[1]):
            break
        v = int(GS.unhash64(np.uint64(x))[0])
        if v < 4**k and bool(GS.is_canonical(v, k)[0] or v == int(GS.revcomp_value(v, k)[0])):
            return bytes(b"ACGT"[j] for j in GS.codes_of(v, k)), x
    raise AssertionError("no k-mer near %d" % h)


@pytest.mark.parametrize("paired", [False, True])
def test_kmers_at_part_bounds_count_once(ctx, monkeypatch, paired):
    """k-mers whose hashes are the nearest valid ones below and at every part's lo, and at its hi - 1, each in reads
    with duplicate pair-key histories; every one is counted as the oracle counts it"""
    from oracle import oracle as O
    k, c, P = 31, 10, 7
    g = D.Gen(77 + paired, k, c)
    n_reads = 2400
    bases_per = 150
    bounds = part_bounds(n_reads * bases_per * (2 if paired else 1), n_reads * (2 if paired else 1), k, c, P)
    targets = []
    for p, (lo, hi) in enumerate(bounds):
        if p:
            targets.append(kmer_near(lo - 1, k, -1, (bounds[p - 1][0], lo)))
        targets.append(kmer_near(lo, k, 1, (lo, hi)))
        targets.append(kmer_near(hi - 1, k, -1, (lo, hi)))
    keys = [g.key() for _ in range(3)]
    r1, r2 = [], []
    for i in range(n_reads):
        t, _ = targets[i % len(targets)]
        a, b = keys[i % 3], keys[(i // 3) % 3]
        if paired:
            m1 = g.mate(t, (a[0], a[1]), 1, i % 2 == 1)
            m2 = g.mate(t, (b[0], b[1]), (i // 5) % 2, i % 4 == 0)
            r1.append(m1 + g.bases(bases_per - len(m1)))
            r2.append(m2 + g.bases(bases_per - len(m2)))
        else:  # pair_kmer_single keys from bases 0 and 75, the target between them
            read = bytearray(g.bases(bases_per))
            read[0:32] = D._interleave(a[0], b[0])
            read[75:107] = D._interleave(a[1], b[1])
            read[36:36 + k] = D.revcomp(t) if i % 2 else t
            r1.append(bytes(read))
    assert all(len(x) == bases_per for x in r1 + r2)
    set_env(monkeypatch, {}, P)
    if paired:
        flat = flatten(r1) + flatten(r2)
        eh, ec, emean, end = O.sketch_read_pairs(*flat, k=k, c=c)
        got = result(sketch(ctx, flat, "device", k=k, c=c))
    else:
        buf, off = flatten(r1)
        eh, ec, emean, end = O.sketch_reads(buf, off, k=k, c=c)
        got = result(sketch_single(ctx, buf, off, "device", k=k, c=c))
    assert ctx.sample_parts() == P
    same(got, (eh, ec, end, got[3]), "bounds")
    hashes = set(got[0].tolist())
    for _, h in targets:
        assert h in hashes
        assert int(ec[np.searchsorted(eh, h)]) == int(got[1][np.searchsorted(got[0], h)])


# ---- memory ----------------------------------------------------------------------------------------------------------
def big_pairs(n_pairs, seed=5):
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    b1 = acgt[rng.integers(0, 4, n_pairs * 150, dtype=np.uint8)]
    b2 = acgt[rng.integers(0, 4, n_pairs * 150, dtype=np.uint8)]
    off = np.arange(n_pairs + 1, dtype=np.uint64) * 150
    return b1, off, b2, off.copy()


def test_quarter_budget_is_met_by_parts(monkeypatch):
    """0.6 Gbp of host pairs at c = 25 within a quarter of the one-pass peak (block cache plus staging rings)"""
    import sylph_b200
    set_env(monkeypatch, {})
    flat = big_pairs(2_000_000)
    a = sylph_b200.Context(0)
    a.device_bytes(reset_peak=True)
    one = result(a.sketch_pair_sequences(*flat, c=25))
    peak1 = a.device_bytes()[1] + a.ingest_ring_bytes()[0]
    assert a.sample_parts() == 1
    a.close()
    budget = peak1 // 4
    b = sylph_b200.Context(0)
    b.set_sample_memory(budget)
    assert b.sample_memory()[0] == budget
    b.device_bytes(reset_peak=True)
    got = result(b.sketch_pair_sequences(*flat, c=25))
    peak = b.device_bytes()[1] + b.ingest_ring_bytes()[0]
    print("one pass %d B, budget %d B, %d parts: %d B" % (peak1, budget, b.sample_parts(), peak))
    assert b.sample_parts() > 1 and peak <= budget, (peak1, budget, peak, b.sample_parts())
    same(got, one, "quarter budget")
    b.close()


def test_budget_below_the_floor_is_refused(ctx, monkeypatch):
    import sylph_b200
    set_env(monkeypatch, {})
    buf, off = flatten(dup_reads(9))
    ctx.set_sample_memory(1 << 20)
    before = ctx.device_bytes()
    try:
        for mem in ("host", "device"):
            with pytest.raises(sylph_b200.SylphError) as e:
                sketch_single(ctx, buf, off, mem, c=10)
            assert e.value.code == 3 and "bytes of device memory" in str(e.value)
            assert ctx.device_bytes() == before
    finally:
        ctx.set_sample_memory(0)
    result(sketch_single(ctx, buf, off, "host", c=10))   # the default budget takes one pass again
    assert ctx.sample_parts() == 1


def test_query_and_profile_rows_unchanged(ctx, monkeypatch):
    from sylph_b200.api import ANI_ROW_DTYPE  # noqa: F401
    gs = []
    for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "e.coli-o157.fasta.gz"):
        recs = read_fastx(os.path.join(DATA, f))
        buf, off = flatten([s for _, s in recs])
        gs.append(ctx.sketch_genomes(buf, off, np.array([0, len(recs)], dtype=np.uint64), c=100))
    db = ctx.build_db(ctx.concat_genomes(gs))
    reads = [s for _, s in read_fastx(os.path.join(DATA, "o157_reads.fastq.gz"))]
    buf, off = flatten(reads)
    set_env(monkeypatch, {})
    one = ctx.sketch_sequences(buf, off, c=100)
    set_env(monkeypatch, {}, 5)
    five = ctx.sketch_sequences(buf, off, c=100)
    assert ctx.sample_parts() == 5
    q1, q5 = ctx.query(db, [one]), ctx.query(db, [five])
    p1, p5 = ctx.profile(db, [one]), ctx.profile(db, [five])
    assert len(q1) > 0 and q1.tobytes() == q5.tobytes()
    assert len(p1) > 0 and p1.tobytes() == p5.tobytes()


def test_driver_sketch_files_identical_in_parts(exe, d, sk):  # noqa: F811
    """sylph-b200 sketch with SYL_SAMPLE_PARTS=5: byte-identical .sylsp files for reads and pairs, with one context and
    with --devices 0,0"""
    one, _ = _sketch(exe, d, "sp_one", [])
    for tag, extra in (("sp_five", []), ("sp_five_dev", ["--devices", "0,0"])):
        got, _ = _sketch(exe, d, tag, extra, env={"SYL_SAMPLE_PARTS": "5"})
        assert got == one, tag
