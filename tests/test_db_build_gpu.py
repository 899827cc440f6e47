"""GPU: the containment index built by bucket scatter (syl_db_build, syl_db_build_arrays) against a numpy reference,
bit for bit, from device genomes, host arrays in one chunk and in chunks that straddle genomes and the k-mer / tracked
boundary, and device arrays; rows of a db built from host arrays against the oracle; the build's device memory; its
argument checks; and the driver's output with tiny build chunks."""
import ctypes as C

import numpy as np
import pytest

from tests import contain_scripts as S
from tests.test_contain_scripts_gpu import CASES, check
from tests.test_driver_gpu import GENOMES, SAMPLES, d, exe, run  # noqa: F401  (d, exe: fixtures)

pytestmark = pytest.mark.gpu

U64_MAX = 2**64 - 1
TINY_CHUNK = "997"        # entries per host chunk: genomes and the k-mer / tracked boundary straddle chunks
BIG_CHUNK = "999983"      # the same for the ~10^8-entry input, in ~100 chunks instead of 10^5


# ---- the reference index ------------------------------------------------------------------------------------------

def _mulhi(a, m):
    """(a * m) >> 64 for a uint64 array and a Python int m, exact (32-bit limbs)"""
    m_lo, m_hi = np.uint64(m & 0xFFFFFFFF), np.uint64(m >> 32)
    a_lo, a_hi = a & np.uint64(0xFFFFFFFF), a >> np.uint64(32)
    ll, hl, lh, hh = a_lo * m_lo, a_hi * m_lo, a_lo * m_hi, a_hi * m_hi
    cross = (ll >> np.uint64(32)) + (hl & np.uint64(0xFFFFFFFF)) + lh
    return hh + (hl >> np.uint64(32)) + (cross >> np.uint64(32))


def reference_index(db):
    """stable sort of the entries in the layout all genomes' k-mers (genome order), then all tracked k-mers; NB, M
    with Python integers; bstart from searchsorted"""
    koff = db["kmer_off"].astype(np.int64)
    G = len(koff) - 1
    keys = [db["kmers"]]
    gid = [np.repeat(np.arange(G, dtype=np.uint32) << 1, np.diff(koff))]
    if db["tracked_off"] is not None:
        keys.append(db["tracked"])
        gid.append(np.repeat((np.arange(G, dtype=np.uint32) << 1) | 1, np.diff(db["tracked_off"].astype(np.int64))))
    keys = np.concatenate(keys).astype(np.uint64)
    gid = np.concatenate(gid).astype(np.uint32)
    o = np.argsort(keys, kind="stable")
    keys, gid = keys[o], gid[o]
    N = len(keys)
    NB = 1024
    while NB < N // 4:
        NB <<= 1
    if N == 0:
        return dict(keys=keys, gid=gid, bstart=np.zeros(NB + 1, np.uint32), NB=NB)
    M = min((NB << 64) // (int(keys[-1]) + 1), U64_MAX)
    b = np.minimum(_mulhi(keys, M), np.uint64(NB - 1))
    probe = np.linspace(0, N - 1, min(N, 1000)).astype(np.int64)
    assert all(int(b[i]) == min((int(keys[i]) * M) >> 64, NB - 1) for i in probe)
    bstart = np.searchsorted(b, np.arange(NB + 1, dtype=np.uint64), side="left").astype(np.uint32)
    return dict(keys=keys, gid=gid, bstart=bstart, NB=NB)


def assert_index(got, want, what):
    assert len(got["keys"]) == len(want["keys"]), what
    assert len(got["bstart"]) == want["NB"] + 1, what
    assert np.array_equal(got["keys"], want["keys"]), what
    assert np.array_equal(got["gid"], want["gid"]), what
    assert np.array_equal(got["bstart"], want["bstart"]), what


# ---- inputs ---------------------------------------------------------------------------------------------------------

def csr(per_genome_kmers, per_genome_tracked=None, gn=None):
    koff = np.concatenate([[0], np.cumsum([len(x) for x in per_genome_kmers])]).astype(np.uint64)
    kmers = np.concatenate([np.asarray(x, np.uint64) for x in per_genome_kmers] + [np.zeros(0, np.uint64)])
    d = dict(kmers=kmers, kmer_off=koff, tracked=None, tracked_off=None,
             gn_size=np.asarray(gn if gn is not None else [1000 + i for i in range(len(per_genome_kmers))], np.uint64))
    if per_genome_tracked is not None:
        d["tracked_off"] = np.concatenate([[0], np.cumsum([len(x) for x in per_genome_tracked])]).astype(np.uint64)
        d["tracked"] = np.concatenate([np.asarray(x, np.uint64) for x in per_genome_tracked] + [np.zeros(0, np.uint64)])
    return d


def rand_keys(rng, n, hi):
    return rng.integers(0, hi, n, dtype=np.uint64, endpoint=False)


def inp_empty(rng):
    return csr([[], [], []], [[], [], []])


def inp_empty_genomes(rng):
    ks = [rand_keys(rng, int(n), 2**60) if n else [] for n in rng.choice([0, 0, 3, 40, 700], 60)]
    ts = [rand_keys(rng, int(n), 2**60) if n else [] for n in rng.choice([0, 0, 5, 90], 60)]
    ks[0], ts[-1] = [], []
    return csr(ks, ts)


def inp_no_tracked(rng):
    return csr([rand_keys(rng, int(n), 2**60) for n in rng.integers(0, 900, 40)])


def inp_tracked_equal_kept(rng):
    ks = [rand_keys(rng, int(n), 2**58) for n in rng.integers(50, 600, 30)]
    pool = np.concatenate(ks)
    ts = [rng.choice(pool, int(n)) for n in rng.integers(0, 300, 30)]   # other genomes' kept keys (and their own)
    ks = [np.concatenate([k, rng.choice(pool, 20)]) for k in ks]        # and kept keys shared between genomes
    return csr(ks, ts)


def inp_shared_key(rng):
    G = 2**16 + 5
    key = 0x0123456789ABCDEF
    ks = [[key] for _ in range(G)]
    ts = [[key] for _ in range(G)]
    for g in rng.integers(0, G, 3000):                                  # a few other keys around it
        ks[g] = [key, int(rng.integers(0, 2**62))]
    return csr(ks, ts)


def inp_crowded_bucket(rng):
    G = 400
    ks = [list(rand_keys(rng, 50, 2**64 - 2)) for _ in range(G)]
    base, base2 = 0x7000000000000000, 0x3000000000000000
    crowd = np.arange(base, base + 6000, dtype=np.uint64)              # > 2048 distinct keys in one bucket
    crowd2 = np.arange(base2, base2 + 700, dtype=np.uint64)            # a middle-sized one
    ts = [[] for _ in range(G)]
    for i, x in enumerate(rng.permutation(np.concatenate([crowd, crowd2]))):
        (ks if i % 3 else ts)[int(rng.integers(0, G))].append(int(x))
    ks[7].append(2**64 - 2)
    return csr(ks, ts)


def inp_extreme_keys(rng):
    ks = [list(rand_keys(rng, 100, 2**64 - 2)) + [0, 2**64 - 2] for _ in range(20)]
    ts = [[0, 2**64 - 2, 2**64 - 2] for _ in range(20)]
    return csr(ks, ts)


def inp_small_maxkey(rng):
    return csr([rand_keys(rng, int(n), 1000) for n in rng.integers(0, 400, 30)],
               [rand_keys(rng, int(n), 1000) for n in rng.integers(0, 100, 30)])


def inp_full_range(rng):
    return csr([rand_keys(rng, int(n), 2**64 - 1) for n in rng.integers(1000, 30000, 50)],
               [rand_keys(rng, int(n), 2**64 - 1) for n in rng.integers(0, 3000, 50)])


def fracminhash_db(seed, G=5000, mean=17400, tracked_share=0.15):
    """FracMinHash-like sketches (c = 200): ~G * mean * (1 + tracked_share) keys below 2^64 / 200, 3 % of them drawn
    from a shared pool so that some keys recur across genomes"""
    rng = np.random.default_rng(seed)
    nk = np.maximum(rng.normal(mean, mean / 4, G), 0).astype(np.int64)
    nt = (nk * tracked_share * rng.random(G) * 2).astype(np.int64)
    hi = (2**64 - 1) // 200
    kmers = rand_keys(rng, int(nk.sum()), hi)
    tracked = rand_keys(rng, int(nt.sum()), hi)
    pool = rand_keys(rng, 200_000, hi)
    for a in (kmers, tracked):
        sel = rng.random(len(a)) < 0.03
        a[sel] = pool[rng.integers(0, len(pool), int(sel.sum()))]
    return dict(kmers=kmers, kmer_off=np.concatenate([[0], np.cumsum(nk)]).astype(np.uint64), tracked=tracked,
                tracked_off=np.concatenate([[0], np.cumsum(nt)]).astype(np.uint64),
                gn_size=rng.integers(10**6, 10**7, G).astype(np.uint64))


def inp_fracminhash(rng):
    return fracminhash_db(11)


INPUTS = {"empty": inp_empty, "empty_genomes": inp_empty_genomes, "no_tracked": inp_no_tracked,
          "tracked_equal_kept": inp_tracked_equal_kept, "shared_key": inp_shared_key,
          "crowded_bucket": inp_crowded_bucket, "extreme_keys": inp_extreme_keys, "small_maxkey": inp_small_maxkey,
          "full_range": inp_full_range, "fracminhash_1e8": inp_fracminhash}


def _args(db):
    return (db["kmers"], db["kmer_off"], db["tracked"], db["tracked_off"], db["gn_size"])


# ---- 1. bit identity ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(INPUTS))
def test_index_bit_identical_to_reference(ctx, monkeypatch, name):
    import torch
    db = INPUTS[name](np.random.default_rng(list(INPUTS).index(name)))
    want = reference_index(db)
    if name == "shared_key":
        assert np.diff(want["bstart"].astype(np.int64)).max() > 10**5
    if name == "small_maxkey":
        assert (want["NB"] << 64) // (int(want["keys"][-1]) + 1) > U64_MAX
    monkeypatch.delenv("SYL_DB_CHUNK", raising=False)
    g = ctx.upload_genomes(*_args(db), c=200)
    got = ctx.build_db(g)
    assert_index(got.download(), want, "syl_db_build")
    got.free()
    g.free()
    host = ctx.build_db_arrays(*_args(db))
    assert_index(host.download(), want, "host arrays, one chunk")
    host.free()
    monkeypatch.setenv("SYL_DB_CHUNK", BIG_CHUNK if len(want["keys"]) > 10**7 else TINY_CHUNK)
    chunked = ctx.build_db_arrays(*_args(db))
    assert_index(chunked.download(), want, "host arrays, small chunks")
    chunked.free()
    monkeypatch.delenv("SYL_DB_CHUNK")
    dev = [None if a is None else torch.from_numpy(a.view(np.int64)).cuda() for a in _args(db)]
    on_dev = ctx.build_db_arrays(*dev)
    assert_index(on_dev.download(), want, "device arrays")
    on_dev.free()


# ---- 2. rows --------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def chunked_world(ctx):
    """the scripted world's db built from host arrays in 997-entry chunks, and the same db from uploaded genomes"""
    import os
    w = S.world()
    d = w.db()
    old = os.environ.get("SYL_DB_CHUNK")
    os.environ["SYL_DB_CHUNK"] = TINY_CHUNK
    try:
        db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=1)
    finally:
        if old is None:
            os.environ.pop("SYL_DB_CHUNK")
        else:
            os.environ["SYL_DB_CHUNK"] = old
    assert d["kmer_off"][-1] + d["tracked_off"][-1] > 10 * int(TINY_CHUNK)
    smp = {n: ctx.upload_sample(*w.sample_arrays(n), c=1) for n in S.SAMPLES}
    return db, smp


@pytest.mark.parametrize("csr_env", [None, "1"], ids=["hist", "csr"])
@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("name,pi", CASES)
def test_rows_from_chunked_host_build(ctx, chunked_world, monkeypatch, name, pi, pseudotax, csr_env):
    from sylph_b200.api import contain_params
    monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)
    monkeypatch.delenv("SYL_BOOT_REPLAY", raising=False)
    if csr_env:
        monkeypatch.setenv("SYL_CONTAIN_CSR", csr_env)
    db, smp = chunked_world
    p = contain_params(pseudotax=pseudotax, **S.params_for(name)[pi])
    rows = ctx.profile(db, [smp[name]], p) if pseudotax else ctx.query(db, [smp[name]], p)
    assert check(rows, name, pseudotax, pi) > 0


# ---- 3. bounded memory ----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def big_db():
    return fracminhash_db(5)


def _round(b):
    return (max(b, 1) + 255) // 256 * 256


def test_build_memory_is_bounded(monkeypatch, big_db):
    import sylph_b200
    C_ = 1 << 24
    monkeypatch.setenv("SYL_DB_CHUNK", str(C_))
    N = int(big_db["kmer_off"][-1] + big_db["tracked_off"][-1])
    G = len(big_db["kmer_off"]) - 1
    assert N > 9 * 10**7
    NB = 1024
    while NB < N // 4:
        NB <<= 1
    index = _round(8 * N) + _round(4 * N) + _round(4 * (NB + 2)) + _round(4 * G)
    staging = 2 * _round(8 * (C_ + 2 * min(C_, G)))
    small = 2 << 20    # directory scan storage and the list of large buckets (none in this input)
    ctx = sylph_b200.Context(0)
    try:
        held0, peak0 = ctx.device_bytes(reset_peak=True)
        assert held0 == 0 and peak0 == 0
        stats0 = ctx.ingest_stats()
        db1 = ctx.build_db_arrays(*_args(big_db))
        held, peak = ctx.device_bytes(reset_peak=True)
        assert peak <= index + staging + small, (peak, index + staging + small)
        assert held <= index + (1 << 20), (held, index)
        db2 = ctx.build_db_arrays(*_args(big_db))
        held2, peak2 = ctx.device_bytes()
        assert held2 <= 2 * index + (1 << 20), (held2, 2 * index)
        assert peak2 <= index + held + staging + small
        # the chunks cross on the ctx's copy stream, straight from the arrays: no staging ring, no ingest bytes counted
        assert ctx.ingest_ring_bytes() == (0, 0)
        assert ctx.ingest_stats() == stats0
        db2.free()
        db1.free()
        assert ctx.device_bytes()[0] == held2      # freed handles return their blocks to the ctx cache
    finally:
        ctx.close()


# ---- 4. errors ------------------------------------------------------------------------------------------------------

def test_build_arrays_argument_errors(ctx):
    import torch
    from sylph_b200 import _lib
    from sylph_b200.api import SylphError
    L = _lib.lib()
    ctx.device_bytes(reset_peak=True)
    held, peak = ctx.device_bytes()

    def raw(mem, kmers, koff, n_genomes):
        h = C.c_void_p()
        return L.syl_db_build_arrays(ctx._h, mem, kmers, koff, None, None, None, n_genomes, 31, 200, 0, C.byref(h))

    keys = np.arange(10, dtype=np.uint64)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    too_many = np.array([0, 2**32 - 1], np.uint64)                     # one past the largest shard
    assert raw(_lib.MEM_HOST, vp(keys), vp(too_many), 1) == _lib.SYL_ERR_ARG
    two = np.array([0, 2**31, 2**32 - 1], np.uint64)
    h = C.c_void_p()
    assert L.syl_db_build_arrays(ctx._h, _lib.MEM_HOST, vp(keys), vp(np.array([0, 2**31], np.uint64)), vp(keys),  # together
                                 vp(np.array([0, 2**31], np.uint64)), None, 1, 31, 200, 0, C.byref(h)) == _lib.SYL_ERR_ARG
    assert raw(_lib.MEM_HOST, vp(keys), vp(two), 2**31 - 1) == _lib.SYL_ERR_ARG  # genomes: checked before reading offsets
    assert ctx.device_bytes() == (held, peak)
    assert raw(7, vp(keys), vp(np.array([0, 10], np.uint64)), 1) == _lib.SYL_ERR_ARG
    for bad in ([0, 5, 3, 10], [1, 4, 10]):
        with pytest.raises(SylphError) as e:
            ctx.build_db_arrays(keys, np.array(bad, np.uint64))
        assert e.value.code == _lib.SYL_ERR_ARG
        with pytest.raises(SylphError) as e:
            ctx.build_db_arrays(torch.arange(10, device="cuda"), torch.tensor(bad, device="cuda"))
        assert e.value.code == _lib.SYL_ERR_ARG
        with pytest.raises(SylphError) as e:
            ctx.build_db_arrays(keys, np.array([0, 4, 10], np.uint64), keys, np.array(bad, np.uint64))
        assert e.value.code == _lib.SYL_ERR_ARG
    with pytest.raises(SylphError) as e:
        ctx.build_db_arrays(None, np.array([0, 4], np.uint64))
    assert e.value.code == _lib.SYL_ERR_ARG
    assert ctx.device_bytes()[1] == peak


# ---- 5. driver ------------------------------------------------------------------------------------------------------

def test_driver_profile_with_tiny_build_chunks(exe, d):  # noqa: F811
    args = ["profile"] + SAMPLES + GENOMES
    default = run(exe, args, d).stdout
    tiny = run(exe, args, d, env={"SYL_DB_CHUNK": TINY_CHUNK}).stdout
    assert tiny == default
    assert len(default.splitlines()) > 5
