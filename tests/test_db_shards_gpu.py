"""GPU: a host-memory database swept shard by shard (syl_db_shards_*, Context.db_shards).  query / profile rows equal
the one-index call bit for bit, in both formulations, at caps giving one shard, 2-3 uneven shards and one genome per
shard: on the scripted families (and the oracle), the ANI near-tie pairs in separate shards in both orders, a synthetic
community spread over every shard (with empty genomes), a db without tracked k-mers, -u, no_ci and all samples of
unequal size in one call.  The capacity protocol (a retry copies the kept rows out and builds nothing), the split of a
sample batch whose survivors together pass the cap, device memory bounded by one shard's build, and the argument
checks."""
import ctypes as C

import numpy as np
import pytest

from tests import ani_ties as T
from tests import contain_scripts as S
from tests.contain_compare import compare, cr_params
from tests.test_contain_scripts_gpu import Gpu, check, same
from tests.test_db_build_gpu import fracminhash_db

pytestmark = pytest.mark.gpu

CAPS = ["one", "uneven", "per_genome"]


def cap_for(kind, d):
    """max_entries that cuts db `d` into one shard, 2-3 uneven shards, or one genome per shard"""
    n = int(d["kmer_off"][-1]) + (int(d["tracked_off"][-1]) if d.get("tracked_off") is not None else 0)
    return {"one": 0, "uneven": max(n * 9 // 20, 1), "per_genome": 1}[kind]


def shards_of(ctx, d, kind, k=31, c=1):
    sh = ctx.db_shards(d["kmers"], d["kmer_off"], d.get("tracked"), d.get("tracked_off"), d["gn_size"], k=k, c=c,
                       max_entries=cap_for(kind, d))
    G = len(d["kmer_off"]) - 1
    n = {"one": 1, "uneven": None, "per_genome": G}[kind]
    if n is None:
        assert 2 <= len(sh) <= 3, sh.ranges()
        assert len({e for _, _, e in sh.ranges()}) > 1
    else:
        assert len(sh) == n
    r = sh.ranges()
    assert r[0][0] == 0 and sum(g for _, g, _ in r) == G and all(a + g == b for (a, g, _), (b, _, _) in zip(r, r[1:]))
    return sh


@pytest.fixture(params=["hist", "csr"])
def formulation(request, monkeypatch):
    monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)
    monkeypatch.delenv("SYL_BOOT_REPLAY", raising=False)
    monkeypatch.delenv("SYL_DB_SHARD_ENTRIES", raising=False)
    if request.param == "csr":
        monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
    return request.param


@pytest.fixture(scope="module")
def world(ctx):
    g = Gpu(ctx)
    for i, n in enumerate(S.SAMPLES):
        g.smp[n].mean_read_length = 150.0 + 7 * i   # -u reads it
    return g


PARAM_SETS = sorted({tuple(sorted(P.items())) for n in S.SAMPLES for P in S.params_for(n)}) + [
    (("estimate_unknown", 1), ("minimum_ani", 0.0), ("read_seq_id", 98.0))]


def one_index_and_shards(ctx, db, sh, handles, pseudotax, P):
    from sylph_b200.api import contain_params
    p = contain_params(pseudotax=pseudotax, **P)
    if pseudotax:
        return ctx.profile(db, handles, p), sh.profile(handles, p)
    return ctx.query(db, handles, p), sh.query(handles, p)


@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("kind", CAPS)
def test_scripted_rows_equal_one_index(ctx, world, formulation, kind, pseudotax):
    """every scripted sample in one call (sizes 100 to 501 000 keys), under every parameter set the families are built
    for, plus -u: rows bit-identical to the one-index call; at the uneven cut also each sample's rows == the oracle"""
    sh = shards_of(ctx, world.d, kind)
    handles = [world.smp[n] for n in S.SAMPLES]
    try:
        for P in map(dict, PARAM_SETS):
            want, got = one_index_and_shards(ctx, world.db, sh, handles, pseudotax, P)
            same(got, want, (kind, P))
            if kind != "uneven" or "estimate_unknown" in P:
                continue
            for si, name in enumerate(S.SAMPLES):
                if P in S.params_for(name):
                    sub = got[got["sample"] == si].copy()
                    sub["sample"] = 0
                    check(sub, name, pseudotax, S.params_for(name).index(P))
        assert len(want) > 50
    finally:
        sh.free()


PAIRS = [("adjacent",) + p for p in T.WINNER_PAIRS] + [("equal",) + p for p in T.TIE_PAIRS]


@pytest.mark.parametrize("swap", [False, True], ids=["a_first", "b_first"])
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s_k%d_%d" % (p[0], p[1], p[2][1]))
def test_near_tied_genomes_in_separate_shards(ctx, formulation, pair, swap):
    """two genomes of adjacent or equal ANIs sharing hit k-mers, one per shard: the pass-2 winner, kmers_lost and the
    abundances equal the one-index call's and the oracle's"""
    from oracle import oracle as O
    from sylph_b200.api import contain_params
    kind, k, a, b = pair
    case = T.Case([b, a] if swap else [a, b], shared=3)
    d = case.db
    db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], k=k, c=1)
    sh = shards_of(ctx, d, "per_genome", k=k)
    smp = ctx.upload_sample(case.hash, case.count, k=k, c=1)
    try:
        for pseudotax in (False, True):
            p = contain_params(k=k, pseudotax=pseudotax, minimum_ani=0.0)
            want = ctx.profile(db, [smp], p) if pseudotax else ctx.query(db, [smp], p)
            got = sh.profile([smp], p) if pseudotax else sh.query([smp], p)
            same(got, want, (pair, swap, pseudotax))
            if pseudotax:
                exp = O.contain_sample(cr_params(k=k, pseudotax=True, minimum_ani=0.0), d["kmers"], d["kmer_off"],
                                       d["tracked"], d["tracked_off"], d["gn_size"], O.Sample(case.hash, case.count))
                compare(got, exp, True)
                assert sorted(int(x) for x in got["kmers_lost"]) == [0, 3]
    finally:
        smp.free()
        sh.free()
        db.free()


def community(seed=4, G=240, empty_every=17):
    """a FracMinHash-like db with empty genomes (no k-mers, or no k-mers and no tracked k-mers) at regular places and
    tracked k-mers taken from other genomes' k-mers; samples drawing most k-mers of genomes spread over the whole db at
    unequal coverages, plus k-mers shared between those genomes (winner decisions in pass 2)"""
    rng = np.random.default_rng(seed)
    hi = (2**64 - 1) // 200
    nk = rng.integers(300, 4000, G)
    nk[::empty_every] = 0
    ks = [rng.integers(0, hi, int(n), dtype=np.uint64) for n in nk]
    pool = np.concatenate(ks)
    nt = rng.integers(0, 200, G)
    nt[::2 * empty_every] = 0
    ts = [rng.choice(pool, int(n)) if n else np.zeros(0, np.uint64) for n in nt]
    shared = rng.integers(0, hi, 150, dtype=np.uint64)
    members = [g for g in range(3, G, 11) if nk[g]]
    for g in members:                        # genomes of the community share some k-mers
        ks[g] = np.unique(np.concatenate([ks[g], shared[rng.random(150) < 0.5]]))
    d = dict(kmers=np.concatenate(ks).astype(np.uint64),
             kmer_off=np.concatenate([[0], np.cumsum([len(x) for x in ks])]).astype(np.uint64),
             tracked=np.concatenate(ts).astype(np.uint64),
             tracked_off=np.concatenate([[0], np.cumsum(nt)]).astype(np.uint64),
             gn_size=rng.integers(10**6, 10**7, G).astype(np.uint64))
    samples = []
    for si in range(5):
        keys = {}
        for g in members[si::2]:
            cov = float(rng.choice([0.3, 1.0, 2.5, 6.0]))
            for x in ks[g][rng.random(len(ks[g])) < 0.9]:
                keys[int(x)] = int(max(1, rng.poisson(cov)))
        for x in rng.integers(0, hi, 500 * (si + 1), dtype=np.uint64):   # k-mers of no genome
            keys[int(x)] = 1
        samples.append((np.array(list(keys), np.uint64), np.array(list(keys.values()), np.uint32)))
    return d, samples


@pytest.fixture(scope="module")
def comm(ctx):
    d, raw = community()
    db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200)
    smp = [ctx.upload_sample(h, c, c=200) for h, c in raw]
    for i, s in enumerate(smp):
        s.mean_read_length = 120.0 + 30 * i
    return d, db, smp


@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("kind", CAPS)
def test_community_spread_over_every_shard(ctx, comm, formulation, kind, pseudotax):
    """five samples of unequal size in one call and each alone, default parameters, no_ci, -m 0 and -u: rows equal
    the one-index call's; most shards hold no survivor of a sample"""
    d, db, smp = comm
    sh = shards_of(ctx, d, kind, c=200)
    try:
        for P in ({}, {"no_ci": 1}, {"minimum_ani": 0.0}, {"estimate_unknown": 1, "read_seq_id": 97.5}):
            want, got = one_index_and_shards(ctx, db, sh, smp, pseudotax, P)
            same(got, want, (kind, P))
            assert len(set(want["sample"].tolist())) == 5 and len(want) >= 20
        for s in smp[::2]:
            want, got = one_index_and_shards(ctx, db, sh, [s], pseudotax, {})
            same(got, want, kind)
        if pseudotax:
            assert (want["kmers_lost"] > 0).any()
    finally:
        sh.free()


def test_db_without_tracked_kmers(ctx, comm):
    """query rows equal the one-index call's; profile refuses the db with syl_profile's code and message"""
    from sylph_b200 import _lib
    from sylph_b200.api import SylphError
    d, _, smp = comm
    db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], None, None, d["gn_size"], c=200)
    sh = ctx.db_shards(d["kmers"], d["kmer_off"], None, None, d["gn_size"], c=200, max_entries=cap_for("uneven", dict(d, tracked_off=None)))
    try:
        assert len(sh) >= 2
        same(sh.query(smp), ctx.query(db, smp), "no tracked")
        errs = []
        for fn in (lambda: ctx.profile(db, smp), lambda: sh.profile(smp)):
            with pytest.raises(SylphError) as e:
                fn()
            errs.append((e.value.code, str(e.value)))
        assert errs[0] == errs[1] and errs[0][0] == _lib.SYL_ERR_ARG and "disable-profiling" in errs[0][1]
    finally:
        sh.free()
        db.free()


def _raw(fn, ctx, sh, handles, p, cap):
    from sylph_b200.api import ANI_ROW_DTYPE
    arr = (C.c_void_p * len(handles))(*[s._h for s in handles])
    rows = np.empty(max(cap, 1), dtype=ANI_ROW_DTYPE)
    n = C.c_uint64(0)
    rc = fn(ctx._h, sh._h, arr, len(handles), C.byref(p), rows.ctypes.data_as(C.c_void_p), cap, C.byref(n))
    return rc, n.value, rows[: n.value]


@pytest.mark.parametrize("pseudotax", [False, True])
def test_capacity_retry_builds_nothing(ctx, comm, pseudotax):
    """cap = 1: SYL_ERR_CAPACITY with the size; the retry with that size and the same arguments launches no kernel and
    returns the rows of an ordinary call.  A call with other params in between drops the kept rows."""
    from sylph_b200 import _lib
    from sylph_b200.api import contain_params
    d, _, smp = comm
    L = _lib.lib()
    fn = L.syl_profile_shards if pseudotax else L.syl_query_shards
    sh = shards_of(ctx, d, "uneven", c=200)
    try:
        p = contain_params(pseudotax=pseudotax)
        want = sh.profile(smp, p) if pseudotax else sh.query(smp, p)
        rc, need, _ = _raw(fn, ctx, sh, smp, p, 1)
        assert rc == _lib.SYL_ERR_CAPACITY and need == len(want) > 1
        before = ctx.launches
        rc, n, rows = _raw(fn, ctx, sh, smp, p, need)
        assert rc == _lib.SYL_OK and n == need and ctx.launches == before
        same(rows, want, "retry")
        rc, _, _ = _raw(fn, ctx, sh, smp, p, 1)
        assert rc == _lib.SYL_ERR_CAPACITY
        p2 = contain_params(pseudotax=pseudotax, no_ci=1)
        rc, _, _ = _raw(fn, ctx, sh, smp, p2, 1 << 20)       # another call: the kept rows are dropped
        assert rc == _lib.SYL_OK
        before = ctx.launches
        rc, n, rows = _raw(fn, ctx, sh, smp, p, need)
        assert rc == _lib.SYL_OK and ctx.launches > before   # swept again
        same(rows, want, "after another call")
    finally:
        sh.free()


def test_survivor_union_split(ctx, comm, formulation):
    """two samples whose survivors fit the cap each but not together are profiled on two survivor indexes (two more
    statistics launches per pass), with the rows of the one-index call"""
    from sylph_b200.api import contain_params
    d, db, smp = comm
    pair = [smp[0], smp[1]]
    p = contain_params(pseudotax=True)
    want = ctx.profile(db, pair, p)
    ent = lambda g: int(d["kmer_off"][g + 1] - d["kmer_off"][g] + d["tracked_off"][g + 1] - d["tracked_off"][g])  # noqa: E731
    q = ctx.query(db, pair, contain_params(pseudotax=False, minimum_ani=95.0, no_ci=1))
    own = [sum(ent(int(g)) for g in q["genome"][q["sample"] == i]) for i in range(2)]
    assert set(q["genome"][q["sample"] == 0].tolist()).isdisjoint(q["genome"][q["sample"] == 1].tolist())
    stats = {}
    ctx.enable_timing()
    try:
        for cap in (sum(own), max(own)):                 # fits together / only one at a time
            sh = ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200,
                               max_entries=cap)
            ctx.kernel_time("stats")
            got = sh.profile(pair, p)
            stats[cap] = ctx.kernel_time("stats")[1] - len(sh)   # minus one pass-1 launch per shard
            same(got, want, cap)
            sh.free()
    finally:
        ctx.enable_timing(False)
    assert stats == {sum(own): 2, max(own): 4}, stats


def _r(b):
    return (max(b, 1) + 255) // 256 * 256


def _index_bytes(N, G):
    NB = 1024
    while NB < N // 4:
        NB <<= 1
    return _r(8 * N) + _r(4 * N) + _r(4 * (NB + 2)) + _r(4 * G)


def test_device_memory_bounded_by_one_shard(monkeypatch):
    """10^8 entries in 8-9 shards: the profile's peak stays within the largest shard's build (index + two staging
    chunks) plus the survivor index and the joins' scratch, and is under a quarter of the one-index build's peak"""
    import sylph_b200
    from sylph_b200.api import contain_params
    chunk = 1 << 22
    monkeypatch.setenv("SYL_DB_CHUNK", str(chunk))
    monkeypatch.delenv("SYL_DB_SHARD_ENTRIES", raising=False)
    d = fracminhash_db(5)
    N = int(d["kmer_off"][-1] + d["tracked_off"][-1])
    assert N > 9 * 10**7
    hits = [7, 2400, 4990]
    h = np.concatenate([d["kmers"][int(d["kmer_off"][g]):int(d["kmer_off"][g + 1])] for g in hits])
    h = np.unique(h)
    c = np.full(len(h), 3, np.uint32)
    peaks = {}
    for mode in ("shards", "one"):
        ctx = sylph_b200.Context(0)
        try:
            smp = ctx.upload_sample(h, c, c=200)
            held0, _ = ctx.device_bytes(reset_peak=True)
            if mode == "shards":
                sh = ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200,
                                   max_entries=N // 8 + 1)
                assert 8 <= len(sh) <= 9
                rows = sh.profile([smp], contain_params(pseudotax=True))
                assert sorted(rows["genome"].tolist()) == hits
                shard = max(_index_bytes(e, g) + 2 * _r(8 * (min(chunk, e) + 2 * min(chunk, g))) for _, g, e in sh.ranges())
                surv = sum(int(d["kmer_off"][x + 1] - d["kmer_off"][x] + d["tracked_off"][x + 1] - d["tracked_off"][x])
                           for x in hits)
                bound = shard + _index_bytes(surv, 3) + 2 * _r(8 * (surv + 6)) + (64 << 20)
                peaks[mode] = ctx.device_bytes()[1] - held0
                assert peaks[mode] <= bound, (peaks[mode], bound)
                sh.free()
            else:
                db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200)
                peaks[mode] = ctx.device_bytes()[1] - held0
                db.free()
            smp.free()
        finally:
            ctx.close()
    assert 4 * peaks["shards"] <= peaks["one"], peaks


def test_argument_errors(ctx):
    """NULL arrays, offsets that do not start at 0 or decrease, a genome over 2^32-3 entries below a small cap, and
    device pointers: SYL_ERR_ARG before anything is allocated.  A genome of exactly 2^32-3 entries is its own shard."""
    import torch
    from sylph_b200 import _lib
    from sylph_b200.api import SylphError
    L = _lib.lib()
    ctx.device_bytes(reset_peak=True)
    held, peak = ctx.device_bytes()
    keys = np.arange(10, dtype=np.uint64)
    vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731

    def raw(kmers, koff, G, tracked=None, toff=None, cap=0):
        h = C.c_void_p()
        rc = L.syl_db_shards_create(ctx._h, kmers, koff, tracked, toff, None, G, 31, 200, cap, C.byref(h))
        if rc == _lib.SYL_OK:
            L.syl_db_shards_free(h)
        return rc

    off = np.array([0, 4, 10], np.uint64)
    assert raw(vp(keys), vp(off), 2) == _lib.SYL_OK
    assert raw(vp(keys), None, 2) == _lib.SYL_ERR_ARG                         # kmer_off NULL
    assert raw(None, vp(off), 2) == _lib.SYL_ERR_ARG                          # k-mers counted, none given
    assert raw(vp(keys), vp(off), 2, None, vp(off)) == _lib.SYL_ERR_ARG       # tracked counted, none given
    for bad in ([0, 5, 3, 10], [1, 4, 10]):
        b = np.array(bad, np.uint64)
        assert raw(vp(keys), vp(b), len(bad) - 1) == _lib.SYL_ERR_ARG
        assert raw(vp(keys), vp(off), 2, vp(keys), vp(np.array(bad[-3:], np.uint64))) == _lib.SYL_ERR_ARG
    huge = np.array([0, 3, 3 + 2**32 - 2], np.uint64)                         # genome 1: 2^32-2 entries
    assert raw(vp(keys), vp(huge), 2, cap=5) == _lib.SYL_ERR_ARG
    fits = np.array([0, 3, 3 + 2**32 - 3, 2**32 + 3], np.uint64)               # genome 1: exactly 2^32-3
    h = C.c_void_p()
    assert L.syl_db_shards_create(ctx._h, vp(keys), vp(fits), None, None, None, 3, 31, 200, 5, C.byref(h)) == _lib.SYL_OK
    got = []
    for i in range(int(L.syl_db_shards_count(h))):
        a, n, e = C.c_uint64(), C.c_uint64(), C.c_uint64()
        assert L.syl_db_shards_range(h, i, C.byref(a), C.byref(n), C.byref(e)) == _lib.SYL_OK
        got.append((a.value, n.value, e.value))
    assert got == [(0, 1, 3), (1, 1, 2**32 - 3), (2, 1, 3)]
    assert L.syl_db_shards_range(h, 3, None, None, None) == _lib.SYL_ERR_ARG
    L.syl_db_shards_free(h)
    dk, do = torch.arange(10, device="cuda"), torch.tensor([0, 4, 10], device="cuda")
    assert raw(C.c_void_p(dk.data_ptr()), vp(off), 2) == _lib.SYL_ERR_ARG    # device k-mers
    assert raw(vp(keys), C.c_void_p(do.data_ptr()), 2) == _lib.SYL_ERR_ARG   # device offsets
    with pytest.raises(SylphError) as e:
        ctx.db_shards(dk, do)
    assert e.value.code == _lib.SYL_ERR_ARG
    assert ctx.device_bytes() == (held, peak)
