"""GPU: pass 1 of a db-shards call by the scan formulation (SYL_DB_SCAN=1): the genome k-mers streamed chunk by chunk
past every sample's lookup table instead of an index build.  Rows bit-identical to the same call under SYL_DB_SCAN=0
and to the one-index handle path, and equal to the oracle: the scripted families in both formulations (a count >= 256
redone in CSR inside one chunk, -u -I, no_ci, -m 0, -M at a genome's k-mer count, tracked-only winners, derep at its
threshold), the ANI near-tie pairs in different chunks, chunk edges (1, 997 and the default, empty genomes, a genome
larger than a chunk), sample-table edges (empty sample, keys 0 and 2^64-2, count 0, 1 to 10^5 keys, 17 unequal
samples, keys sharing a bucket and their fingerprint), host samples from pageable and pinned arrays, device memory of
a 10^8-entry scan, the default rule, and the driver's TSVs."""
import numpy as np
import pytest

from tests import ani_ties as T
from tests import contain_scripts as S
from tests.contain_compare import compare, cr_params
from tests.test_contain_scripts_gpu import check, same
from tests.test_db_shards_gpu import PARAM_SETS, comm, community, world  # noqa: F401  (fixtures)
from tests.test_sample_stream_gpu import pinned_copy

pytestmark = pytest.mark.gpu

CHUNKS = ["1", "997", None]   # SYL_DB_SCAN_CHUNK: one genome per chunk, 997 k-mers, the default 2^25


@pytest.fixture(params=["hist", "csr"])
def formulation(request, monkeypatch):
    for k in ("SYL_CONTAIN_CSR", "SYL_BOOT_REPLAY", "SYL_DB_SHARD_ENTRIES", "SYL_DB_SCAN", "SYL_DB_SCAN_CHUNK",
              "SYL_SAMPLE_BATCH"):
        monkeypatch.delenv(k, raising=False)
    if request.param == "csr":
        monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
    return request.param


def shards(ctx, d, k=31, c=1):
    return ctx.db_shards(d["kmers"], d["kmer_off"], d.get("tracked"), d.get("tracked_off"), d["gn_size"], k=k, c=c)


def scan_build_one(ctx, monkeypatch, db, sh, handles, pseudotax, P, chunk):
    """rows of the scan call, after checking them equal to the build call and the one-index call"""
    from sylph_b200.api import contain_params
    p = contain_params(pseudotax=pseudotax, **P)
    call = (lambda: sh.profile(handles, p)) if pseudotax else (lambda: sh.query(handles, p))
    want = ctx.profile(db, handles, p) if pseudotax else ctx.query(db, handles, p)
    monkeypatch.setenv("SYL_DB_SCAN", "0")
    ctx.kernel_time("scan", reset=True)
    built = call()
    assert ctx.kernel_time("scan")[1] == 0
    monkeypatch.setenv("SYL_DB_SCAN", "1")
    if chunk:
        monkeypatch.setenv("SYL_DB_SCAN_CHUNK", chunk)
    ctx.enable_timing(True)
    ctx.kernel_time("scan", reset=True)
    ctx.kernel_time("join", reset=True)
    got = call()
    n_scan, n_join = ctx.kernel_time("scan")[1], ctx.kernel_time("join")[1]
    ctx.enable_timing(False)
    monkeypatch.delenv("SYL_DB_SCAN_CHUNK", raising=False)
    monkeypatch.delenv("SYL_DB_SCAN")
    same(built, want, ("build", P))
    same(got, want, ("scan", P, chunk))
    assert n_scan > 0
    if not pseudotax:
        assert n_join == 0   # no index was probed: pass 1 only scanned
    return got


@pytest.mark.parametrize("chunk", CHUNKS, ids=["chunk1", "chunk997", "chunk_default"])
@pytest.mark.parametrize("pseudotax", [False, True])
def test_scripted_rows(ctx, world, formulation, monkeypatch, pseudotax, chunk):  # noqa: F811
    """every scripted sample in one call under every parameter set the families are built for, plus -u -I: scan rows ==
    build rows == one-index rows; at the default chunk also each sample's rows == the oracle"""
    handles = [world.smp[n] for n in S.SAMPLES]
    sh = shards(ctx, world.d)
    try:
        for P in map(dict, PARAM_SETS):
            got = scan_build_one(ctx, monkeypatch, world.db, sh, handles, pseudotax, P, chunk)
            if chunk is not None or "estimate_unknown" in P:
                continue
            for si, name in enumerate(S.SAMPLES):
                if P in S.params_for(name):
                    sub = got[got["sample"] == si].copy()
                    sub["sample"] = 0
                    check(sub, name, pseudotax, S.params_for(name).index(P))
    finally:
        sh.free()


PAIRS = [("adjacent",) + p for p in T.WINNER_PAIRS] + [("equal",) + p for p in T.TIE_PAIRS]


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s_k%d_%d" % (p[0], p[1], p[2][1]))
def test_near_tied_genomes_in_different_chunks(ctx, monkeypatch, formulation, pair):
    """two genomes of adjacent or equal ANIs sharing hit k-mers, each in a chunk of its own, in both orders"""
    from oracle import oracle as O
    kind, k, a, b = pair
    for order in ([a, b], [b, a]):
        case = T.Case(order, shared=3)
        d = case.db
        db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], k=k, c=1)
        sh = shards(ctx, d, k=k)
        smp = ctx.upload_sample(case.hash, case.count, k=k, c=1)
        try:
            for pseudotax in (False, True):
                got = scan_build_one(ctx, monkeypatch, db, sh, [smp], pseudotax, {"k": k, "minimum_ani": 0.0}, "1")
                if pseudotax:
                    exp = O.contain_sample(cr_params(k=k, pseudotax=True, minimum_ani=0.0), d["kmers"], d["kmer_off"],
                                           d["tracked"], d["tracked_off"], d["gn_size"], O.Sample(case.hash, case.count))
                    compare(got, exp, True)
        finally:
            smp.free()
            sh.free()
            db.free()


@pytest.mark.parametrize("chunk", CHUNKS, ids=["chunk1", "chunk997", "chunk_default"])
def test_community_with_empty_genomes(ctx, comm, formulation, monkeypatch, chunk):  # noqa: F811
    """five samples of unequal size and each alone, on a db with empty genomes at regular places (so at chunk starts and
    ends), default parameters, no_ci, -m 0 and -u"""
    d, db, smp = comm
    sh = shards(ctx, d, c=200)
    try:
        for pseudotax in (False, True):
            for P in ({}, {"no_ci": 1}, {"minimum_ani": 0.0}, {"estimate_unknown": 1, "read_seq_id": 97.5}):
                got = scan_build_one(ctx, monkeypatch, db, sh, smp, pseudotax, P, chunk)
                assert len(set(got["sample"].tolist())) == 5
            for s in smp[::2]:
                scan_build_one(ctx, monkeypatch, db, sh, [s], pseudotax, {}, chunk)
    finally:
        sh.free()


def crafted_world(seed=9):
    """a db whose genomes hold keys 0 and 2^64-2, keys sharing a table bucket and their low 32 bits, one genome larger
    than 997 k-mers, empty genomes at the start and end; samples: empty, one key, count-0 entries, 1 to 10^5 keys, and
    17 samples of unequal size"""
    rng = np.random.default_rng(seed)
    hi = 2**64 - 2
    crafted = np.array([0, hi] + [(1 << 40) + (i << 32) + 77 for i in range(8)], np.uint64)
    ks = [np.zeros(0, np.uint64)]
    for g in range(30):
        n = 5000 if g == 7 else int(rng.integers(60, 900))
        x = rng.integers(0, hi, n, dtype=np.uint64)
        if g % 5 == 0:
            x = np.concatenate([x, crafted])
        ks.append(np.unique(x))
    ks.append(np.zeros(0, np.uint64))
    G = len(ks)
    pool = np.concatenate(ks)
    d = dict(kmers=np.concatenate(ks), kmer_off=np.concatenate([[0], np.cumsum([len(x) for x in ks])]).astype(np.uint64),
             tracked=rng.choice(pool, 40 * G).astype(np.uint64), tracked_off=(np.arange(G + 1) * 40).astype(np.uint64),
             gn_size=rng.integers(10**5, 10**6, G).astype(np.uint64))

    def sample(n, frac_db=0.7, zero=0.0):
        m = int(n * frac_db)
        keys = np.unique(np.concatenate([rng.choice(pool, m) if m else np.zeros(0, np.uint64),
                                         rng.integers(0, hi, n - m, dtype=np.uint64)]))
        cnt = rng.integers(1, 6, len(keys)).astype(np.uint32)
        cnt[rng.random(len(keys)) < zero] = 0
        return keys, cnt

    samples = [(np.zeros(0, np.uint64), np.zeros(0, np.uint32)), (crafted.copy(), np.arange(1, 11, dtype=np.uint32)),
               sample(1), sample(2000, zero=0.3), sample(100_000, frac_db=0.05)]
    samples += [sample(int(n)) for n in rng.integers(1, 4000, 17)]
    return d, samples


@pytest.mark.parametrize("chunk", ["997", None], ids=["chunk997", "chunk_default"])
def test_sample_table_edges(ctx, formulation, monkeypatch, chunk):
    d, raw = crafted_world()
    db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=1)
    sh = shards(ctx, d)
    smp = [ctx.upload_sample(h, c, c=1) for h, c in raw]
    try:
        for pseudotax in (False, True):
            for P in ({"minimum_ani": 0.0}, {}):
                got = scan_build_one(ctx, monkeypatch, db, sh, smp, pseudotax, P, chunk)
                if P and not pseudotax:
                    assert 1 in set(got["sample"].tolist())   # the crafted keys hit
            for s in smp[:5]:
                scan_build_one(ctx, monkeypatch, db, sh, [s], pseudotax, {"minimum_ani": 0.0}, chunk)
    finally:
        for s in smp:
            s.free()
        sh.free()
        db.free()


def test_host_samples_pageable_and_pinned_db(ctx, comm, monkeypatch):  # noqa: F811
    """syl_query_host_samples / syl_profile_host_samples with shards of a db in pageable and in pinned host arrays"""
    for k in ("SYL_CONTAIN_CSR", "SYL_DB_SCAN_CHUNK", "SYL_SAMPLE_BATCH"):
        monkeypatch.delenv(k, raising=False)
    d, db, smp = comm
    _, raw = community()
    hashes = np.concatenate([h for h, _ in raw])
    counts = np.concatenate([c for _, c in raw])
    off = np.concatenate([[0], np.cumsum([len(h) for h, _ in raw])]).astype(np.uint64)
    mrl = np.array([120.0 + 30 * i for i in range(len(raw))])
    keep = []
    pinned = dict(d)
    for key in ("kmers", "kmer_off", "tracked", "tracked_off", "gn_size"):
        pinned[key], t = pinned_copy(np.ascontiguousarray(d[key]))
        keep.append(t)
    for arrays in (d, pinned):
        sh = shards(ctx, arrays, c=200)
        try:
            for pseudotax in (False, True):
                fn = ctx.profile_host_samples if pseudotax else ctx.query_host_samples
                want = (ctx.profile if pseudotax else ctx.query)(db, smp)
                for scan in ("0", "1"):
                    monkeypatch.setenv("SYL_DB_SCAN", scan)
                    for chunk in ("997", None):
                        if chunk:
                            monkeypatch.setenv("SYL_DB_SCAN_CHUNK", chunk)
                        same(fn(sh, hashes, counts, off, 200, mrl), want, (scan, chunk, pseudotax))
                        monkeypatch.delenv("SYL_DB_SCAN_CHUNK", raising=False)
        finally:
            monkeypatch.delenv("SYL_DB_SCAN", raising=False)
            sh.free()


def big_db(n_entries, G, seed=1):
    rng = np.random.default_rng(seed)
    kmers = rng.integers(0, (2**64 - 1) // 200, n_entries, dtype=np.uint64)
    kmer_off = np.linspace(0, n_entries, G + 1).astype(np.uint64)
    return kmers, kmer_off, rng


def test_device_memory_of_a_large_scan(monkeypatch):
    """a scan over a 10^8-entry db peaks within DESIGN §3's bound (two staging chunks + the sample tables + one chunk's
    per-pair buffers and row tables), far below the build's ~14 bytes per entry, and holds nothing after the call"""
    import sylph_b200
    for k in ("SYL_CONTAIN_CSR", "SYL_DB_SCAN_CHUNK"):
        monkeypatch.delenv(k, raising=False)
    N, G = 10**8, 5000
    kmers, kmer_off, rng = big_db(N, G)
    ctx = sylph_b200.Context(0)
    try:
        g = 123
        a, b = int(kmer_off[g]), int(kmer_off[g + 1])
        h = np.unique(np.concatenate([kmers[a:b], rng.integers(0, 2**60, 10**5, dtype=np.uint64)]))
        smp = ctx.upload_sample(h, np.full(len(h), 3, np.uint32), c=200)
        sh = ctx.db_shards(kmers, kmer_off, gn_size=np.full(G, 10**6, np.uint64), c=200)
        held0, _ = ctx.device_bytes(reset_peak=True)
        monkeypatch.setenv("SYL_DB_SCAN", "1")
        rows = sh.query([smp])
        held1, peak = ctx.device_bytes(reset_peak=True)
        assert list(rows["genome"]) == [g]
        chunk = 2**25
        G_chunk = -(-chunk * G // N) + 1
        bound = (2 * (chunk * 8 + G_chunk * 12) + len(h) * 7 + 4096
                 + G_chunk * (1 + 1024) + 64 * 2**20)   # per-pair histograms of one chunk; row tables, bootstrap, scratch
        assert peak - held0 <= bound, (peak - held0, bound)
        assert peak - held0 < N * 14 / 2
        assert held1 <= held0
        monkeypatch.setenv("SYL_DB_SCAN", "0")
        assert (sh.query([smp]) == rows).all()
        sh.free()
        smp.free()
    finally:
        ctx.close()


def test_default_rule(monkeypatch):
    """above the size floor a 1-sample call scans (scan launches, no index join); 80 samples of 10 genomes each, whose
    tables outgrow L2, build; the plan the library reports agrees"""
    import sylph_b200
    for k in ("SYL_CONTAIN_CSR", "SYL_DB_SCAN_CHUNK", "SYL_DB_SCAN"):
        monkeypatch.delenv(k, raising=False)
    N, G = 2**28 + 1000, 20000
    kmers, kmer_off, rng = big_db(N, G, seed=2)
    ctx = sylph_b200.Context(0)
    try:
        smp, genomes, sk = [], [], 0
        for i in range(80):
            gs = [int(g) for g in rng.choice(G, 10, replace=False)]
            h = np.unique(np.concatenate([kmers[int(kmer_off[g]):int(kmer_off[g + 1])] for g in gs]))
            smp.append(ctx.upload_sample(h, np.full(len(h), 2, np.uint32), c=200))
            genomes.append(gs)
            sk += len(h)
        assert ctx.db_scan_plan(N, 0, G, 1, N // G * 10)
        assert not ctx.db_scan_plan(N, 0, G, 80, sk)
        assert not ctx.db_scan_plan(2**28 - 1, 0, G, 1, N // G * 10)
        sh = ctx.db_shards(kmers, kmer_off, gn_size=np.full(G, 10**6, np.uint64), c=200)
        ctx.enable_timing(True)
        for n, scans in ((1, True), (80, False)):
            ctx.kernel_time("scan", reset=True)
            ctx.kernel_time("join", reset=True)
            rows = sh.query(smp[:n])
            assert (ctx.kernel_time("scan")[1] > 0) == scans
            assert (ctx.kernel_time("join")[1] == 0) == scans
            want = sorted((i, g) for i in range(n) for g in genomes[i])
            assert sorted(zip(rows["sample"].tolist(), rows["genome"].tolist())) == want
        sh.free()
        for s in smp:
            s.free()
    finally:
        ctx.close()


from tests.test_driver_gpu import d, exe, sk  # noqa: E402,F401  (fixtures)


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_driver_tsv(exe, d, sk, cmd):  # noqa: F811
    """`sylph-b200 query | profile` prints the same TSV with SYL_DB_SCAN=1, =0 and the default (one index), also with
    --devices 0,0"""
    from tests.test_driver_gpu import SK_PAIRS, SK_SAMPLES, run
    args = [cmd] + SK_SAMPLES + SK_PAIRS + ["sk/db.syldb"]
    one = run(exe, args, d).stdout
    assert len(one.splitlines()) > 10
    for env in ({"SYL_DB_SCAN": "1"}, {"SYL_DB_SCAN": "0"}, {"SYL_DB_SCAN": "1", "SYL_DB_SCAN_CHUNK": "997"}):
        assert run(exe, args, d, env=env).stdout == one, env
        assert run(exe, args[:1] + ["--devices", "0,0"] + args[1:], d, env=env).stdout == one, env


@pytest.mark.parametrize("batch", ["2", "5"])
def test_forced_scan_of_host_samples_in_several_batches(ctx, comm, monkeypatch, batch):  # noqa: F811
    """SYL_DB_SCAN=1 with host samples that do not fit one batch (SYL_SAMPLE_BATCH=2 for five samples) builds instead,
    since a scan stages every sample at once: no scan launch, rows equal to SYL_DB_SCAN=0 and to the handle path.  With
    all five in one batch (SYL_SAMPLE_BATCH=5) the forced call scans, with the same rows; syl_db_scan_plan agrees."""
    for k in ("SYL_CONTAIN_CSR", "SYL_DB_SCAN_CHUNK"):
        monkeypatch.delenv(k, raising=False)
    d, db, smp = comm
    _, raw = community()
    hashes = np.concatenate([h for h, _ in raw])
    counts = np.concatenate([c for _, c in raw])
    off = np.concatenate([[0], np.cumsum([len(h) for h, _ in raw])]).astype(np.uint64)
    mrl = np.array([120.0 + 30 * i for i in range(len(raw))])
    monkeypatch.setenv("SYL_SAMPLE_BATCH", batch)
    sh = shards(ctx, d, c=200)
    try:
        for pseudotax in (False, True):
            fn = ctx.profile_host_samples if pseudotax else ctx.query_host_samples
            want = (ctx.profile if pseudotax else ctx.query)(db, smp)
            monkeypatch.setenv("SYL_DB_SCAN", "0")
            same(fn(sh, hashes, counts, off, 200, mrl), want, ("build", batch, pseudotax))
            monkeypatch.setenv("SYL_DB_SCAN", "1")
            ctx.enable_timing(True)
            ctx.kernel_time("scan", reset=True)
            got = fn(sh, hashes, counts, off, 200, mrl)
            launches = ctx.kernel_time("scan")[1]
            ctx.enable_timing(False)
            same(got, want, ("forced scan", batch, pseudotax))
            assert (launches > 0) == (batch == "5"), (batch, launches)
            assert ctx.db_scan_plan(len(d["kmers"]), len(d["tracked"]), len(d["gn_size"]), len(raw), len(hashes)) == (batch == "5")
    finally:
        monkeypatch.delenv("SYL_DB_SCAN", raising=False)
        sh.free()
