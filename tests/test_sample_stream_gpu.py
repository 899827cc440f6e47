"""GPU: query and profile samples from host memory (syl_query_host_samples / syl_profile_host_samples).  Rows equal
the handle path's (syl_sample_upload + syl_query / syl_profile, or the _shards calls) bit for bit, at one sample per
batch, three per batch and the budget's own batches, on one index and on forced shards, for query, profile and profile
-u -I 98, with samples of c below the db's, empty samples and unsorted input, from pinned and pageable arrays.  Also:
shard builds in small chunks against one-sample batches, equal to the one-index call in both formulations; the capacity
protocol on both db kinds, every argument error, the device-memory bound, and one build per shard per call."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_contain_scripts_gpu import same
from tests.test_db_shards_gpu import cap_for, community

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = {"query": (False, {}), "profile": (True, {}), "profile_u": (True, {"estimate_unknown": 1, "read_seq_id": 98.0})}


def host_set(raw, rng):
    """the community's samples (plus copies at c = 100 and empty samples), each shuffled: hashes, counts, off, c, mrl"""
    smp = []
    for i, (h, c) in enumerate(raw):
        smp.append((h, c, 200))
        if i % 2 == 0:
            smp.append((h[: len(h) // 2], c[: len(h) // 2], 100))   # c below the db's
    smp.insert(3, (np.zeros(0, np.uint64), np.zeros(0, np.uint32), 200))
    smp.append((np.zeros(0, np.uint64), np.zeros(0, np.uint32), 200))
    hs, cs = [], []
    for h, c, _ in smp:
        p = rng.permutation(len(h))
        hs.append(h[p])
        cs.append(c[p])
    off = np.concatenate([[0], np.cumsum([len(h) for h in hs])]).astype(np.uint64)
    return dict(hashes=np.concatenate(hs).astype(np.uint64), counts=np.concatenate(cs).astype(np.uint32), off=off,
                c=np.array([c for _, _, c in smp], np.uint64), mrl=np.array([110.0 + 13 * i for i in range(len(smp))]))


def pinned_copy(a):
    import torch
    t = torch.empty(a.nbytes, dtype=torch.uint8, pin_memory=True)
    out = t.numpy().view(a.dtype)
    out[:] = a
    return out, t


@pytest.fixture(scope="module")
def world(ctx):
    d, raw = community()
    hs = host_set(raw, np.random.default_rng(3))
    db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200)
    off = hs["off"]
    handles = []
    for i in range(len(off) - 1):
        s = ctx.upload_sample(hs["hashes"][off[i]:off[i + 1]], hs["counts"][off[i]:off[i + 1]], c=int(hs["c"][i]))
        s.mean_read_length = float(hs["mrl"][i])
        handles.append(s)
    ph, kh = pinned_copy(hs["hashes"])
    pc, kc = pinned_copy(hs["counts"])
    yield dict(d=d, db=db, hs=hs, handles=handles, pinned=(ph, pc), keep=(kh, kc))
    for s in handles:
        s.free()
    db.free()


def run_host(ctx, target, hs, arrays, mode, cap=None):
    from sylph_b200.api import contain_params
    pseudotax, P = MODES[mode]
    p = contain_params(pseudotax=pseudotax, **P)
    fn = ctx.profile_host_samples if pseudotax else ctx.query_host_samples
    return fn(target, arrays[0], arrays[1], hs["off"], hs["c"], hs["mrl"], p, cap=cap)


def run_handles(ctx, target, handles, mode, shards):
    from sylph_b200.api import contain_params
    pseudotax, P = MODES[mode]
    p = contain_params(pseudotax=pseudotax, **P)
    if shards:
        return target.profile(handles, p) if pseudotax else target.query(handles, p)
    return ctx.profile(target, handles, p) if pseudotax else ctx.query(target, handles, p)


@pytest.mark.parametrize("batch", ["1", "3", None], ids=["batch1", "batch3", "budget"])
@pytest.mark.parametrize("kind", ["one", "shards"])
def test_rows_equal_handle_path(ctx, world, monkeypatch, batch, kind):
    monkeypatch.delenv("SYL_SAMPLE_BATCH", raising=False)
    monkeypatch.delenv("SYL_DB_SHARD_ENTRIES", raising=False)
    d, hs = world["d"], world["hs"]
    target = world["db"]
    if kind == "shards":
        monkeypatch.setenv("SYL_DB_SHARD_ENTRIES", str(cap_for("uneven", d)))
        target = ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200)
        assert len(target) >= 2
    if batch:
        monkeypatch.setenv("SYL_SAMPLE_BATCH", batch)
    try:
        for mode in MODES:
            want = run_handles(ctx, target, world["handles"], mode, kind == "shards")
            assert len(set(want["sample"].tolist())) >= 5, mode
            for arrays, what in (((hs["hashes"], hs["counts"]), "pageable"), (world["pinned"], "pinned")):
                same(run_host(ctx, target, hs, arrays, mode), want, (kind, batch, mode, what))
    finally:
        if kind == "shards":
            target.free()


@pytest.mark.parametrize("csr", [False, True], ids=["hist", "csr"])
def test_shard_builds_share_the_copy_stream_with_batches(ctx, world, monkeypatch, csr):
    """index chunks of 4096 entries and one sample per batch: each shard build's chunk copies and the staging of the next
    batch take turns on the ctx's copy stream; rows equal the one-index call's, from pageable and pinned arrays"""
    for v in ("SYL_DB_SHARD_ENTRIES", "SYL_CONTAIN_CSR", "SYL_BOOT_REPLAY"):
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setenv("SYL_DB_CHUNK", "4096")
    monkeypatch.setenv("SYL_SAMPLE_BATCH", "1")
    if csr:
        monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
    d, hs = world["d"], world["hs"]
    sh = ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200,
                       max_entries=cap_for("uneven", d))
    try:
        assert len(sh) >= 2 and all(e > 4 * 4096 for _, _, e in sh.ranges())
        for mode in MODES:
            want = run_handles(ctx, world["db"], world["handles"], mode, False)
            for arrays, what in (((hs["hashes"], hs["counts"]), "pageable"), (world["pinned"], "pinned")):
                same(run_host(ctx, sh, hs, arrays, mode), want, (csr, mode, what))
    finally:
        sh.free()


@pytest.mark.parametrize("kind", ["one", "shards"])
def test_capacity_retry(ctx, world, monkeypatch, kind):
    """a row buffer that is too small: SYL_ERR_CAPACITY with the size needed; the retry returns the same rows"""
    monkeypatch.setenv("SYL_SAMPLE_BATCH", "2")
    d, hs = world["d"], world["hs"]
    target = world["db"] if kind == "one" else ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"],
                                                             d["gn_size"], c=200, max_entries=cap_for("uneven", d))
    try:
        for mode in ("query", "profile"):
            want = run_handles(ctx, target, world["handles"], mode, kind == "shards")
            got = run_host(ctx, target, hs, (hs["hashes"], hs["counts"]), mode, cap=3)
            same(got, want, (kind, mode))
            assert len(want) > 3
    finally:
        if kind == "shards":
            target.free()


def _raw_call(ctx, db, shards, s, p, cap=16):
    import ctypes as C
    from sylph_b200 import _lib
    from sylph_b200.api import ANI_ROW_DTYPE
    rows = np.empty(cap, dtype=ANI_ROW_DTYPE)
    n = C.c_uint64(0)
    fn = _lib.lib().syl_profile_host_samples if p.pseudotax else _lib.lib().syl_query_host_samples
    return fn(ctx._h, db, shards, C.byref(s), C.byref(p), rows.ctypes.data_as(C.c_void_p), cap, C.byref(n))


def test_argument_errors(ctx, world):
    import ctypes as C
    import torch
    from sylph_b200 import _lib
    from sylph_b200.api import contain_params
    d, hs = world["d"], world["hs"]
    db = world["db"]
    sh = ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200)
    nt = ctx.build_db_arrays(d["kmers"], d["kmer_off"], None, None, d["gn_size"], c=200)
    dev = torch.zeros(len(hs["hashes"]), dtype=torch.int64, device="cuda")

    def make(off=None, c=None, k=31, hashes=None):
        off = hs["off"] if off is None else np.asarray(off, np.uint64)
        c = hs["c"] if c is None else np.asarray(c, np.uint64)
        keep = [hs["hashes"], hs["counts"], off, c, hs["mrl"]]
        h = hashes if hashes is not None else hs["hashes"].ctypes.data
        return _lib.HostSamples(h, hs["counts"].ctypes.data, off.ctypes.data, c.ctypes.data, hs["mrl"].ctypes.data,
                                len(off) - 1, k), keep

    def code(db_h, sh_h, s, p):
        return _raw_call(ctx, db_h, sh_h, s[0], p)

    q, pr = contain_params(pseudotax=False), contain_params(pseudotax=True)
    try:
        bad_off = hs["off"].copy()
        bad_off[2] = bad_off[1] - 1 if bad_off[1] else 5
        cases = [
            ("no db", (None, None, make(), q), _lib.SYL_ERR_ARG, "exactly one"),
            ("both dbs", (db._h, sh._h, make(), q), _lib.SYL_ERR_ARG, "exactly one"),
            ("k", (db._h, None, make(k=21), q), _lib.SYL_ERR_ARG, "k parameter"),
            ("c", (db._h, None, make(c=np.full(len(hs["c"]), 300)), q), _lib.SYL_ERR_ARG, "c parameter"),
            ("c shards", (None, sh._h, make(c=np.full(len(hs["c"]), 300)), q), _lib.SYL_ERR_ARG, "c parameter"),
            ("-u without -I", (db._h, None, make(), contain_params(pseudotax=False, estimate_unknown=1)), _lib.SYL_ERR_UNSUPPORTED, "-u"),
            ("no tracked", (nt._h, None, make(), pr), _lib.SYL_ERR_ARG, "disable-profiling"),
            ("off[0]", (db._h, None, make(off=np.concatenate([[1], hs["off"][1:]])), q), _lib.SYL_ERR_ARG, "offsets"),
            ("decreasing off", (db._h, None, make(off=bad_off), q), _lib.SYL_ERR_ARG, "offsets"),
            ("device pointer", (db._h, None, make(hashes=dev.data_ptr()), q), _lib.SYL_ERR_ARG, "device pointer"),
        ]
        for what, (a, b, s, p), want, msg in cases:
            rc = code(a, b, s, p)
            assert rc == want, (what, rc)
            assert msg in _lib.lib().syl_last_error().decode(), what
    finally:
        nt.free()
        sh.free()


def test_device_memory_bounded_by_budget(monkeypatch):
    """samples totalling over 4 B under a budget of B: the call's peak above what the ctx held stays within B plus the
    staging rings, while the same samples as resident handles exceed that; rows equal the handles' rows.  A sample that
    does not fit alone is SYL_ERR_OOM, naming its bytes."""
    import sylph_b200
    from sylph_b200 import _lib
    from sylph_b200.api import SylphError, contain_params
    monkeypatch.delenv("SYL_SAMPLE_BATCH", raising=False)
    d, raw = community(seed=9, G=60)
    rng = np.random.default_rng(5)
    hi = (2**64 - 1) // 200
    n, S = 250_000, 90
    hs = [np.unique(rng.integers(0, hi, n, dtype=np.uint64)) for _ in range(S)]
    hs[0] = np.unique(np.concatenate([hs[0], raw[0][0]]))
    cs = [np.full(len(h), 3, np.uint32) for h in hs]
    off = np.concatenate([[0], np.cumsum([len(h) for h in hs])]).astype(np.uint64)
    H, Cn = np.concatenate(hs), np.concatenate(cs)
    B = 64 << 20
    assert 12 * len(H) >= 4 * B
    ctx = sylph_b200.Context(0)
    try:
        db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200)
        ctx.set_sample_memory(B)
        held0, _ = ctx.device_bytes(reset_peak=True)
        got = ctx.profile_host_samples(db, H, Cn, off, 200, 150.0)
        peak = ctx.device_bytes()[1] - held0
        ring = ctx.ingest_ring_bytes()[0]
        assert peak <= B + ring, (peak, B, ring)
        handles = [ctx.upload_sample(h, c, c=200) for h, c in zip(hs, cs)]
        for s in handles:
            s.mean_read_length = 150.0
        want = ctx.profile(db, handles, contain_params(pseudotax=True))
        same(got, want, "budget")
        assert len(want) > 0
        assert ctx.device_bytes()[1] - held0 > B + ring
        for s in handles:
            s.free()
        ctx.set_sample_memory(8 << 20)
        with pytest.raises(SylphError) as e:
            ctx.query_host_samples(db, H, Cn, off, 200, 150.0)
        assert e.value.code == _lib.SYL_ERR_OOM and "sample 0 needs" in str(e.value) and "budget is 8388608" in str(e.value)
        db.free()
    finally:
        ctx.close()


SHARD_SCRIPT = r"""
import numpy as np, sylph_b200
from sylph_b200.api import contain_params
from tests.test_db_shards_gpu import community
d, raw = community()
ctx = sylph_b200.Context(0)
sh = ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200,
                   max_entries=int(d["kmer_off"][-1] + d["tracked_off"][-1]) // 4 + 1)
H = np.concatenate([h for h, _ in raw]); C = np.concatenate([c for _, c in raw])
off = np.concatenate([[0], np.cumsum([len(h) for h, _ in raw])]).astype(np.uint64)
print("SHARDS", len(sh), flush=True)
for pseudotax in (False, True):
    print("CALL", flush=True)
    fn = ctx.profile_host_samples if pseudotax else ctx.query_host_samples
    rows = fn(sh, H, C, off, 200, 150.0, contain_params(pseudotax=pseudotax))
    assert len(rows) > 0
sh.free()
ctx.close()
"""


def test_one_build_per_shard_per_call():
    """one sample per batch (SYL_SAMPLE_BATCH=1): query and profile each build every shard once, counted from the
    [db shard] lines of SYL_DEBUG_TIMING"""
    env = dict(os.environ, SYL_DEBUG_TIMING="1", SYL_SAMPLE_BATCH="1", PYTHONPATH=REPO)
    env.pop("SYL_DB_SHARD_ENTRIES", None)
    r = subprocess.run([sys.executable, "-c", SHARD_SCRIPT], cwd=REPO, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    lines = r.stdout.splitlines()
    n = int(next(x for x in lines if x.startswith("SHARDS")).split()[1])
    assert n >= 3
    calls = "\n".join(lines).split("CALL")[1:]
    assert len(calls) == 2
    for c in calls:
        built = [x.split("]")[0] for x in c.splitlines() if x.startswith("[db shard")]
        assert built == ["[db shard %d/%d" % (i + 1, n) for i in range(n)], c[-2000:]
