"""GPU: samples streamed from host memory (syl_query_host_samples / syl_profile_host_samples) branch by branch.

Scripted statistics (tests/contain_scripts.py): every scripted sample in one host-samples call, in a shuffled order
with `big` (counts >= 256) in a middle batch, at 1, 2 and 3 samples per batch and the budget's one batch, in both
formulations, from pageable, pinned and half-pinned arrays, under every parameter set of the families and -u: rows
bit-equal to the handle path and each sample's rows == the C oracle; the statistics launches show that only the batch
of `big` is redone (in the CSR formulation, after the next batch was staged); SYL_BOOT_REPLAY=1 on the replay
samples; the same over db shards, with survivor batches inside plan batches, staged again and found in a slot, and the
ANI near-tie pairs in separate shards.

Segment-sort regimes: one batch of 640 samples of every size from 0 to 400 k-mers and a few of 10^3 to 10^5, so that
cub::DeviceSegmentedSort partitions them into small, medium and large segments; keys 0 and 2^64 - 2 and keys shared
between samples; input shuffled, sorted and reversed: rows == the handle path and the plain join mapping, a
stratified subset == the oracle; calls of empty samples; H2D bytes of exactly one copy of each batch.

Memory bound: a db of 600 genomes sharing a core and samples drawn from it, at a budget of 16 MB: the CSR hit values
and the rows past the plan's 96 per sample would pass the budget, so the batches are split in halves; the peak stays
within the budget and the rows equal the handle path's and the oracle's.  A sample that does not fit alone is
SYL_ERR_OOM, naming its bytes."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import ani_ties as T
from tests import contain_scripts as S
from tests.contain_compare import compare, cr_params
from tests.test_contain_scripts_gpu import Gpu, check, same
from tests.test_db_shards_gpu import PAIRS, PARAM_SETS, shards_of
from tests.test_sample_stream_gpu import pinned_copy

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = ("SYL_CONTAIN_CSR", "SYL_BOOT_REPLAY", "SYL_SAMPLE_BATCH", "SYL_DB_SHARD_ENTRIES", "SYL_JOIN_PLAIN")
BATCHES = ["1", "2", "3", None]
BATCH_IDS = ["batch1", "batch2", "batch3", "budget"]
# (hash pinned, count pinned): the call decides each array's copy path on its own
MEMS = {"pageable": (False, False), "pinned": (True, True), "hash_pinned": (True, False), "count_pinned": (False, True)}


def row_bytes():
    """contain.hpp ROW_BYTES: two row tables, the bootstrap's results and its histogram"""
    from sylph_b200.api import ANI_ROW_DTYPE
    return 2 * ANI_ROW_DTYPE.itemsize + 100 * 17 + 17 * 4 + 8


@pytest.fixture(params=["hist", "csr"])
def formulation(request, monkeypatch):
    for k in HOOKS:
        monkeypatch.delenv(k, raising=False)
    if request.param == "csr":
        monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
    return request.param


def stream_order(seed=11):
    """every scripted sample, shuffled, with `big` fifth: in a middle batch at 1, 2 and 3 samples per batch"""
    rest = [n for n in S.SAMPLES if n != "big"]
    rest = [rest[i] for i in np.random.default_rng(seed).permutation(len(rest))]
    return rest[:4] + ["big"] + rest[4:]


def host_arrays(w, names):
    hs, cs = zip(*(w.sample_arrays(n) for n in names))
    off = np.concatenate([[0], np.cumsum([len(h) for h in hs])]).astype(np.uint64)
    mrl = np.array([150.0 + 7 * S.SAMPLES.index(n) for n in names])
    return dict(hashes=np.concatenate(hs).astype(np.uint64), counts=np.concatenate(cs).astype(np.uint32), off=off,
                c=np.ones(len(names), np.uint64), mrl=mrl)


class Stream:
    """The scripted world as one db and handles (Gpu), and its samples as host arrays in stream_order()."""

    def __init__(self, ctx):
        self.ctx, self.g = ctx, Gpu(ctx)
        for i, n in enumerate(S.SAMPLES):
            self.g.smp[n].mean_read_length = 150.0 + 7 * i
        self.order = stream_order()
        self.hs = host_arrays(self.g.w, self.order)
        ph, kh = pinned_copy(self.hs["hashes"])
        pc, kc = pinned_copy(self.hs["counts"])
        self.pinned, self.keep = (ph, pc), (kh, kc)
        self.want = {}

    def arrays(self, mem):
        ph, pc = MEMS[mem]
        return (self.pinned[0] if ph else self.hs["hashes"]), (self.pinned[1] if pc else self.hs["counts"])

    def handles(self, target, pseudotax, P, key):
        """handle-path rows of the samples in stream order (cached per target, formulation and parameters)"""
        k = (key, os.environ.get("SYL_CONTAIN_CSR"), pseudotax, tuple(sorted(P.items())))
        if k not in self.want:
            from sylph_b200.api import contain_params
            p = contain_params(pseudotax=pseudotax, **P)
            hl = [self.g.smp[n] for n in self.order]
            if key == "one":
                self.want[k] = self.ctx.profile(target, hl, p) if pseudotax else self.ctx.query(target, hl, p)
            else:
                self.want[k] = target.profile(hl, p) if pseudotax else target.query(hl, p)
        return self.want[k]


@pytest.fixture(scope="module")
def sw(ctx):
    return Stream(ctx)


def run_host(ctx, target, hs, arrays, pseudotax, P):
    from sylph_b200.api import contain_params
    p = contain_params(pseudotax=pseudotax, **P)
    fn = ctx.profile_host_samples if pseudotax else ctx.query_host_samples
    return fn(target, arrays[0], arrays[1], hs["off"], hs["c"], hs["mrl"], p)


def check_each(rows, names, pseudotax, P):
    """each sample's rows == the oracle (parameter sets its family is built for; -u is held to the handle path)"""
    n = 0
    for si, name in enumerate(names):
        if P in S.params_for(name):
            sub = rows[rows["sample"] == si].copy()
            sub["sample"] = 0
            n += check(sub, name, pseudotax, S.params_for(name).index(P))
    return n


def n_batches(batch, S_):
    return 1 if batch is None else -(-S_ // int(batch))


@pytest.mark.parametrize("mem", list(MEMS))
@pytest.mark.parametrize("batch", BATCHES, ids=BATCH_IDS)
def test_scripted_rows_streamed(sw, formulation, monkeypatch, batch, mem):
    """query and profile of every scripted sample in one host-samples call, under every parameter set and -u: rows
    bit-equal to the handle path, each sample's rows == the oracle"""
    if batch:
        monkeypatch.setenv("SYL_SAMPLE_BATCH", batch)
    arrays = sw.arrays(mem)
    for pseudotax in (False, True):
        checked = 0
        for P in map(dict, PARAM_SETS):
            got = run_host(sw.ctx, sw.g.db, sw.hs, arrays, pseudotax, P)
            same(got, sw.handles(sw.g.db, pseudotax, P, "one"), (batch, mem, pseudotax, P))
            checked += check_each(got, sw.order, pseudotax, P)
        assert checked > 300


@pytest.mark.parametrize("batch", BATCHES, ids=BATCH_IDS)
def test_only_the_batch_of_big_is_redone(sw, monkeypatch, batch):
    """one statistics launch per pass and batch, plus one more per pass for the batch of `big` (a middle one: its CSR
    redo runs after the next batch was staged), none under SYL_CONTAIN_CSR=1; so no batch is split either.  The H2D
    bytes of the call are one copy of each batch: 12 bytes per k-mer and 8 per offset (S + batches of them)."""
    for k in HOOKS:
        monkeypatch.delenv(k, raising=False)
    if batch:
        monkeypatch.setenv("SYL_SAMPLE_BATCH", batch)
    ctx, hs = sw.ctx, sw.hs
    nS = len(sw.order)
    nb = n_batches(batch, nS)
    assert batch is None or 0 < sw.order.index("big") // int(batch) < nb - 1
    ctx.enable_timing()
    try:
        for csr in (False, True):
            if csr:
                monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
            for pseudotax in (False, True):
                passes = 2 if pseudotax else 1
                ctx.kernel_time("stats")
                h2d = ctx.ingest_stats()[0]
                run_host(ctx, sw.g.db, hs, sw.arrays("pageable"), pseudotax, {})
                assert ctx.ingest_stats()[0] - h2d == 12 * len(hs["hashes"]) + 8 * (nS + nb)
                _, n = ctx.kernel_time("stats")
                assert n == passes * (nb + (0 if csr else 1)), (csr, pseudotax, n)
    finally:
        ctx.enable_timing(False)


@pytest.mark.parametrize("batch", ["1", None], ids=["batch1", "budget"])
def test_boot_replay_streamed(sw, formulation, monkeypatch, batch):
    """SYL_BOOT_REPLAY=1 on the replay samples (with `big` between them) streamed from host memory: rows bit-equal to
    the counter-based bootstrap's and == the oracle, every bootstrapped row replayed"""
    names = [S.REPLAY_SAMPLES[0], "big", S.REPLAY_SAMPLES[1]]
    hs = host_arrays(sw.g.w, names)
    if batch:
        monkeypatch.setenv("SYL_SAMPLE_BATCH", batch)
    P = {"minimum_ani": 0.0}
    for pseudotax in (False, True):
        base = run_host(sw.ctx, sw.g.db, hs, (hs["hashes"], hs["counts"]), pseudotax, P)
        monkeypatch.setenv("SYL_BOOT_REPLAY", "1")
        replay = run_host(sw.ctx, sw.g.db, hs, (hs["hashes"], hs["counts"]), pseudotax, P)
        monkeypatch.delenv("SYL_BOOT_REPLAY")
        same(replay, base, (batch, pseudotax))
        check_each(replay, names, pseudotax, P)
        for si, name in enumerate(names):
            if name in S.REPLAY_SAMPLES:
                want = sum(1 for _, r in S.classify(name, P) if r is not None and r["emitted"] and r["boot"] >= 50)
                assert int(replay["ci_valid"][replay["sample"] == si].sum()) == want and want >= 2


def shard_cap(d):
    """a third of the entries outside `huge`: at least three shards besides the one of `huge`'s genome, and survivor
    indexes of one or two samples"""
    n = int(d["kmer_off"][-1] + d["tracked_off"][-1])
    return (n - (2**20 + 1)) // 3


@pytest.mark.parametrize("batch", ["3", "5"])
def test_scripted_rows_streamed_over_shards(sw, formulation, monkeypatch, batch):
    """the scripted world over db shards: rows bit-equal to the one-index handle path, profile rows == the oracle.
    At 3 samples per batch the survivor batches (one or two samples each) are staged again, into the slot the last
    join did not use; at 5 both plan batches are still in the slots, so each survivor batch is found there."""
    monkeypatch.setenv("SYL_SAMPLE_BATCH", batch)
    ctx, d = sw.ctx, sw.g.d
    sh = ctx.db_shards(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=1,
                       max_entries=shard_cap(d))
    try:
        assert len(sh) >= 4
        for pseudotax in (False, True):
            for P in map(dict, PARAM_SETS):
                got = run_host(ctx, sh, sw.hs, (sw.hs["hashes"], sw.hs["counts"]), pseudotax, P)
                same(got, sw.handles(sw.g.db, pseudotax, P, "one"), (batch, pseudotax, P))
                if pseudotax:
                    check_each(got, sw.order, pseudotax, P)
    finally:
        sh.free()


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s_k%d_%d" % (p[0], p[1], p[2][1]))
def test_near_tied_pairs_streamed_over_shards(ctx, formulation, monkeypatch, pair):
    """the ANI near-tie pairs, one genome per shard, with the pair's sample between two empty samples at one sample per
    batch: the pass-2 winner, kmers_lost and the abundances == the one-index handle path and the oracle"""
    from oracle import oracle as O
    from sylph_b200.api import contain_params
    monkeypatch.setenv("SYL_SAMPLE_BATCH", "1")
    _, k, a, b = pair
    case = T.Case([a, b], shared=3)
    d = case.db
    db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], k=k, c=1)
    sh = shards_of(ctx, d, "per_genome", k=k)
    smp = ctx.upload_sample(case.hash, case.count, k=k, c=1)
    n = len(case.hash)
    off = np.array([0, 0, n, n], np.uint64)
    try:
        for pseudotax in (False, True):
            p = contain_params(k=k, pseudotax=pseudotax, minimum_ani=0.0)
            want = ctx.profile(db, [smp], p) if pseudotax else ctx.query(db, [smp], p)
            fn = ctx.profile_host_samples if pseudotax else ctx.query_host_samples
            got = fn(sh, case.hash, case.count, off, 1, 150.0, p)
            assert (got["sample"] == 1).all()
            got["sample"] = 0
            same(got, want, (pair, pseudotax))
            if pseudotax:
                exp = O.contain_sample(cr_params(k=k, pseudotax=True, minimum_ani=0.0), d["kmers"], d["kmer_off"],
                                       d["tracked"], d["tracked_off"], d["gn_size"], O.Sample(case.hash, case.count))
                compare(got, exp, True)
                assert sorted(int(x) for x in got["kmers_lost"]) == [0, 3]
    finally:
        smp.free()
        sh.free()
        db.free()


# ---- segment-sort regimes ---------------------------------------------------------------------------------------

def regime_world(seed=21):
    """40 genomes (c = 1, keys over [0, 2^64 - 2], key 0 in genome 0 and 2^64 - 2 in genome 1) and 640 samples: every
    size 0..400, 233 more sizes drawn below 400 and 2 each of 10^3, 10^4 and 10^5; keys are hits from random genomes,
    shared keys of a common pool and misses; counts 1-40"""
    rng = np.random.default_rng(seed)
    G = 40
    ks = [np.unique(rng.integers(1, S.MAX_KEY, int(n), dtype=np.uint64)) for n in rng.integers(200, 3000, G)]
    ks[0] = np.unique(np.concatenate([ks[0], [0]]).astype(np.uint64))
    ks[1] = np.unique(np.concatenate([ks[1], [S.MAX_KEY]]).astype(np.uint64))
    ts = [rng.choice(ks[(g + 1) % G], 20) if g % 3 == 0 else np.zeros(0, np.uint64) for g in range(G)]
    d = dict(kmers=np.concatenate(ks), kmer_off=np.concatenate([[0], np.cumsum([len(x) for x in ks])]).astype(np.uint64),
             tracked=np.concatenate(ts).astype(np.uint64),
             tracked_off=np.concatenate([[0], np.cumsum([len(x) for x in ts])]).astype(np.uint64),
             gn_size=rng.integers(10**6, 10**7, G).astype(np.uint64))
    pool = np.unique(rng.integers(1, S.MAX_KEY, 3000, dtype=np.uint64))
    sizes = list(range(401)) + rng.integers(0, 400, 233).tolist() + [1000, 1000, 10**4, 10**4, 10**5, 10**5]
    sizes = [sizes[i] for i in rng.permutation(len(sizes))]
    samples = []
    for i, n in enumerate(sizes):
        genomes = rng.choice(G, 3, replace=False)
        parts = [ks[g][rng.random(len(ks[g])) < 0.6] for g in genomes] + [rng.choice(pool, min(n, 40))]
        parts.append(rng.integers(1, S.MAX_KEY, n, dtype=np.uint64))
        if i % 7 == 0:
            parts.append(np.array([0, S.MAX_KEY], np.uint64))
        h = np.unique(np.concatenate(parts).astype(np.uint64))
        h = h[rng.permutation(len(h))][:n]
        samples.append((h, rng.integers(1, 41, len(h)).astype(np.uint32)))
    return d, samples


def ordered(samples, how):
    out = []
    for h, c in samples:
        p = {"shuffled": np.random.default_rng(len(h)).permutation(len(h)), "sorted": np.argsort(h, kind="stable"),
             "reversed": np.argsort(h, kind="stable")[::-1]}[how]
        out.append((h[p], c[p]))
    return out


def pack(samples):
    off = np.concatenate([[0], np.cumsum([len(h) for h, _ in samples])]).astype(np.uint64)
    H = np.concatenate([h for h, _ in samples]).astype(np.uint64) if samples else np.zeros(0, np.uint64)
    C_ = np.concatenate([c for _, c in samples]).astype(np.uint32) if samples else np.zeros(0, np.uint32)
    return H, C_, off


REGIME_PLAIN = r"""
import sys
import numpy as np
import sylph_b200
from sylph_b200.api import contain_params
from tests.test_sample_stream_scripts_gpu import ordered, pack, regime_world
d, samples = regime_world()
ctx = sylph_b200.Context(0)
db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=1)
H, C, off = pack(ordered(samples, "reversed"))
for pseudotax in (False, True):
    fn = ctx.profile_host_samples if pseudotax else ctx.query_host_samples
    np.save(sys.argv[1] + "_%d.npy" % pseudotax, fn(db, H, C, off, 1, 150.0, contain_params(pseudotax=pseudotax, minimum_ani=0.0)))
ctx.close()
"""


@pytest.fixture(scope="module")
def regime(ctx):
    d, samples = regime_world()
    db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=1)
    handles = [ctx.upload_sample(h, c, c=1) for h, c in samples]
    for s in handles:
        s.mean_read_length = 150.0
    yield d, samples, db, handles
    for s in handles:
        s.free()
    db.free()


def test_segment_sort_regimes(ctx, regime, monkeypatch, tmp_path):
    """640 samples in one batch (small, medium and large segments of the segmented sort), fed shuffled, sorted and
    reversed: rows == the handle path, == a child process under SYL_JOIN_PLAIN=1, and a stratified subset == the
    oracle; the call's H2D bytes are one copy of the batch"""
    from oracle import oracle as O
    from sylph_b200.api import contain_params
    from tests.contain_compare import sort_query_rows
    for k in HOOKS:
        monkeypatch.delenv(k, raising=False)
    d, samples, db, handles = regime
    nS = len(samples)
    assert nS >= 600 and sum(1 for h, _ in samples if len(h) <= 400) >= 600
    assert sum(len(h) == 0 for h, _ in samples) >= 1 and max(len(h) for h, _ in samples) == 10**5
    want = {}
    for pseudotax in (False, True):
        p = contain_params(pseudotax=pseudotax, minimum_ani=0.0)
        want[pseudotax] = ctx.profile(db, handles, p) if pseudotax else ctx.query(db, handles, p)
        assert len(set(want[pseudotax]["sample"].tolist())) > 500
    for how in ("shuffled", "sorted", "reversed"):
        H, C_, off = pack(ordered(samples, how))
        for pseudotax in (False, True):
            p = contain_params(pseudotax=pseudotax, minimum_ani=0.0)
            fn = ctx.profile_host_samples if pseudotax else ctx.query_host_samples
            h2d = ctx.ingest_stats()[0]
            got = fn(db, H, C_, off, 1, 150.0, p)
            assert ctx.ingest_stats()[0] - h2d == 12 * len(H) + 8 * (nS + 1), how
            same(got, want[pseudotax], (how, pseudotax))
    out = str(tmp_path / "plain")
    r = subprocess.run([sys.executable, "-c", REGIME_PLAIN, out], cwd=ROOT, env=dict(os.environ, SYL_JOIN_PLAIN="1"),
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    by_size = sorted(range(nS), key=lambda i: len(samples[i][0]))
    subset = sorted(set(by_size[::40] + by_size[-6:]))
    for pseudotax in (False, True):
        same(np.load(out + "_%d.npy" % pseudotax), want[pseudotax], ("plain", pseudotax))
        rows = want[pseudotax]
        for i in subset:
            sub = rows[rows["sample"] == i].copy()
            sub["sample"] = 0
            if not pseudotax:
                sub = sort_query_rows(sub)
            exp = O.contain_sample(cr_params(pseudotax=pseudotax, minimum_ani=0.0), d["kmers"], d["kmer_off"],
                                   d["tracked"], d["tracked_off"], d["gn_size"], O.Sample(*samples[i]))
            compare(sub, exp, pseudotax)


def test_empty_samples(ctx, regime, monkeypatch):
    """a call of only empty samples (no rows, one copy of its offsets), and a batch of only empty samples between
    non-empty ones (three per batch): rows == the handle path"""
    from sylph_b200.api import contain_params
    for k in HOOKS:
        monkeypatch.delenv(k, raising=False)
    d, samples, db, handles = regime
    big = [i for i, (h, _) in enumerate(samples) if 50 <= len(h) <= 400][:6]
    empty = [i for i, (h, _) in enumerate(samples) if len(h) == 0]
    e = np.zeros(0, np.uint64)
    for pseudotax in (False, True):
        p = contain_params(pseudotax=pseudotax, minimum_ani=0.0)
        fn = ctx.profile_host_samples if pseudotax else ctx.query_host_samples
        h2d = ctx.ingest_stats()[0]
        assert len(fn(db, e, np.zeros(0, np.uint32), np.zeros(6, np.uint64), 1, 150.0, p)) == 0
        assert ctx.ingest_stats()[0] - h2d == 8 * (5 + 1)
        monkeypatch.setenv("SYL_SAMPLE_BATCH", "3")
        idx = big[:3] + [empty[0]] * 3 + big[3:]
        H, C_, off = pack([samples[i] for i in idx])
        got = fn(db, H, C_, off, 1, 150.0, p)
        monkeypatch.delenv("SYL_SAMPLE_BATCH")
        hl = [handles[i] for i in idx]
        want = ctx.profile(db, hl, p) if pseudotax else ctx.query(db, hl, p)
        same(got, want, pseudotax)
        assert set(got["sample"].tolist()) == {0, 1, 2, 6, 7, 8}


# ---- memory bound -----------------------------------------------------------------------------------------------

MEM_G, MEM_CORE, MEM_N, MEM_MISS, MEM_B = 600, 2000, 1800, 2100, 16 << 20


def memory_world(deep=False, seed=31):
    """MEM_G genomes sharing a core of MEM_CORE k-mers (each keeps 98 % of it, plus 10 of its own); samples of MEM_N
    core k-mers and MEM_MISS misses, count 3 (deep: one count of 300 per sample), 4 x MEM_B bytes of them in all"""
    rng = np.random.default_rng(seed)
    hi = (2**64 - 1) // 200
    core = np.unique(rng.integers(0, hi, MEM_CORE, dtype=np.uint64))
    ks = [np.unique(np.concatenate([core[rng.random(len(core)) < 0.98], rng.integers(0, hi, 10, dtype=np.uint64)]))
          for _ in range(MEM_G)]
    d = dict(kmers=np.concatenate(ks), kmer_off=np.concatenate([[0], np.cumsum([len(x) for x in ks])]).astype(np.uint64),
             tracked=np.zeros(0, np.uint64), tracked_off=np.zeros(MEM_G + 1, np.uint64),
             gn_size=rng.integers(10**6, 10**7, MEM_G).astype(np.uint64))
    nS = -(-4 * MEM_B // (12 * (MEM_N + MEM_MISS)))
    hs, cs = [], []
    for _ in range(nS):
        h = np.concatenate([rng.choice(core, MEM_N, replace=False), rng.integers(0, hi, MEM_MISS, dtype=np.uint64)])
        c = np.full(len(h), 3, np.uint32)
        if deep:
            c[0] = 300   # a core k-mer
        p = rng.permutation(len(h))
        hs.append(h[p])
        cs.append(c[p])
    return d, hs, cs


MEMORY_SCRIPT = r"""
import json, sys
import numpy as np
import sylph_b200
from sylph_b200 import _lib
from sylph_b200.api import SylphError, contain_params
from tests.test_sample_stream_scripts_gpu import MEM_B, memory_world
case, out = sys.argv[1], sys.argv[2]
d, hs, cs = memory_world(deep=case == "deep")
H, C = np.concatenate(hs), np.concatenate(cs)
off = np.concatenate([[0], np.cumsum([len(h) for h in hs])]).astype(np.uint64)
ctx = sylph_b200.Context(0)
db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200)
ctx.set_sample_memory(MEM_B)
res = {}
for pseudotax in (False, True):
    fn = ctx.profile_host_samples if pseudotax else ctx.query_host_samples
    held0, _ = ctx.device_bytes(reset_peak=True)
    print("CALL", pseudotax, file=sys.stderr, flush=True)
    rows = fn(db, H, C, off, 200, 150.0, contain_params(pseudotax=pseudotax))
    res[str(pseudotax)] = dict(peak=ctx.device_bytes()[1] - held0, held=held0, ring=ctx.ingest_ring_bytes()[0])
    np.save(out + "_%d.npy" % pseudotax, rows)
if case == "csr":   # one sample whose hit values alone pass a budget that its plan fits
    u, n = np.unique(d["kmers"], return_counts=True)
    one = u[n > len(d["kmer_off"]) // 2]   # the core
    ctx.set_sample_memory(5 << 20)
    try:
        ctx.profile_host_samples(db, one, np.full(len(one), 3, np.uint32), np.array([0, len(one)], np.uint64), 200, 150.0)
        res["oom"] = "no error"
    except SylphError as e:
        res["oom"] = [e.code, str(e)]
print("RESULT " + json.dumps(res), flush=True)
db.free()
ctx.close()
"""

MEMORY_CASES = {"csr": {"SYL_CONTAIN_CSR": "1"}, "deep": {}, "rows": {}}


@pytest.mark.parametrize("case", list(MEMORY_CASES))
def test_device_memory_bounded_when_joins_outgrow_the_plan(ctx, monkeypatch, case, tmp_path):
    """600 genomes sharing a core, samples of 4 x the 16 MB budget drawn from it: (csr) under SYL_CONTAIN_CSR=1 and
    (deep) with one count of 300 per sample, the CSR hit values (4 bytes per hit) pass the budget, so batches are split
    in halves ([join split] lines); (rows) each sample has 600 rows, past the plan's 96.  The call's peak above what the
    ctx held stays within the budget plus the staging ring, and the rows equal the handle path's and, for two samples,
    the oracle's.  (csr) also: a sample whose hit values alone pass a budget its plan fits is SYL_ERR_OOM, naming its
    bytes."""
    from oracle import oracle as O
    from sylph_b200 import _lib
    from sylph_b200.api import contain_params
    from tests.contain_compare import sort_query_rows
    for k in HOOKS:
        monkeypatch.delenv(k, raising=False)
    d, hs, cs = memory_world(deep=case == "deep")
    assert sum(12 * len(h) for h in hs) >= 4 * MEM_B
    # the joins' bytes the plan does not charge: 4 per hit in the CSR formulation, ROW_BYTES per row past 96 per sample
    u, n = np.unique(d["kmers"], return_counts=True)
    allh = np.concatenate(hs)
    i = np.minimum(np.searchsorted(u, allh), len(u) - 1)
    hits = int(n[i][u[i] == allh].sum())
    unplanned = 4 * hits if case != "rows" else len(hs) * (MEM_G - 96) * row_bytes()
    assert unplanned > 8 * MEM_B, unplanned
    env = dict(os.environ, SYL_DEBUG_TIMING="1", PYTHONPATH=ROOT, **MEMORY_CASES[case])
    out = str(tmp_path / "rows")
    r = subprocess.run([sys.executable, "-c", MEMORY_SCRIPT, case, out], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads(next(x for x in r.stdout.splitlines() if x.startswith("RESULT "))[7:])
    splits = [log.count("[join split]") for log in r.stderr.split("CALL")[1:]]
    print("memory", case, "unplanned", unplanned, "budget", MEM_B, "splits", splits, res)
    for pseudotax, k in zip((False, True), splits):
        m = res[str(pseudotax)]
        assert m["peak"] <= MEM_B + m["ring"], (case, pseudotax, m)
        assert k >= 1 or case == "rows", (case, pseudotax)
    if case == "csr":
        code, msg = res["oom"]
        assert code == _lib.SYL_ERR_OOM and "sample 0 needs" in msg and "the budget is 5242880" in msg, msg
    for k, v in MEMORY_CASES[case].items():
        monkeypatch.setenv(k, v)
    handles = [ctx.upload_sample(h, c, c=200) for h, c in zip(hs, cs)]
    db = ctx.build_db_arrays(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=200)
    try:
        for s in handles:
            s.mean_read_length = 150.0
        for pseudotax in (False, True):
            p = contain_params(pseudotax=pseudotax)
            want = ctx.profile(db, handles, p) if pseudotax else ctx.query(db, handles, p)
            same(np.load(out + "_%d.npy" % pseudotax), want, (case, pseudotax))
            if not pseudotax:
                assert len(want) == len(hs) * MEM_G
            for i in (0, len(hs) // 2):
                sub = want[want["sample"] == i].copy()
                sub["sample"] = 0
                if not pseudotax:
                    sub = sort_query_rows(sub)
                exp = O.contain_sample(cr_params(pseudotax=pseudotax), d["kmers"], d["kmer_off"], d["tracked"],
                                       d["tracked_off"], d["gn_size"], O.Sample(hs[i], cs[i]))
                compare(sub, exp, pseudotax)
    finally:
        for s in handles:
            s.free()
        db.free()
