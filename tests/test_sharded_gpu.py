"""GPU: the genome-sharded query and profile (sylph_b200/dist.py, include/sylph_b200.h section (5)) at 2-15 ranks on
one GPU.

Every rank is a thread with its own Context (and so its own stream), its own db shard built with
build_db(genome_base=...) and its own copies of the samples.  The rank threads call the real dist.* functions, which
drive the real library.  Inside each test, torch.distributed is replaced by an in-process group of those threads
(FakeGroup): all_gather, all_gather_into_tensor and all_reduce(MIN) put each rank's tensor in a slot, wait on a
barrier, build every rank's output from all slots with device copies, and wait again.  all_gather_into_tensor and
all_reduce assert NCCL's rule that every rank brings the same number of elements.  Backend "nccl", so the
device-tensor paths of dist.py run.

In every case all ranks return the same rows, those rows equal the single-GPU ctx.query / ctx.profile on the whole db
bit for bit in every field (the statistics come from the same integer histograms, and the bootstrap stream depends
only on the row, not on where it sits in a table), and they equal the CPU oracle."""
import os
import threading

import numpy as np
import pytest

from tests import ani_ties as T
from tests import contain_scripts as S
from tests.contain_compare import compare, cr_params, sort_query_rows
from tests.util import DATA, flatten, read_fastx

pytestmark = pytest.mark.gpu

BARRIER_TIMEOUT = 120.0
TABLE_HEADER, ROW_BYTES = 32, 144     # contain.cu ShardTable, syl_ani_row


# ---- the in-process process group -----------------------------------------------------------------------------------

class FakeGroup:
    """torch.distributed for `world` threads of one process on one GPU (see the module docstring)."""

    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=BARRIER_TIMEOUT)
        self.slots = [None] * world
        self.calls = [[] for _ in range(world)]   # per rank: (collective, elements in)
        self.local = threading.local()

    def rank(self):
        return self.local.rank

    def install(self, monkeypatch):
        import torch.distributed as dist
        fns = dict(is_available=lambda: True, is_initialized=lambda: True, get_rank=lambda *a, **k: self.rank(),
                   get_world_size=lambda *a, **k: self.world, get_backend=lambda *a, **k: "nccl",
                   all_gather=self.all_gather, all_gather_into_tensor=self.all_gather_into_tensor,
                   all_reduce=self.all_reduce)
        for name, fn in fns.items():
            monkeypatch.setattr(dist, name, fn)

    def _exchange(self, name, t):
        import torch
        self.calls[self.rank()].append((name, t.numel()))
        torch.cuda.current_stream().synchronize()
        self.slots[self.rank()] = t
        self.barrier.wait()
        return list(self.slots)

    def _done(self):
        import torch
        torch.cuda.synchronize()
        self.barrier.wait()

    def all_gather(self, out, t, *a, **k):
        ins = self._exchange("all_gather", t)
        assert len(out) == self.world
        for o, i in zip(out, ins):
            assert o.shape == i.shape and o.dtype == i.dtype, (o.shape, i.shape)
            o.copy_(i)
        self._done()

    def all_gather_into_tensor(self, out, t, *a, **k):
        ins = self._exchange("all_gather_into_tensor", t)
        sizes = [i.numel() for i in ins]
        assert sizes == [t.numel()] * self.world, "all_gather_into_tensor: ranks bring %s elements" % sizes
        assert out.numel() == self.world * t.numel() and out.dtype == t.dtype
        view = out.view(self.world, -1)
        for r, i in enumerate(ins):
            view[r].copy_(i.reshape(-1))
        self._done()

    def all_reduce(self, t, op=None, *a, **k):
        import torch
        import torch.distributed as dist
        assert op == dist.ReduceOp.MIN
        ins = self._exchange("all_reduce", t)
        sizes = [i.numel() for i in ins]
        assert sizes == [t.numel()] * self.world, "all_reduce: ranks bring %s elements" % sizes
        res = ins[0].clone()
        for i in ins[1:]:
            torch.minimum(res, i, out=res)
        torch.cuda.synchronize()
        self.barrier.wait()          # every rank has read every slot before any rank overwrites its own
        t.copy_(res)
        self._done()


def run_ranks(monkeypatch, world, fn):
    """fn(rank) on `world` threads under a FakeGroup -> ([result per rank], group).  A rank that raises breaks the
    barrier so the others fail at once; every thread is joined before this returns."""
    grp = FakeGroup(world)
    grp.install(monkeypatch)
    out, errs = [None] * world, [None] * world

    def body(r):
        grp.local.rank = r
        try:
            out[r] = fn(r)
        except BaseException as e:  # noqa: B036 - reported by the main thread
            errs[r] = e
            grp.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,), name="rank%d" % r) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    errs = [e for e in errs if e is not None]
    if errs:   # the rank that failed first, not the ones it released from the barrier
        raise next((e for e in errs if not isinstance(e, threading.BrokenBarrierError)), errs[0])
    return out, grp


# ---- ranks and their inputs ------------------------------------------------------------------------------------------

def csr_slice(d, b0, b1):
    """genomes [b0, b1) of a CSR dict (Genomes.download layout)"""
    k0, k1, t0, t1 = (int(d["kmer_off"][b0]), int(d["kmer_off"][b1]), int(d["tracked_off"][b0]), int(d["tracked_off"][b1]))
    return dict(kmers=d["kmers"][k0:k1], kmer_off=d["kmer_off"][b0:b1 + 1] - np.uint64(k0), tracked=d["tracked"][t0:t1],
                tracked_off=d["tracked_off"][b0:b1 + 1] - np.uint64(t0), gn_size=d["gn_size"][b0:b1])


def upload(ctx, d, c):
    return ctx.upload_genomes(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=c)


class SampleData:
    """A sample's sketch on the host: (hash, count), c and mean read length (for -u)."""

    def __init__(self, h, cnt, c, mrl=0.0):
        self.hc, self.c, self.mrl = (np.asarray(h, np.uint64), np.asarray(cnt, np.uint32)), c, mrl

    @staticmethod
    def of(smp, c):
        return SampleData(*smp.download(), c, smp.mean_read_length)

    def to(self, ctx):
        s = ctx.upload_sample(*self.hc, c=self.c)
        s.mean_read_length = self.mrl
        return s


class Rank:
    def __init__(self, base, end, make_genomes, samples):
        import sylph_b200
        self.base, self.end = base, end
        self.ctx = sylph_b200.Context(0)
        self.g = make_genomes(self.ctx, base, end)
        assert len(self.g) == end - base and self.g.has_tracked
        self.db = self.ctx.build_db(self.g, genome_base=base)
        self.samples = [s.to(self.ctx) for s in samples]

    def close(self):
        for s in self.samples:
            s.free()
        self.db.free()
        self.g.free()
        self.ctx.close()


class Sharded:
    """One rank per consecutive pair of `cuts`; rank r holds genomes [cuts[r], cuts[r + 1])."""

    def __init__(self, cuts, make_genomes, samples):
        self.cuts, self.world = list(cuts), len(cuts) - 1
        self.ranks = []
        try:
            for r in range(self.world):
                self.ranks.append(Rank(cuts[r], cuts[r + 1], make_genomes, samples))
        except BaseException:
            self.close()
            raise

    def close(self):
        for r in self.ranks:
            r.close()
        self.ranks = []

    def log_jobs(self):
        """Wrap every rank's profile_shard_begin: -> per rank, one dict per job (R = table rows, csr = the formulation the
        caller asked for, rc / need of finish)."""
        logs = [[] for _ in self.ranks]
        for rk, log in zip(self.ranks, logs):
            begin = rk.ctx.profile_shard_begin

            def logged(db, samples, params, world, rank, rows_per_rank, csr, _begin=begin, _log=log):
                job = _begin(db, samples, params, world, rank, rows_per_rank, csr)
                entry = {"R": (job.buffers()["table1"].numel() - TABLE_HEADER) // ROW_BYTES, "csr": csr}
                _log.append(entry)
                finish = job.finish

                def logged_finish(*fa, **fk):
                    rows, rc, need = finish(*fa, **fk)
                    entry.update(rc=rc, need=need)
                    return rows, rc, need

                job.finish = logged_finish
                return job

            rk.ctx.profile_shard_begin = logged
        return logs


def shard_cuts(n, world):
    from sylph_b200.dist import shard_range
    return [shard_range(n, r, world)[0] for r in range(world)] + [n]


# ---- running and checking ---------------------------------------------------------------------------------------------

def same(a, b, what):
    assert len(a) == len(b), (what, len(a), len(b))
    for f in a.dtype.names:
        assert a[f].tobytes() == b[f].tobytes(), (what, f)


def params(pseudotax, kw):
    from sylph_b200.api import contain_params
    return contain_params(pseudotax=pseudotax, **kw)


def run_sharded(monkeypatch, sh, kw=None, rows_per_rank=0, which=("query", "profile")):
    """The sharded calls on every rank -> {call: rows}, after checking that every rank returned the same rows."""
    from sylph_b200 import dist as D
    kw = kw or {}

    def rank_fn(r):
        rk, out = sh.ranks[r], {}
        if "query" in which:
            out["query"] = D.query_sharded(rk.ctx, rk.db, rk.samples, params(False, kw))
        if "profile" in which:
            out["profile"] = D.profile_sharded(rk.ctx, rk.g, rk.db, rk.samples, rk.base, params(True, kw), rows_per_rank)
        return out

    res, grp = run_ranks(monkeypatch, sh.world, rank_fn)
    for r in range(1, sh.world):
        for call in which:
            same(res[r][call], res[0][call], "rank %d %s" % (r, call))
    return res[0], grp


class Whole:
    """The single-GPU reference: the whole db on the session context, and the oracle."""

    def __init__(self, ctx, d, c, samples):
        self.ctx, self.d, self.samples = ctx, d, samples
        self.g = upload(ctx, d, c)
        self.db = ctx.build_db(self.g)
        self.handles = [s.to(ctx) for s in samples]

    def rows(self, call, kw=None):
        kw = kw or {}
        if call == "query":
            return self.ctx.query(self.db, self.handles, params(False, kw))
        return self.ctx.profile(self.db, self.handles, params(True, kw))

    def oracle(self, si, pseudotax, kw):
        from oracle import oracle as O
        kw = dict(kw)
        unknown = None
        if kw.pop("estimate_unknown", 0):
            unknown = O.Unknown(kw.pop("read_seq_id"), self.samples[si].mrl, self.samples[si].c)
        d = self.d
        return O.contain_sample(cr_params(pseudotax=pseudotax, **kw), d["kmers"], d["kmer_off"], d["tracked"],
                                d["tracked_off"], d["gn_size"], O.Sample(*self.samples[si].hc), unknown=unknown)

    def check(self, got, kw=None):
        """got: {call: rows} of the sharded run -> number of rows; == ctx.query / ctx.profile bit for bit, == oracle"""
        kw = kw or {}
        n = 0
        for call, rows in got.items():
            pseudotax = call != "query"
            same(rows, self.rows("query" if call == "query" else "profile", kw), call)
            for si in range(len(self.samples)):
                sub = rows[rows["sample"] == si]
                compare(sort_query_rows(sub) if not pseudotax else sub, self.oracle(si, pseudotax, kw), pseudotax)
            n = max(n, len(rows))
        return n

    def close(self):
        for s in self.handles:
            s.free()
        self.db.free()
        self.g.free()


def with_csr(values):
    """parameter sets (value, csr): every value as it is, then every value again with the id suffix -csr, where the
    test sets SYL_CONTAIN_CSR=1 and every rank runs the CSR formulation"""
    return [pytest.param(v, False, id=str(v)) for v in values] + [pytest.param(v, True, id="%s-csr" % v) for v in values]


def set_csr(monkeypatch, csr):
    if csr:
        monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
    else:
        monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)


# ---- synthetic communities spread over every shard (scripts/dist_check.py) ----------------------------------------

G_SYN, GLEN_SYN, C_SYN = 200, 50000, 20


def synth_sample(ctx, n_reads, seed, n_comm, G, glen, c):
    import torch
    from sylph_b200 import synth
    comm = synth.community_ids(n_comm, G, seed=seed)
    rb, ro = synth.reads(n_reads, n_comm=n_comm, genome_len=glen, seed=seed, device="cuda", comm=comm)
    smp = ctx.sketch_sequences(rb, ro, c=c)
    torch.cuda.synchronize()
    out = SampleData.of(smp, c)
    smp.free()
    return out


def synth_genomes(ctx, b0, b1, glen, c):
    import torch
    from sylph_b200 import synth
    bases, off = synth.db_chunk(b0, b1, glen, device="cuda")
    goff = torch.arange(b1 - b0 + 1, dtype=torch.int64, device="cuda")
    return ctx.sketch_genomes(bases, off, goff, c=c)


@pytest.fixture(scope="module")
def syn(ctx):
    from sylph_b200 import synth
    g = synth_genomes(ctx, 0, G_SYN, GLEN_SYN, C_SYN)
    d = g.download()
    g.free()
    samples = [synth_sample(ctx, 40000, synth.SEED_READS + 0x10 + si, G_SYN // 2, G_SYN, GLEN_SYN, C_SYN) for si in range(3)]
    whole = Whole(ctx, d, C_SYN, samples)
    yield whole
    whole.close()


@pytest.mark.parametrize("world,csr", with_csr([2, 3, 4, 8]))
def test_communities_over_every_shard(ctx, syn, monkeypatch, world, csr):
    """G = 200 at c = 20, three samples whose communities span every shard, shard_range splits; the shards are
    sketched by their own ranks.  The profile keeps genomes of every shard."""
    set_csr(monkeypatch, csr)
    sh = Sharded(shard_cuts(G_SYN, world), lambda c, b0, b1: synth_genomes(c, b0, b1, GLEN_SYN, C_SYN), syn.samples)
    try:
        got, grp = run_sharded(monkeypatch, sh)
    finally:
        sh.close()
    assert syn.check(got) > 100
    shards = {int(np.searchsorted(sh.cuts, g, side="right")) - 1 for g in got["profile"]["genome"]}
    assert shards == set(range(world))
    assert [n for n, _ in grp.calls[0]].count("all_reduce") == 1        # one pass of the three-collective profile


def test_mixed_formulations(ctx, syn, monkeypatch):
    """The odd ranks ask for the CSR formulation and the even ranks run the histograms: the ranks' row tables meet in
    the same collectives and give ctx.profile's rows."""
    world = 4
    sh = Sharded(shard_cuts(G_SYN, world), lambda cx, b0, b1: upload(cx, csr_slice(syn.d, b0, b1), C_SYN), syn.samples)
    logs = sh.log_jobs()
    for r in range(1, world, 2):
        begin = sh.ranks[r].ctx.profile_shard_begin
        sh.ranks[r].ctx.profile_shard_begin = lambda *a, _begin=begin: _begin(*a[:6], True)
    try:
        got, _ = run_sharded(monkeypatch, sh, which=("profile",))
    finally:
        sh.close()
    assert syn.check(got) > 20
    assert [[e["csr"] for e in lg] for lg in logs] == [[r % 2 == 1] for r in range(world)]


HIST_PAIRS = (8 << 30) // (S.COV_BINS * 4)      # the most (sample, genome) pairs whose count histograms fit 8 GB


def test_one_rank_past_the_histogram_limit(ctx, syn, monkeypatch):
    """64 samples (the `syn` ones, small ones and empty ones).  Rank 0 holds 100 `syn` genomes and enough filler genomes
    to pass the 8 GB histogram limit, rank 1 the other 100 `syn` genomes: rank 0 runs the CSR formulation, rank 1 the
    histograms, with no error and no retry.  Each filler genome has one kept and one tracked k-mer above the FracMinHash
    threshold, so no sample hits it.  The rows equal ctx.profile on the concatenated db and the oracle."""
    from sylph_b200 import _lib
    from sylph_b200 import synth
    from sylph_b200.dist import _merge_csr
    n_samples, half = 64, G_SYN // 2
    n_fill = HIST_PAIRS // n_samples + 1 - half          # rank 0: 131 073 genomes
    assert n_samples * (half + n_fill) > HIST_PAIRS >= n_samples * half
    lo = np.uint64((2**64 - 1) // C_SYN + 1)            # sample hashes stay below (2^64 - 1) / c
    fill = dict(kmers=lo + np.arange(0, 2 * n_fill, 2, dtype=np.uint64), kmer_off=np.arange(n_fill + 1, dtype=np.uint64),
                tracked=lo + np.arange(1, 2 * n_fill, 2, dtype=np.uint64), tracked_off=np.arange(n_fill + 1, dtype=np.uint64),
                gn_size=np.full(n_fill, 100000, np.uint64))
    parts = [csr_slice(syn.d, 0, half), fill, csr_slice(syn.d, half, G_SYN)]
    d = _merge_csr({k: [p[k] for p in parts] for k in fill})
    small = [synth_sample(ctx, 300, synth.SEED_READS + 0x60 + i, 10, G_SYN, GLEN_SYN, C_SYN) for i in range(5)]
    empty = SampleData(np.zeros(0, np.uint64), np.zeros(0, np.uint32), C_SYN)
    samples = syn.samples + small + [empty] * (n_samples - len(syn.samples) - len(small))
    whole = Whole(ctx, d, C_SYN, samples)
    sh = Sharded([0, half + n_fill, G_SYN + n_fill], lambda cx, b0, b1: upload(cx, csr_slice(d, b0, b1), C_SYN), samples)
    logs = sh.log_jobs()
    try:
        got, _ = run_sharded(monkeypatch, sh, which=("profile",))
        assert whole.check(got) > 20
    finally:
        sh.close()
        whole.close()
    assert [[(e["csr"], e["rc"]) for e in lg] for lg in logs] == [[(False, _lib.SYL_OK)]] * 2
    genomes = got["profile"]["genome"]
    assert (genomes < half).any() and (genomes >= half + n_fill).any() and not ((genomes >= half) & (genomes < half + n_fill)).any()


def parent_default_rows(S, G):
    """what the row table defaulted to before it stopped depending on the shard: min(S * G, 256 + 96 S), rounded up"""
    return (max(min(S * G, 256 + 96 * S), 256) + 255) // 256 * 256


@pytest.mark.parametrize("G,n_samples", [(513, 1), (257, 2)])
def test_uneven_shards_around_the_default_table_size(ctx, monkeypatch, G, n_samples):
    """shard_range over 2 ranks gives shards of (G + 1) / 2 and (G - 1) / 2 genomes, on either side of the size where a
    row table sized from the shard would grow from 256 to 512 rows: every rank must still bring tables of one size."""
    from sylph_b200 import synth
    glen, c = 20000, 20
    cuts = shard_cuts(G, 2)
    assert parent_default_rows(n_samples, cuts[1]) != parent_default_rows(n_samples, G - cuts[1])
    g = synth_genomes(ctx, 0, G, glen, c)
    d = g.download()
    g.free()
    samples = [synth_sample(ctx, 30000, synth.SEED_READS + 0x40 + si, G // 2, G, glen, c) for si in range(n_samples)]
    whole = Whole(ctx, d, c, samples)
    sh = Sharded(cuts, lambda cx, b0, b1: upload(cx, csr_slice(d, b0, b1), c), samples)
    logs = sh.log_jobs()
    try:
        got, _ = run_sharded(monkeypatch, sh)
        assert whole.check(got) > 20
    finally:
        sh.close()
        whole.close()
    assert [[e["R"] for e in lg] for lg in logs] == [[(256 + 96 * n_samples + 255) // 256 * 256]] * 2


def test_undersized_row_table_is_redone_on_every_rank(ctx, monkeypatch):
    """rows_per_rank = 256 where one shard has more than 256 pass-1 rows and the other fewer: every rank's finish
    reports SYL_ERR_CAPACITY with the same need, and every rank redoes the call once with the same table size."""
    from sylph_b200 import _lib
    rng = np.random.default_rng(0x5A4D)
    G, nk, hit = 600, 60, 340                       # genomes 0..339 are in the sample: 300 rows in shard 0, 40 in shard 1
    kmers = rng.permutation(np.unique(rng.integers(1, 2**63, size=G * nk + 1000, dtype=np.uint64)))[:G * nk]
    tracked = np.unique(rng.integers(2**63, 2**64 - 2, size=G * 3 + 100, dtype=np.uint64))[:G * 3]
    d = dict(kmers=kmers, kmer_off=np.arange(0, G * nk + 1, nk, dtype=np.uint64), tracked=tracked,
             tracked_off=np.arange(0, G * 3 + 1, 3, dtype=np.uint64), gn_size=np.full(G, 2_000_000, np.uint64) + np.arange(G, dtype=np.uint64))
    sh_keys = kmers[: hit * nk]
    counts = (3 + rng.poisson(2.0, size=len(sh_keys))).astype(np.uint32)
    samples = [SampleData(sh_keys, counts, 200)]
    whole = Whole(ctx, d, 200, samples)
    cuts = shard_cuts(G, 2)
    sh = Sharded(cuts, lambda cx, b0, b1: upload(cx, csr_slice(d, b0, b1), 200), samples)
    try:
        p1 = params(True, {"no_ci": 1})
        n1 = [len(rk.ctx.query(rk.db, rk.samples, p1)) for rk in sh.ranks]     # pass 1 of profile on each shard
        assert n1 == [300, 40]
        logs = sh.log_jobs()
        got, _ = run_sharded(monkeypatch, sh, rows_per_rank=256, which=("profile",))
        assert whole.check(got) == hit
    finally:
        sh.close()
        whole.close()
    for lg in logs:
        assert [e["R"] for e in lg] == [256, (max(n1) + 256 + 255) // 256 * 256]
        assert (lg[0]["rc"], lg[0]["need"]) == (_lib.SYL_ERR_CAPACITY, max(n1))
        assert lg[1]["rc"] == _lib.SYL_OK


# ---- empty shards ------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def ecoli(ctx):
    bufs, coffs, goff = [], [0], [0]
    for name in ("e.coli-EC590.fasta.gz", "e.coli-o157.fasta.gz", "e.coli-K12.fasta.gz"):
        for _, s in read_fastx(os.path.join(DATA, name)):
            bufs.append(s)
            coffs.append(coffs[-1] + len(s))
        goff.append(len(coffs) - 1)
    g = ctx.sketch_genomes(np.frombuffer(b"".join(bufs), dtype=np.uint8), np.array(coffs, np.uint64), np.array(goff, np.uint64))
    d = g.download()
    g.free()
    rb, ro = flatten([s for _, s in read_fastx(os.path.join(DATA, "o157_reads.fastq.gz"))])
    smp = ctx.sketch_sequences(rb, ro)
    samples = [SampleData.of(smp, 200)]
    smp.free()
    whole = Whole(ctx, d, 200, samples)
    yield whole
    whole.close()


def empty_genomes(ctx, kind, b):
    """a shard of no genome, the way scripts/dist_check.py makes one (db_chunk(b, b) sketched) or uploaded"""
    if kind == "sketch":
        return synth_genomes(ctx, b, b, 1000, 200)
    z = np.zeros(0, np.uint64)
    return ctx.upload_genomes(z, np.zeros(1, np.uint64), z, np.zeros(1, np.uint64), z, c=200)


@pytest.mark.parametrize("kind,csr", with_csr(["sketch", "upload"]))
@pytest.mark.parametrize("cuts", [[0, 1, 2, 3, 3], [0, 0, 3], [0, 3, 3], [0, 1, 1, 3]], ids=["W4", "0|3", "3|0", "1|0|2"])
def test_empty_shards(ctx, ecoli, monkeypatch, cuts, kind, csr):
    """The three config-1 E. coli genomes and o157_reads with a rank that holds no genome: that rank runs every stage
    and every collective the others run, and all ranks return the single-GPU rows."""
    set_csr(monkeypatch, csr)
    if cuts == [0, 1, 2, 3, 3]:
        assert cuts == shard_cuts(3, 4)

    def make(cx, b0, b1):
        return empty_genomes(cx, kind, b0) if b0 == b1 else upload(cx, csr_slice(ecoli.d, b0, b1), 200)

    sh = Sharded(cuts, make, ecoli.samples)
    try:
        got, grp = run_sharded(monkeypatch, sh)
    finally:
        sh.close()
    assert ecoli.check(got) == 3
    for r in range(1, sh.world):
        assert grp.calls[r] == grp.calls[0], r
    names = [n for n, _ in grp.calls[0]]
    assert names.count("all_gather_into_tensor") == 2 and names.count("all_reduce") == 1


# ---- scripted statistics (tests/contain_scripts.py) ---------------------------------------------------------------

def scripted(ctx, names, sel):
    """the scripted world restricted to the genomes `sel`, one sample holding the keys of every family in `names`"""
    w = S.world()
    d = w.db(sel)
    keys = {}
    for n in names:
        keys.update(w.samples[n])
    h = np.array(list(keys), dtype=np.uint64)
    c = np.array(list(keys.values()), dtype=np.uint32)
    p = np.random.default_rng(len(h)).permutation(len(h))
    samples = [SampleData(h[p], c[p], 1)]
    return d, samples, Whole(ctx, d, 1, samples)


def run_scripted(ctx, monkeypatch, names, sel, cuts, kws):
    """every parameter set in `kws`, in the formulation each rank picks and with SYL_CONTAIN_CSR=1"""
    d, samples, whole = scripted(ctx, names, sel)
    sh = Sharded(cuts, lambda cx, b0, b1: upload(cx, csr_slice(d, b0, b1), 1), samples)
    try:
        for csr in (False, True):
            set_csr(monkeypatch, csr)
            for kw in kws:
                got, _ = run_sharded(monkeypatch, sh, kw)
                assert whole.check(got, kw) > 0, (kw, csr)
    finally:
        sh.close()
        whole.close()


def test_scripted_winner_each_genome_alone(ctx, monkeypatch):
    """Every genome of the `winner` family on a rank of its own: the three-way ANI tie is decided across three ranks
    (the lowest global genome index wins), a tracked-only winner sits on another rank than the genome it takes k-mers
    from, and derep at floor(t * glen) counts k-mers won on another rank."""
    sel = tuple(S.world().local["winner"])
    run_scripted(ctx, monkeypatch, ["winner"], sel, list(range(len(sel) + 1)), S.params_for("winner"))


@pytest.mark.parametrize("world", [3, 4])
@pytest.mark.parametrize("name", ["probe", "suc"])
def test_scripted_shard_range(ctx, monkeypatch, name, world):
    """`probe` (equal ranges of up to 33 genomes with kept and tracked entries, spread over the shards) and `suc`
    (bootstrap success counts of exactly 50, 49 and 45) under shard_range splits of their own genomes."""
    sel = tuple(S.world().local[name])
    run_scripted(ctx, monkeypatch, [name], sel, shard_cuts(len(sel), world), S.params_for(name))


def test_scripted_big_is_redone_in_csr_on_every_rank(ctx, monkeypatch):
    """`big` (counts >= 256) on two ranks and the `median` genomes, which see no count >= 256, on a third: every rank's
    first finish returns SYL_ERR_UNSUPPORTED, every rank redoes the job with csr set and gets ctx.profile's rows.  The
    redo runs the same three collectives again and moves no sketch."""
    from sylph_b200 import _lib
    w = S.world()
    big, med = w.local["big"], w.local["median"]
    sel = tuple(big + med)
    d, samples, whole = scripted(ctx, ["big", "median"], sel)
    assert max(w.samples["median"].values()) < S.COV_BINS
    cuts = shard_cuts(len(big), 2) + [len(sel)]
    sh = Sharded(cuts, lambda cx, b0, b1: upload(cx, csr_slice(d, b0, b1), 1), samples)
    logs = sh.log_jobs()
    try:
        got, grp = run_sharded(monkeypatch, sh, which=("profile",))
        assert whole.check(got) > 5
    finally:
        sh.close()
        whole.close()
    assert [[(e["csr"], e["rc"]) for e in lg] for lg in logs] == [[(False, _lib.SYL_ERR_UNSUPPORTED), (True, _lib.SYL_OK)]] * 3
    for r in range(3):
        assert [n for n, _ in grp.calls[r]] == ["all_gather_into_tensor", "all_reduce", "all_gather_into_tensor"] * 2, r


# ---- parameters -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kw", [dict(estimate_unknown=1, read_seq_id=98.0), dict(no_ci=1), dict(minimum_ani=0.0)],
                         ids=["u98", "no_ci", "min_ani0"])
def test_parameters_at_three_ranks(ctx, syn, monkeypatch, kw):
    sh = Sharded(shard_cuts(G_SYN, 3), lambda cx, b0, b1: upload(cx, csr_slice(syn.d, b0, b1), C_SYN), syn.samples)
    try:
        got, _ = run_sharded(monkeypatch, sh, kw)
    finally:
        sh.close()
    assert syn.check(got, kw) > 100


def test_five_samples_of_unequal_size_one_call(ctx, syn, monkeypatch):
    """As test_several_samples_of_unequal_size_one_call, over three shards: an empty sample and one of 50 reads among
    five in one call (the tiled join mapping on every rank)."""
    mid = synth_sample(ctx, 15000, 0x5EED0011, 40, G_SYN, GLEN_SYN, C_SYN)
    tiny = synth_sample(ctx, 50, 0x5EED0012, 5, G_SYN, GLEN_SYN, C_SYN)
    empty = SampleData(np.zeros(0, np.uint64), np.zeros(0, np.uint32), C_SYN)
    samples = [mid, empty, syn.samples[0], tiny, mid]
    whole = Whole(ctx, syn.d, C_SYN, samples)
    sh = Sharded(shard_cuts(G_SYN, 3), lambda cx, b0, b1: upload(cx, csr_slice(syn.d, b0, b1), C_SYN), samples)
    try:
        got, _ = run_sharded(monkeypatch, sh)
        assert whole.check(got) > 40
    finally:
        sh.close()
        whole.close()
    for call, rows in got.items():
        assert set(rows["sample"].tolist()) >= {0, 2, 4}, call
        assert 1 not in set(rows["sample"].tolist()), call


@pytest.mark.parametrize("pair", [T.WINNER_PAIRS[-1], T.TIE_PAIRS[0]], ids=["adjacent", "equal"])
def test_near_tied_winner_across_two_ranks(ctx, monkeypatch, pair):
    """Two genomes whose ANIs are adjacent doubles or equal (tests/ani_ties.py), sharing hit k-mers, one per rank: the
    gathered k_rank_rows orders them like the oracle, in both genome orders."""
    k, a, b = pair
    assert k == 31
    for specs in ([a, b], [b, a]):
        case = T.Case(specs, shared=3)
        samples = [SampleData(case.hash, case.count, 1)]
        whole = Whole(ctx, case.db, 1, samples)
        sh = Sharded([0, 1, 2], lambda cx, b0, b1: upload(cx, csr_slice(case.db, b0, b1), 1), samples)
        try:
            got, _ = run_sharded(monkeypatch, sh, {"minimum_ani": 0.0})
            assert whole.check(got, {"minimum_ani": 0.0}) == 2
            assert sorted(int(x) for x in got["profile"]["kmers_lost"]) == [0, 3]
        finally:
            sh.close()
            whole.close()
