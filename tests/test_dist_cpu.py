"""CPU suite: the N>1 host logic (sharding, variable-length all-gather, row merge, survivor-db
gather) over gloo with world_size 2 and 3.  Compute kernels are not involved (no GPU here)."""
import os
import socket

import numpy as np
import pytest


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sylph_b200 import dist as D
    from sylph_b200.api import ANI_ROW_DTYPE
    try:
        # 1. variable-length all-gather (rank r contributes r*3+1 rows; rank 1 of 2 also tests empty->nonempty mix)
        rows = np.zeros(rank * 3 + (0 if rank == 0 else 1), dtype=ANI_ROW_DTYPE)
        rows["sample"] = np.arange(len(rows)) % 2
        rows["genome"] = 1000 * rank + np.arange(len(rows))[::-1]
        rows["final_est_ani"] = 0.9 + 0.01 * rank
        parts = D.all_gather_bytes(rows)
        assert [len(p) for p in parts] == [r * 3 + (0 if r == 0 else 1) for r in range(world)]
        merged = D.merge_rows(parts)
        key = list(zip(merged["sample"].tolist(), merged["genome"].tolist()))
        assert key == sorted(key) and len(merged) == sum(len(p) for p in parts)
        # 2. survivor-db gather: each rank owns 2 genomes with rank-dependent sizes
        nk = [3 + rank, 1 + 2 * rank]
        sub = {"kmers": np.arange(sum(nk), dtype=np.uint64) + 100 * rank,
               "kmer_off": np.array([0, nk[0], sum(nk)], dtype=np.uint64),
               "tracked": np.arange(rank + 1, dtype=np.uint64) + 7000 * rank,
               "tracked_off": np.array([0, rank + 1, rank + 1], dtype=np.uint64),
               "gn_size": np.array([10 + rank, 20 + rank], dtype=np.uint64)}
        gid = np.array([50 * rank + 1, 50 * rank + 9], dtype=np.uint64)
        m, ids = D.gather_survivor_genomes(sub, gid)
        e_ids, e_koff, e_toff, e_km, e_gn = [], [0], [0], [], []
        for r in range(world):  # what the concatenation in rank order must look like
            e_ids += [50 * r + 1, 50 * r + 9]
            e_koff += [e_koff[-1] + 3 + r, e_koff[-1] + 3 + r + 1 + 2 * r]
            e_toff += [e_toff[-1] + r + 1, e_toff[-1] + r + 1]
            e_km += list(range(100 * r, 100 * r + 4 + 3 * r))
            e_gn += [10 + r, 20 + r]
        assert ids.tolist() == e_ids
        assert m["kmer_off"].tolist() == e_koff
        assert m["tracked_off"].tolist() == e_toff
        assert m["kmers"].tolist() == e_km
        assert m["gn_size"].tolist() == e_gn
        if world == 2:  # literal pins
            assert ids.tolist() == [1, 9, 51, 59] and m["kmer_off"].tolist() == [0, 3, 4, 8, 11]
            assert m["kmers"].tolist() == [0, 1, 2, 3, 100, 101, 102, 103, 104, 105, 106]
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_shard_range():
    from sylph_b200.dist import shard_range
    for n in (0, 1, 7, 8, 100000, 113104):
        for w in (1, 2, 3, 8):
            r = [shard_range(n, i, w) for i in range(w)]
            assert r[0][0] == 0 and r[-1][1] == n
            assert all(r[i][1] == r[i + 1][0] for i in range(w - 1))
            sizes = [b - a for a, b in r]
            assert max(sizes) - min(sizes) <= 1


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_gather_and_merge(world):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(r, "ok") for r in range(world)], res


class _FakeJob:
    """Stand-in for api.ProfileJob on CPU tensors: records the order of the stages and checks, stage by stage, that the
    collective before it delivered every rank's contribution (what the library's kernels rely on)."""

    def __init__(self, ctx, rows_per_rank, csr):
        import torch
        self.ctx, self.R, self.csr = ctx, rows_per_rank if rows_per_rank else 4, csr
        w, r = ctx.world, ctx.rank
        self.b = dict(table1=torch.full((8,), 10 + r, dtype=torch.uint8), gathered1=torch.zeros(8 * w, dtype=torch.uint8),
                      winner=torch.full((5,), 1000, dtype=torch.int32), table2=torch.zeros(8, dtype=torch.uint8),
                      gathered2=torch.zeros(8 * w, dtype=torch.uint8))
        ctx.log.append("begin(R=%d, csr=%d)" % (self.R, self.csr))

    def buffers(self):
        return self.b

    def rank(self):
        w, r = self.ctx.world, self.ctx.rank
        assert self.b["gathered1"].view(w, 8)[:, 0].tolist() == [10 + i for i in range(w)]   # every rank's pass-1 table
        self.b["winner"][:] = 1000
        self.b["winner"][r % 5] = 7 + r          # this shard's best order for "its" keys
        self.ctx.log.append("rank")

    def pass2(self):
        w = self.ctx.world
        want = [1000] * 5
        for i in range(w):
            want[i % 5] = min(want[i % 5], 7 + i)
        assert self.b["winner"].tolist() == want                                             # MIN over the shards
        self.b["table2"][:] = 50 + self.ctx.rank
        self.ctx.log.append("pass2")

    def finish(self):
        from sylph_b200 import _lib
        from sylph_b200.api import ANI_ROW_DTYPE
        w = self.ctx.world
        assert self.b["gathered2"].view(w, 8)[:, 0].tolist() == [50 + i for i in range(w)]   # every rank's pass-2 table
        self.ctx.log.append("finish")
        if self.ctx.mode == "unsupported" and not self.csr:     # a count >= 256 in the histogram formulation
            return None, _lib.SYL_ERR_UNSUPPORTED, 0
        if self.R < 300:                                   # same verdict on every rank (the headers were gathered)
            return None, _lib.SYL_ERR_CAPACITY, 300
        rows = np.zeros(w, dtype=ANI_ROW_DTYPE)
        rows["genome"] = np.arange(w)
        return rows, _lib.SYL_OK, 0

    def free(self):
        self.ctx.log.append("free")


class _FakeCtx:
    def __init__(self, rank, world, mode):
        self.rank, self.world, self.mode, self.log, self._stream = rank, world, mode, [], 0

    def profile_shard_begin(self, db, samples, params, world, rank, rows_per_rank, csr):
        assert (world, rank) == (self.world, self.rank)
        return _FakeJob(self, rows_per_rank, csr)

    def sync(self):
        pass


def _worker_profile(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sylph_b200 import dist as D
    try:
        # 1. an undersized row table: every rank retries once with the size the gathered headers ask for
        ctx = _FakeCtx(rank, world, "ok")
        rows = D.profile_sharded(ctx, None, None, [], 0, params=object())
        assert len(rows) == world
        stage = ["rank", "pass2", "finish", "free"]
        assert ctx.log == ["begin(R=4, csr=0)"] + stage + ["begin(R=556, csr=0)"] + stage, ctx.log
        # 2. the >= 256-count case: every rank redoes the job in the CSR formulation, through the same collectives,
        #    and keeps that formulation for the row-table retry that follows
        ctx = _FakeCtx(rank, world, "unsupported")
        rows = D.profile_sharded(ctx, None, None, [], 0, params=object())
        assert len(rows) == world
        assert ctx.log == (["begin(R=4, csr=0)"] + stage + ["begin(R=4, csr=1)"] + stage + ["begin(R=556, csr=1)"] + stage), ctx.log
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_profile_sharded_control_flow(world):
    """The three collectives of the sharded profile sit between the library's stages in the right order, move every
    rank's table / the minimum of the winner orders, and all ranks take the same retry decisions (a larger row table, the
    CSR formulation)."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_profile, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(r, "ok") for r in range(world)], res
