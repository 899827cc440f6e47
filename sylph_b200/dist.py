"""Multi-GPU host logic: one process per GPU over torch.distributed (NCCL on GPUs, gloo in the
CPU tests).  The path shards naturally:

  sketching : independent samples / genome batches per rank, no collective
  query     : db sharded by genome (syl_db_build(genome_base=...)), samples replicated, every rank
              emits its rows; ONE all-gather of the row tables at the end (the only collective)
  profile   : profile_sharded — three fixed-size collectives between the library's compute stages, all
              enqueued on one stream with no host synchronisation in between (include/sylph_b200.h (5)):
                pass 1 per shard -> all_gather of the per-rank row tables
                order of the survivors + per-key local winner -> all_reduce(MIN) of the winner array
                pass 2 per shard + bootstrap -> all_gather of the pass-2 row tables -> host finish
              every rank picks its own join formulation; a k-mer count >= 256 makes every rank redo the job
              in the CSR formulation.
  sketches  : gather_survivor_genomes (with all_gather_bytes / all_gather_device) gathers genome sketches of
              every rank into one database, identical on every rank; bench.py's multi-GPU parity step gathers
              the whole database with it to compare the sharded profile with a single-GPU one.

torch is plumbing here (process group, collectives); all compute goes through the C ABI.
"""
import numpy as np

from .api import ANI_ROW_DTYPE, contain_params


def shard_range(n, rank, world):
    """Contiguous split of n units: -> (begin, end) of `rank`."""
    base, rem = divmod(n, world)
    b = rank * base + min(rank, rem)
    return b, b + base + (1 if rank < rem else 0)


def _dev():
    import torch
    import torch.distributed as dist
    return torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")


def all_gather_bytes(arr):
    """All-gather variable-length numpy arrays (any dtype): -> list of per-rank arrays (same dtype).
    Two collectives: sizes, then the payload padded to the largest size."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return [arr]
    world, dev = dist.get_world_size(), _dev()
    raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    n = torch.tensor([raw.size], dtype=torch.int64, device=dev)
    sizes = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(sizes, n)
    sizes = [int(s.item()) for s in sizes]
    mx = max(max(sizes), 1)
    buf = torch.zeros(mx, dtype=torch.uint8, device=dev)
    if raw.size:
        buf[: raw.size] = torch.from_numpy(raw.copy()).to(dev)
    out = [torch.empty(mx, dtype=torch.uint8, device=dev) for _ in range(world)]
    dist.all_gather(out, buf)
    return [o[:s].cpu().numpy().view(arr.dtype) for o, s in zip(out, sizes)]


def merge_rows(parts):
    """Concatenate per-rank row tables and order them by (sample, genome) like a single-GPU syl_query."""
    parts = [p for p in parts if len(p)]
    if not parts:
        return np.zeros(0, dtype=ANI_ROW_DTYPE)
    rows = np.concatenate(parts)
    order = np.lexsort((rows["genome"], rows["sample"]))
    return rows[order]


def query_sharded(ctx, db, samples, params=None):
    """`sylph query` over a genome-sharded db: local syl_query + one all-gather of the rows."""
    params = params or contain_params(pseudotax=False)
    local = ctx.query(db, samples, params)
    return merge_rows(all_gather_bytes(local))


def all_gather_device(t):
    """All-gather variable-length 1-D int64 CUDA tensors (NCCL): -> list of per-rank tensors."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size()
    n = torch.tensor([t.numel()], dtype=torch.int64, device=t.device)
    sizes = [torch.zeros(1, dtype=torch.int64, device=t.device) for _ in range(world)]
    dist.all_gather(sizes, n)
    sizes = [int(x.item()) for x in sizes]
    mx = max(max(sizes), 1)
    buf = torch.zeros(mx, dtype=torch.int64, device=t.device)
    buf[: t.numel()] = t
    out = [torch.empty(mx, dtype=torch.int64, device=t.device) for _ in range(world)]
    dist.all_gather(out, buf)
    return [o[:s] for o, s in zip(out, sizes)]


def _merge_csr(parts):
    """parts: per-rank dicts of arrays (numpy or torch, same kind) -> merged dict in rank order."""
    first = parts["kmers"][0]
    if type(first).__module__.startswith("torch"):
        import torch
        cat, zero = torch.cat, lambda: torch.zeros(1, dtype=torch.int64, device=first.device)
    else:
        cat, zero = np.concatenate, lambda: np.zeros(1, dtype=np.uint64)
    out = {"kmers": cat(parts["kmers"]), "tracked": cat(parts["tracked"]), "gn_size": cat(parts["gn_size"])}
    for name in ("kmer_off", "tracked_off"):
        offs, base = [zero()], 0
        for p in parts[name]:
            offs.append(p[1:] + base)
            base += int(p[-1]) if len(p) else 0
        out[name] = cat(offs)
    return out


def gather_survivor_genomes(sub, global_ids):
    """sub: this rank's pass-1 survivors as a dict of CSR arrays — numpy (gloo / tests) or torch CUDA
    int64 tensors (NCCL, stays on the device) — global_ids: their global genome ids (numpy).
    -> (merged dict, merged global ids), identical on every rank (rank order)."""
    keys = ("kmers", "kmer_off", "tracked", "tracked_off", "gn_size")
    on_device = type(sub["kmers"]).__module__.startswith("torch")
    if on_device:
        parts = {k: all_gather_device(sub[k]) for k in keys}
    else:
        parts = {k: all_gather_bytes(np.ascontiguousarray(sub[k], dtype=np.uint64)) for k in keys}
    ids = all_gather_bytes(np.ascontiguousarray(global_ids, dtype=np.uint64))
    return _merge_csr(parts), np.concatenate(ids)


def profile_sharded(ctx, genomes, db, samples, genome_base, params=None, rows_per_rank=0):
    """`sylph profile` over a genome-sharded db: three collectives (module docstring).  Returns all rows on
    every rank, per sample sorted by rel_abund descending; row.genome is the GLOBAL genome id.
    `genomes` and `genome_base` are unused; they stay because existing callers (bench.py) pass them."""
    import torch
    import torch.distributed as dist
    from . import _lib
    rank = dist.get_rank() if dist.is_initialized() else 0
    world = dist.get_world_size() if dist.is_initialized() else 1
    params = params or contain_params(pseudotax=True)
    try:
        own_stream = ctx._stream != torch.cuda.current_stream().cuda_stream   # the collectives run on torch's stream
    except Exception:   # no CUDA device: the gloo tests drive this function with a stand-in context
        own_stream = False

    def fence():
        if own_stream:
            ctx.sync()
            torch.cuda.current_stream().synchronize()

    csr = False
    for _ in range(4):   # one formulation switch + capacity retries, as in the single-GPU driver
        job = ctx.profile_shard_begin(db, samples, params, world, rank, rows_per_rank, csr)
        try:
            b = job.buffers()
            if world > 1:
                fence()
                dist.all_gather_into_tensor(b["gathered1"], b["table1"])
                fence()
            job.rank()
            if world > 1:
                fence()
                dist.all_reduce(b["winner"], op=dist.ReduceOp.MIN)
                fence()
            job.pass2()
            if world > 1:
                fence()
                dist.all_gather_into_tensor(b["gathered2"], b["table2"])
                fence()
            rows, rc, need = job.finish()
        finally:
            job.free()
        if rc == _lib.SYL_OK:
            return rows
        # every rank reaches the same verdict (the table headers were gathered)
        if rc == _lib.SYL_ERR_CAPACITY:          # redo with a larger row table
            rows_per_rank = need + 256
        elif rc == _lib.SYL_ERR_UNSUPPORTED and not csr:   # a count >= 256: redo in the CSR formulation
            csr = True
        else:
            _lib.check(rc)
    raise RuntimeError("profile_sharded: row table kept overflowing")

