"""Run under torchrun (N ranks, one GPU each): query / profile over a genome-sharded db must equal the single-GPU
result on the whole db — for the three-collective profile (dist.profile_sharded) in the formulation each rank picks
and with every rank in the CSR formulation (SYL_CONTAIN_CSR=1).  The samples' communities are spread over ALL shards.
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 scripts/dist_check.py
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sylph_b200  # noqa: E402
from sylph_b200 import dist as D  # noqa: E402
from sylph_b200 import synth  # noqa: E402
from sylph_b200.api import contain_params  # noqa: E402

INT_FIELDS = ("sample", "genome", "contain", "glen", "kmers_lost", "lambda_status", "ci_valid")
FLT_FIELDS = ("final_est_ani", "final_est_cov", "naive_ani", "mean_cov", "median_cov", "lambda", "rel_abund", "seq_abund")


def same_rows(a, b):
    if len(a) != len(b):
        return False
    ok = all(bool(np.array_equal(a[f], b[f])) for f in INT_FIELDS)
    ok &= all(bool(np.allclose(a[f], b[f], rtol=1e-9, atol=0)) for f in FLT_FIELDS)
    return ok and bool(np.allclose(a["ci"], b["ci"], rtol=1e-9, atol=0))


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ctx = sylph_b200.Context(local, stream=torch.cuda.current_stream().cuda_stream)
    ok = True
    # G = 513 with one sample: 2 ranks hold 257 and 256 genomes, where a row table sized from the shard would differ
    for G, glen, c, n_reads, n_samples in ((200, 120000, 20, 60000, 3), (96, 150000, 1000, 300000, 2), (513, 20000, 20, 30000, 1)):
        b0, b1 = D.shard_range(G, rank, world)
        bases, off = synth.db_chunk(b0, b1, glen, device="cuda")
        goff = torch.arange(b1 - b0 + 1, dtype=torch.int64, device="cuda")
        genomes = ctx.sketch_genomes(bases, off, goff, c=c)
        db = ctx.build_db(genomes, genome_base=b0)
        samples = []
        for si in range(n_samples):
            comm = synth.community_ids(G // 2, G, seed=synth.SEED_READS + 0x10 + si)   # spans every shard
            rb, ro = synth.reads(n_reads, n_comm=G // 2, genome_len=glen, seed=synth.SEED_READS + 0x10 + si, device="cuda", comm=comm)
            samples.append(ctx.sketch_sequences(rb, ro, c=c))
        q = D.query_sharded(ctx, db, samples)
        p = D.profile_sharded(ctx, genomes, db, samples, b0)
        prev = os.environ.get("SYL_CONTAIN_CSR")
        os.environ["SYL_CONTAIN_CSR"] = "1"         # read by the library per call
        pc = D.profile_sharded(ctx, genomes, db, samples, b0)
        if prev is None:
            del os.environ["SYL_CONTAIN_CSR"]
        if rank == 0:  # single-GPU reference with the whole db
            fb, fo = synth.db_chunk(0, G, glen, device="cuda")
            fg = ctx.sketch_genomes(fb, fo, torch.arange(G + 1, dtype=torch.int64, device="cuda"), c=c)
            fdb = ctx.build_db(fg)
            q1 = ctx.query(fdb, samples, contain_params(pseudotax=False))
            p1 = ctx.profile(fdb, samples, contain_params(pseudotax=True))
            shards_hit = len(set(int(g) * world // G for g in p1["genome"]))
            for name, a, b in (("query", q, q1), ("profile (3 collectives)", p, p1), ("profile (3 collectives, CSR)", pc, p1)):
                same = same_rows(a, b)
                print("G=%d c=%d %s: sharded(%d ranks) rows=%d single rows=%d genomes from %d shards equal=%s"
                      % (G, c, name, world, len(a), len(b), shards_hit, same), flush=True)
                ok &= same and len(b) > 0
            fdb.free()
            fg.free()
        for s in samples:
            s.free()
        db.free()
        genomes.free()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
