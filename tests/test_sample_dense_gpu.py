"""GPU parity: how the read-sketch post-pass assembles its result (k_group_dedup stages every in-kernel group's uniques,
k_compact_uniq builds the exact-size sketch; sylph_b200/csrc/sample.cu, SampleBuilder::finish).

SYL_GROUP_CAP=700 (just above the expected group size): groups that fall back to the generic path sit
between groups written by the kernel, on the single-end and on the paired path, so the result is assembled from the
staged uniques and the generic path's (k_fallback_place, k_compact_uniq).
Against the CPU oracle: hashes, counts and num_dup_removed equal.  The library reads SYL_GROUP_CAP once per
process, hence the subprocess."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MIXED = r"""
import numpy as np
import torch
import sylph_b200
from sylph_b200 import synth
from oracle import oracle as O
ctx = sylph_b200.Context(0)
def cuda(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a).view(dt)).cuda()
b1, o1 = synth.reads(40000, n_comm=4, genome_len=200000)
b2, o2 = synth.reads(40000, n_comm=4, genome_len=200000, seed=synth.SEED_READS + 1000)
b1, o1, b2, o2 = b1.numpy(), o1.numpy().astype(np.uint64), b2.numpy(), o2.numpy().astype(np.uint64)
for k, c in ((31, 200), (21, 50)):
    eh, ec, _, nd = O.sketch_reads(b1, o1, k=k, c=c)
    s = ctx.sketch_sequences(cuda(b1, np.uint8), cuda(o1, np.int64), k=k, c=c)
    h, cnt = s.download()
    assert len(h) > 1000 and np.array_equal(h, eh) and np.array_equal(cnt, ec), ("reads", k, c, len(h), len(eh))
    assert s.num_dup_removed == nd, ("reads", s.num_dup_removed, nd)
    s.free()
    eh, ec, _, nd = O.sketch_read_pairs(b1, o1, b2, o2, k=k, c=c)
    s = ctx.sketch_pair_sequences(cuda(b1, np.uint8), cuda(o1, np.int64), cuda(b2, np.uint8), cuda(o2, np.int64), k=k, c=c)
    h, cnt = s.download()
    assert len(h) > 1000 and np.array_equal(h, eh) and np.array_equal(cnt, ec), ("pairs", k, c, len(h), len(eh))
    assert s.num_dup_removed == nd, ("pairs", s.num_dup_removed, nd)
    s.free()
print("ok")
"""


def test_fallback_groups_between_in_kernel_groups():
    env = dict(os.environ, SYL_GROUP_CAP="700")
    r = subprocess.run([sys.executable, "-c", MIXED], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
