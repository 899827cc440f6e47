"""GPU parity: read sketches whose post-pass group slots overflow on an ordinary sample.

SYL_GROUP_CAP shrinks every group's slot, so the events the seeding kernel flushes past it land in the
overflow list and their groups take the generic path.  The library reads the variable once per process,
hence the subprocess."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import numpy as np
import sylph_b200
from sylph_b200 import synth
from oracle import oracle as O
ctx = sylph_b200.Context(0)
b, o = synth.reads(40000, n_comm=4, genome_len=200000)
b, o = b.numpy(), o.numpy().astype(np.uint64)
db, do = synth.reads(40000, n_comm=4, genome_len=200000, device="cuda")
src = (b, o) if SOURCE == "host" else (db, do)  # host memory: packed ingest, 2-bit k_seed; device memory: ASCII k_seed
for k, c in ((31, 200), (21, 50)):
    eh, ec, _, nd = O.sketch_reads(b, o, k=k, c=c)
    s = ctx.sketch_sequences(*src, k=k, c=c)
    h, cnt = s.download()
    assert len(h) > 1000 and np.array_equal(h, eh) and np.array_equal(cnt, ec), (k, c, len(h), len(eh))
    assert s.num_dup_removed == nd, (s.num_dup_removed, nd)
    s.free()
# scripted duplicate-removal histories (tests/dedup_scripts.py): every in-kernel replay, every fallback
import torch
from tests import dedup_scripts as D
for name in D.SAMPLES:
    b, o = D.single_sample(name, c=10).flat()
    eh, ec, _, nd = O.sketch_reads(b, o, k=31, c=10)
    src = (b, o) if SOURCE == "host" else (torch.from_numpy(b).cuda(), torch.from_numpy(o.view(np.int64)).cuda())
    s = ctx.sketch_sequences(*src, k=31, c=10)
    h, cnt = s.download()
    assert np.array_equal(h, eh) and np.array_equal(cnt, ec), name
    assert s.num_dup_removed == nd, (name, s.num_dup_removed, nd)
    s.free()
print("ok")
"""


# 32: nearly every group overflows; 700: just above the expected group size, so in-kernel groups and
# overflowing groups alternate along the hash range and the generic path's pairs are slotted between them
@pytest.mark.parametrize("source", ["host", "device"])
@pytest.mark.parametrize("group_cap", ["32", "700"])
def test_reads_overflowing_group_slots(source, group_cap):
    env = dict(os.environ, SYL_GROUP_CAP=group_cap)
    r = subprocess.run([sys.executable, "-c", "SOURCE = %r\n" % source + SCRIPT], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
