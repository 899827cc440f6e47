"""GPU parity: paired-end sample sketch with the exact pair set (sketch_pair_sequences, --fpr 0; src/sketch.rs:771-895)."""
import os

import numpy as np
import pytest

from tests.test_oracle_cpu import make_pairs, rand_seq
from tests.util import DATA, flatten, read_fastx

pytestmark = pytest.mark.gpu


def check_pairs(ctx, r1, r2, device=False, **kw):
    from oracle import oracle as O
    b1, o1 = flatten(r1)
    b2, o2 = flatten(r2)
    eh, ec, emean, end = O.sketch_read_pairs(b1, o1, b2, o2, **kw)
    if device:
        import torch
        t = lambda a, dt: torch.from_numpy(a.astype(dt) if a.dtype != dt else a).cuda()
        s = ctx.sketch_pair_sequences(t(b1, np.uint8), t(o1, np.int64), t(b2, np.uint8), t(o2, np.int64), **kw)
    else:
        s = ctx.sketch_pair_sequences(b1, o1, b2, o2, **kw)
    h, c = s.download()
    assert np.array_equal(h, eh) and np.array_equal(c, ec)
    assert s.num_dup_removed == end
    assert abs(s.mean_read_length - emean) <= 1e-9 * max(1.0, emean)
    return len(h), end


def test_k12_pairs_fixture(ctx):
    r1 = [s for _, s in read_fastx(os.path.join(DATA, "k12_R1.fq"))]
    r2 = [s for _, s in read_fastx(os.path.join(DATA, "k12_R2.fq"))]
    n, _ = check_pairs(ctx, r1, r2, c=20)
    assert n == 9916
    check_pairs(ctx, r1, r2, c=200)
    check_pairs(ctx, r1, r2[:-7], c=20)        # unequal files: pairs = records zipped


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("no_dedup", [False, True])
def test_synthetic_pairs_with_duplicates(ctx, device, no_dedup):
    """duplicate pairs, pairs with the same mate 1 only (no key in common), overlapping mates (k-mer in both mates:
    counted once), mates < 33 bp (no key), one k-mer with hundreds of events (dedup set far beyond 4: no
    MAX_DEDUP_COUNT for pairs)"""
    rng = np.random.default_rng(31)
    genome = rand_seq(rng, 30000, b"ACGT")
    r1, r2 = make_pairs(rng, 4000, genome)
    hot = genome[1000:1150]
    for i in range(300):                       # deep k-mers: same mate 1, varying mate 2
        r1.append(hot)
        r2.append(genome[2000 + (i % 37) * 50:2150 + (i % 37) * 50])
    r1 += [b"A" * 150, b"A" * 150, b"", b"ACGTN" * 30]
    r2 += [b"A" * 150, b"A" * 150, b"ACGT" * 20, b"acgtn" * 30]
    order = rng.permutation(len(r1))
    r1, r2 = [r1[i] for i in order], [r2[i] for i in order]
    n, nd = check_pairs(ctx, r1, r2, device=device, c=5, no_dedup=no_dedup)
    if not no_dedup:
        assert nd > 2000
    else:
        assert nd == 0


def test_pairs_k21_scalar(ctx):
    rng = np.random.default_rng(32)
    genome = rand_seq(rng, 20000, b"ACGT")
    r1, r2 = make_pairs(rng, 1500, genome)
    check_pairs(ctx, r1, r2, k=21, c=9, sem=0)
