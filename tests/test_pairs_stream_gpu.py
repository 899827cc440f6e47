"""GPU parity: read pairs from host memory through the chunked feeder, and their duplicate removal in the group
post-pass (k_group_dedup<PAIRED>), against oracle.sketch_read_pairs: hashes, counts, num_dup_removed equal.

Tiny SYL_INGEST_CHUNK makes a sample dozens of pair chunks, so pairs straddle every kind of edge, under each ingest
setting; SYL_SAMPLE_POSTPASS=sort (read per call) is the generic post-pass the group path is compared with."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tests import dedup_scripts as D
from tests import pair_scripts as P
from tests.test_driver_gpu import exe, run  # noqa: F401 (exe: the fixture that builds the driver)
from tests.test_oracle_cpu import make_pairs, rand_seq
from tests.util import DATA, flatten, read_fastx

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INGEST = {"default": {}, "ascii": {"SYL_HOST_INGEST": "ascii"}, "packed-only": {"SYL_HOST_INGEST": "packed-only"},
          "steal": {"SYL_INGEST_FORCE_STEAL": "1"}}
ENV = ("SYL_HOST_INGEST", "SYL_INGEST_FORCE_STEAL", "SYL_INGEST_CHUNK", "SYL_SAMPLE_POSTPASS")


def set_env(monkeypatch, ingest="default", chunk=None, postpass=None):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in INGEST[ingest].items():
        monkeypatch.setenv(k, v)
    if chunk:
        monkeypatch.setenv("SYL_INGEST_CHUNK", str(chunk))
    if postpass:
        monkeypatch.setenv("SYL_SAMPLE_POSTPASS", postpass)


def _pinned(a, dt):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(dt)).pin_memory()


def _cuda(a, dt):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(dt)).cuda()


def sketch(ctx, flat, source, **kw):
    from sylph_b200.api import pack2
    b1, o1, b2, o2 = flat
    if source == "host":
        return ctx.sketch_pair_sequences(b1, o1, b2, o2, **kw)
    if source == "pinned":
        return ctx.sketch_pair_sequences(_pinned(b1, np.uint8), _pinned(o1, np.int64), _pinned(b2, np.uint8),
                                         _pinned(o2, np.int64), **kw)
    if source == "device":
        return ctx.sketch_pair_sequences(_cuda(b1, np.uint8), _cuda(o1, np.int64), _cuda(b2, np.uint8),
                                         _cuda(o2, np.int64), **kw)
    w1, w2 = pack2(b1), pack2(b2)
    if source == "host-packed":
        return ctx.sketch_pair_sequences(w1, o1, w2, o2, packed=True, **kw)
    assert source == "device-packed"
    return ctx.sketch_pair_sequences(_cuda(w1, np.int32), _cuda(o1, np.int64), _cuda(w2, np.int32), _cuda(o2, np.int64),
                                     packed=True, **kw)


def check(ctx, r1, r2, source="host", expect=None, **kw):
    """-> (unique k-mers, duplicates removed, the oracle's result for the next call on the same input)"""
    from oracle import oracle as O
    flat = flatten(r1) + flatten(r2)
    n = min(len(r1), len(r2))
    flat = (flat[0][:int(flat[1][n])], flat[1][:n + 1], flat[2][:int(flat[3][n])], flat[3][:n + 1])
    eh, ec, emean, end = expect or O.sketch_read_pairs(*flat, **kw)
    s = sketch(ctx, flat, source, **kw)
    h, c = s.download()
    assert np.array_equal(h, eh) and np.array_equal(c, ec), source
    assert s.num_dup_removed == end, (source, s.num_dup_removed, end)
    assert abs(s.mean_read_length - emean) <= 1e-9 * max(1.0, emean), source
    s.free()
    return len(h), end, (eh, ec, emean, end)


def synthetic_pairs():
    """tests/test_pairs_gpu.py's duplicate-heavy sample: duplicate pairs, a 300-event hot k-mer, short and empty mates"""
    rng = np.random.default_rng(31)
    genome = rand_seq(rng, 30000, b"ACGT")
    r1, r2 = make_pairs(rng, 4000, genome)
    hot = genome[1000:1150]
    for i in range(300):
        r1.append(hot)
        r2.append(genome[2000 + (i % 37) * 50:2150 + (i % 37) * 50])
    r1 += [b"A" * 150, b"A" * 150, b"", b"ACGTN" * 30]
    r2 += [b"A" * 150, b"A" * 150, b"ACGT" * 20, b"acgtn" * 30]
    order = rng.permutation(len(r1))
    return [r1[i] for i in order], [r2[i] for i in order]


# ---- 1. the inputs of tests/test_pairs_gpu.py in dozens of chunks ---------------------------------------------------------

@pytest.mark.parametrize("ingest", list(INGEST))
def test_k12_fixture_in_small_chunks(ctx, monkeypatch, ingest):
    r1 = [s for _, s in read_fastx(os.path.join(DATA, "k12_R1.fq"))]
    r2 = [s for _, s in read_fastx(os.path.join(DATA, "k12_R2.fq"))]
    set_env(monkeypatch, ingest, chunk=4096)
    n, _, _ = check(ctx, r1, r2, "pinned" if ingest == "steal" else "host", c=20)
    assert n == 9916
    nbytes, n_packed, n_ascii = ctx.ingest_stats()
    nb, np_ = sum(map(len, r1)) + sum(map(len, r2)), len(r1)
    assert n_packed + n_ascii >= nb // 4096
    if ingest == "ascii":       # every base once, and per chunk and mate one offset more than pairs
        assert n_packed == 0 and nbytes == nb + 8 * 2 * (np_ + n_ascii)
    elif ingest == "packed-only":
        assert n_ascii == 0 and nb / 4 <= nbytes - 4 * 2 * (np_ + n_packed) <= nb / 4 + 2 * 64 * n_packed + 8 * n_packed
    elif ingest == "steal":
        assert n_packed > 1 and n_ascii > 1
    check(ctx, r1, r2[:-7], c=20)        # unequal files: pairs = records zipped
    check(ctx, r1, r2, c=200)


@pytest.mark.parametrize("source", ["host", "pinned"])
@pytest.mark.parametrize("no_dedup", [False, True])
@pytest.mark.parametrize("ingest", list(INGEST))
def test_synthetic_duplicates_in_small_chunks(ctx, monkeypatch, ingest, no_dedup, source):
    r1, r2 = synthetic_pairs()
    set_env(monkeypatch, ingest, chunk=800)
    _, nd, _ = check(ctx, r1, r2, source, c=5, no_dedup=no_dedup)
    assert (nd > 2000) if not no_dedup else (nd == 0)
    assert sum(ctx.ingest_stats()[1:]) > 100


def test_k21_scalar_in_small_chunks(ctx, monkeypatch):
    rng = np.random.default_rng(32)
    genome = rand_seq(rng, 20000, b"ACGT")
    r1, r2 = make_pairs(rng, 1500, genome)
    for ingest in ("default", "ascii"):
        set_env(monkeypatch, ingest, chunk=640)
        check(ctx, r1, r2, k=21, c=9, sem=0)


# ---- 2. mates of very different lengths -----------------------------------------------------------------------------------

@pytest.mark.parametrize("ingest", ["default", "ascii"])
def test_uneven_mates_and_degenerate_samples(ctx, monkeypatch, ingest):
    rng = np.random.default_rng(77)
    genome = rand_seq(rng, 40000, b"ACGT")
    lens = [30, 250, 0, 5000, 33, 32, 150]
    r1, r2 = [], []
    for i in range(600):
        a, b = int(rng.integers(0, 30000)), int(rng.integers(0, 30000))
        r1.append(genome[a:a + lens[i % 7]])
        r2.append(genome[b:b + lens[(i * 3 + 1) % 7]])
    r1 += r1[:100]                       # duplicate pairs
    r2 += r2[:100]
    set_env(monkeypatch, ingest, chunk=2048)    # a 5 kbp mate is longer than a chunk
    for c in (1, 7):
        check(ctx, r1, r2, c=c)
    assert sum(ctx.ingest_stats()[1:]) > 100
    check(ctx, [], [], c=5)
    check(ctx, [genome[:150]], [genome[100:250]], c=5)
    check(ctx, [b""], [genome[100:250]], c=5)
    check(ctx, [genome[:20000]], [genome[20000:20040]], c=5)


# ---- 3. group path == sorted path == oracle -------------------------------------------------------------------------------

@pytest.mark.parametrize("source", ["host", "device", "host-packed", "device-packed"])
def test_group_path_equals_sorted_path(ctx, monkeypatch, source):
    r1, r2 = synthetic_pairs()
    expect = None
    for postpass in (None, "sort", None):
        set_env(monkeypatch, chunk=8192, postpass=postpass)
        for no_dedup in (False, True):
            _, _, e = check(ctx, r1, r2, source, c=5, no_dedup=no_dedup, expect=expect if not no_dedup else None)
            expect = expect if no_dedup else e


# ---- 4. scripted histories ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("source", ["device", "host", "device-packed"])
@pytest.mark.parametrize("name", list(P.SAMPLES))
def test_scripted_pairs(ctx, monkeypatch, name, source):
    from oracle import pyref as R
    s = P.sample(name, c=10)
    set_env(monkeypatch, chunk=8192)
    n, nd, (eh, ec, _, end) = check(ctx, s.r1, s.r2, source, c=10)
    assert nd > 100
    check(ctx, s.r1, s.r2, source, c=10, no_dedup=True)
    if name == "small" and source == "device":      # the slow restatement once
        pc, _, pnd = R.sketch_read_pairs(s.r1, s.r2, 31, 10)
        assert dict(zip(eh.tolist(), ec.tolist())) == pc and pnd == end


PROBE = r"""
import sys
import sylph_b200
from tests import pair_scripts as P
from tests.test_pairs_stream_gpu import check
ctx = sylph_b200.Context(0)
for name in ("in_kernel", "slot"):
    for source in ("device", "host"):
        print("@@ %s %s" % (name, source), file=sys.stderr, flush=True)
        s = P.sample(name, c=10)
        check(ctx, s.r1, s.r2, source, c=10)
        check(ctx, s.r1, s.r2, source, c=10, no_dedup=True)
print("ok")
"""


def _probe(env):
    env = dict({k: v for k, v in os.environ.items() if k not in ENV + ("SYL_GROUP_CAP",)}, SYL_DEBUG_TIMING="1",
               SYL_INGEST_CHUNK="8192", **env)
    r = subprocess.run([sys.executable, "-c", PROBE], cwd=ROOT, env=env, capture_output=True, text=True, timeout=540)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
    handed = {}
    for block in r.stderr.split("@@ ")[1:]:
        head, body = block.split("\n", 1)
        handed[tuple(head.split())] = [int(x) for x in re.findall(r"events handed to the generic path (\d+)", body)]
    return handed


def test_pairs_leave_the_group_kernel_only_past_a_slot():
    """The post-pass's own report (SYL_DEBUG_TIMING): no event of the in-kernel families reaches the generic path, the
    k-mers of more than 1024 events do."""
    handed = _probe({})
    for source in ("device", "host"):
        assert handed[("in_kernel", source)] and all(n == 0 for n in handed[("in_kernel", source)]), handed
        assert all(n > D.SLOT for n in handed[("slot", source)]), handed


def test_scripted_pairs_with_tiny_group_slots():
    """SYL_GROUP_CAP=32 (read once per process): nearly every group is past its slot, its events split between the slot
    and the overflow list, and the generic path's pairs are slotted back between the in-kernel groups."""
    handed = _probe({"SYL_GROUP_CAP": "32"})
    assert all(n > 0 for v in handed.values() for n in v), handed


# ---- 5. device memory is bounded by the rings and the events, not by the sample -------------------------------------------

def test_host_pairs_device_memory_is_bounded(monkeypatch):
    """0.6 Gbp of pairs from host memory: the peak of the ctx's block cache plus the staging rings stays under
    DESIGN.md §3's bound for pair samples, 0.60 B per base + 0.25 GB at c = 200, and under the sample's ASCII.
    A ctx of its own: the session's holds the blocks and the rings earlier tests grew."""
    import torch
    import sylph_b200
    from sylph_b200 import synth
    set_env(monkeypatch)
    ctx = sylph_b200.Context(0)
    n_pairs, c = 2_000_000, 200
    b1, o1 = synth.reads(n_pairs, n_comm=8, genome_len=2_000_000, seed=1)
    b2, o2 = synth.reads(n_pairs, n_comm=8, genome_len=2_000_000, seed=2)
    nb = b1.numel() + b2.numel()
    assert nb >= 500_000_000
    torch.cuda.synchronize()
    ctx.device_bytes(reset_peak=True)
    s = ctx.sketch_pair_sequences(b1.numpy(), o1.numpy().astype(np.uint64), b2.numpy(), o2.numpy().astype(np.uint64), c=c)
    _, peak = ctx.device_bytes()
    ring, _ = ctx.ingest_ring_bytes()
    assert len(s) > 1000 and ring > 0 and sum(ctx.ingest_stats()[1:]) >= nb // (32 << 20)
    s.free()
    ctx.close()
    print("peak %d + rings %d bytes for %d bases" % (peak, ring, nb))
    assert peak + ring < 0.60 * nb + 0.25e9, (peak, ring, nb)
    assert peak + ring < nb, (peak, ring, nb)


# ---- 6. the driver --------------------------------------------------------------------------------------------------------

def test_driver_paired_sketch_is_byte_identical_under_every_ingest(exe, tmp_path):
    r1, r2 = os.path.join(DATA, "k12_R1.fq"), os.path.join(DATA, "k12_R2.fq")
    outs = []
    for i, env in enumerate([{}, {"SYL_INGEST_CHUNK": "4096"}, {"SYL_INGEST_CHUNK": "4096", "SYL_HOST_INGEST": "ascii"},
                             {"SYL_INGEST_CHUNK": "4096", "SYL_HOST_INGEST": "packed-only"},
                             {"SYL_INGEST_CHUNK": "4096", "SYL_SAMPLE_POSTPASS": "sort"}]):
        d = tmp_path / str(i)
        d.mkdir()
        run(exe, ["sketch", "-1", r1, "-2", r2, "--fpr", "0", "-c", "20", "-d", str(d)], str(tmp_path), env=env)
        files = sorted(f for f in os.listdir(d) if f.endswith(".paired.sylsp"))
        assert len(files) == 1, os.listdir(d)
        outs.append(open(d / files[0], "rb").read())
    assert len(outs[0]) > 1000 and all(o == outs[0] for o in outs)
