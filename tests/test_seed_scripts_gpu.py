"""GPU parity on scripted seeding batches (tests/seed_scripts.py): k_seed at its capacity edges (survivors staged per
tile, candidates listed per record chunk, record chunks, runs and their masks, the staging tail, the pair-key rule, a
sample part that overflows the staging buffer) against the C oracle, bit for bit, in every instantiation
k_seed<K, EMIT, W, PACKED>: k = 21 and 31; plain survivors (both window rules, with and without positions), read
sketches (grouped, SYL_SAMPLE_POSTPASS=sort, no_dedup, 2 parts) and read-pair sketches; ASCII and 2-bit input from host
and device memory; W = 24, 30, 32 forced by SYL_SEED_W, which the library reads once per process, so each W runs in a
child process.  And the survivor ABI's capacity: appends past cap are counted, not written."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

from tests import seed_scripts as S

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV = ("SYL_SAMPLE_POSTPASS", "SYL_SAMPLE_PARTS", "SYL_HOST_INGEST", "SYL_INGEST_CHUNK", "SYL_GENOME_POSTPASS")


def _cuda(a, dtype):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(dtype)).cuda()


def _inputs(b):
    """(label, bases, offsets, kwargs) of the four input forms."""
    from sylph_b200.api import pack2
    w = pack2(b.buf)
    od = _cuda(b.off, np.int64)
    return [("host ascii", b.buf, b.off, {}), ("host packed", w, b.off, {"packed_bases": b.n_bases}),
            ("device ascii", _cuda(b.buf, np.uint8), od, {}),
            ("device packed", _cuda(w, np.int32), od, {"packed_bases": b.n_bases})]


def _env(**kv):
    for k in ENV:
        os.environ.pop(k, None)
    os.environ.update(kv)


def _same_sample(s, exp, what):
    h, c = s.download()
    assert np.array_equal(h, exp[0]) and np.array_equal(c, exp[1]), what
    assert s.num_dup_removed == exp[3], (what, s.num_dup_removed, exp[3])
    s.free()


def run_batch(ctx, b):
    """Every output of b against the oracle; -> number of calls."""
    from oracle import oracle as O
    from sylph_b200.api import pack2
    calls = 0
    _env()
    forms = _inputs(b)
    if "emit0" in b.outputs:
        for sem in (0, 1):
            for with_pos in (0, 1):
                exp = S.oracle_survivors(b, sem, with_pos)
                for label, x, o, kw in forms:
                    sv = ctx.extract_markers_batch(x, o, k=b.k, c=b.c, sem=sem, with_pos=with_pos, **kw)
                    got = sorted(zip(sv["rec"].tolist(), sv["pos"].tolist() if with_pos else [0] * len(sv),
                                     sv["hash"].tolist()))
                    assert got == exp, (b.name, label, sem, with_pos, len(got), len(exp))
                    calls += 1
    variants = []
    if "reads" in b.outputs:
        variants.append(("grouped", {}, False))
    if "sort" in b.outputs:
        variants.append(("sort", {"SYL_SAMPLE_POSTPASS": "sort"}, False))
    if "no_dedup" in b.outputs:
        variants += [("grouped no_dedup", {}, True), ("sort no_dedup", {"SYL_SAMPLE_POSTPASS": "sort"}, True)]
    if "parts" in b.outputs:
        variants.append(("parts", {"SYL_SAMPLE_PARTS": str(b.parts)}, False))
    for sem in (0, 1):
        for vname, env, no_dedup in variants:
            exp = O.sketch_reads(b.buf, b.off, k=b.k, c=b.c, no_dedup=no_dedup, sem=sem)
            for label, x, o, kw in forms:
                _env(**env)
                s = ctx.sketch_sequences(x, o, k=b.k, c=b.c, no_dedup=no_dedup, sem=sem, **kw)
                if vname == "parts":
                    assert ctx.sample_parts() == b.parts
                _same_sample(s, exp, (b.name, vname, label, sem))
                calls += 1
        if "pairs" in b.outputs:
            _env()
            exp = O.sketch_read_pairs(b.buf, b.off, b.buf, b.off, k=b.k, c=b.c, sem=sem)
            w = pack2(b.buf)
            od = _cuda(b.off, np.int64)
            for label, x, o, packed in (("host ascii", b.buf, b.off, False), ("host packed", w, b.off, True),
                                        ("device ascii", _cuda(b.buf, np.uint8), od, False),
                                        ("device packed", _cuda(w, np.int32), od, True)):
                s = ctx.sketch_pair_sequences(x, o, x, o, k=b.k, c=b.c, sem=sem, packed=packed)
                _same_sample(s, exp, (b.name, "pairs", label, sem))
                calls += 1
    _env()
    return calls


def run_all():
    """Every family's batches in this process (at the run length SYL_SEED_W forces) -> per family calls and seconds."""
    import sylph_b200
    ctx = sylph_b200.Context(0)
    out = []
    for family in S.FAMILIES:
        t0 = time.time()
        calls = sum(run_batch(ctx, b) for b in S.family_batches(family))
        out.append(dict(family=family, calls=calls, seconds=round(time.time() - t0, 1)))
    ctx.close()
    return dict(W=int(os.environ.get("SYL_SEED_W", "0")), families=out)


CHILD = r"""
import json, sys
sys.path.insert(0, %(root)r)
from tests.test_seed_scripts_gpu import run_all
print("RESULT " + json.dumps(run_all()))
"""


@pytest.mark.parametrize("W", [24, 30, 32])
def test_every_family_in_every_instantiation(W):
    """One child process per run length: SYL_SEED_W selects k_seed<K, EMIT, W, PACKED> for every call in it."""
    assert W in S.run_lengths()
    env = dict(os.environ, SYL_SEED_W=str(W))
    for k in ENV:
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", CHILD % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=580)
    assert r.returncode == 0, (r.stdout[-2000:] + r.stderr[-4000:])
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][7:])
    print(res)
    assert res["W"] == W
    assert [f["family"] for f in res["families"]] == list(S.FAMILIES) and all(f["calls"] > 0 for f in res["families"])


def _seed_abi(ctx, b, cap, guard, sem=1, with_pos=1):
    """syl_seed_batch on device input into a device buffer of cap + guard entries filled with 0xA5: -> (rc, n_out,
    the first cap entries, the guard bytes)."""
    import torch
    from sylph_b200 import _lib
    L = _lib.lib()
    xb, xo = _cuda(b.buf, np.uint8), _cuda(b.off, np.int64)
    out = torch.full(((cap + guard) * 16,), 0xA5, dtype=torch.uint8, device="cuda")
    n = C.c_uint64(0)
    rc = L.syl_seed_batch(ctx._h, _lib.MEM_DEVICE, C.c_void_p(xb.data_ptr()), b.n_bases, C.c_void_p(xo.data_ptr()),
                          b.n_rec, b.k, b.c, sem, with_pos, C.c_void_p(out.data_ptr()), cap, C.byref(n))
    torch.cuda.synchronize()
    a = out.cpu().numpy()
    from sylph_b200.api import SURVIVOR_DTYPE
    return rc, n.value, a[:cap * 16].view(SURVIVOR_DTYPE), a[cap * 16:]


@pytest.mark.parametrize("name", [("stage", 31, 1), ("cand", 31, 1), ("stage", 21, 0)], ids=lambda n: "%s-k%d-%d" % n)
def test_capacity_counts_and_guards(ctx, name):
    """cap = n - 1: SYL_ERR_CAPACITY with the true count n, cap entries written, all of them survivors, nothing past
    them; cap = n: every survivor, nothing past them.  stage513 / cand1025 overflow tile 0's staging buffer, so appends
    come from both the inline path and the flush."""
    from sylph_b200 import _lib
    b = S.batch(*name)
    exp = S.oracle_survivors(b, 1, 1)
    n = len(exp)
    for cap in (n - 1, n):
        rc, got_n, sv, guard = _seed_abi(ctx, b, cap, 64)
        assert got_n == n, (cap, got_n, n)
        assert rc == (_lib.SYL_ERR_CAPACITY if cap < n else 0), (cap, rc)
        assert (guard == 0xA5).all(), cap
        got = sorted(zip(sv["rec"].tolist(), sv["pos"].tolist(), sv["hash"].tolist()))
        assert len(set(got)) == cap and set(got) <= set(exp), cap
