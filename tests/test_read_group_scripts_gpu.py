"""GPU: the read-sketch grouping kernel at its capacity edges, on the samples of tests/read_group_scripts.py.

Every family -- a full hash table, one probe chain over the whole table, a group in one bucket, groups of exactly
slot and slot + 1 events, dedup histories at full occupancy, k-mers at every bucket boundary, a group split by a part
bound -- goes through device ASCII, device 2-bit words, host memory in 8 KB packed chunks (a group's events arrive
from many batches in any order), host ASCII ingest and --no-dedup, and must give the C oracle's sketch: hashes,
counts, num_dup_removed and mean_read_length.  And each sample must take the path it was built for: the post-pass's
own report (SYL_DEBUG_TIMING=1, read once per process, so a child) of the groups, the overflow list, the in-kernel
uniques and the events handed to the generic path equals the model's (read_group_scripts.post_pass), part by part
under SYL_SAMPLE_PARTS, and under SYL_GROUP_CAP = 32, 255, 256, 257 and 700.  SYL_SAMPLE_POSTPASS=sort sends every
event to the generic path and gives the same sketches."""
import os
import pickle
import re
import subprocess
import sys

import numpy as np
import pytest

from tests import read_group_scripts as G

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV = ("SYL_HOST_INGEST", "SYL_INGEST_CHUNK", "SYL_SAMPLE_POSTPASS", "SYL_SAMPLE_PARTS", "SYL_INGEST_FORCE_STEAL")
# form -> (source, no_dedup, environment of the call)
FORMS = {"device": ("device", False, {}), "packed": ("packed", False, {}),
         "host": ("host", False, {"SYL_INGEST_CHUNK": "8192"}),
         "host-ascii": ("host", False, {"SYL_INGEST_CHUNK": "8192", "SYL_HOST_INGEST": "ascii"}),
         "no_dedup": ("device", True, {})}
CASES = [(name, paired) for name in G.FAMILIES for paired in (False, True)]
IDS = ["%s-%s" % (n, "pairs" if p else "single") for n, p in CASES]
LINE = re.compile(r"\[sample post-pass\] groups (\d+) of (\d+) slots, overflow list (\d+) \(cap \d+\): "
                  r"in-kernel uniques (\d+), events handed to the generic path (\d+)")


def _cuda(a, dt):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(dt)).cuda()


def sketch(ctx, s, source, no_dedup):
    from sylph_b200.api import pack2
    kw = dict(k=s.k, c=s.c, no_dedup=no_dedup, sem=G.SEM)
    if not s.paired:
        b, o = s.flat()
        if source == "host":
            return ctx.sketch_sequences(b, o, **kw)
        if source == "device":
            return ctx.sketch_sequences(_cuda(b, np.uint8), _cuda(o, np.int64), **kw)
        return ctx.sketch_sequences(_cuda(pack2(b), np.int32), _cuda(o, np.int64), packed_bases=len(b), **kw)
    b1, o1, b2, o2 = s.flat()
    if source == "host":
        return ctx.sketch_pair_sequences(b1, o1, b2, o2, **kw)
    if source == "device":
        return ctx.sketch_pair_sequences(_cuda(b1, np.uint8), _cuda(o1, np.int64), _cuda(b2, np.uint8),
                                         _cuda(o2, np.int64), **kw)
    return ctx.sketch_pair_sequences(_cuda(pack2(b1), np.int32), _cuda(o1, np.int64), _cuda(pack2(b2), np.int32),
                                     _cuda(o2, np.int64), packed=True, **kw)


def oracle(s, no_dedup):
    from oracle import oracle as O
    f = O.sketch_read_pairs if s.paired else O.sketch_reads
    return f(*s.flat(), k=s.k, c=s.c, no_dedup=no_dedup, sem=G.SEM)


def check(ctx, s, form, env=None, expect=None):
    """sketch s in one form (under env) and compare it with the oracle; -> the oracle's result"""
    source, no_dedup, fenv = FORMS[form]
    saved = {k: os.environ.pop(k) for k in ENV if k in os.environ}
    os.environ.update(fenv)
    os.environ.update(env or {})
    try:
        eh, ec, emean, end = expect or oracle(s, no_dedup)
        x = sketch(ctx, s, source, no_dedup)
        h, c = x.download()
        what = (s.name, s.paired, s.slot, form, env)
        assert np.array_equal(h, eh) and np.array_equal(c, ec), what
        assert x.num_dup_removed == end, (what, x.num_dup_removed, end)
        assert abs(x.mean_read_length - emean) <= 1e-9 * max(1.0, emean), what
        x.free()
    finally:
        for k in ENV:
            os.environ.pop(k, None)
        os.environ.update(saved)
    return eh, ec, emean, end


@pytest.mark.parametrize("name,paired", CASES, ids=IDS)
def test_every_input_form_equals_the_oracle(ctx, name, paired):
    s = G.sample(name, paired)
    for form in FORMS:
        check(ctx, s, form)


@pytest.mark.parametrize("name,paired", [(n, p) for n in ("full_distinct", "slot_plus_one", "parts")
                                         for p in (False, True)])
def test_parts_equal_the_oracle(ctx, name, paired):
    s = G.sample(name, paired)
    expect = oracle(s, False)
    for P in (2, 3, 7):
        for form in ("device", "host"):
            check(ctx, s, form, {"SYL_SAMPLE_PARTS": str(P)}, expect)
        assert ctx.sample_parts() == P


CHILD = r"""
import pickle
import sys
import sylph_b200
from tests.test_read_group_scripts_gpu import check
ctx = sylph_b200.Context(0)
for i, (s, form, env) in enumerate(pickle.load(open(sys.argv[1], "rb"))):
    print("@@ %d" % i, file=sys.stderr, flush=True)
    check(ctx, s, form, env)
print("ok")
"""


def run_jobs(tmp_path, jobs, cap=None):
    """jobs: [(sample, form, env)], each checked against the oracle in a child with SYL_DEBUG_TIMING=1 -> per job the
    (groups, slot, overflow list, in-kernel uniques, events handed to the generic path) of every post-pass line"""
    path = str(tmp_path / "jobs.pkl")
    with open(path, "wb") as f:
        pickle.dump(jobs, f)
    env = {k: v for k, v in os.environ.items() if k not in ENV + ("SYL_GROUP_CAP",)}
    env["SYL_DEBUG_TIMING"] = "1"
    if cap:
        env["SYL_GROUP_CAP"] = str(cap)
    r = subprocess.run([sys.executable, "-c", CHILD, path], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=540)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr[-5000:]
    got = {}
    for block in r.stderr.split("@@ ")[1:]:
        head, body = block.split("\n", 1)
        got[int(head)] = [tuple(map(int, m)) for m in LINE.findall(body)]
    assert sorted(got) == list(range(len(jobs)))
    return [got[i] for i in range(len(jobs))]


def expected(s, form, env, slot=None):
    if (env or {}).get("SYL_SAMPLE_POSTPASS") == "sort":     # no groups: every event to the generic path
        n = sum(sum(e.values()) for e in G.group_events(s).values())
        return [(0, 0, n, 0, n)]
    return G.post_pass(s, slot, FORMS[form][1], int((env or {}).get("SYL_SAMPLE_PARTS", 1)))


def check_paths(jobs, lines, slot=None):
    for (s, form, env), got in zip(jobs, lines):
        assert got == expected(s, form, env, slot), (s.name, s.paired, form, env)


def test_each_family_takes_the_path_it_was_built_for(tmp_path):
    """every family and form at the default slot, the part setups under SYL_SAMPLE_PARTS, and the full and slot
    families through the generic path alone (SYL_SAMPLE_POSTPASS=sort)"""
    jobs = []
    for name, paired in CASES:
        s = G.sample(name, paired)
        jobs += [(s, form, None) for form in FORMS]
    for name in ("parts", "full_distinct", "slot_plus_one"):
        for paired in (False, True):
            for P in (2, 3):
                jobs += [(G.sample(name, paired), form, {"SYL_SAMPLE_PARTS": str(P)}) for form in ("device", "host")]
    for name in G.FULL + ("slot_exact", "slot_plus_one"):
        for paired in (False, True):
            jobs.append((G.sample(name, paired), "device", {"SYL_SAMPLE_POSTPASS": "sort"}))
    lines = run_jobs(tmp_path, jobs)
    check_paths(jobs, lines)
    # the report has power: the families' own claims show in it
    by = {(s.name, s.paired, form, str(env)): got for (s, form, env), got in zip(jobs, lines)}
    for paired in (False, True):
        assert by[("full_distinct", paired, "device", "None")][0][4] == 0
        assert by[("slot_exact", paired, "device", "None")][0][4] == G.SLOT + 1
        assert by[("slot_plus_one", paired, "device", "None")][0][4] == 2 * (G.SLOT + 1)
        parts = by[("parts", paired, "device", str({"SYL_SAMPLE_PARTS": "3"}))]
        assert len(parts) == 3 and parts[1][0] == 4 and parts[0][4] == 0


@pytest.mark.parametrize("cap", G.SMALL_CAPS)
def test_small_slots(tmp_path, cap):
    """SYL_GROUP_CAP (read once per process): groups of exactly slot and slot + 1 events, with the per-thread event rows
    of k_group_dedup partly filled when the slot is not a multiple of 256"""
    jobs = [(G.sample(name, paired, cap), form, None) for name in ("slot_exact", "slot_plus_one")
            for paired in (False, True) for form in FORMS]
    check_paths(jobs, run_jobs(tmp_path, jobs, cap), cap)
