"""GPU parity on scripted duplicate-removal histories (tests/dedup_scripts.py): every device path of the read-sketch
post-pass -- the four-event register replay, the warp-cooperative replay, the generic k_dedup behind the 64-step, the
32-entry and the slot fallbacks, and k_dedup_paired -- against the CPU oracle, bit for bit, on inputs built to reach
it; and proof, from the post-pass's own report, that the fallback ran where it has to and not elsewhere."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tests import dedup_scripts as D
from tests.test_packed_sketch_gpu import _cuda, check_pairs_packed

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C = 10


def check_single(ctx, s, source, k=31, sem=1, no_dedup=False):
    from oracle import oracle as O
    from sylph_b200.api import pack2
    b, o = s.flat()
    eh, ec, mean, nd = O.sketch_reads(b, o, k=k, c=C, no_dedup=no_dedup, sem=sem)
    if source == "host":
        x = ctx.sketch_sequences(b, o, k=k, c=C, no_dedup=no_dedup, sem=sem)
    elif source == "device":
        x = ctx.sketch_sequences(_cuda(b, np.uint8), _cuda(o, np.int64), k=k, c=C, no_dedup=no_dedup, sem=sem)
    else:
        x = ctx.sketch_sequences(_cuda(pack2(b), np.int32), _cuda(o, np.int64), k=k, c=C, no_dedup=no_dedup, sem=sem,
                                 packed_bases=len(b))
    h, cnt = x.download()
    assert np.array_equal(h, eh) and np.array_equal(cnt, ec), source
    assert x.num_dup_removed == nd, (source, x.num_dup_removed, nd)
    assert abs(x.mean_read_length - mean) <= 1e-9 * max(1.0, mean), source
    x.free()
    return nd


# host: packed host ingest in 8 KB chunks, so one k-mer's history spans many batches that arrive in any order
@pytest.mark.parametrize("source", ["device", "host", "packed"])
@pytest.mark.parametrize("name", list(D.SAMPLES))
def test_single_end_parity(ctx, monkeypatch, name, source):
    monkeypatch.setenv("SYL_INGEST_CHUNK", "8192")
    monkeypatch.delenv("SYL_HOST_INGEST", raising=False)
    assert check_single(ctx, D.single_sample(name, c=C), source) > 1000


@pytest.mark.parametrize("name", list(D.SAMPLES))
def test_single_end_parity_no_dedup_and_k21_scalar(ctx, name):
    assert check_single(ctx, D.single_sample(name, c=C), "device", no_dedup=True) == 0
    assert check_single(ctx, D.single_sample(name, k=21, c=C, sem=0), "device", k=21, sem=0) > 1000


PROBE = r"""
import sys
import numpy as np
from tests import dedup_scripts as D
from tests.test_dedup_scripts_gpu import check_single
import sylph_b200
ctx = sylph_b200.Context(0)
for name in NAMES:
    for source in ("device", "host"):
        print("@@ %s %s" % (name, source), file=sys.stderr, flush=True)
        check_single(ctx, D.single_sample(name, c=10), source)
    if ALL_CONFIGS:
        check_single(ctx, D.single_sample(name, c=10), "packed")
        check_single(ctx, D.single_sample(name, c=10), "device", no_dedup=True)
        check_single(ctx, D.single_sample(name, k=21, c=10, sem=0), "device", k=21, sem=0)
print("ok")
"""


def _probe(env, names, all_configs=False):
    unset = ("SYL_SAMPLE_POSTPASS", "SYL_GROUP_CAP", "SYL_HOST_INGEST")
    env = dict({k: v for k, v in os.environ.items() if k not in unset}, **env)
    code = "NAMES = %r\nALL_CONFIGS = %r\n" % (names, all_configs) + PROBE
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=540)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
    return r.stderr


def test_fallback_runs_exactly_where_the_classifier_says():
    """SYL_DEBUG_TIMING=1: the post-pass reports how many events it handed to the generic path.  None for the sample of
    in-kernel families (the classifier finds no fallback k-mer and no group past its slot there), some for the
    64-step, the 32-entry and the slot samples.  The library reads both switches once per process."""
    err = _probe({"SYL_DEBUG_TIMING": "1", "SYL_INGEST_CHUNK": "8192"}, list(D.SAMPLES))
    handed = {}
    for block in err.split("@@ ")[1:]:
        head, body = block.split("\n", 1)
        n = [int(x) for x in re.findall(r"\[sample post-pass\].*events handed to the generic path (\d+)", body)]
        assert n, block
        handed[tuple(head.split())] = n[-1]
    r = D.classify(D.single_sample("in_kernel", c=C), c=C)
    assert all(r["classes"][cls] == 0 for cls in D.FALLBACK) and r["max_group"] <= D.SLOT, r
    for source in ("device", "host"):
        assert handed[("in_kernel", source)] == 0, handed
        for name in ("steps", "set", "slot"):
            assert handed[(name, source)] > 0, handed


def test_generic_postpass_on_every_scripted_sample():
    """SYL_SAMPLE_POSTPASS=sort: every event through the radix sorts and k_dedup."""
    _probe({"SYL_SAMPLE_POSTPASS": "sort", "SYL_INGEST_CHUNK": "8192"}, list(D.SAMPLES), all_configs=True)


@pytest.mark.parametrize("name", list(D.PAIR_SAMPLES))
def test_pair_parity(ctx, name):
    """Host and device memory, ASCII and 2-bit words (check_pairs_packed)."""
    s = D.pair_sample(name, c=C)
    _, nd = check_pairs_packed(ctx, s.r1, s.r2, c=C)
    assert nd > 500
    check_pairs_packed(ctx, s.r1, s.r2, c=C, no_dedup=True)
