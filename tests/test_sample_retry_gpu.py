"""GPU parity: samples with more survivor events than the event array is sized for.  mm_hash64 of a poly-A / poly-T
k-mer is below 2^64 / 2, so at c = 2 every window of such a read survives; the sketch finds that the events did not
fit, and is redone with the exact capacity.  Covered for read pairs from every input form (host ASCII re-fed through
the chunked feeder under each ingest setting, host 2-bit staged once per call, device ASCII and 2-bit used in place)
and for single-end 2-bit input from host and device memory, in both post-pass modes: hashes, counts, num_dup_removed
and mean_read_length equal to the oracle's.  The cases run in a child process under SYL_DEBUG_TIMING, whose
per-attempt report shows that the retry did happen."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tests.test_pairs_stream_gpu import ENV, _cuda, check
from tests.test_sketch_gpu import rand_seqs
from tests.util import flatten

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C = 2
A, T = b"A" * 150, b"T" * 150
# read pairs: name -> (source of tests/test_pairs_stream_gpu.py's sketch(), the ingest setting it runs under)
PAIR_FORMS = {"host": ("host", {}), "host-ascii": ("host", {"SYL_HOST_INGEST": "ascii"}),
              "pinned-steal": ("pinned", {"SYL_INGEST_FORCE_STEAL": "1"}), "host-packed": ("host-packed", {}),
              "device": ("device", {}), "device-packed": ("device-packed", {})}
SINGLE_FORMS = ("host-packed", "device-packed")


def homopolymer_pairs():
    """10 000 pairs of poly-A / poly-T mates among 1 000 random pairs, and mates too short for a pair key"""
    rng = np.random.default_rng(41)
    r1 = [A] * 3000 + [T] * 3000 + [A] * 2000 + [T] * 2000 + rand_seqs(rng, [150] * 1000) + [A[:20], T, b""]
    r2 = [A] * 3000 + [T] * 3000 + [T] * 2000 + [A] * 2000 + rand_seqs(rng, [150] * 1000) + [T, A[:32], A]
    order = rng.permutation(len(r1))
    return [r1[i] for i in order], [r2[i] for i in order]


def homopolymer_reads():
    """tests/test_sketch_gpu.py's homopolymer sample with fewer random reads, so that it overflows without groups too"""
    rng = np.random.default_rng(99)
    seqs = [A] * 5000 + [T] * 4000 + rand_seqs(rng, [150] * 1000) + [b"A" * 60, b"T" * 401, b"C" * 150]
    return flatten([seqs[i] for i in rng.permutation(len(seqs))])


def check_single_packed(ctx, buf, off, source, expect):
    from sylph_b200.api import pack2
    words = pack2(buf)
    if source == "host-packed":
        s = ctx.sketch_sequences(words, off, c=C, packed_bases=len(buf))
        assert ctx.ingest_stats() == (4 * len(words) + 8 * len(off), 0, 0)  # staged whole: words and offsets
    else:
        s = ctx.sketch_sequences(_cuda(words, np.int32), _cuda(off, np.int64), c=C, packed_bases=len(buf))
    eh, ec, emean, end = expect
    h, c = s.download()
    assert np.array_equal(h, eh) and np.array_equal(c, ec), source
    assert s.num_dup_removed == end and abs(s.mean_read_length - emean) <= 1e-9 * max(1.0, emean), source
    s.free()


def run_cases(postpass):
    """child process: every case once, each after a '@@ <kind> <form>' line on stderr"""
    import sylph_b200
    from oracle import oracle as O
    ctx = sylph_b200.Context(0)
    expect = None
    r1, r2 = homopolymer_pairs()
    for name, (source, env) in PAIR_FORMS.items():
        for k in ENV:
            os.environ.pop(k, None)
        os.environ.update(env, SYL_INGEST_CHUNK="32768", **({"SYL_SAMPLE_POSTPASS": postpass} if postpass else {}))
        print("@@ pairs %s" % name, file=sys.stderr, flush=True)
        n, nd, expect = check(ctx, r1, r2, source, expect=expect, c=C)
        assert n > 1000 and nd > 500000
        if source == "host-packed":
            nb1, nb2 = sum(map(len, r1)), sum(map(len, r2))
            assert ctx.ingest_stats() == (4 * ((nb1 + 15) // 16 + (nb2 + 15) // 16) + 2 * 8 * (len(r1) + 1), 0, 0)
        elif source in ("host", "pinned"):
            assert sum(ctx.ingest_stats()[1:]) > 50
    buf, off = homopolymer_reads()
    expect = O.sketch_reads(buf, off, c=C)
    assert expect[3] > 100000
    for source in SINGLE_FORMS:
        print("@@ reads %s" % source, file=sys.stderr, flush=True)
        check_single_packed(ctx, buf, off, source, expect)
    print("ok")


PROBE = r"""
import sys
from tests.test_sample_retry_gpu import run_cases
run_cases(sys.argv[1] or None)
"""


@pytest.mark.parametrize("postpass", ["group", "sort"])
def test_overflowing_samples_are_redone_in_every_input_form(postpass):
    env = dict({k: v for k, v in os.environ.items() if k not in ENV + ("SYL_GROUP_CAP",)}, SYL_DEBUG_TIMING="1")
    r = subprocess.run([sys.executable, "-c", PROBE, "sort" if postpass == "sort" else ""], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
    blocks = r.stderr.split("@@ ")[1:]
    assert len(blocks) == len(PAIR_FORMS) + len(SINGLE_FORMS), r.stderr
    for block in blocks:
        head, body = block.split("\n", 1)
        entry = "syl_sketch_read_pairs" if head.startswith("pairs") else "syl_sketch_reads"
        attempts = [int(x) for x in re.findall(r"\[%s\] feed .* \(attempt (\d+)\)" % entry, body)]
        assert attempts and attempts[0] == 0 and attempts[-1] >= 1, block   # the first attempt did not fit
        handed = [int(x) for x in re.findall(r"events handed to the generic path (\d+)", body)]
        assert handed and handed[-1] > 1000000, block
