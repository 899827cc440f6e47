"""GPU: `sylph-b200 query | profile` in host batches of samples (--max-sample-bytes).  One sample per batch
(--max-sample-bytes 1) prints byte for byte what the default batch prints: on the golden E. coli genomes and reads
together with synthetic .sylsp files (shuffled, subsampled, renamed), on raw reads mixed with sketches, with
--devices 0,0, with --max-db-entries, with SYL_DRIVER_SAMPLES_PER_CALL, and against the oracle's rows."""
import os

import numpy as np
import pytest

from tests import driver_ref as D
from tests.test_driver_gpu import (GENOMES, PAIRS, SAMPLES, SK_PAIRS, SK_SAMPLES, d, exe, ref, run, sk)  # noqa: F401
from tests.util import REPO

pytestmark = pytest.mark.gpu

GOLD = os.path.join(REPO, "tests", "golden", "data")
GOLD_GENOMES = [os.path.join(GOLD, "e.coli-%s.fasta.gz" % g) for g in ("K12", "EC590", "o157")]
GOLD_READS = [os.path.join(GOLD, "o157_reads.fastq.gz"), os.path.join(GOLD, "k12_R1.fq")]


def _one_per_batch(exe, args, d, env=None):  # noqa: F811
    """the run with --max-sample-bytes 1 prints what the default run prints -> that output"""
    one = run(exe, args, d, env=env).stdout
    assert len(one.splitlines()) > 1
    got = run(exe, args[:1] + ["--max-sample-bytes", "1"] + args[1:], d, env=env).stdout
    assert got == one, args
    return one


@pytest.fixture(scope="module")
def golden_sylsp(exe, d):  # noqa: F811
    """the golden reads sketched by the driver, plus synthetic .sylsp files made from them: pairs shuffled, every
    other pair dropped, a sample name set, and one sketch without any k-mer"""
    from sylph_b200 import formats as F
    out = os.path.join(d, "gold_sk")
    if not os.path.exists(out):
        run(exe, ["sketch", "-d", out] + GOLD_READS, d)
    base = sorted(os.path.join(out, f) for f in os.listdir(out) if f.endswith(".sylsp") and not f.startswith("syn_"))
    assert len(base) == 2
    rng = np.random.default_rng(11)
    files = []
    for i, f in enumerate(base):
        s = F.read_sylsp(f)
        p = rng.permutation(len(s["hashes"]))
        for tag, sel in (("shuf", p), ("half", p[::2])):
            t = dict(s, hashes=s["hashes"][sel], counts=s["counts"][sel], sample_name="syn %d %s" % (i, tag))
            files.append(os.path.join(out, "syn_%d_%s.sylsp" % (i, tag)))
            F.write_sylsp(files[-1], t)
    s = F.read_sylsp(base[0])
    files.append(os.path.join(out, "syn_empty.sylsp"))
    F.write_sylsp(files[-1], dict(s, hashes=s["hashes"][:0], counts=s["counts"][:0], sample_name="syn empty"))
    return base + files


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_golden_with_synthetic_sketches(exe, d, golden_sylsp, cmd):  # noqa: F811
    out = _one_per_batch(exe, [cmd] + golden_sylsp + GOLD_READS + GOLD_GENOMES, d)
    assert "syn 1 half" in out and "syn 1 shuf" in out
    _one_per_batch(exe, [cmd, "-u", "-I", "98"] + golden_sylsp + GOLD_GENOMES, d)


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_raw_reads_mixed_with_sketches(exe, d, sk, cmd):  # noqa: F811
    args = [cmd, "sk/db.syldb", SK_SAMPLES[1], SK_PAIRS[0], SAMPLES[0]] + GENOMES[:5] + [SAMPLES[2]] + SK_PAIRS[1:]
    one = _one_per_batch(exe, args, d)
    assert run(exe, args, d, env={"SYL_DRIVER_SAMPLES_PER_CALL": "2"}).stdout == one
    assert run(exe, args[:1] + ["--devices", "0,0", "--max-sample-bytes", "1"] + args[1:], d).stdout == one
    assert run(exe, args[:1] + ["--max-db-entries", "10000", "--max-sample-bytes", "1"] + args[1:], d).stdout == one
    assert run(exe, args[:1] + ["--devices", "0,0", "--max-db-entries", "10000"] + args[1:], d).stdout == one


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_one_sample_per_batch_against_the_oracle(exe, d, ref, sk, cmd):  # noqa: F811
    pt = cmd == "profile"
    want = D.contain(ref.genomes(GENOMES), [ref.sample(s) for s in SAMPLES], pt)
    out = run(exe, [cmd, "--max-sample-bytes", "1"] + SAMPLES + GENOMES, d).stdout
    D.compare_tsv(out, want, pt)
    sk_out = run(exe, [cmd, "--max-sample-bytes", "1", "--max-db-entries", "10000"] + SK_SAMPLES + ["sk/db.syldb"], d).stdout
    assert sk_out == out
