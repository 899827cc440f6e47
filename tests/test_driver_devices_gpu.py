"""GPU: `sylph-b200 --devices` deals sketching, query and profile over several contexts and writes exactly what one
context writes: the .sylsp / .syldb files byte for byte, and the TSVs byte for byte.  Several contexts on device 0 stand
in for several GPUs (the work split is the same); a run on devices 0 and 1 is added when two are visible.  The inputs and
the one-context runs, which tests/test_driver_gpu.py ties to the oracle, are those of that file."""
import os
import subprocess
import sys

import pytest

from tests.test_driver_gpu import (GENOMES, PAIRS, SAMPLES, SK_PAIRS, SK_SAMPLES, big, d, exe, ref, run, sk)  # noqa: F401
from tests.util import REPO

pytestmark = pytest.mark.gpu


def _tree(path):
    """{relative name: bytes} of every file under path"""
    out = {}
    for root, _, files in os.walk(path):
        for f in files:
            p = os.path.join(root, f)
            out[os.path.relpath(p, path)] = open(p, "rb").read()
    return out


def _sketch(exe, d, tag, extra, env=None):  # noqa: F811
    args = ["sketch"] + extra + GENOMES + SAMPLES + ["-1", PAIRS[0][0], PAIRS[1][0], "-2", PAIRS[0][1], PAIRS[1][1],
                                                     "--fpr", "0", "-d", "dv_" + tag, "-o", "dv_%s/db" % tag]
    r = run(exe, args, d, env=env)
    return _tree(os.path.join(d, "dv_" + tag)), r


def _named(exe, d, tag, devices, env=None):  # noqa: F811
    names = ["n_pair_a", "n_pair_b"] + ["named/%d" % i for i in range(len(SAMPLES))]
    args = ["sketch", "-1", PAIRS[0][0], PAIRS[1][0], "-2", PAIRS[0][1], PAIRS[1][1], "--fpr", "0", "-S"] + names + \
        ["-d", "nm_" + tag] + SAMPLES + devices
    run(exe, args, d, env=env)
    return _tree(os.path.join(d, "nm_" + tag))


def test_sketch_files_identical(exe, d, sk):  # noqa: F811
    """--devices 0,0,0 and 0,0 at -t 1 and -t 8: every .sylsp and the .syldb equal the one-context run's bytes"""
    one, r1 = _sketch(exe, d, "one", [])
    assert len(one) == len(SAMPLES) + len(PAIRS) + 1
    for tag, extra in (("three", ["--devices", "0,0,0"]), ("t1", ["--devices", "0,0", "-t", "1"]),
                       ("t8", ["--devices", "0,0", "-t", "8"])):
        got, r = _sketch(exe, d, tag, extra)
        assert got == one, tag
        # the lines that name a file are the same lines (their order on stderr may differ)
        named = lambda e: sorted(ln.replace("dv_%s" % tag, "dv_one") for ln in e.splitlines() if "Sketching " in ln)  # noqa: E731
        assert named(r.stderr) == named(r1.stderr), tag


def test_sketch_one_file_per_batch_and_names(exe, d, sk):  # noqa: F811
    """SYL_DRIVER_BATCH_BASES=1: one genome file per batch, so batches finish out of order; -S sample names"""
    env = {"SYL_DRIVER_BATCH_BASES": "1"}
    one, _ = _sketch(exe, d, "b1_one", [], env)
    got, _ = _sketch(exe, d, "b1_three", ["--devices", "0,0,0"], env)
    assert got == one and len(one) == len(SAMPLES) + len(PAIRS) + 1
    assert one["db.syldb"] == _sketch(exe, d, "b1_default", [])[0]["db.syldb"]
    a, b = _named(exe, d, "one", []), _named(exe, d, "three", ["--devices", "0,0,0"])
    assert a == b and len(a) == len(SAMPLES) + len(PAIRS)


def _same(exe, d, args, devices=("0,0", "0,0,0,0"), env=None):  # noqa: F811
    one = run(exe, args, d, env=env).stdout
    assert len(one.splitlines()) > 1
    for dv in devices:
        assert run(exe, args[:1] + ["--devices", dv] + args[1:], d, env=env).stdout == one, (dv, env)
    return one


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_raw_sketched_and_mixed_inputs(exe, d, sk, cmd):  # noqa: F811
    _same(exe, d, [cmd] + SAMPLES + GENOMES)
    _same(exe, d, [cmd] + SK_SAMPLES + SK_PAIRS + ["sk/db.syldb"])
    _same(exe, d, [cmd, "sk/db.syldb", SK_SAMPLES[1], SK_PAIRS[0], SAMPLES[0]] + GENOMES[:5] + [SAMPLES[2]])


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_more_contexts_than_samples(exe, d, sk, cmd):  # noqa: F811
    _same(exe, d, [cmd, SK_SAMPLES[0], "sk/db.syldb"], devices=("0,0", "0,0,0,0"))
    _same(exe, d, [cmd, SAMPLES[0], SK_SAMPLES[2]] + GENOMES, devices=("0,0,0,0",))


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_samples_of_very_different_size(exe, d, sk, big, cmd):  # noqa: F811
    """~72 Mbp of reads first, then small samples: the later blocks finish first and wait for it"""
    _same(exe, d, [cmd, big] + SAMPLES + SK_SAMPLES + ["sk/db.syldb"])


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_batches_row_buffer_and_u(exe, d, sk, cmd):  # noqa: F811
    args = [cmd] + SK_SAMPLES + SK_PAIRS + ["sk/db.syldb"]
    one = _same(exe, d, args, env={"SYL_DRIVER_SAMPLES_PER_CALL": "1"})
    assert run(exe, args, d).stdout == one
    _same(exe, d, args, env={"SYL_DRIVER_ROWS": "1"})
    _same(exe, d, [cmd, "-u", "-I", "98"] + SK_SAMPLES + SAMPLES[:2] + ["sk/db.syldb"])


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_sharded_database(exe, d, sk, cmd):  # noqa: F811
    args = [cmd] + SK_SAMPLES + SK_PAIRS + ["sk/db.syldb"]
    one = run(exe, args, d).stdout
    for extra, env in ((["--max-db-entries", "10000"], None), ([], {"SYL_DRIVER_SHARD_ENTRIES": "3000"})):
        r1 = run(exe, args[:1] + extra + args[1:], d, env=env)
        shards = [ln for ln in r1.stderr.splitlines() if "Database shard " in ln]
        assert r1.stdout == one and len(shards) >= 3
        for dv in ("0,0", "0,0,0"):
            r = run(exe, args[:1] + ["--devices", dv] + extra + args[1:], d, env=env)
            assert r.stdout == one, (dv, extra, env)
            # an explicit cap is the cap of every context: the same shards
            assert [ln for ln in r.stderr.splitlines() if "Database shard " in ln] == shards
    _same(exe, d, [cmd, "--max-db-entries", "10000"] + SAMPLES[:3] + GENOMES, devices=("0,0",))


def test_damaged_gzip_among_good_files(exe, d, sk):  # noqa: F811
    for f, src in (("dv_bad.fq.gz", SAMPLES[1]), ("dv_bad.fa.gz", GENOMES[1])):
        raw = open(os.path.join(d, src), "rb").read()
        with open(os.path.join(d, f), "wb") as fh:
            fh.write(raw[:len(raw) // 2])
    args = ["query", SAMPLES[0], "dv_bad.fq.gz", SAMPLES[2]] + GENOMES[:10] + ["dv_bad.fa.gz"] + GENOMES[10:20]
    one = run(exe, args, d)
    warns = sorted(ln for ln in one.stderr.splitlines() if ln.startswith("WARN"))
    assert len(warns) == 2
    for dv in ("0,0", "0,0,0"):
        r = run(exe, args[:1] + ["--devices", dv] + args[1:], d)
        assert r.stdout == one.stdout and sorted(ln for ln in r.stderr.splitlines() if ln.startswith("WARN")) == warns
    sk_args = ["sketch", "-d", "dv_badsk", SAMPLES[0], "dv_bad.fq.gz", "dv_bad.fa.gz", GENOMES[0], "-o", "dv_badsk/db"]
    r = run(exe, sk_args[:1] + ["--devices", "0,0"] + sk_args[1:], d)
    assert sum("is not a valid fasta/fastq file; skipping." in ln for ln in r.stderr.splitlines()) == 2


def test_library_error_on_one_context_exits(exe, d, sk):  # noqa: F811
    """a k = 21 sketch among k = 31 ones: the context holding it fails, the process exits 1 with the one-context
    message (and does not hang: run() has a timeout)"""
    if not os.path.exists(os.path.join(d, "dv_k21", SAMPLES[3] + ".sylsp")):
        run(exe, ["sketch", "-k", "21", "-d", "dv_k21", SAMPLES[3]], d)
    k21 = "dv_k21/%s.sylsp" % SAMPLES[3]
    for cmd in ("query", "profile"):
        args = [cmd] + SK_SAMPLES + [k21] + SK_SAMPLES + ["sk/db.syldb"]
        one = run(exe, args, d, rc=1)
        err = [ln for ln in one.stderr.splitlines() if ln.startswith("ERROR")]
        assert len(err) == 1 and "k parameter for reads != k parameter for genome" in err[0]
        for dv in ("0,0", "0,0,0"):
            r = run(exe, args[:1] + ["--devices", dv] + args[1:], d, rc=1)
            assert [ln for ln in r.stderr.splitlines() if ln.startswith("ERROR")] == err, dv


def test_missing_device_exits_before_reading(exe, d):  # noqa: F811
    r = run(exe, ["query", "--devices", "0,4096", "nonexistent.fq", "nonexistent.fa"], d, rc=1)
    assert "syl_ctx_create (device 4096): bad device index" in r.stderr and r.stdout == ""


PACK_SCRIPT = r"""
import ctypes as C, threading, numpy as np, sys
sys.path.insert(0, %(repo)r)
import sylph_b200
from sylph_b200 import _lib, synth
from oracle import oracle as O
L = _lib.lib()
a = sylph_b200.Context(0)
one = L.syl_pack_threads()
b = sylph_b200.Context(0)
two = L.syl_pack_threads()
assert two == max(1, one // 2), (one, two)
rb, ro = synth.reads(60000, n_comm=8, genome_len=100000, seed=%(seed)d)
rb, ro = rb.numpy(), ro.numpy().astype(np.uint64)
eh, ec, _, nd = O.sketch_reads(rb, ro, c=50)
res = {}
def work(name, ctx):
    s = ctx.sketch_sequences(rb, ro, c=50)
    res[name] = s.download() + (s.num_dup_removed, ctx.ingest_stats())
ts = [threading.Thread(target=work, args=(n, c)) for n, c in (("a", a), ("b", b))]
[t.start() for t in ts]
[t.join() for t in ts]
for n in "ab":
    h, c, dup, st = res[n]
    assert np.array_equal(h, eh) and np.array_equal(c, ec) and dup == nd, n
    assert st[1] > 0, st            # packed chunks: two contexts on one host still pack (<= 4 producers)
b.close()
assert L.syl_pack_threads() == one
print("ok", one, two)
"""


def test_packer_pool_shared_by_contexts(tmp_path):
    """two live contexts: a new packer pool gets half the one-context default; one host-memory sketch on each context,
    run at once from two threads, equals the oracle"""
    env = dict(os.environ)
    for k in ("SYL_PACK_THREADS", "SYL_HOST_INGEST", "LOCAL_WORLD_SIZE"):
        env.pop(k, None)
    env["SYL_INGEST_CHUNK"] = "65536"       # many chunks, so the pools work through the ring
    r = subprocess.run([sys.executable, "-c", PACK_SCRIPT % dict(repo=REPO, seed=11)], env=env, cwd=str(tmp_path),
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.startswith("ok"), r.stderr[-3000:]


def _device_count():
    import torch
    return torch.cuda.device_count()


def test_two_real_devices(exe, d, sk):  # noqa: F811
    if _device_count() < 2:
        pytest.skip("one CUDA device visible")
    one, _ = _sketch(exe, d, "dev1", [])
    got, _ = _sketch(exe, d, "dev01", ["--devices", "0,1"])
    assert got == one
    _same(exe, d, ["profile"] + SAMPLES + SK_SAMPLES + GENOMES, devices=("0,1",))
