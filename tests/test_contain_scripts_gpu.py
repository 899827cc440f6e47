"""GPU parity on scripted containment statistics (tests/contain_scripts.py): query and profile of every scripted
sample against the CPU oracle, in both formulations (per-pair count histograms, CSR), with the parameter sets each
family is built for; the two formulations bit-identical; one call of all samples (tiled join mapping), the plain
mapping and each sample alone bit-identical; the statistics launches showing which formulation ran; and the
sequential bootstrap replay (k_boot_seq) forced on every row by SYL_BOOT_REPLAY=1."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import contain_scripts as S
from tests.test_contain_gpu import compare, sort_query_rows

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FORMULATIONS = {"hist": None, "csr": "1"}


@pytest.fixture(params=list(FORMULATIONS))
def formulation(request, monkeypatch):
    """Per-pair count histograms (the default; the CSR formulation only where a count >= 256 asks for it) or the CSR
    formulation throughout (SYL_CONTAIN_CSR=1, read per call)."""
    monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)
    monkeypatch.delenv("SYL_BOOT_REPLAY", raising=False)
    if FORMULATIONS[request.param]:
        monkeypatch.setenv("SYL_CONTAIN_CSR", FORMULATIONS[request.param])
    return request.param


class Gpu:
    """The scripted world on the device: one db of every genome, one sample handle per sample."""

    def __init__(self, ctx):
        self.ctx, self.w = ctx, S.world()
        self.d = self.w.db()
        self.g = ctx.upload_genomes(self.d["kmers"], self.d["kmer_off"], self.d["tracked"], self.d["tracked_off"],
                                    self.d["gn_size"], c=1)
        self.db = ctx.build_db(self.g)
        self.smp = {n: ctx.upload_sample(*self.w.sample_arrays(n), c=1) for n in S.SAMPLES}

    def run(self, names, pseudotax, P, db=None):
        from sylph_b200.api import contain_params
        p = contain_params(pseudotax=pseudotax, **P)
        handles = [self.smp[n] for n in names]
        return self.ctx.profile(db or self.db, handles, p) if pseudotax else self.ctx.query(db or self.db, handles, p)


@pytest.fixture(scope="module")
def gpu(ctx):
    return Gpu(ctx)


@functools.lru_cache(maxsize=None)
def oracle(name, pseudotax, pi, sel=None):
    from oracle import oracle as O
    w = S.world()
    d = w.db(sel)
    P = S.params_for(name)[pi]
    return O.contain_sample(O.default_params(pseudotax=pseudotax, **P), d["kmers"], d["kmer_off"], d["tracked"],
                            d["tracked_off"], d["gn_size"], O.Sample(*w.sample_arrays(name)))


def check(rows, name, pseudotax, pi, sel=None):
    if not pseudotax:
        rows = sort_query_rows(rows)
    exp = oracle(name, pseudotax, pi, sel)
    compare(rows, exp, pseudotax)
    return len(exp)


def same(a, b, what):
    assert len(a) == len(b), (what, len(a), len(b))
    for f in a.dtype.names:
        assert np.array_equal(a[f], b[f]), (what, f)


CASES = [(n, i) for n in S.SAMPLES for i in range(len(S.params_for(n)))]


@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("name,pi", CASES)
def test_scripted_sample_against_oracle(gpu, formulation, name, pi, pseudotax):
    rows = gpu.run([name], pseudotax, S.params_for(name)[pi])
    n = check(rows, name, pseudotax, pi)
    assert n > 0


@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("name,pi", CASES)
def test_histogram_and_csr_rows_bit_identical(gpu, monkeypatch, name, pi, pseudotax):
    """Both formulations hand the same integers to stats_emit: every field of every row is equal, not just close."""
    P = S.params_for(name)[pi]
    monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)
    hist = gpu.run([name], pseudotax, P)
    monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
    csr = gpu.run([name], pseudotax, P)
    same(hist, csr, name)


PLAIN = r"""
import sys
import numpy as np
import sylph_b200
from tests.test_contain_scripts_gpu import Gpu
from tests import contain_scripts as S
g = Gpu(sylph_b200.Context(0))
np.save(sys.argv[1], g.run(S.SAMPLES, PSEUDOTAX, {"minimum_ani": 0.0}))
"""


@pytest.mark.parametrize("pseudotax", [False, True])
def test_one_call_plain_mapping_and_each_sample_alone(gpu, monkeypatch, tmp_path, pseudotax):
    """All samples in one call (the tiled (hash range, sample) join mapping; `big` sends the call to the CSR
    formulation), the same call with SYL_JOIN_PLAIN=1 (read once per process, so in a child process) and every sample
    alone: the same rows, bit for bit, and each sample's rows equal to the oracle."""
    monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)
    monkeypatch.delenv("SYL_BOOT_REPLAY", raising=False)
    P = {"minimum_ani": 0.0}
    allrows = gpu.run(S.SAMPLES, pseudotax, P)
    for si, name in enumerate(S.SAMPLES):
        sub = allrows[allrows["sample"] == si]
        alone = gpu.run([name], pseudotax, P)
        sub = sub.copy()
        sub["sample"] = 0
        same(sub, alone, name)
        check(sub, name, pseudotax, S.params_for(name).index(P))
    out = tmp_path / "plain.npy"
    env = dict(os.environ, SYL_JOIN_PLAIN="1")
    code = ("PSEUDOTAX = %r\n" % pseudotax) + PLAIN
    r = subprocess.run([sys.executable, "-c", code, str(out)], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    same(np.load(out), allrows, "plain mapping")


@pytest.mark.parametrize("pseudotax", [False, True])
def test_statistics_launches_show_the_formulation(gpu, monkeypatch, pseudotax):
    """One statistics launch per get_stats pass: a sample whose counts are all below 256 is not redone, `big` is
    redone once in the CSR formulation, and SYL_CONTAIN_CSR=1 runs it there from the start."""
    monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)
    monkeypatch.delenv("SYL_BOOT_REPLAY", raising=False)
    passes = 2 if pseudotax else 1
    ctx = gpu.ctx
    ctx.enable_timing()
    try:
        for name in S.SAMPLES:
            ctx.kernel_time("stats")
            gpu.run([name], pseudotax, {})
            _, n = ctx.kernel_time("stats")
            assert n == (2 * passes if name in S.CSR_SAMPLES else passes), (name, n)
        monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
        gpu.run(["big"], pseudotax, {})
        assert ctx.kernel_time("stats")[1] == passes
    finally:
        ctx.enable_timing(False)


@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("name", S.REPLAY_SAMPLES)
def test_boot_replay_on_every_row(gpu, formulation, monkeypatch, name, pseudotax):
    """SYL_BOOT_REPLAY=1 flags every bootstrapped row, so k_boot_seq recomputes all of them with the sequential
    WyRand stream (the path a Lemire redraw takes): rows bit-identical to the counter-based bootstrap, and == oracle."""
    P = {"minimum_ani": 0.0}
    pi = S.params_for(name).index(P)
    base = gpu.run([name], pseudotax, P)
    monkeypatch.setenv("SYL_BOOT_REPLAY", "1")
    replay = gpu.run([name], pseudotax, P)
    same(replay, base, name)
    check(replay, name, pseudotax, pi)
    want = sum(1 for _, r in S.classify(name, P) if r is not None and r["emitted"] and r["boot"] >= 50)
    assert int(replay["ci_valid"].sum()) == want and want >= 2


def test_probe_keys_above_maxkey(gpu, monkeypatch):
    """A db without the genome that holds 2^64 - 3 and 2^64 - 2: the probe sample's keys above the db's largest key
    miss (the bucket directory clamps them), and the rows equal the oracle on that db."""
    monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)
    w = gpu.w
    top = [g for g in w.local["probe"] if w.scripts[g].tag == "top_keys"]
    sel = tuple(g for g in range(len(w.scripts)) if g not in top)
    d = w.db(sel)
    g = gpu.ctx.upload_genomes(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], c=1)
    db = gpu.ctx.build_db(g)
    assert int(d["kmers"].max()) < S.MAX_KEY - 1
    for pseudotax in (False, True):
        rows = gpu.run(["probe"], pseudotax, {"minimum_ani": 0.0}, db=db)
        assert check(rows, "probe", pseudotax, S.params_for("probe").index({"minimum_ani": 0.0}), sel) > 30
