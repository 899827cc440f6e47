"""CPU suite: scripted containment statistics (tests/contain_scripts.py).

Every sample reaches the get_stats branches it is built for (read off the scripts by the classifier); the C oracle and
the pure-Python restatement (oracle/pyref.py) agree on every scripted pair, query and profile, with the parameter sets
the GPU suite uses; and the oracle's rows agree with what the classifier derives from the count multisets."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import pyref as R
from tests import contain_scripts as S


def _has(t, **want):
    for k, v in want.items():
        assert t[k] >= v, (k, t[k], v, dict(t))


def test_families_reach_their_classes():
    t = S.tally("median")
    _has(t, n_even=7, n_odd=7, status_1=10, status_2=4, final_mean=4, final_median=6, final_lambda=4, cut_removes=12)
    for m in (1, 2, 3, 14, 15, 29, 30):
        assert t["median_%d" % m] == 2, m
    assert S.tally("median", {"mean_coverage": 1})["final_mean_param"] == 6
    t = S.tally("cut")
    assert all(t["median_%d" % m] == 1 for m in range(1, 30)) and t["cut_removes"] == 29
    t = S.tally("ratio")
    _has(t, low_distinct=2, low_nz=1, low_p1_absent=4, low_count_p1=2, status_2=5, **{"mode_8-14": 2})
    t1 = S.tally("ratio", {"min_count_correct": 1.0}, with_boot=False)
    assert t1["status_2"] == t["status_2"] + 2 and t1["low_count_p1"] == 0          # cp1 = 1 and 2 pass at 1
    t = S.tally("boot")
    _has(t, status_2=21, no_zero=2, **{"mode_1-3": 5, "mode_4-7": 5, "mode_8-14": 3})
    for v in (3, 7, 8, 11, 15):
        assert t["max_kept_%d" % v] >= 1, v
    assert t["emitted"] == 21 and t["filtered"] == 0
    t = S.tally("suc")
    assert (t["boot_50"], t["boot_49"], t["boot_45"]) == (2, 1, 1)
    t = S.tally("huge", with_boot=False)
    assert t["status_2"] == 1 and t["mode_1-3"] == 1
    t = S.tally("filter")
    assert (t["emitted"], t["filtered"]) == (3, 1)
    assert S.tally("filter", {"minimum_ani": 100.0})["emitted"] == 2                 # glen50 and ani_exactly_1
    t = S.tally("big")
    _has(t, csr=11, sum_wraps=4, status_2=1, cut_removes=2)
    assert t["median_%d" % (2**31)] == 1 and t["median_%d" % (2**32 - 1)] == 1
    t = S.tally("probe")
    assert t["emitted"] == 38 and t["csr"] == 0
    for name in S.SAMPLES:                                                            # only `big` needs CSR
        assert (S.tally(name, with_boot=False)["csr"] > 0) == (name in S.CSR_SAMPLES), name


def test_scripts_are_well_formed():
    w = S.world()
    keys = [k for s in w.scripts for k in s.kmers + s.tracked]
    assert max(keys) == S.MAX_KEY and min(keys) == 0
    for name in S.SAMPLES:
        h, c = w.sample_arrays(name)
        assert len(np.unique(h)) == len(h) and int(h.max()) < 2**64 - 1
        if name not in S.CSR_SAMPLES:
            assert int(c.max()) < S.COV_BINS, name
    for name in S.REPLAY_SAMPLES:
        assert all(len(w.scripts[g].kmers) <= S.REPLAY_MAX for g in w.local[name])


def local_db(name):
    w = S.world()
    sel = w.local[name]
    return w.db(sel), [dict(kmers=w.scripts[g].kmers, tracked=w.scripts[g].tracked, gn_size=int(gs))
                       for g, gs in zip(sel, w.db(sel)["gn_size"])]


def oracle_local(name, pseudotax, P):
    d, _ = local_db(name)
    h, c = S.world().sample_arrays(name)
    return O.contain_sample(O.default_params(pseudotax=pseudotax, **P), d["kmers"], d["kmer_off"], d["tracked"],
                            d["tracked_off"], d["gn_size"], O.Sample(h, c))


CASES = [(n, i, pt) for n in S.SAMPLES if n != "huge" for i in range(len(S.params_for(n))) for pt in (False, True)]


@pytest.mark.parametrize("name,pi,pseudotax", CASES)
def test_oracle_equals_pyref(name, pi, pseudotax):
    """All integer fields equal; floats within 1e-12 relative; CI columns too (pyref bootstraps every row here)."""
    P = S.params_for(name)[pi]
    got = oracle_local(name, pseudotax, P)
    _, genomes = local_db(name)
    kw = {k: (bool(v) if k in ("no_ci", "no_adj", "mean_coverage") else v) for k, v in P.items()}
    exp = R.contain_sample(genomes, S.world().samples[name], pseudotax=pseudotax, **kw)
    assert [r.genome for r in got] == [e["genome"] for e in exp]
    close = lambda a, b: abs(a - b) <= 1e-12 * max(1.0, abs(b))  # noqa: E731
    for r, e in zip(got, exp):
        assert (r.contain, r.glen, r.median_cov) == (e["contain"], e["glen"], e["median_cov"])
        assert ["LOW", "HIGH", "LAMBDA"][r.lambda_status] == e["status"]
        assert r.kmers_lost == (e["kmers_lost"] if pseudotax else -1)
        for f in ("naive_ani", "final_est_ani", "final_est_cov", "mean_cov"):
            assert close(getattr(r, f), e[f]), (f, getattr(r, f), e[f])
        if e["lam"] is not None:
            assert close(r.lambda_, e["lam"])
        assert bool(r.ci_valid) == (e["ci"] is not None)
        if e["ci"]:
            assert all(close(a, b) for a, b in zip(r.ci, e["ci"]))
        if pseudotax:
            assert close(r.rel_abund, e["rel_abund"]) and close(r.seq_abund, e["seq_abund"])


@pytest.mark.parametrize("name", S.SAMPLES)
def test_oracle_rows_follow_the_classifier(name):
    """Query at minimum_ani = 0: the oracle emits a row exactly for the classifier's emitted pairs, with its status,
    median and hit count; mean_cov * contain rounds to the kept sum wrapped mod 2^32; the CI is valid exactly when the
    classifier counts 50 or more successful bootstrap iterations."""
    P = {"minimum_ani": 0.0}
    cls = {g - S.world().local[name][0]: r for g, r in S.classify(name, P, with_boot=name != "huge")}
    got = {r.genome: r for r in oracle_local(name, False, P)}
    assert set(got) == {g for g, r in cls.items() if r is not None and r["emitted"]}
    for g, r in got.items():
        c = cls[g]
        assert (r.lambda_status, r.median_cov, r.contain) == (c["status"], c["median"], c["n"])
        assert int(round(r.mean_cov * r.contain)) == c["sum"], (g, r.mean_cov, c["sum"])
        if c["boot"] is not None:
            assert bool(r.ci_valid) == (c["boot"] >= 50), (g, c["boot"])
    if name == "huge":
        assert [r.ci_valid for r in got.values()] == [1]


def test_profile_winner_cases():
    """The winner family in the oracle: a tracked-only winner takes its k-mers from the loser, a tracked genome that
    is not a pass-1 survivor takes none; of three tied genomes the first keeps the shared k-mers; derep keeps
    floor(t * glen) reassigned k-mers and drops one more."""
    w = S.world()
    tags = [w.scripts[g].tag for g in w.local["winner"]]
    for ra in (99.0, 95.0):
        rows = {tags[r.genome]: r for r in oracle_local("winner", True, {"redundant_ani": ra})}
        assert rows["tracked_loser_B"].kmers_lost == 5 and rows["tracked_keeper_B"].kmers_lost == 0
        assert "tracked_filtered_A" not in rows
        assert rows["tie3_0"].kmers_lost == 0 and rows["tie3_1"].kmers_lost == 10 and rows["tie3_2"].kmers_lost == 10
        for r2 in (99.0, 95.0):
            d = int(np.floor((r2 / 100.0) ** S.K * 100))
            assert ("derep%d_B_%d" % (r2, d) in rows) == (r2 <= ra)
            assert ("derep%d_B_%d" % (r2, d + 1) in rows) == (r2 < ra)
