"""CPU: how a read or pair sketch is cut into hash-range parts within a device memory budget
(sylph_b200/csrc/sample_parts.hpp, built on the host).  One part whenever the one-pass estimate fits; otherwise the
fewest parts (at most 64) whose largest pass fits.  The parts are disjoint, contiguous, cover [0, thr) and start on
bucket boundaries of the one-pass group map, every part's event array stays below 2^32-2 entries, and a budget that
64 parts exceed is refused with the bytes needed."""
import os
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "sylph_b200", "csrc")
U64 = 2**64 - 1
MAX_EVENTS = 2**32 - 2
GB = 10**9


@pytest.fixture(scope="module")
def plan_exe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("sample_parts") / "sample_parts_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", CSRC, "-o", exe,
                           os.path.join(REPO, "tests", "cpp", "sample_parts_check.cpp")])
    return exe


def plan(exe, cases):
    """cases: [(bases, records, mates, k, c, grouped, budget, fixed, forced)] -> per case ("ok", head, parts) |
    ("events",) | ("oom", need)"""
    inp = "\n".join(" ".join(str(int(x)) for x in cs) for cs in cases) + "\n"
    lines = subprocess.run([exe], input=inp, stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines()
    out, i = [], 0
    while i < len(lines):
        f = lines[i].split()
        i += 1
        if f[0] == "events":
            out.append(("events",))
        elif f[0] == "oom":
            out.append(("oom", int(f[1])))
        else:
            thr, nbk, mb, need, n = map(int, f[1:])
            parts = [tuple(map(int, lines[i + j].split())) for j in range(n)]
            i += n
            out.append(("ok", dict(thr=thr, nbk=nbk, Mb=mb, need=need), parts))
    assert len(out) == len(cases)
    return out


def bucket(h, mb, nbk):
    return min((h * mb) >> 64, nbk - 1)


def check_parts(head, parts, budget, fixed, grouped=True):
    thr, nbk, mb = head["thr"], head["nbk"], head["Mb"]
    assert parts[0][0] == 0 and parts[-1][1] == thr
    for (lo, hi, g0, ng, ev, by), nxt in zip(parts, parts[1:] + [None]):
        assert lo <= hi
        if nxt is not None:
            assert nxt[0] == hi                       # contiguous and disjoint
        assert ev < MAX_EVENTS
        assert fixed + by <= head["need"]
        if budget:
            assert head["need"] <= budget
        if lo > 0 and lo < thr:                       # a bucket starts at lo
            assert bucket(lo, mb, nbk) > bucket(lo - 1, mb, nbk)
        if lo < hi and grouped:                       # the part's hashes fall in its groups
            assert g0 == bucket(lo, mb, nbk) // 32
            assert g0 <= bucket(hi - 1, mb, nbk) // 32 < g0 + ng
        if not grouped:
            assert ng == 0


def test_one_part_whenever_the_estimate_fits(plan_exe):
    cases = []
    for bases, reads, mates, c in [(10**6, 6667, 1, 200), (6 * 10**8, 2 * 10**6, 2, 200), (10**9, 6666667, 1, 50),
                                   (0, 0, 1, 200), (150, 1, 1, 1)]:
        cases.append((bases, reads, mates, 31, c, 1, U64, 0, 0))
    for r in plan(plan_exe, cases):
        assert r[0] == "ok" and len(r[2]) == 1
        check_parts(r[1], r[2], U64, 0)
    # exactly the one-pass need: one part; one byte less: more parts, each fitting
    (_, head, parts), = plan(plan_exe, [(10**9, 6666667, 1, 31, 200, 1, U64, 10**8, 0)])
    need1 = head["need"]
    (_, h1, p1), (_, h2, p2) = plan(plan_exe, [(10**9, 6666667, 1, 31, 200, 1, need1, 10**8, 0),
                                              (10**9, 6666667, 1, 31, 200, 1, need1 - 1, 10**8, 0)])
    assert len(p1) == 1 and len(p2) == 2 and h2["need"] <= need1 - 1
    check_parts(h2, p2, need1 - 1, 10**8)


def test_parts_cover_the_threshold_on_bucket_boundaries(plan_exe):
    cases = []
    for bases, reads, mates, k, c, grouped in [(10**9, 6666667, 1, 31, 200, 1), (6 * 10**8, 2 * 10**6, 2, 21, 50, 1),
                                               (3 * 10**6, 10**4, 2, 31, 1000, 0), (5 * 10**4, 300, 1, 31, 3, 1),
                                               (10**10, 10**5, 1, 31, 7, 1)]:
        for P in (2, 3, 7, 16, 64, 100000):
            cases.append((bases, reads, mates, k, c, grouped, U64, 0, P))
    for cs, r in zip(cases, plan(plan_exe, cases)):
        assert r[0] == "ok", cs
        head, parts = r[1], r[2]
        assert len(parts) == min(cs[8], head["nbk"])   # at most one part per bucket
        check_parts(head, parts, 0, 0, grouped=bool(cs[5]))


def test_budget_picks_the_fewest_parts_that_fit(plan_exe):
    base = (10**9, 6666667, 1, 31, 200, 1)
    (_, h1, _), = plan(plan_exe, [base + (U64, 0, 0)])
    per_event = (h1["need"] - (16 << 20)) / (10**9 / 200)
    assert 90 < per_event < 160                     # about 120 B per expected event, derived from the allocations
    cases = [base + (h1["need"] // d, 0, 0) for d in (2, 3, 4)]
    prev = 1
    for (tag, head, parts), cs in zip(plan(plan_exe, cases), cases):
        assert tag == "ok" and head["need"] <= cs[6]
        assert len(parts) >= max(prev, 2)
        prev = len(parts)
        check_parts(head, parts, cs[6], 0)
        (t2, h2, p2), = plan(plan_exe, [base + (U64, 0, len(parts) - 1)])
        assert h2["need"] > cs[6]                   # one part fewer would not fit


def test_budget_below_the_floor_is_refused(plan_exe):
    r = plan(plan_exe, [(10**9, 6666667, 1, 31, 200, 1, 10**6, 0, 0),
                        (10**9, 6666667, 1, 31, 200, 1, 10**10, 10**10, 0),
                        (6 * 10**8, 2 * 10**6, 2, 31, 200, 1, 1, 0, 0)])
    for x, budget in zip(r, (10**6, 10**10, 1)):
        assert x[0] == "oom" and x[1] > budget


def test_a_terabase_plans_without_overflow(plan_exe):
    """10^12 bases at c from 1 to 1000: a valid plan, or a refusal, never a wrapped size"""
    cs = [1, 2, 3, 5, 10, 20, 50, 100, 200, 500, 1000]
    cases = [(10**12, 10**12 // 150, 1, 31, c, 1, budget, 10**9, 0) for c in cs for budget in (80 * GB, U64)]
    cases += [(10**12, 10**12 // 150, 2, 21, c, 1, 80 * GB, 0, 64) for c in cs]
    for cs_, r in zip(cases, plan(plan_exe, cases)):
        c, budget = cs_[4], cs_[6]
        n_exp = (10**12 - cs_[1] * cs_[2] * (cs_[3] - 1)) // c
        if r[0] == "ok":
            head, parts = r[1], r[2]
            check_parts(head, parts, budget if not cs_[8] else 0, cs_[7])
            assert 1 <= len(parts) <= 64 and head["thr"] == U64 // c
            assert sum(p[4] for p in parts) >= n_exp      # the parts' slots and lists hold every expected event
            assert head["need"] < 2**63
        elif r[0] == "oom":
            assert budget < U64 and budget < r[1] < 2**63
        else:
            assert n_exp / 64 > MAX_EVENTS / 2            # events refused only where a 64th of them approaches 2^32
    # c = 1000 fits a terabase into 80 GB in a few parts; c = 1 cannot be cut finely enough
    got = dict(zip([(x[4], x[6]) for x in cases[:22]], plan(plan_exe, cases[:22])))
    assert got[(1000, 80 * GB)][0] == "ok" and 1 < len(got[(1000, 80 * GB)][2]) <= 64
    assert got[(1, U64)][0] == "events"
