"""ANI near-ties without a GPU: the correctly rounded pow / exp of the device (sylph_b200/csrc/crmath.cuh, built for
the host) against libquadmath and Python's decimal, and the pinned near-tie inputs of tests/ani_ties.py against the
oracle, pyref, glibc and the decimal reference."""
import math
import os
import re
import subprocess
from decimal import Decimal

import numpy as np
import pytest

from tests import ani_ties as T

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "sylph_b200", "csrc")


@pytest.fixture(scope="module")
def crmath_exe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("crmath") / "crmath_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", CSRC, "-o", exe, os.path.join(REPO, "tests", "cpp", "crmath_check.cpp"),
                           "-lquadmath"])
    return exe


def cr_eval(exe, calls):
    """[("pow", x, c) | ("exp", z)] -> the host build's cr_pow / cr_exp"""
    text = "".join("pow %s %s\n" % (a[1].hex(), a[2].hex()) if a[0] == "pow" else "exp %s\n" % a[1].hex() for a in calls)
    out = subprocess.run([exe, "eval"], input=text, stdout=subprocess.PIPE, text=True, check=True).stdout.split()
    assert len(out) == len(calls)
    return [float.fromhex(v) for v in out]


def test_crmath_sweep_against_quad(crmath_exe):
    """10^6 inputs of each shape, each refined from libm's value and from it moved by up to 2 ulp either way: every
    refinement is the correctly rounded value.  glibc's own misroundings are the count libm_bad (0.52-ulp pow)."""
    out = subprocess.run([crmath_exe, "sweep", "1000000"], stdout=subprocess.PIPE, text=True, check=True, timeout=600).stdout
    tallies = dict(re.findall(r"tally (\w+) (.*)", out))
    assert set(tallies) == {"naive", "exp", "adjusted"}, out
    for shape, t in tallies.items():
        f = dict(kv.split("=") for kv in t.split())
        assert int(f["n"]) == 1000000 and int(f["cr_bad"]) == 0 and int(f["undecided"]) == 0, (shape, t)
        assert int(f["libm_bad"]) < 5000, (shape, t)   # glibc misrounds about 1 in 1000 of these


def shapes(n, seed=11):
    """n seeded inputs of each shape (naive pow, exp(-lambda), adjusted pow), as in crmath_check's sweep"""
    rng = np.random.default_rng(seed)
    calls = []
    for i in range(n):
        c = 1.0 / (21 if i & 1 else 31)
        gl = int(rng.integers(50, 1 << 24))
        calls.append(("pow", int(rng.integers(1, gl + 1)) / gl, c))
        cm = int(rng.integers(3, 100000))
        lam = int(rng.integers(3, cm + 1)) / cm * int(rng.integers(2, 17))
        calls.append(("exp", -lam))
        nfull = int(rng.integers(50, 1 << 24))
        calls.append(("pow", int(rng.integers(1, nfull + 1)) / (1.0 - math.exp(-lam)) / nfull, c))
    return calls


def decimal_of(call):
    return T.cr_pow(call[1], call[2]) if call[0] == "pow" else T.cr_exp(call[1])


def test_crmath_against_decimal(crmath_exe):
    """The host build against the 50-digit decimal reference on 6000 seeded inputs and on every pinned tuple's pow /
    exp calls."""
    calls = shapes(2000) + T.pinned_calls()
    got = cr_eval(crmath_exe, calls)
    bad = [(c, g.hex()) for c, g in zip(calls, got) if g != decimal_of(c)]
    assert not bad, bad[:5]


def test_crmath_log_table_and_ln2():
    """crmath.cuh's double-double log(1 + j/128) table and log 2: hi the nearest double, lo the nearest double to
    the rest."""
    import decimal
    ctx = decimal.Context(prec=60)
    src = open(os.path.join(CSRC, "crmath.cuh")).read()
    body = src[src.index("#define CRM_LOG_TAB {"):src.index("#if defined(__CUDACC__)\n__constant__")]
    vals = [float.fromhex(v) for v in re.findall(r"-?0x[0-9a-f.]+p[-+]\d+", body)]
    assert len(vals) == 256

    def split(v):
        hi = float(v)
        return hi, float(ctx.subtract(v, Decimal(hi)))

    for j in range(128):
        assert (vals[2 * j], vals[2 * j + 1]) == split(ctx.ln(1 + Decimal(j) / 128)), j
    ln2 = re.search(r"ln2 = \{(\S+), (\S+)\}", src)
    assert (float.fromhex(ln2.group(1)), float.fromhex(ln2.group(2))) == split(ctx.ln(Decimal(2)))


@pytest.mark.parametrize("k,spec", list(T.pinned_specs(misrounded=False)), ids=lambda v: str(v))
def test_pin_oracle_and_pyref_reproduce_the_ani(k, spec):
    """The oracle's and pyref's rows for the pinned genome carry its glibc ANI bit for bit, and glibc's value is the
    correctly rounded one at every pow / exp call along the way."""
    from oracle import oracle as O
    from oracle import pyref as R
    a = T.glibc_ani(spec, k)
    assert a == T.cr_ani(spec, k)
    for call in T.calls_of(spec, k):
        glibc = call[1] ** call[2] if call[0] == "pow" else math.exp(call[1])
        assert glibc == decimal_of(call), call
    case = T.Case([spec])
    d = case.db
    rows = O.contain_sample(O.default_params(k=k, minimum_ani=0.0, no_ci=1), d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"],
                            d["gn_size"], O.Sample(case.hash, case.count))
    assert len(rows) == 1 and rows[0].final_est_ani == a
    assert rows[0].lambda_status == (1 if spec[0] == "naive" else 2)
    r = R.get_stats(d["kmers"].tolist(), case.sample, k=k, min_ani=0.0, no_ci=True)
    assert r["final_est_ani"] == a


@pytest.mark.parametrize("gate", T.GATES, ids=lambda g: str(g[:2]))
def test_gate_percents_map_to_the_gate(gate):
    k, spec, a, p, p_up, p_dn = gate
    assert T.glibc_ani(spec, k) == a
    assert p / 100.0 == a
    assert p_up / 100.0 == math.nextafter(a, math.inf)
    assert p_dn / 100.0 == math.nextafter(a, -math.inf)


def test_pairs_are_adjacent_or_equal():
    assert T.WINNER_PAIRS and T.TIE_PAIRS
    for k, a, b in T.WINNER_PAIRS:
        assert math.nextafter(T.glibc_ani(a, k), math.inf) == T.glibc_ani(b, k), (k, a, b)
    for k, a, b in T.TIE_PAIRS:
        assert T.glibc_ani(a, k) == T.glibc_ani(b, k) and a != b, (k, a, b)


def misrounded_call(spec, k):
    """the pow / exp calls along spec's ANI where glibc and the decimal reference differ"""
    return [c for c in T.calls_of(spec, k) if (c[1] ** c[2] if c[0] == "pow" else math.exp(c[1])) != decimal_of(c)]


@pytest.mark.parametrize("pin", T.MISROUNDED, ids=lambda m: "k%d_%s" % (m[0], "_".join(map(str, m[1]))))
def test_misrounded_pin_against_decimal_and_glibc(crmath_exe, pin):
    """glibc's ANI and the correctly rounded one are the pinned adjacent doubles, a glibc call along the way is the
    misrounded one, and crmath.cuh's host build rounds every call as decimal does.  The oracle and pyref print
    glibc's ANI in their default mode and the correctly rounded one in their correctly rounded mode."""
    from oracle import oracle as O
    from oracle import pyref as R
    k, spec, a_glibc, a_cr = pin
    assert T.glibc_ani(spec, k) == a_glibc and T.cr_ani(spec, k) == a_cr
    assert a_glibc in (math.nextafter(a_cr, math.inf), math.nextafter(a_cr, -math.inf))
    assert misrounded_call(spec, k)
    calls = T.calls_of(spec, k)
    assert cr_eval(crmath_exe, calls) == [decimal_of(c) for c in calls]
    case = T.Case([spec])
    d = case.db
    for cr, a in ((0, a_glibc), (1, a_cr)):
        rows = O.contain_sample(O.default_params(k=k, minimum_ani=0.0, no_ci=1, cr_math=cr), d["kmers"], d["kmer_off"],
                                d["tracked"], d["tracked_off"], d["gn_size"], O.Sample(case.hash, case.count))
        assert len(rows) == 1 and rows[0].final_est_ani == a
        r = R.get_stats(d["kmers"].tolist(), case.sample, k=k, min_ani=0.0, no_ci=True, cr_math=bool(cr))
        assert r["final_est_ani"] == a


@pytest.mark.parametrize("gate", T.MISROUNDED_GATES, ids=lambda g: "k%d_%s" % (g[0], "_".join(map(str, g[1]))))
def test_misrounded_gate_keeps_only_the_correctly_rounded_row(gate):
    """RN(p / 100) is the correctly rounded ANI and glibc's ANI the double below it: at -m p the correctly rounded
    oracle keeps the row and the glibc oracle drops it."""
    from oracle import oracle as O
    k, spec, p = gate
    a = T.cr_ani(spec, k)
    assert p / 100.0 == a and T.glibc_ani(spec, k) == math.nextafter(a, -math.inf)
    case = T.Case([spec])
    d = case.db
    for cr in (0, 1):
        rows = O.contain_sample(O.default_params(k=k, minimum_ani=p, cr_math=cr), d["kmers"], d["kmer_off"], d["tracked"],
                                d["tracked_off"], d["gn_size"], O.Sample(case.hash, case.count))
        assert len(rows) == cr


@pytest.mark.parametrize("pair", T.MISROUNDED_WINNERS, ids=lambda w: "k%d_%s_%s" % (w[0], w[1][1], w[2][1]))
def test_misrounded_winner_differs(pair):
    """A (genome 0) and B: the pass-2 winner is the pinned one in each mode (the greater ANI, A on equal ANIs), in
    the decimal / glibc restatement and in the oracle."""
    from oracle import oracle as O
    k, a, b, win_glibc, win_cr = pair
    assert win_glibc != win_cr
    for ani, win in (((T.glibc_ani(a, k), T.glibc_ani(b, k)), win_glibc), ((T.cr_ani(a, k), T.cr_ani(b, k)), win_cr)):
        assert abs(ani[0] - ani[1]) <= math.ulp(ani[0])
        assert (0 if ani[0] >= ani[1] else 1) == win
    case = T.Case([a, b], shared=3)
    d = case.db
    for cr, win in ((0, win_glibc), (1, win_cr)):
        rows = O.contain_sample(O.default_params(k=k, pseudotax=True, minimum_ani=0.0, cr_math=cr), d["kmers"],
                                d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], O.Sample(case.hash, case.count))
        assert {r.genome: r.kmers_lost for r in rows} == {win: 0, 1 - win: 3}
