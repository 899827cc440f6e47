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


@pytest.mark.parametrize("k,spec", list(T.pinned_specs()), ids=lambda v: str(v))
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
