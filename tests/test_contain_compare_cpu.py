"""The containment comparator (tests/contain_compare.py) without a GPU: fed the correctly rounded oracle's own rows,
laid out as the device returns them, for every scripted family (tests/contain_scripts.py) and every ANI pin
(tests/ani_ties.py), it passes; moved by one ulp in any float field of a row, it fails.  So no slack can come back into
the comparison unnoticed.  On the pins where glibc misrounds, the glibc oracle's rows fail it too."""
import math

import numpy as np
import pytest

from tests import ani_ties as T
from tests import contain_scripts as S
from tests.contain_compare import FLOATS, compare, cr_params, sort_query_rows


def as_rows(exp, sample=0):
    """oracle rows in the device's row layout (sylph_b200.api.ANI_ROW_DTYPE)"""
    from sylph_b200.api import ANI_ROW_DTYPE
    rows = np.zeros(len(exp), ANI_ROW_DTYPE)
    for i, e in enumerate(exp):
        r = rows[i]
        r["sample"] = sample
        for f in ("genome", "lambda_status", "ci_valid", "contain", "glen", "kmers_lost", "rel_abund", "seq_abund") + FLOATS:
            r[f] = getattr(e, f)
        r["lambda"] = e.lambda_
        r["ci"] = list(e.ci)
    return rows


def contain(d, hc, pseudotax, k=31, cr=True, **P):
    from oracle import oracle as O
    p = cr_params(k=k, pseudotax=pseudotax, **P) if cr else O.default_params(k=k, pseudotax=pseudotax, **P)
    return O.contain_sample(p, d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], O.Sample(*hc))


def cases():
    """(id, k, db, (hash, count), P): every scripted sample against the scripted db, and every pinned genome (pairs
    sharing hit k-mers)"""
    w = S.world()
    d = w.db()
    for name in S.SAMPLES:
        yield "script_" + name, 31, d, w.sample_arrays(name), {"minimum_ani": 0.0}
    for k, spec in T.pinned_specs():
        c = T.Case([spec])
        yield "pin_k%d_%s" % (k, "_".join(map(str, spec))), k, c.db, (c.hash, c.count), {"minimum_ani": 0.0}
    for k, a, b, *_ in T.WINNER_PAIRS + T.TIE_PAIRS + T.MISROUNDED_WINNERS:
        c = T.Case([a, b], shared=3)
        yield "pair_k%d_%s_%s" % (k, "_".join(map(str, a[1:])), "_".join(map(str, b[1:]))), k, c.db, (c.hash, c.count), {"minimum_ani": 0.0}


CASES = list(cases())


def moved(rows, i, field, j, up):
    """a copy of rows with field (element j of ci) of row i one ulp up or down"""
    out = rows.copy()
    v = float(out[field][i] if j is None else out[field][i][j])
    v = math.nextafter(v, math.inf if up else -math.inf)
    if j is None:
        out[field][i] = v
    else:
        out[field][i][j] = v
    return out


def checked_fields(e, pseudotax):
    """the float fields compare() defines for oracle row e"""
    fields = [(f, None) for f in FLOATS]
    if e.lambda_status == 2:
        fields.append(("lambda", None))
    if e.ci_valid:
        fields += [("ci", j) for j in range(4)]
    if pseudotax:
        fields += [("rel_abund", None), ("seq_abund", None)]
    return fields


@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_rows_pass_and_one_ulp_fails(case, pseudotax):
    _, k, d, hc, P = case
    exp = contain(d, hc, pseudotax, k=k, **P)
    assert exp
    rows = as_rows(exp)
    compare(sort_query_rows(rows) if not pseudotax else rows, exp, pseudotax)
    # the row with the most fields defined: a lambda row with a bootstrap interval where there is one
    i = max(range(len(exp)), key=lambda n: (exp[n].ci_valid, exp[n].lambda_status == 2, -n))
    fields = checked_fields(exp[i], pseudotax)
    for field, j in fields:
        for up in (False, True):
            with pytest.raises(AssertionError):
                compare(moved(rows, i, field, j, up), exp, pseudotax)


def test_the_guard_reaches_every_float_field():
    """Across the cases, the mutated row has lambda, a bootstrap interval and (in profile) abundances: every float
    field compare() reads is moved somewhere."""
    seen = set()
    for _, k, d, hc, P in CASES[:len(S.SAMPLES)]:
        exp = contain(d, hc, True, k=k, **P)
        i = max(range(len(exp)), key=lambda n: (exp[n].ci_valid, exp[n].lambda_status == 2, -n))
        seen |= {(f, j) for f, j in checked_fields(exp[i], True)}
    assert seen == {(f, None) for f in FLOATS + ("lambda", "rel_abund", "seq_abund")} | {("ci", j) for j in range(4)}


@pytest.mark.parametrize("pin", T.MISROUNDED, ids=lambda m: "k%d_%s" % (m[0], "_".join(map(str, m[1]))))
def test_glibc_rows_fail_where_glibc_misrounds(pin):
    """the reference's arithmetic (the oracle's glibc mode) is one ulp off on these pins, and compare() sees it"""
    k, spec, _, _ = pin
    c = T.Case([spec])
    exp = contain(c.db, (c.hash, c.count), False, k=k, minimum_ani=0.0)
    ref = contain(c.db, (c.hash, c.count), False, k=k, cr=False, minimum_ani=0.0)
    with pytest.raises(AssertionError):
        compare(as_rows(ref), exp, False)
