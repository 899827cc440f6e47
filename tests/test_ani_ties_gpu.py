"""ANI near-ties on the device (tests/ani_ties.py): the -m gate at a pinned ANI and one ulp either side, the profile
winner between genomes whose ANIs are adjacent doubles or equal (both genome orders), and the query order of those
genomes; in both formulations (per-pair count histograms, CSR).  The device's rows equal the correctly rounded oracle's
bit for bit.  On the MISROUNDED pins glibc is one ulp off, and the glibc oracle (the reference's arithmetic) prints
another ANI, drops the row at the gate, or gives the shared k-mers to the other genome: the device must not."""
import numpy as np
import pytest

from tests import ani_ties as T
from tests.contain_compare import compare, cr_params, sort_query_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["hist", "csr"])
def formulation(request, monkeypatch):
    monkeypatch.delenv("SYL_CONTAIN_CSR", raising=False)
    if request.param == "csr":
        monkeypatch.setenv("SYL_CONTAIN_CSR", "1")
    return request.param


def glibc_rows(case, k, pseudotax, **P):
    """the oracle's rows with the reference's glibc pow / exp"""
    from oracle import oracle as O
    d = case.db
    return O.contain_sample(O.default_params(k=k, pseudotax=pseudotax, **P), d["kmers"], d["kmer_off"], d["tracked"],
                            d["tracked_off"], d["gn_size"], O.Sample(case.hash, case.count))


def run(ctx, case, k, pseudotax, **P):
    """the device's rows of case == the correctly rounded oracle's -> (rows, oracle rows)"""
    from oracle import oracle as O
    from sylph_b200.api import contain_params
    d = case.db
    g = ctx.upload_genomes(d["kmers"], d["kmer_off"], d["tracked"], d["tracked_off"], d["gn_size"], k=k, c=1)
    db = ctx.build_db(g)
    smp = ctx.upload_sample(case.hash, case.count, k=k, c=1)
    try:
        p = contain_params(k=k, pseudotax=pseudotax, **P)
        rows = ctx.profile(db, [smp], p) if pseudotax else sort_query_rows(ctx.query(db, [smp], p))
    finally:
        smp.free()
        db.free()
        g.free()
    exp = O.contain_sample(cr_params(k=k, pseudotax=pseudotax, **P), d["kmers"], d["kmer_off"], d["tracked"],
                           d["tracked_off"], d["gn_size"], O.Sample(case.hash, case.count))
    compare(rows, exp, pseudotax)
    return rows, exp


def gate_id(g):
    return "k%d_%s_%s" % (g[0], g[1][0], "_".join(map(str, g[1][1:])))


@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("gate", T.GATES, ids=gate_id)
def test_gate_at_the_pinned_ani(ctx, formulation, gate, pseudotax):
    """-m p with RN(p / 100) == the genome's ANI keeps the row; the percent of the next double up drops it, the
    percent of the next double down keeps it."""
    k, spec, a, p, p_up, p_dn = gate
    case = T.Case([spec])
    for pct, present in ((p, True), (p_up, False), (p_dn, True)):
        rows, exp = run(ctx, case, k, pseudotax, minimum_ani=pct)
        assert len(exp) == int(present) and len(rows) == int(present), (pct, present)
        if present:
            assert float(rows["final_est_ani"][0]) == a


def pair_id(p):
    return "k%d_%s_%s" % (p[0], "_".join(map(str, p[1][1:])), "_".join(map(str, p[2][1:])))


PAIRS = [("adjacent",) + p for p in T.WINNER_PAIRS] + [("equal",) + p for p in T.TIE_PAIRS]
SHARED = 3


@pytest.mark.parametrize("swap", [False, True], ids=["a_first", "b_first"])
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: p[0] + "_" + pair_id(p[1:]))
def test_winner_between_near_tied_genomes(ctx, formulation, pair, swap):
    """Two genomes sharing SHARED hit k-mers: in pass 2 they all go to the genome of the greater ANI (the lower genome
    index on equal ANIs), and the other counts them as lost.  Rows == oracle: presence, contain, kmers_lost and the
    abundances."""
    kind, k, a, b = pair
    specs = [b, a] if swap else [a, b]
    rows, exp = run(ctx, T.Case(specs, shared=SHARED), k, True, minimum_ani=0.0)
    ani = [T.glibc_ani(s, k) for s in specs]
    win = 0 if ani[0] >= ani[1] else 1
    assert (ani[0] == ani[1]) == (kind == "equal")
    lost = {int(r["genome"]): int(r["kmers_lost"]) for r in rows}
    assert lost == {win: 0, 1 - win: SHARED}


@pytest.mark.parametrize("swap", [False, True], ids=["a_first", "b_first"])
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: p[0] + "_" + pair_id(p[1:]))
def test_query_order_of_near_tied_genomes(ctx, formulation, pair, swap):
    """query rows in ANI-descending order: the genome of the greater ANI first, on equal ANIs the lower index first
    (the reference's stable sort)."""
    kind, k, a, b = pair
    specs = [b, a] if swap else [a, b]
    rows, exp = run(ctx, T.Case(specs), k, False, minimum_ani=0.0)
    ani = [T.glibc_ani(s, k) for s in specs]
    want = [0, 1] if ani[0] >= ani[1] else [1, 0]
    assert [int(g) for g in rows["genome"]] == want == [e.genome for e in exp]
    assert np.array_equal(rows["final_est_ani"], [ani[i] for i in want])


def spec_id(v):
    return "_".join(map(str, v[1:])) if isinstance(v, tuple) else str(v)


@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("pin", T.MISROUNDED, ids=lambda m: "k%d_%s_%s" % (m[0], m[1][0], spec_id(m[1])))
def test_ani_where_glibc_misrounds(ctx, formulation, pin, pseudotax):
    """The device's ANI is the correctly rounded one; the glibc oracle's is one ulp away (the naive ANI too where it
    is final)."""
    k, spec, a_glibc, a_cr = pin
    case = T.Case([spec])
    rows, _ = run(ctx, case, k, pseudotax, minimum_ani=0.0)
    ref = glibc_rows(case, k, pseudotax, minimum_ani=0.0)
    assert len(rows) == len(ref) == 1
    assert float(rows["final_est_ani"][0]) == a_cr and ref[0].final_est_ani == a_glibc != a_cr
    if spec[0] == "naive":
        assert float(rows["naive_ani"][0]) == a_cr and ref[0].naive_ani == a_glibc


@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("gate", T.MISROUNDED_GATES, ids=lambda g: "k%d_%s_%s" % (g[0], g[1][0], spec_id(g[1])))
def test_gate_where_glibc_misrounds(ctx, formulation, gate, pseudotax):
    """-m p with RN(p / 100) == the correctly rounded ANI: the device keeps the row, the glibc oracle (whose ANI is
    the double below) drops it."""
    k, spec, p = gate
    case = T.Case([spec])
    rows, _ = run(ctx, case, k, pseudotax, minimum_ani=p)
    assert len(rows) == 1 and float(rows["final_est_ani"][0]) == p / 100.0
    assert glibc_rows(case, k, pseudotax, minimum_ani=p) == []


@pytest.mark.parametrize("pair", T.MISROUNDED_WINNERS, ids=lambda w: "k%d_%s_%s" % (w[0], spec_id(w[1]), spec_id(w[2])))
def test_winner_where_glibc_misrounds(ctx, formulation, pair):
    """Genomes A (index 0) and B sharing SHARED hit k-mers whose ANIs are equal or adjacent doubles, where one glibc
    misrounding reverses the order: in pass 2 the device gives the shared k-mers to the correctly rounded winner, the
    glibc oracle to the other genome."""
    k, a, b, win_glibc, win_cr = pair
    case = T.Case([a, b], shared=SHARED)
    rows, _ = run(ctx, case, k, True, minimum_ani=0.0)
    lost = {int(r["genome"]): int(r["kmers_lost"]) for r in rows}
    assert win_cr != win_glibc and lost == {win_cr: 0, 1 - win_cr: SHARED}
    ref = glibc_rows(case, k, True, minimum_ani=0.0)
    assert {e.genome: e.kmers_lost for e in ref} == {win_glibc: 0, 1 - win_glibc: SHARED}
