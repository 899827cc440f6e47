"""Containment rows against the CPU oracle, field for field and bit for bit (a test helper module, not a conftest).

The device rounds every ANI's pow and exp correctly (sylph_b200/csrc/crmath.cuh), so its rows are held to the oracle
in its correctly rounded mode (`cr_params`: libquadmath's powq / expq rounded to the nearest double, sylph_oracle.h
cr_math), where they must agree in every bit, ANIs and bootstrap percentiles included.  The oracle's default mode calls
glibc as the reference does; it differs from the correctly rounded mode where glibc misrounds (about 1 in 1000 pow /
exp calls), and tests/ani_ties.py pins inputs where that difference decides a row or a winner.
"""


def cr_params(**kw):
    """oracle parameters (O.default_params keywords) in the correctly rounded mode the device's rows must equal"""
    from oracle import oracle as O
    return O.default_params(cr_math=1, **kw)


def oracle_rows(db, sample_hc, pseudotax, nthreads=1, **kw):
    """the correctly rounded oracle's rows of one sample (hashes, counts) against db (the download() dict layout)"""
    from oracle import oracle as O
    return O.contain_sample(cr_params(pseudotax=pseudotax, **kw), db["kmers"], db["kmer_off"], db["tracked"],
                            db["tracked_off"], db["gn_size"], O.Sample(*sample_hc), nthreads=nthreads)


FLOATS = ("naive_ani", "final_est_ani", "final_est_cov", "mean_cov", "median_cov")


def compare(rows, exp, pseudotax):
    """Row by row against the correctly rounded oracle: every field bit-equal.  The integers; naive_ani,
    final_est_ani, the coverages and the median; lambda where the status defines it; ci_valid and, where it is set, all
    four bootstrap percentiles; in profile the two abundances."""
    assert len(rows) == len(exp), (len(rows), len(exp))
    for i, (r, e) in enumerate(zip(rows, exp)):
        where = (i, int(e.genome))
        assert int(r["genome"]) == e.genome, where
        assert int(r["contain"]) == e.contain and int(r["glen"]) == e.glen, where
        assert int(r["lambda_status"]) == e.lambda_status, where
        assert int(r["kmers_lost"]) == e.kmers_lost, where
        for f in FLOATS:
            assert float(r[f]) == getattr(e, f), (where, f, float(r[f]).hex(), getattr(e, f).hex())
        if e.lambda_status == 2:
            assert float(r["lambda"]) == e.lambda_, (where, "lambda", float(r["lambda"]).hex(), e.lambda_.hex())
        assert int(r["ci_valid"]) == e.ci_valid, where
        if e.ci_valid:
            for j in range(4):
                assert float(r["ci"][j]) == e.ci[j], (where, "ci", j, float(r["ci"][j]).hex(), e.ci[j].hex())
        if pseudotax:
            for f in ("rel_abund", "seq_abund"):
                assert float(r[f]) == getattr(e, f), (where, f, float(r[f]).hex(), getattr(e, f).hex())


def sort_query_rows(rows):
    """syl_query returns (sample, genome) order; the reference prints by ANI descending (stable)."""
    order = sorted(range(len(rows)), key=lambda i: (-float(rows[i]["final_est_ani"]), i))
    return rows[order]
