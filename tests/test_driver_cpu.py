"""CPU suite: the driver's TSV format restated in tests/driver_ref.py against the oracle's, and the argument errors
`sylph-b200` reports before it needs a device."""
import os
import subprocess

import pytest

from tests import driver_ref as D
from tests.util import REPO


def _row(**kw):
    from oracle import oracle as O
    r = O.AniResult(genome=0, lambda_status=D.LAMBDA_HIGH, contain=812, glen=1000, kmers_lost=0, naive_ani=0.99321,
                    final_est_ani=0.99412, final_est_cov=12.3456, mean_cov=12.5, median_cov=12., lambda_=0., ci_valid=0,
                    rel_abund=41.23456, seq_abund=40.98765)
    for a, b in kw.items():
        if a == "ci":
            for i, v in enumerate(b):
                r.ci[i] = v
        else:
            setattr(r, a, b)
    return r


ROWS = {
    "high": {},
    "low": dict(lambda_status=D.LAMBDA_LOW, median_cov=1.),
    "lambda_ci": dict(lambda_status=D.LAMBDA_VALUE, lambda_=0.73251, ci_valid=1, ci=[0.97123, 0.98877, 0.61234, 0.84999]),
    "lambda_no_ci": dict(lambda_status=D.LAMBDA_VALUE, lambda_=1.0005, median_cov=2.5, mean_cov=2.0625),
    "ani_above_100": dict(final_est_ani=1.0213, naive_ani=1.0),
    "ani_rounds_to_100": dict(final_est_ani=0.999996),
    "kmers_lost_large": dict(kmers_lost=123456789012, contain=2 ** 40, glen=2 ** 41),
    "query_row": dict(kmers_lost=-1, rel_abund=0., seq_abund=0.),
    "median_half": dict(median_cov=2.5, final_est_cov=0.0005),
}


@pytest.mark.parametrize("pseudotax", [False, True])
@pytest.mark.parametrize("case", list(ROWS))
def test_row_format_restatement_matches_oracle(case, pseudotax):
    from oracle import oracle as O
    r = _row(**ROWS[case])
    want = O.format_row(r, pseudotax, "reads/s 1.fq", "g.fa.gz", "NC_000913.3 Escherichia coli")
    assert D.format_row(r, pseudotax, "reads/s 1.fq", "g.fa.gz", "NC_000913.3 Escherichia coli") == want
    fields = want.split("\t")
    assert len(fields) == (15 if pseudotax else 12) and len(fields) == len(D.header(pseudotax).split("\t"))
    ani = fields[4 if pseudotax else 2]
    assert float(ani) <= 100. and (case != "ani_above_100" or ani == "100.00")
    if case in ("high", "low"):
        assert fields[7 if pseudotax else 5] == ("HIGH" if case == "high" else "LOW") and fields.count("NA-NA") == 2
    if case == "lambda_ci":
        assert "97.12-98.88" in fields and "0.61-0.85" in fields and "0.733" in fields
    if pseudotax and case == "kmers_lost_large":
        assert fields[13] == "123456789012" and fields[11] == "%d/%d" % (2 ** 40, 2 ** 41)


def test_headers():
    q, p, pu = D.header(False), D.header(True), D.header(True, estimate_unknown=True)
    assert D.header(False, estimate_unknown=True) == q and "\tEff_cov\t" in q
    assert p.split("\t")[5] == "Eff_cov" and pu.split("\t")[5] == "True_cov"
    assert p.replace("Eff_cov", "True_cov") == pu and p.split("\t")[:2] == q.split("\t")[:2]


def test_compare_tsv_ties_and_boundaries():
    from oracle import oracle as O
    a, b = _row(), _row(contain=811)
    rows = [(0, 0.5, D.row_fields(a, True, "s", "g1", "c")), (0, 0.5, D.row_fields(b, True, "s", "g2", "c")),
            (1, 0.5, D.row_fields(a, True, "t", "g1", "c"))]
    lines = [D.format_row(a, True, "s", "g1", "c"), D.format_row(b, True, "s", "g2", "c"),
             D.format_row(a, True, "t", "g1", "c")]
    txt = D.header(True) + "\n" + "\n".join(lines) + "\n"
    assert D.compare_tsv(txt, rows, True) == []
    swapped = D.header(True) + "\n" + "\n".join([lines[1], lines[0], lines[2]]) + "\n"
    assert D.compare_tsv(swapped, rows, True) == []          # a tie group is a set
    with pytest.raises(AssertionError):                      # ... but samples are not
        D.compare_tsv(D.header(True) + "\n" + "\n".join([lines[2], lines[1], lines[0]]) + "\n", rows, True)
    # a value on the rounding boundary of its column may print either way; one off it may not
    c = _row(final_est_cov=0.0125)
    exp = [(0, 0.5, D.row_fields(c, False, "s", "g", "c"))]
    line = O.format_row(c, False, "s", "g", "c")
    assert "\t0.013\t" in line
    other = line.replace("\t0.013\t", "\t0.012\t")
    with pytest.warns(UserWarning):
        assert len(D.compare_tsv(D.header(False) + "\n" + other + "\n", exp, False)) == 1
    far = _row(final_est_cov=0.0121)
    line = O.format_row(far, False, "s", "g", "c").replace("\t0.012\t", "\t0.013\t")
    with pytest.raises(AssertionError):
        D.compare_tsv(D.header(False) + "\n" + line + "\n", [(0, 0.5, D.row_fields(far, False, "s", "g", "c"))], False)


@pytest.fixture(scope="module")
def exe():
    from sylph_b200 import build
    build.build()
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    subprocess.check_call(["make", "-C", os.path.join(REPO, "host"), "-s"], env=env)
    return os.path.join(REPO, "host", "sylph-b200")


PAIRS_MSG = "query/profile do not sketch read pairs (-1/-2) here"


@pytest.mark.parametrize("args,msg", [
    (["sketch", "-k", "25", "g.fa"], "Only k = 21, 31 are currently supported"),
    (["query", "-k", "25", "r.fq", "g.fa"], "Only k = 21, 31 are currently supported"),
    (["sketch", "-1", "a_1.fq", "b_1.fq", "-2", "a_2.fq", "--fpr", "0"], "Different number of paired sequences"),
    (["profile", "-u", "r.fq", "g.fa"], "-u needs -I/--read-seq-id"),
    (["query", "-u", "-I", "0", "r.fq", "g.fa"], "-u needs -I/--read-seq-id"),
    (["sketch", "-1", "a_1.fq", "-2", "a_2.fq", "--fpr", "0.5"], "paired-end reads need --fpr 0"),
    (["sketch", "-1", "a_1.fq", "-2", "a_2.fq"], "paired-end reads need --fpr 0"),
    (["sketch", "--fpr", "1"], "Invalid value for --fpr"),
    (["query", "g.fa", "-1", "a_1.fq", "-2", "a_2.fq"], PAIRS_MSG),
    (["profile", "-1", "a_1.fq", "-2", "a_2.fq", "--fpr", "0", "g.fa", "r.fq"], PAIRS_MSG),
    (["profile", "--bogus", "g.fa"], "unknown option --bogus"),
])
def test_argument_errors_before_the_device(exe, tmp_path, args, msg):
    """Each is refused with exit code 1 and its message while parsing, so no GPU (and no input file) is needed."""
    r = subprocess.run([exe] + args, cwd=tmp_path, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 1 and msg in r.stderr and r.stdout == "", r.stderr


def test_truncated_gzip_is_an_invalid_file(exe, tmp_path):
    """A gzip stream cut short makes the file invalid, not shorter: FASTA (where a shorter file still parses) and
    FASTQ cut exactly after a record, read by zlib (-t 1) and by the BGZF path (-t 4)."""
    import gzip
    import zlib
    from tests.util import read_fastx
    fa = b"".join(b">c%d contig\n" % i + b"ACGT" * 5000 + b"\n" for i in range(40))
    rec = [b"@r%04d\n" % i + b"ACGTTGCA" * 20 + b"\n+\n" + b"I" * 160 + b"\n" for i in range(4000)]
    for name, data in (("a.fa.gz", fa), ("r.fq.gz", b"".join(rec))):
        z = gzip.compress(data, 6)
        (tmp_path / name).write_bytes(z)
        (tmp_path / ("cut_" + name)).write_bytes(z[:len(z) // 2])
    co = zlib.compressobj(6, zlib.DEFLATED, 31)     # gzip header, no trailer: the inflated bytes are 2000 whole records
    (tmp_path / "cut_rec.fq.gz").write_bytes(co.compress(b"".join(rec[:2000])) + co.flush(zlib.Z_SYNC_FLUSH))
    files = ["a.fa.gz", "cut_a.fa.gz", "r.fq.gz", "cut_r.fq.gz", "cut_rec.fq.gz"]
    for t in ("1", "4"):
        out = subprocess.run([exe, "fastx-stats", "-t", t] + files, cwd=tmp_path, stdout=subprocess.PIPE, text=True,
                             check=True).stdout.strip().split("\n")
        assert [ln.split("\t")[1] == "INVALID" for ln in out] == [False, True, False, True, True], out
        assert int(out[0].split("\t")[1]) == len(read_fastx(str(tmp_path / "a.fa.gz"))) == 40
