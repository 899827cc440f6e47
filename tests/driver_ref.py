"""What `sylph-b200 query | profile` should print, built from the oracle (tests/test_driver_*.py).

The header and row formats restate the reference's print_header (src/contain.rs:461-480) and
print_ani_result (src/contain.rs:18-94); tests/test_driver_cpu.py holds the row format against
oracle.format_row.  `compare_tsv` checks a driver's TSV against the expected rows."""
import math
import warnings

import numpy as np

from tests.util import flatten, read_fastx

QUERY_HEADER = ["Sample_file", "Genome_file", "Adjusted_ANI", "Eff_cov", "ANI_5-95_percentile", "Eff_lambda",
                "Lambda_5-95_percentile", "Median_cov", "Mean_cov_geq1", "Containment_ind", "Naive_ANI", "Contig_name"]
LAMBDA_LOW, LAMBDA_HIGH, LAMBDA_VALUE = 0, 1, 2


def header(pseudotax, estimate_unknown=False):
    """print_header: query has one header; profile names the coverage column True_cov under -u."""
    if not pseudotax:
        return "\t".join(QUERY_HEADER)
    return "\t".join(["Sample_file", "Genome_file", "Taxonomic_abundance", "Sequence_abundance", "Adjusted_ANI",
                      "True_cov" if estimate_unknown else "Eff_cov", "ANI_5-95_percentile", "Eff_lambda",
                      "Lambda_5-95_percentile", "Median_cov", "Mean_cov_geq1", "Containment_ind", "Naive_ANI",
                      "kmers_reassigned", "Contig_name"])


def row_fields(r, pseudotax, seq_name, gn_name, contig_name):
    """print_ani_result as a list of (text, [(value, decimals), ...]) per column; the list holds the unrounded
    values behind a printed float (empty for text and integer columns)."""
    def f(v, d):
        return ("%.*f" % (d, v), [(v, d)])
    ani = f(min(r.final_est_ani * 100., 100.), 2)
    if r.lambda_status == LAMBDA_VALUE:
        lam = f(r.lambda_, 3)
    else:
        lam = ("HIGH" if r.lambda_status == LAMBDA_HIGH else "LOW", [])
    if r.ci_valid:
        ci_ani = ("%.2f-%.2f" % (r.ci[0] * 100., r.ci[1] * 100.), [(r.ci[0] * 100., 2), (r.ci[1] * 100., 2)])
        ci_lam = ("%.2f-%.2f" % (r.ci[2], r.ci[3]), [(r.ci[2], 2), (r.ci[3], 2)])
    else:
        ci_ani = ci_lam = ("NA-NA", [])
    cols = [(seq_name, []), (gn_name, [])]
    if pseudotax:
        cols += [f(r.rel_abund, 4), f(r.seq_abund, 4)]
    cols += [ani, f(r.final_est_cov, 3), ci_ani, lam, ci_lam, f(r.median_cov, 0), f(r.mean_cov, 3),
             ("%d/%d" % (r.contain, r.glen), []), f(r.naive_ani * 100., 2)]
    if pseudotax:
        cols.append(("%d" % r.kmers_lost, []))
    cols.append((contig_name, []))
    return cols


def format_row(r, pseudotax, seq_name, gn_name, contig_name):
    return "\t".join(t for t, _ in row_fields(r, pseudotax, seq_name, gn_name, contig_name))


# ---- sketches the driver should build ----------------------------------------------------------------

def genome_sketches(path, name, k=31, c=200, min_spacing=30, pseudotax=True, individual=False):
    """-> list of dicts in the .syldb layout of sylph_b200.formats: one per file, or one per record with -i"""
    from oracle import oracle as O
    recs = read_fastx(path)
    groups = [[r] for r in recs] if individual else [recs]
    out = []
    for g in groups:
        km, tr, gs = O.sketch_genome(*flatten([s for _, s in g]), k=k, c=c, min_spacing=min_spacing, pseudotax=pseudotax)
        out.append(dict(genome_kmers=km, tracked=tr if pseudotax else None, file_name=name,
                        first_contig_name=g[0][0].decode() if g else "", c=c, k=k, gn_size=gs, min_spacing=min_spacing))
    return out


def read_sketch(path, name, k=31, c=200, no_dedup=False):
    """-> dict in the .sylsp layout (+ num_dup_removed)"""
    from oracle import oracle as O
    h, ct, mean, nd = O.sketch_reads(*flatten([s for _, s in read_fastx(path)]), k=k, c=c, no_dedup=no_dedup,
                                     nthreads=8)
    return dict(hashes=h, counts=ct, c=c, k=k, file_name=name, sample_name=None, paired=False, mean_read_length=mean,
                num_dup_removed=nd)


def pair_sketch(path1, path2, name, k=31, c=200, no_dedup=False):
    from oracle import oracle as O
    b1, o1 = flatten([s for _, s in read_fastx(path1)])
    b2, o2 = flatten([s for _, s in read_fastx(path2)])
    h, ct, mean, nd = O.sketch_read_pairs(b1, o1, b2, o2, k=k, c=c, no_dedup=no_dedup)
    return dict(hashes=h, counts=ct, c=c, k=k, file_name=name, sample_name=None, paired=True, mean_read_length=mean,
                num_dup_removed=nd)


def contain(genomes, samples, pseudotax, min_ani=-1., min_number_kmers=50., min_count_correct=3., redundant_ani=99.,
            no_ci=False, no_adj=False, mean_cov=False, read_seq_id=None):
    """Expected rows of query / profile: per sample in the given order, the oracle's rows (with the ANI's pow / exp
    correctly rounded, as the product computes them) sorted as the reference sorts them (src/contain.rs:329-334).  samples: dicts in the .sylsp layout; the printed sample name is
    sample_name if set, else file_name.  -> list of (sample_index, sort_key, row_fields)"""
    from oracle import oracle as O
    k = int(genomes[0]["k"])
    kmers = np.concatenate([g["genome_kmers"] for g in genomes]).astype(np.uint64)
    koff = np.concatenate([[0], np.cumsum([len(g["genome_kmers"]) for g in genomes])]).astype(np.uint64)
    has_tr = genomes[0]["tracked"] is not None
    tr = np.concatenate([g["tracked"] for g in genomes]).astype(np.uint64) if has_tr else None
    toff = np.concatenate([[0], np.cumsum([len(g["tracked"]) for g in genomes])]).astype(np.uint64) if has_tr else None
    gsz = np.array([g["gn_size"] for g in genomes], np.uint64)
    p = O.default_params(k=k, pseudotax=pseudotax, minimum_ani=float(min_ani), min_number_kmers=float(min_number_kmers),
                         min_count_correct=float(min_count_correct), redundant_ani=float(redundant_ani), no_ci=int(no_ci),
                         no_adj=int(no_adj), mean_coverage=int(mean_cov), cr_math=1)
    out = []
    for si, s in enumerate(samples):
        u = None if read_seq_id is None else O.Unknown(read_seq_id, s["mean_read_length"], int(s["c"]))
        rows = O.contain_sample(p, kmers, koff, tr, toff, gsz, O.Sample(s["hashes"], s["counts"]), nthreads=8, unknown=u)
        name = s["sample_name"] if s.get("sample_name") is not None else s["file_name"]
        for r in rows:
            g = genomes[r.genome]
            out.append((si, r.rel_abund if pseudotax else r.final_est_ani,
                        row_fields(r, pseudotax, name, g["file_name"], g["first_contig_name"])))
    return out


# ---- comparison ----------------------------------------------------------------------------------------

def _near_boundary(v, d):
    """v lies within 1e-9 (relative) of a rounding boundary of %.{d}f"""
    x = v * 10 ** d
    b = (math.floor(x) + 0.5) / 10 ** d
    return abs(v - b) <= 1e-9 * max(abs(v), 1e-300)


def _match(got, want, boundary):
    """got: list of str; want: row_fields.  Fields must be equal; a printed float may differ only when the
    expected value sits on a rounding boundary (such cases are appended to `boundary`)."""
    if len(got) != len(want):
        return False
    cases = []
    for i, (g, (t, raws)) in enumerate(zip(got, want)):
        if g == t:
            continue
        gp, tp = g.split("-"), t.split("-")
        if not raws or len(gp) != len(raws) or len(tp) != len(raws):
            return False
        for gv, tv, (v, d) in zip(gp, tp, raws):
            if gv != tv:
                if not _near_boundary(v, d):
                    return False
                cases.append((i, gv, tv, v))
    boundary += cases
    return True


def compare_tsv(text, expected, pseudotax, estimate_unknown=False):
    """The driver's TSV `text` against contain()'s rows: the header, then every line field for field.  Rows whose
    sort key ties with a neighbour's in the same sample form a group compared as a set (the reference's order
    inside a tie is unspecified).  Returns the rounding-boundary cases it let through, and warns about each."""
    lines = text.split("\n")
    assert lines[-1] == "", "output does not end with a newline"
    lines = lines[:-1]
    assert lines[0] == header(pseudotax, estimate_unknown), lines[0]
    got = [ln.split("\t") for ln in lines[1:]]
    assert len(got) == len(expected), "%d rows, expected %d:\n%s\n--- expected ---\n%s" % (
        len(got), len(expected), "\n".join(lines[1:]), "\n".join("\t".join(t for t, _ in w) for _, _, w in expected))
    boundary = []
    i = 0
    while i < len(expected):
        j = i + 1
        while j < len(expected) and expected[j][:2] == expected[i][:2]:
            j += 1
        pool = got[i:j]
        for _, _, want in expected[i:j]:
            hit = next((n for n, g in enumerate(pool) if _match(g, want, boundary)), None)
            assert hit is not None, "row %d..%d: no line matches\n%s\namong\n%s" % (
                i, j, "\t".join(t for t, _ in want), "\n".join("\t".join(g) for g in pool))
            pool.pop(hit)
        i = j
    for c in boundary:
        warnings.warn("printed float differs on a rounding boundary: column %d %s vs %s (value %r)" % c)
    return boundary
