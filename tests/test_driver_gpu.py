"""GPU: `sylph-b200 sketch | query | profile` end to end against the oracle, option by option.

Inputs are written into a temporary directory: about 40 synthetic genomes of 100-300 kbp (sylph_b200.synth; genomes
g % 100 == 99 are ~97 %-identity mutants of g - 1, one file holds the same records as another) in 1-3 records each, as plain,
gzip and BGZF files; four read samples of different communities (one without a genome in the db); synthetic read
pairs and the committed k12 pairs.  tests/driver_ref.py turns the oracle's sketches and rows into the lines the
reference would print, and compares them with the driver's field for field."""
import gzip
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import driver_ref as D
from tests.test_host_cpu import _bgzf
from tests.util import DATA, REPO

pytestmark = pytest.mark.gpu

GIDS = list(range(32)) + [98, 99, 198, 199, 298, 299, 398, 399]
COPY = "g005_copy.fa"                      # the records of g005: ties with it in query, loses every k-mer in profile
COMMUNITIES = {                            # sample -> [(genome id, coverage)]
    "s1.fq": [(0, 8.), (1, 3.), (2, 1.), (3, .4), (98, 2.), (5, 5.)],
    "s2.fq.gz": [(99, 4.), (10, 1.5), (11, .6), (12, 10.)],
    "s3.fastq.gz": [(198, 3.), (199, 2.), (20, 1.), (21, .3), (298, 6.)],
    "s4.fastq": [(700, 2.), (701, 1.)],    # no genome of the db
}
SAMPLES = list(COMMUNITIES)
PAIRS = [("p_1.fq", "p_2.fq"), ("k12_R1.fq", "k12_R2.fq")]
RL = 150
_LUT = np.frombuffer(b"ACGT", np.uint8)
_COMP = np.zeros(256, np.uint8)
_COMP[list(b"ACGT")] = list(b"TGCA")


def glen(g):
    src = g - 1 if g % 100 == 99 else g
    return 100_000 + (src * 7919 % 41) * 5_000


_SEQ = {}


def genome_seq(g):
    if g not in _SEQ:
        import torch
        from sylph_b200 import synth
        _SEQ[g] = _LUT[synth.genome_codes(g, torch.arange(glen(g), dtype=torch.int64)).numpy()]
    return _SEQ[g]


def gname(i, g):
    return "g%03d.%s" % (g, ("fa", "fa.gz", "fasta.gz")[i % 3])


GENOMES = [gname(i, g) for i, g in enumerate(GIDS)] + [COPY]


def fasta_bytes(g):
    s = genome_seq(g)
    n = 1 + g % 3
    cut = [len(s) * i // n for i in range(n + 1)]
    out = b""
    for c in range(n):
        part = s[cut[c]:cut[c + 1]].tobytes()
        out += b">g%03d_c%d synthetic genome %d\n" % (g, c, g) + b"\n".join(part[i:i + 80] for i in range(0, len(part), 80)) + b"\n"
    return out


def sample_reads(comm, seed, dup=0.02):
    """reads of length RL from the genomes of `comm` at the given coverages: uniform starts, either strand, 0.5 %
    substitutions, `dup` of them exact duplicates -> uint8 (n, RL)"""
    rng = np.random.default_rng(seed)
    parts = []
    for g, cov in comm:
        s = genome_seq(g)
        n = int(cov * len(s) / RL)
        st = rng.integers(0, len(s) - RL + 1, n)
        r = s[st[:, None] + np.arange(RL)[None, :]]
        rev = rng.random(n) < .5
        r[rev] = _COMP[r[rev][:, ::-1]]
        sub = rng.random(r.shape) < .005
        r[sub] = _LUT[rng.integers(0, 4, int(sub.sum()))]
        parts.append(r)
    r = np.concatenate(parts)
    r = r[rng.permutation(len(r))]
    d = rng.random(len(r)) < dup
    r[d] = r[rng.integers(0, len(r), int(d.sum()))]
    return r


def fastq_bytes(r):
    n = len(r)
    h = 12                                           # "@r%09d\n"
    rec = np.empty((n, h + RL + 3 + RL + 1), np.uint8)
    rec[:, :h] = np.frombuffer(b"".join(b"@r%09d\n" % i for i in range(n)), np.uint8).reshape(n, h)
    rec[:, h:h + RL] = r
    rec[:, h + RL:h + 3 + RL] = np.frombuffer(b"\n+\n", np.uint8)
    rec[:, h + 3 + RL:h + 3 + 2 * RL] = ord("I")
    rec[:, -1] = ord("\n")
    return rec.tobytes()


def write(path, data):
    if path.endswith("fastq.gz") or path.endswith("fasta.gz"):    # BGZF
        data = _bgzf(data)
    elif path.endswith(".gz"):
        data = gzip.compress(data, 6)
    with open(path, "wb") as f:
        f.write(data)


@pytest.fixture(scope="module")
def exe():
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    subprocess.check_call(["make", "-C", os.path.join(REPO, "host"), "-s"], env=env)
    return os.path.join(REPO, "host", "sylph-b200")


def run(exe, args, cwd, env=None, rc=0):
    e = dict(os.environ)
    for k in ("SYL_DRIVER_BATCH_BASES", "SYL_DRIVER_SAMPLES_PER_CALL", "SYL_DRIVER_ROWS", "SYL_INGEST_CHUNK", "SYL_HOST_INGEST"):
        e.pop(k, None)
    e.update(env or {})
    r = subprocess.run([exe] + args, cwd=cwd, env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == rc, r.stderr[-3000:]
    return r


@pytest.fixture(scope="module")
def d(tmp_path_factory):
    """the input files, written once"""
    d = str(tmp_path_factory.mktemp("driver"))
    for i, g in enumerate(GIDS):
        write(os.path.join(d, gname(i, g)), fasta_bytes(g))
    write(os.path.join(d, COPY), fasta_bytes(5))
    for i, (s, comm) in enumerate(COMMUNITIES.items()):
        write(os.path.join(d, s), fastq_bytes(sample_reads(comm, 100 + i)))
    # synthetic pairs: 400 bp fragments of genomes 4 and 6, with duplicate pairs
    rng = np.random.default_rng(7)
    r1, r2 = [], []
    for g, cov in ((4, 3.), (6, 1.)):
        s = genome_seq(g)
        st = rng.integers(0, len(s) - 400 + 1, int(cov * len(s) / 400))
        r1.append(s[st[:, None] + np.arange(RL)])
        r2.append(_COMP[s[st[:, None] + 400 - 1 - np.arange(RL)]])
    r1, r2 = np.concatenate(r1), np.concatenate(r2)
    dup = np.flatnonzero(rng.random(len(r1)) < .03)
    src = rng.integers(0, len(r1), len(dup))
    r1[dup], r2[dup] = r1[src], r2[src]
    write(os.path.join(d, "p_1.fq"), fastq_bytes(r1))
    write(os.path.join(d, "p_2.fq"), fastq_bytes(r2))
    for f in ("k12_R1.fq", "k12_R2.fq", "o157_reads.fastq.gz", "e.coli-K12.fasta.gz", "e.coli-o157.fasta.gz"):
        shutil.copy(os.path.join(DATA, f), os.path.join(d, f))
    return d


class Ref:
    """the oracle's sketches of the inputs, computed once per (file, k, c, ...)"""

    def __init__(self, d):
        self.d, self._g, self._s = d, {}, {}

    def genomes(self, names, k=31, c=200, individual=False, pseudotax=True):
        out = []
        for n in names:
            key = (n, k, c, individual, pseudotax)
            if key not in self._g:
                self._g[key] = D.genome_sketches(os.path.join(self.d, n), n, k=k, c=c, individual=individual,
                                                 pseudotax=pseudotax)
            out += self._g[key]
        return out

    def sample(self, name, k=31, c=200):
        key = (name, k, c)
        if key not in self._s:
            self._s[key] = D.read_sketch(os.path.join(self.d, name), name, k=k, c=c)
        return self._s[key]

    def pair(self, f1, f2):
        key = (f1, f2)
        if key not in self._s:
            self._s[key] = D.pair_sketch(os.path.join(self.d, f1), os.path.join(self.d, f2), f1)
        return self._s[key]


@pytest.fixture(scope="module")
def ref(d):
    return Ref(d)


@pytest.fixture(scope="module")
def sk(exe, d):
    """`sketch` of every genome, sample and pair into sk/ -> the run"""
    args = ["sketch"] + GENOMES + SAMPLES + ["-1", PAIRS[0][0], PAIRS[1][0], "-2", PAIRS[0][1], PAIRS[1][1], "--fpr", "0",
                                             "-d", "sk", "-o", "sk/db"]
    return run(exe, args, d)


SK_SAMPLES = ["sk/%s.sylsp" % s for s in SAMPLES]
SK_PAIRS = ["sk/%s.paired.sylsp" % p[0] for p in PAIRS]


def assert_syldb(path, want):
    from sylph_b200 import formats as F
    got = F.read_syldb(path)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for f in ("file_name", "first_contig_name", "c", "k", "gn_size", "min_spacing"):
            assert g[f] == w[f], (f, g[f], w[f])
        assert np.array_equal(g["genome_kmers"], w["genome_kmers"]), w["file_name"]
        assert (g["tracked"] is None) == (w["tracked"] is None)
        assert w["tracked"] is None or np.array_equal(g["tracked"], w["tracked"]), w["file_name"]


def assert_sylsp(path, want):
    from sylph_b200 import formats as F
    g = F.read_sylsp(path)
    for f in ("c", "k", "file_name", "sample_name", "paired"):
        assert g[f] == want[f], (f, g[f], want[f])
    assert abs(g["mean_read_length"] - want["mean_read_length"]) <= 1e-9 * want["mean_read_length"]
    o = np.argsort(g["hashes"])
    assert np.array_equal(g["hashes"][o], want["hashes"]) and np.array_equal(g["counts"][o], want["counts"]), path


def test_sketch_files_equal_oracle(sk, d, ref):
    """genomes + single-end + paired (-1 a b -2 c d --fpr 0) with -d and -o: which files, and what they hold"""
    assert sorted(os.listdir(os.path.join(d, "sk"))) == sorted(
        ["db.syldb"] + [s + ".sylsp" for s in SAMPLES] + [p[0] + ".paired.sylsp" for p in PAIRS])
    assert_syldb(os.path.join(d, "sk/db.syldb"), ref.genomes(GENOMES))
    for s, p in zip(SAMPLES, SK_SAMPLES):
        assert_sylsp(os.path.join(d, p), ref.sample(s))
    for (f1, f2), p in zip(PAIRS, SK_PAIRS):
        w = ref.pair(f1, f2)
        assert_sylsp(os.path.join(d, p), w)
    assert ref.pair(*PAIRS[0])["num_dup_removed"] > 0    # the synthetic pairs exercise the exact dedup set


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_raw_and_sketched_inputs(exe, d, ref, sk, cmd):
    pt = cmd == "profile"
    want = D.contain(ref.genomes(GENOMES), [ref.sample(s) for s in SAMPLES], pt)
    raw = run(exe, [cmd] + SAMPLES + GENOMES, d).stdout
    D.compare_tsv(raw, want, pt)
    assert {w[0] for w in want} == {0, 1, 2}                       # s4 has no hit, the other three have some
    assert any(w[2][1][0] == COPY for w in want) == (not pt)       # the byte copy ties in query, is derep'd in profile
    assert run(exe, [cmd] + SK_SAMPLES + ["sk/db.syldb"], d).stdout == raw


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_mixed_sketch_and_raw_inputs(exe, d, ref, sk, cmd):
    """one .syldb plus raw genomes; .sylsp files (one carrying a sample_name, one of pairs) plus raw reads: raw reads
    come first, then the sketches (src/contain.rs:258-260)"""
    from sylph_b200 import formats as F
    pt = cmd == "profile"
    if not os.path.exists(os.path.join(d, "sk/db20.syldb")):
        run(exe, ["sketch"] + GENOMES[:20] + ["-o", "sk/db20"], d)
        s = F.read_sylsp(os.path.join(d, SK_PAIRS[0]))
        s["sample_name"] = "named pairs"
        F.write_sylsp(os.path.join(d, "named.sylsp"), s)
    named = dict(ref.pair(*PAIRS[0]), sample_name="named pairs")
    out = run(exe, [cmd, "sk/db20.syldb", SK_SAMPLES[1], "named.sylsp", SAMPLES[0]] + GENOMES[20:] + [SAMPLES[2]], d).stdout
    want = D.contain(ref.genomes(GENOMES), [ref.sample(SAMPLES[0]), ref.sample(SAMPLES[2]), ref.sample(SAMPLES[1]), named],
                     pt)
    D.compare_tsv(out, want, pt)
    assert any(w[0] == 3 for w in want)


def _kmers_of(ref, name):
    return len(ref.genomes([name])[0]["genome_kmers"])


OPTIONS = [  # (id, args, oracle keywords)
    ("m0", ["-m", "0"], dict(min_ani=0.)),
    ("m97.5", ["-m", "97.5"], dict(min_ani=97.5)),
    ("M_at", ["-M", "@"], {}),
    ("M_above", ["-M", "@+1"], {}),
    ("mcc1", ["--min-count-correct", "1"], dict(min_count_correct=1.)),
    ("mcc6", ["--min-count-correct", "6"], dict(min_count_correct=6.)),
    ("R90", ["-R", "90"], dict(redundant_ani=90.)),
    ("no_ci", ["--no-ci"], dict(no_ci=True)),
    ("no_adjust", ["--no-adjust"], dict(no_adj=True)),
    ("mean_cov", ["--mean-coverage"], dict(mean_cov=True)),
    ("u_I98", ["-u", "-I", "98"], dict(read_seq_id=98.)),
]


@pytest.mark.parametrize("cmd", ["query", "profile"])
@pytest.mark.parametrize("opt", OPTIONS, ids=[o[0] for o in OPTIONS])
def test_contain_option(exe, d, ref, sk, cmd, opt):
    """each contain option alone, pre-sketched inputs (four samples and a pair sketch) against the oracle"""
    pt = cmd == "profile"
    name, args, kw = opt
    # -M at and one above the k-mer count of g001 (present in s1 at 3x): kept at, dropped above
    n1 = _kmers_of(ref, GENOMES[1])
    args = [a.replace("@+1", str(n1 + 1)).replace("@", str(n1)) for a in args]
    if name.startswith("M_"):
        kw = dict(min_number_kmers=float(args[1]))
    samples = [ref.sample(s) for s in SAMPLES] + [ref.pair(*PAIRS[0])]
    want = D.contain(ref.genomes(GENOMES), samples, pt, **kw)
    out = run(exe, [cmd] + args + SK_SAMPLES + [SK_PAIRS[0], "sk/db.syldb"], d).stdout
    D.compare_tsv(out, want, pt, estimate_unknown="-u" in args)
    has_g1 = any(w[2][1][0] == GENOMES[1] for w in want)
    if name == "M_at":
        assert has_g1
    if name == "M_above":
        assert not has_g1
    if name == "R90" and pt:   # -R 90 removes a genome that the default keeps
        assert len(want) < len(D.contain(ref.genomes(GENOMES), samples, pt))
    if name == "u_I98":
        assert out.split("\n")[0].split("\t")[5 if pt else 3] == ("True_cov" if pt else "Eff_cov")


def test_k21_end_to_end(exe, d, ref):
    g = GENOMES[:12]
    run(exe, ["sketch", "-k", "21", "-d", "k21", "-o", "k21/db", SAMPLES[0]] + g, d)
    assert_syldb(os.path.join(d, "k21/db.syldb"), ref.genomes(g, k=21))
    assert_sylsp(os.path.join(d, "k21", SAMPLES[0] + ".sylsp"), ref.sample(SAMPLES[0], k=21))
    for cmd in ("query", "profile"):
        want = D.contain(ref.genomes(g, k=21), [ref.sample(SAMPLES[0], k=21)], cmd == "profile")
        assert want
        D.compare_tsv(run(exe, [cmd, "-k", "21", SAMPLES[0], "k21/db.syldb"], d).stdout, want, cmd == "profile")
        D.compare_tsv(run(exe, [cmd, "k21/%s.sylsp" % SAMPLES[0], "k21/db.syldb"], d).stdout, want, cmd == "profile")
    # raw reads are sketched with -k or not at all (src/contain.rs:578-584)
    r = run(exe, ["query", SAMPLES[0], "k21/db.syldb"], d)
    assert "-k 31 is not equal to -k 21" in r.stderr and r.stdout == D.header(False) + "\n"


def test_c_mismatch(exe, d, ref, sk):
    g = GENOMES[:12]
    # -c 100 reads against a c = 200 db
    want = D.contain(ref.genomes(GENOMES), [ref.sample(SAMPLES[0], c=100)], False)
    D.compare_tsv(run(exe, ["query", "-c", "100", SAMPLES[0], "sk/db.syldb"], d).stdout, want, False)
    # the reverse: c = 200 reads (raw and sketched) against a c = 100 db are skipped with the reference's warnings
    run(exe, ["sketch", "-c", "100", "-o", "c100/db", "-d", "c100", SAMPLES[0]] + g, d)
    assert_syldb(os.path.join(d, "c100/db.syldb"), ref.genomes(g, c=100))
    r = run(exe, ["query", SAMPLES[0], "c100/db.syldb"], d)
    assert "value of -c for contain is greater than the smallest value of -c" in r.stderr
    assert r.stdout == D.header(False) + "\n"
    r = run(exe, ["profile", SK_SAMPLES[0], "c100/db.syldb"], d)
    assert "value of -c is greater than the smallest value of -c" in r.stderr and r.stdout == D.header(True) + "\n"
    # a c = 100 .sylsp against the c = 200 db with -u: the sample's own c enters the estimate
    s100 = ref.sample(SAMPLES[0], c=100)
    assert_sylsp(os.path.join(d, "c100", SAMPLES[0] + ".sylsp"), s100)
    for cmd in ("query", "profile"):
        pt = cmd == "profile"
        want = D.contain(ref.genomes(GENOMES), [s100], pt, read_seq_id=98.)
        out = run(exe, [cmd, "-u", "-I", "98", "c100/%s.sylsp" % SAMPLES[0], "sk/db.syldb"], d).stdout
        D.compare_tsv(out, want, pt, estimate_unknown=True)


def test_individual_records(exe, d, ref):
    """-i: one genome per record, contig names from the records"""
    g = GENOMES[:10]
    assert sum(1 + x % 3 for x in GIDS[:10]) > 10
    run(exe, ["sketch", "-i", "-o", "ind_db"] + g, d)
    want_db = ref.genomes(g, individual=True)
    assert_syldb(os.path.join(d, "ind_db.syldb"), want_db)
    assert len({w["first_contig_name"] for w in want_db}) == len(want_db)
    for cmd in ("query", "profile"):
        want = D.contain(want_db, [ref.sample(SAMPLES[0])], cmd == "profile")
        assert want
        D.compare_tsv(run(exe, [cmd, "-i", SAMPLES[0]] + g, d).stdout, want, cmd == "profile")


def test_disable_profiling(exe, d, ref, sk):
    run(exe, ["sketch", "--disable-profiling", "-o", "np_db"] + GENOMES, d)
    assert_syldb(os.path.join(d, "np_db.syldb"), ref.genomes(GENOMES, pseudotax=False))
    q = run(exe, ["query"] + SK_SAMPLES + ["np_db.syldb"], d).stdout
    assert q == run(exe, ["query"] + SK_SAMPLES + ["sk/db.syldb"], d).stdout
    D.compare_tsv(q, D.contain(ref.genomes(GENOMES, pseudotax=False), [ref.sample(s) for s in SAMPLES], False), False)
    r = run(exe, ["profile"] + SK_SAMPLES + ["np_db.syldb"], d, rc=1)
    assert "Attempting profiling, but *.syldb was sketched with the --disable-profiling option. Exiting" in r.stderr


def test_list_files(exe, d, ref, sk):
    with open(os.path.join(d, "genomes.txt"), "w") as f:
        f.write("\n".join(GENOMES) + "\n")
    with open(os.path.join(d, "all.txt"), "w") as f:
        f.write("\n".join(SAMPLES + GENOMES) + "\n")
    run(exe, ["sketch", "-l", "genomes.txt", "-o", "lst_db"], d)
    assert open(os.path.join(d, "lst_db.syldb"), "rb").read() == open(os.path.join(d, "sk/db.syldb"), "rb").read()
    out = run(exe, ["profile", "-l", "all.txt"], d).stdout
    D.compare_tsv(out, D.contain(ref.genomes(GENOMES), [ref.sample(s) for s in SAMPLES], True), True)


@pytest.fixture(scope="module")
def big(d):
    """~72 Mbp of reads in one FASTQ (three 32 M-base ingest chunks) -> name"""
    comm = [(g, 1.) for g in GIDS[:30]] + [(98, 40.), (199, 60.)]
    r = sample_reads(comm, 5, dup=.01)
    reps = -(-480_000 // len(r))
    r = np.concatenate([r] * reps)[:480_000]        # repeated reads: deep counts for the dedup-free query path
    write(os.path.join(d, "big.fq"), fastq_bytes(r))
    return "big.fq"


def test_host_ingest_variants(exe, d, ref, sk, big):
    """the library's ingest paths inside the driver: default (packed), tiny chunks, ASCII"""
    outs = [run(exe, ["profile", big, "sk/db.syldb"], d, env=e).stdout
            for e in ({}, {"SYL_INGEST_CHUNK": "8192"}, {"SYL_HOST_INGEST": "ascii"})]
    assert outs[1] == outs[0] and outs[2] == outs[0]
    D.compare_tsv(outs[0], D.contain(ref.genomes(GENOMES), [ref.sample(big)], True), True)


def test_threads_give_identical_output(exe, d, sk, big):
    """-t 1, 3, 8: the big file first, so parses finish out of order; sketches and rows byte-identical"""
    outs = []
    for t in ("1", "3", "8"):
        run(exe, ["sketch", "-t", t, "-d", "t" + t, "-o", "t%s/db" % t, big] + SAMPLES + GENOMES, d)
        q = run(exe, ["query", "-t", t, big] + SAMPLES + GENOMES, d).stdout
        files = sorted(os.listdir(os.path.join(d, "t" + t)))
        outs.append((q, files, [open(os.path.join(d, "t" + t, f), "rb").read() for f in files]))
    assert outs[1] == outs[0] and outs[2] == outs[0]
    assert outs[0][2][outs[0][1].index("db.syldb")] == open(os.path.join(d, "sk/db.syldb"), "rb").read()


def test_truncated_gzip_among_good_files(exe, d, sk):
    with open(os.path.join(d, SAMPLES[1]), "rb") as f:
        raw = f.read()
    with open(os.path.join(d, "bad.fq.gz"), "wb") as f:
        f.write(raw[:len(raw) // 2])
    with open(os.path.join(d, GENOMES[1]), "rb") as f:
        raw = f.read()
    with open(os.path.join(d, "bad.fa.gz"), "wb") as f:
        f.write(raw[:len(raw) // 2])
    good = run(exe, ["query", SAMPLES[0], SAMPLES[2]] + GENOMES[:20], d).stdout
    r = run(exe, ["query", SAMPLES[0], "bad.fq.gz", SAMPLES[2]] + GENOMES[:10] + ["bad.fa.gz"] + GENOMES[10:20], d)
    assert "bad.fq.gz is not a valid fasta/fastq file; skipping." in r.stderr
    assert "bad.fa.gz is not a valid fasta/fastq file; skipping." in r.stderr
    assert r.stdout == good and good.count("\n") > 1


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_sample_batches_and_row_buffer(exe, d, sk, cmd):
    """5 samples through calls of 1 and 2 samples, and a row buffer of 1 that takes the capacity retry"""
    args = [cmd] + SK_SAMPLES + SK_PAIRS + ["sk/db.syldb"]
    one = run(exe, args, d).stdout
    assert len({ln.split("\t")[0] for ln in one.split("\n")[1:-1]}) >= 4
    for env in ({"SYL_DRIVER_SAMPLES_PER_CALL": "1"}, {"SYL_DRIVER_SAMPLES_PER_CALL": "2"}, {"SYL_DRIVER_ROWS": "1"},
                {"SYL_DRIVER_ROWS": "1", "SYL_DRIVER_SAMPLES_PER_CALL": "2"}):
        assert run(exe, args, d, env=env).stdout == one, env


@pytest.mark.parametrize("individual", [False, True], ids=["files", "records"])
def test_genome_batches(exe, d, ref, sk, individual):
    """a batch threshold of 1 base (one file per syl_sketch_genomes call) and of 300 kbp (batches that close
    mid-list): the same .syldb and the same rows"""
    i = ["-i"] if individual else []
    want_db = ref.genomes(GENOMES, individual=individual)
    res = []
    for env in ({}, {"SYL_DRIVER_BATCH_BASES": "1"}, {"SYL_DRIVER_BATCH_BASES": "300000"}):
        tag = env.get("SYL_DRIVER_BATCH_BASES", "0")
        run(exe, ["sketch"] + i + ["-o", "gb%s_%d" % (tag, individual)] + GENOMES, d, env=env)
        path = os.path.join(d, "gb%s_%d.syldb" % (tag, individual))
        assert_syldb(path, want_db)
        res.append((open(path, "rb").read(), run(exe, ["profile"] + i + SAMPLES[:3] + GENOMES, d, env=env).stdout))
    assert res[1] == res[0] and res[2] == res[0]
    D.compare_tsv(res[0][1], D.contain(want_db, [ref.sample(s) for s in SAMPLES[:3]], True), True)


def test_ecoli_genomes_and_fixture_reads(exe, d, ref, sk):
    """the committed E. coli genomes against the o157 reads and the k12 pair sketch"""
    g = ["e.coli-K12.fasta.gz", "e.coli-o157.fasta.gz"]
    out = run(exe, ["profile", "o157_reads.fastq.gz", SK_PAIRS[1]] + g, d).stdout
    D.compare_tsv(out, D.contain(ref.genomes(g), [ref.sample("o157_reads.fastq.gz"), ref.pair(*PAIRS[1])], True), True)


def test_profile_u_header_and_pairs_refused(exe, d, sk):
    r = run(exe, ["profile", "-u", "-I", "98"] + SK_SAMPLES[:1] + ["sk/db.syldb"], d)
    assert r.stdout.split("\n")[0] == D.header(True, estimate_unknown=True)
    for cmd in ("query", "profile"):
        r = run(exe, [cmd, "sk/db.syldb", "-1", PAIRS[0][0], "-2", PAIRS[0][1], "--fpr", "0"], d, rc=1)
        assert "sketch -1 ... -2 ... --fpr 0" in r.stderr and r.stdout == ""


def test_unwritable_sketch_path_exits_1(exe, d):
    r = run(exe, ["sketch", "-o", "missing_dir/db", GENOMES[0]], d, rc=1)
    assert "missing_dir/db.syldb path not valid; exiting." in r.stderr
