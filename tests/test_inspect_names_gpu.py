"""GPU: sample names (-S / --lS), list inputs (--l1 --l2 --gl --rl) and `inspect`, end to end on the driver.

The first tests replay sylph's own integration tests of these options (tests/integration_test.rs: test_sample_names,
test_sketch lines 81-109, test_sketch_list lines 181-206, test_inspect) in a temporary directory whose `test_files`
links to tests/golden/data, as the committed lists name `test_files/...`.  Every run that sketches read pairs adds
`--fpr 0`: the driver sketches pairs with the exact dedup set only.  Beyond the reference's existence checks, the
sketches are compared with the oracle's (tests/driver_ref.py) with the sample name set, and inspect's YAML with
tests/inspect_ref.py."""
import os
import shutil
import subprocess

import pytest

from tests import driver_ref as D
from tests import inspect_ref as I
from tests.test_driver_gpu import assert_syldb, assert_sylsp
from tests.util import DATA, REPO

pytestmark = pytest.mark.gpu

T1, T2 = "test_files/t1.fq", "test_files/t2.fq"
K1, K2 = "test_files/k12_R1.fq", "test_files/k12_R2.fq"
O157 = "test_files/o157_reads.fastq.gz"
EC590, K12G, O157G = ("test_files/e.coli-%s.fasta.gz" % g for g in ("EC590", "K12", "o157"))


@pytest.fixture(scope="module")
def exe():
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    subprocess.check_call(["make", "-C", os.path.join(REPO, "host"), "-s"], env=env)
    return os.path.join(REPO, "host", "sylph-b200")


@pytest.fixture(scope="module")
def d(tmp_path_factory):
    d = tmp_path_factory.mktemp("names")
    os.symlink(DATA, str(d / "test_files"))
    return str(d)


def run(exe, args, cwd, rc=0):
    e = dict(os.environ)
    for k in ("SYL_DRIVER_BATCH_BASES", "SYL_DRIVER_SAMPLES_PER_CALL", "SYL_DRIVER_ROWS", "SYL_INGEST_CHUNK", "SYL_HOST_INGEST"):
        e.pop(k, None)
    r = subprocess.run([exe] + args, cwd=cwd, env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == rc, r.stderr[-3000:]
    return r


class Ref:
    """the oracle's sketches, once per input"""

    def __init__(self, d):
        self.d, self.m = d, {}

    def _get(self, key, f):
        if key not in self.m:
            self.m[key] = f()
        return self.m[key]

    def reads(self, f, name=None):
        s = self._get(("r", f), lambda: D.read_sketch(os.path.join(self.d, f), f))
        return dict(s, sample_name=name)

    def pair(self, f1, f2, name=None):
        s = self._get(("p", f1, f2), lambda: D.pair_sketch(os.path.join(self.d, f1), os.path.join(self.d, f2), f1))
        return dict(s, sample_name=name)

    def genomes(self, files):
        return sum((self._get(("g", f), lambda: D.genome_sketches(os.path.join(self.d, f), f)) for f in files), [])


@pytest.fixture(scope="module")
def ref(d):
    return Ref(d)


def out(d, sub, f):
    return os.path.join(d, sub, f)


def test_reference_sample_names(exe, d, ref):
    """test_sample_names: --lS with a pair, --lS with two read files, -S with one and two pairs"""
    run(exe, ["sketch", "-1", T1, "-2", T2, "-d", "sn", "--lS", "test_files/single_sample.txt", "--fpr", "0"], d)
    assert_sylsp(out(d, "sn", "SAMPLE_TEST.paired.sylsp"), ref.pair(T1, T2, "SAMPLE_TEST"))
    run(exe, ["sketch", T1, O157, "-d", "sn", "--lS", "test_files/sample_list.txt"], d)
    assert_sylsp(out(d, "sn", "S1.sylsp"), ref.reads(T1, "S1"))
    assert_sylsp(out(d, "sn", "S2.sylsp"), ref.reads(O157, "S2"))
    prof = run(exe, ["profile", "sn/S2.sylsp", EC590], d).stdout
    assert "S2" in prof and "o157_reads" not in prof
    D.compare_tsv(prof, D.contain(ref.genomes([EC590]), [ref.reads(O157, "S2")], True), True)
    run(exe, ["sketch", "-1", T1, "-2", T2, "-d", "sn", "-S", "SAMPLE_TEST_S", "--fpr", "0"], d)
    assert_sylsp(out(d, "sn", "SAMPLE_TEST_S.paired.sylsp"), ref.pair(T1, T2, "SAMPLE_TEST_S"))
    run(exe, ["sketch", "-1", T1, T1, "-2", T2, T2, "-d", "sn", "-S", "SAMPLE_TEST_S", "SAMPLE_TEST_S1", "--fpr", "0"], d)
    assert_sylsp(out(d, "sn", "SAMPLE_TEST_S1.paired.sylsp"), ref.pair(T1, T2, "SAMPLE_TEST_S1"))
    assert sorted(os.listdir(os.path.join(d, "sn"))) == sorted(
        ["SAMPLE_TEST.paired.sylsp", "S1.sylsp", "S2.sylsp", "SAMPLE_TEST_S.paired.sylsp", "SAMPLE_TEST_S1.paired.sylsp"])


def test_reference_lists(exe, d, ref):
    """test_sketch: --l1/--l2 and -g t1.fq -r t2.fq; test_sketch_list: --gl and --rl of list.txt"""
    run(exe, ["sketch", "--l1", "test_files/pair_list1.txt", "--l2", "test_files/pair_list2.txt", "-d", "l12", "--fpr", "0"], d)
    assert os.listdir(os.path.join(d, "l12")) == ["t1.fq.paired.sylsp"]
    assert_sylsp(out(d, "l12", "t1.fq.paired.sylsp"), ref.pair(T1, T2))
    run(exe, ["sketch", "-g", T1, "-r", T2, "-d", "gr", "-o", "gr/testdb"], d)
    assert sorted(os.listdir(os.path.join(d, "gr"))) == ["t2.fq.sylsp", "testdb.syldb"]
    assert_syldb(out(d, "gr", "testdb.syldb"), ref.genomes([T1]))
    assert_sylsp(out(d, "gr", "t2.fq.sylsp"), ref.reads(T2))
    listed = [ln for ln in open(os.path.join(DATA, "list.txt")).read().split("\n") if ln]
    assert listed == [EC590, K12G, O157G, O157]
    os.makedirs(os.path.join(d, "gl"))
    run(exe, ["sketch", "--gl", "test_files/list.txt", "-o", "gl/db"], d)
    assert os.listdir(os.path.join(d, "gl")) == ["db.syldb"]
    assert_syldb(out(d, "gl", "db.syldb"), ref.genomes(listed))                     # the .fastq.gz is a genome too
    run(exe, ["sketch", "--rl", "test_files/list.txt", "-o", "rl/db", "-d", "rl"], d)
    assert sorted(os.listdir(os.path.join(d, "rl"))) == sorted(os.path.basename(f) + ".sylsp" for f in listed)
    for f in (EC590, O157):                                                          # the .fasta.gz is a sample too
        assert_sylsp(out(d, "rl", os.path.basename(f) + ".sylsp"), ref.reads(f))


def test_reference_inspect(exe, d, ref):
    """test_inspect: a db of two genomes (plus a sample), a pair sketch; then inspect's YAML against the restatement"""
    run(exe, ["sketch", EC590, K12G, O157, "-o", "ins/db", "-d", "ins"], d)
    run(exe, ["sketch", "-1", K1, "-2", K2, "-d", "ins", "--fpr", "0"], d)
    paired = run(exe, ["inspect", "./ins/k12_R1.fq.paired.sylsp"], d).stdout
    assert "k12_R1.fq" in paired
    db = run(exe, ["inspect", "./ins/db.syldb"], d).stdout
    assert "e.coli-EC590.fasta.gz" in db and "e.coli-K12.fasta.gz" in db
    files = ["ins/db.syldb", "ins/o157_reads.fastq.gz.sylsp", "ins/k12_R1.fq.paired.sylsp"]
    cwd = os.getcwd()
    os.chdir(d)
    try:
        want = I.inspect(files)
    finally:
        os.chdir(cwd)
    assert run(exe, ["inspect"] + files, d).stdout == want
    assert "  paired: true\n" in want and "  sample_name: null\n" in want and "    genome_size: " in want


def _mixed(exe, d, t, sub):
    """names from every source at once: a pair, -l (a read and a genome), a positional read, -r and --rl"""
    with open(os.path.join(d, "mixed_l.txt"), "w") as f:
        f.write("%s\n\n%s\n" % (T1, K12G))
    with open(os.path.join(d, "mixed_rl.txt"), "w") as f:
        f.write(EC590 + "\n")
    return run(exe, ["sketch", "-t", t, "-l", "mixed_l.txt", T2, "-r", K2, "--rl", "mixed_rl.txt",
                     "-S", "pair", "from_l", "positional", "dir/from_r", "from_rl/", "-1", K1, "-2", K2, "--fpr", "0",
                     "-d", sub, "-o", sub + "/db"], d)


def test_names_follow_the_reference_order(exe, d, ref):
    """name i goes to pair i, then to the reads in the order -l, positional, -r, --rl; a name is written under its last
    path component; query/profile print the names"""
    os.makedirs(os.path.join(d, "mx1"))
    _mixed(exe, d, "1", "mx1")
    assert sorted(os.listdir(os.path.join(d, "mx1"))) == sorted(
        ["pair.paired.sylsp", "from_l.sylsp", "positional.sylsp", "from_r.sylsp", "from_rl.sylsp", "db.syldb"])
    want = {"pair.paired.sylsp": ref.pair(K1, K2, "pair"), "from_l.sylsp": ref.reads(T1, "from_l"),
            "positional.sylsp": ref.reads(T2, "positional"), "from_r.sylsp": ref.reads(K2, "dir/from_r"),
            "from_rl.sylsp": ref.reads(EC590, "from_rl/")}
    for f, w in want.items():
        assert_sylsp(out(d, "mx1", f), w)
    assert_syldb(out(d, "mx1", "db.syldb"), ref.genomes([K12G]))
    # -t 8 writes the same bytes
    os.makedirs(os.path.join(d, "mx8"))
    _mixed(exe, d, "8", "mx8")
    for f in os.listdir(os.path.join(d, "mx1")):
        assert open(out(d, "mx1", f), "rb").read() == open(out(d, "mx8", f), "rb").read(), f
    # query / profile rows of named sketches carry the names
    named = ["mx1/" + f for f in want]
    genomes = [EC590, K12G, O157G]
    for cmd in ("query", "profile"):
        pt = cmd == "profile"
        text = run(exe, [cmd] + named + genomes, d).stdout
        rows = D.contain(ref.genomes(genomes), list(want.values()), pt)
        assert "from_rl/" in {w[2][0][0] for w in rows}
        D.compare_tsv(text, rows, pt)
    # inspect of the driver's sketches
    files = named + ["mx1/db.syldb"]
    cwd = os.getcwd()
    os.chdir(d)
    try:
        assert run(exe, ["inspect"] + files, d).stdout == I.inspect(files)
    finally:
        os.chdir(cwd)


def test_unnamed_runs_unchanged(exe, d, ref):
    """without names, -l reads and genomes land where they always did: one sketch per read file, genomes in -g,
    positional, -l, --gl order"""
    with open(os.path.join(d, "un_l.txt"), "w") as f:
        f.write("%s\n%s\n" % (K12G, T1))
    with open(os.path.join(d, "un_gl.txt"), "w") as f:
        f.write(O157G + "\n")
    os.makedirs(os.path.join(d, "un"))
    run(exe, ["sketch", "-l", "un_l.txt", EC590, T2, "-g", K1, "--gl", "un_gl.txt", "-d", "un", "-o", "un/db"], d)
    assert sorted(os.listdir(os.path.join(d, "un"))) == ["db.syldb", "t1.fq.sylsp", "t2.fq.sylsp"]
    assert_syldb(out(d, "un", "db.syldb"), ref.genomes([K1, EC590, K12G, O157G]))
    assert_sylsp(out(d, "un", "t1.fq.sylsp"), ref.reads(T1))
    shutil.rmtree(os.path.join(d, "un"))
