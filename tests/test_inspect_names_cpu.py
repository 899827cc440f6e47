"""CPU suite: `sylph-b200 inspect` against its Python restatement (tests/inspect_ref.py) on crafted sketches, its
refusals of bad files, and the argument errors of sample names (-S / --lS) and pair lists (--l1 / --l2), which are
all reported before a device is needed."""
import os
import struct
import subprocess

import numpy as np
import pytest

from tests import inspect_ref as I
from tests.util import REPO

NO_GPU = dict(os.environ, CUDA_VISIBLE_DEVICES="")


@pytest.fixture(scope="module")
def exe():
    from sylph_b200 import build
    build.build()
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    subprocess.check_call(["make", "-C", os.path.join(REPO, "host"), "-s"], env=env)
    return os.path.join(REPO, "host", "sylph-b200")


def run(exe, args, cwd, rc=0):
    r = subprocess.run([exe] + args, cwd=cwd, env=NO_GPU, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=120)
    assert r.returncode == rc, r.stderr.decode()[-3000:]
    return r.stdout.decode("utf-8"), r.stderr.decode("utf-8")


# names that serde_yaml writes plain, single-quoted or double-quoted
NAMES = ["", "plain name.fq", "123", "-17", "+5", "0x1F", "0o17", "0b101", "-0x10", "007", "1e3", "1.", ".5", "-2.5E-3",
         "1e400", "inf", "nan", ".inf", "-.inf", "+.inf", ".nan", ".NaN", "true", "False", "null", "~", "Null", "yes",
         "a: b", "a:b", "a:", "key #c", "key#c", "#c", "-x", "- x", "-", "*x", "&x", "!x", "'x", '"x', "%x", "@x", "`x",
         "?x", "? x", ":x", "[x", "{x", "|x", ">x", ",x", "x,y[z]", "---x", "...", " lead", "trail ", "tab\there",
         "e.coli ünïcode Øresund", "emoji 😀", "nbsp\u00a0here", "bom\ufeffhere", "del\x7f", "nul\x00byte",
         "bell\x07", "esc\x1b", "c1\u0085nel", "back\\slash \"quoted\"", "it's", "line\nbreak", "cr\rhere",
         "ls\u2028here", "x" * 300 + " long words " * 20, "340282366920938463463374607431768211455",
         "340282366920938463463374607431768211456", "-170141183460469231731687303715884105728",
         "0x" + "f" * 32, "0x1" + "0" * 32, "NZ_CP016182.2 Escherichia coli strain EC590 chromosome, complete genome"]


def _genome(rng, name, contig, tracked, c=200, k=31, gs=None, ms=30):
    n = int(rng.integers(0, 50))
    return dict(genome_kmers=rng.integers(0, 2 ** 63, n, dtype=np.uint64),
                tracked=rng.integers(0, 2 ** 63, int(rng.integers(0, 20)), dtype=np.uint64) if tracked else None,
                file_name=name, first_contig_name=contig, c=c, k=k, gn_size=gs if gs is not None else n * 200, min_spacing=ms)


def _sample(rng, n, c, k, mrl, file_name="reads.fq", name=None, paired=False):
    return dict(hashes=rng.integers(0, 2 ** 63, n, dtype=np.uint64), counts=rng.integers(1, 9, n, dtype=np.uint32), c=c,
                k=k, file_name=file_name, sample_name=name, paired=paired, mean_read_length=mrl)


@pytest.fixture(scope="module")
def sketches(tmp_path_factory):
    """-> (directory, database files, sample files, an unrelated file)"""
    from sylph_b200 import formats as F
    d = tmp_path_factory.mktemp("inspect")
    rng = np.random.default_rng(11)
    dbs, samples = [], []
    half = len(NAMES) // 2
    F.write_syldb(str(d / "many.syldb"), [_genome(rng, NAMES[i], NAMES[-1 - i], True) for i in range(half)])
    F.write_syldb(str(d / "untracked.sylqueries"),
                  [_genome(rng, "g%d.fa" % i, NAMES[half + i], False, c=1000, k=21, ms=7) for i in range(len(NAMES) - half)])
    F.write_syldb(str(d / "empty.syldb"), [])
    F.write_syldb(str(d / "one.syldb"), [_genome(rng, "ref genomes/a.fna.gz", "", True, gs=2 ** 40 + 3)])
    dbs = ["many.syldb", "untracked.sylqueries", "empty.syldb", "one.syldb"]
    # (n, c, k, mean read length): 0 with and without k-mers (inf, nan), 150, 1/3 and f32 products that round
    cases = [(0, 200, 31, 0.), (5, 200, 31, 0.), (40, 200, 31, 150.), (7, 200, 21, 1 / 3), (16777217, 3, 31, 99.7),
             (12345, 1000, 31, 151.123456789), (3, 200, 31, 1e-7), (3, 200, 31, 1e17), (3, 200, 31, 0.001),
             (3, 200, 31, 1e-5), (3, 200, 31, 5e-324), (3, 200, 31, -0.), (3, 200, 31, float("nan")),
             (3, 200, 31, float("inf")), (3, 200, 31, 123456789012345680.), (3, 200, 31, 1234567890123456.7),
             (3, 7, 31, 12345678.9), (1, 1, 31, -30.), (3, 2 ** 40, 31, 1e300)]
    for i, (n, c, k, mrl) in enumerate(cases):
        name = None if i % 3 == 0 else NAMES[(7 * i) % len(NAMES)]
        s = _sample(rng, min(n, 50), c, k, mrl, "reads %d.fq" % i, name, paired=i % 2 == 1)
        path = d / ("s%02d.%s" % (i, "sylsample" if i == 4 else "sylsp"))
        F.write_sylsp(str(path), s)
        if n > 50:   # more entries than were written: the same file with a longer (sparse) run of zero entries
            tail = path.read_bytes()[8 + 12 * 50:]
            with open(path, "wb") as f:
                f.write(struct.pack("<Q", n))
                f.seek(8 + 12 * n)
                f.write(tail)
        samples.append(path.name)
    for i, nm in enumerate(NAMES):   # every name once as a sample name, once as a file name
        F.write_sylsp(str(d / ("n%03d.sylsp" % i)), _sample(rng, 2, 200, 31, 150., nm, nm, paired=bool(i % 2)))
        samples.append("n%03d.sylsp" % i)
    (d / "notes.txt").write_text("not a sketch\n")
    return d, dbs, samples, "notes.txt"


def test_inspect_matches_restatement(exe, sketches):
    d, dbs, samples, other = sketches
    files = [samples[0], dbs[0], other] + samples[1:] + dbs[1:]     # databases are printed first whatever the order
    out, err = run(exe, ["inspect"] + files, d)
    cwd = os.getcwd()
    try:
        os.chdir(d)
        want = I.inspect(files)
    finally:
        os.chdir(cwd)
    assert out == want
    assert "notes.txt file is not a .sylsp or .syldb file. Skipping..." in err
    assert "The database sketch `empty.syldb` is empty. Skipping..." in err
    # the shapes the restatement is meant to produce, spelled out
    assert out.startswith("- database_file: many.syldb\n  c: 200\n  k: 31\n  min_spacing_parameter: 30\n  genome_files:\n"
                          "  - file_name: ''\n    genome_kmers_num: ")
    assert "- database_file: ''\n  c: 0\n  k: 0\n  min_spacing_parameter: 0\n  genome_files: []\n" in out
    assert "- database_file: untracked.sylqueries\n  c: 1000\n  k: 21\n  min_spacing_parameter: 7\n" in out
    assert "    first_contig_name: ''\n    genome_size: 1099511627779\n" in out
    for line in ("  approximate_number_bases: .nan\n  mean_read_length: 0.0\n  sample_name: null\n  paired: false\n",
                 "  approximate_number_bases: .inf\n  mean_read_length: 0.0\n",
                 "  mean_read_length: 150.0\n", "  mean_read_length: 0.3333333333333333\n",
                 "  mean_read_length: 1e-7\n", "  mean_read_length: 1e17\n", "  mean_read_length: 0.001\n",
                 "  mean_read_length: -0.0\n", "  mean_read_length: .nan\n", "  mean_read_length: .inf\n",
                 "  mean_read_length: 5e-324\n", "  num_sketched_kmers: 16777217\n", "  paired: true\n",
                 "- file_name: '123'\n", "- file_name: 'true'\n", "- file_name: 'null'\n", "- file_name: '1e3'\n",
                 "- file_name: '007'\n", "- file_name: '.inf'\n", "- file_name: 1e400\n", "- file_name: nan\n",
                 "- file_name: 'a: b'\n", "- file_name: a:b\n", "- file_name: 'key #c'\n", "- file_name: key#c\n",
                 "- file_name: -x\n", "- file_name: '- x'\n", "- file_name: '-'\n", "- file_name: '*x'\n", "- file_name: '''x'\n",
                 "- file_name: ' lead'\n", "- file_name: 'trail '\n", "- file_name: \"tab\\there\"\n",
                 "- file_name: e.coli ünïcode Øresund\n", "- file_name: \"emoji \\U0001F600\"\n",
                 "- file_name: \"nul\\0byte\"\n", "- file_name: it's\n", "- file_name: plain name.fq\n",
                 "  sample_name: '-17'\n"):
        assert line in out, line
    assert "- file_name: NZ_CP016182.2 Escherichia coli strain EC590 chromosome, complete genome\n" in out


def test_inspect_output_file(exe, sketches, tmp_path):
    d, dbs, samples, _ = sketches
    files = [str(d / f) for f in dbs[:2] + samples[:3]]
    out, _ = run(exe, ["inspect", "-o", str(tmp_path / "out.yaml")] + files, tmp_path)
    assert out == ""
    assert (tmp_path / "out.yaml").read_text("utf-8") == I.inspect(files)
    only_samples, _ = run(exe, ["inspect"] + files[2:], tmp_path)
    assert only_samples == I.samples_yaml([I.read_sample(f) for f in files[2:]]) and only_samples.startswith("- file_name: ")
    nothing, err = run(exe, ["inspect", "notes.txt"], d)
    assert nothing == "" and "Skipping" in err


def test_inspect_bad_files(exe, sketches, tmp_path):
    d, dbs, samples, _ = sketches
    good = (d / samples[2]).read_bytes()
    for cut in (7, 30, len(good) - 1):
        (tmp_path / "cut.sylsp").write_bytes(good[:cut])
        with pytest.raises(I.InvalidSketch):
            I.read_sample(str(tmp_path / "cut.sylsp"))
        out, err = run(exe, ["inspect", "cut.sylsp"], tmp_path, rc=1)
        assert out == ""
        assert "The sequence sketch `cut.sylsp` is not a valid sketch. Perhaps it is an older, incompatible version" in err
    db = (d / dbs[0]).read_bytes()
    (tmp_path / "cut.syldb").write_bytes(db[:len(db) // 2])
    out, err = run(exe, ["inspect", "cut.syldb"], tmp_path, rc=1)
    assert "The database sketch `cut.syldb` is not a valid sketch. Perhaps it is an older, incompatible version" in err
    (tmp_path / "tag.sylsp").write_bytes(good[:-9] + b"\x02" + good[-8:])           # a paired flag of 2
    run(exe, ["inspect", "tag.sylsp"], tmp_path, rc=1)
    bad_utf8 = bytearray(good)
    bad_utf8[good.index(b"reads 2.fq")] = 0xFF                                        # not UTF-8
    (tmp_path / "utf8.sylsp").write_bytes(bytes(bad_utf8))
    with pytest.raises(I.InvalidSketch):
        I.read_sample(str(tmp_path / "utf8.sylsp"))
    run(exe, ["inspect", "utf8.sylsp"], tmp_path, rc=1)
    out, err = run(exe, ["inspect", "missing.sylsp"], tmp_path, rc=1)
    assert out == "" and "The sketch `missing.sylsp` could not be opened. Exiting" in err


def test_ryu_layout_of_the_restatement():
    """the float layouts the restatement claims for ryu, on values whose text is known"""
    f64 = [(150., "150.0"), (14904.243243243243, "14904.243243243243"), (0.1, "0.1"), (1e16, "1e16"),
           (1e15, "1000000000000000.0"), (1.5e-7, "1.5e-7"), (0.0001, "0.0001"), (1e-5, "0.00001"), (1e-6, "1e-6"), (-2.5, "-2.5"),
           (123456789012345680., "1.2345678901234568e17"), (5e-324, "5e-324"), (0., "0.0")]
    for v, t in f64:
        assert I.yaml_float(v, False) == t, v
    f32 = [(70., "70.0"), (0.1, "0.1"), (1e13, "1e13"), (1e12, "1000000000000.0"), (16777217., "16777216.0"),
           (1e-6, "0.000001"), (1e-7, "1e-7"), (3.4028235e38, "3.4028235e38")]
    for v, t in f32:
        assert I.yaml_float(v, True) == t, v


LIST_ERRORS = [  # (args, list files to write, message)
    (["sketch", "r.fq", "-S", "a", "b"], {}, "Sample name length is not equal to the number of reads. Exiting"),
    (["sketch", "r1.fq", "r2.fq", "g.fa", "-S", "only"], {}, "Sample name length is not equal to the number of reads"),
    (["sketch", "-1", "a_1.fq", "-2", "a_2.fq", "--fpr", "0", "r.fq", "-S", "pair"], {},
     "Sample name length is not equal to the number of reads"),
    (["sketch", "r1.fq", "r2.fq", "--lS", "names.txt", "-S", "a", "b"], {"names.txt": "a\nb\nc\n"},
     "Sample name length is not equal to the number of reads"),                  # --lS wins over a -S that would fit
    (["sketch", "-l", "lst.txt", "--rl", "rl.txt", "-S", "a", "b"], {"lst.txt": "x.fq\n\ny.fa\n", "rl.txt": "z.fa\n\n"},
     "Sample name length is not equal to the number of reads"),                  # -l skips empty lines, --rl keeps them
    (["sketch", "--l1", "l1.txt", "--l2", "l2.txt", "--fpr", "0"], {"l1.txt": "a_1.fq\nb_1.fq\n", "l2.txt": "a_2.fq\n"},
     "Different number of paired sequences. Exiting."),
    (["sketch", "-1", "a_1.fq", "-2", "a_2.fq", "--l1", "l1.txt", "--fpr", "0"], {"l1.txt": "b_1.fq"},
     "Different number of paired sequences. Exiting."),
    (["sketch", "--l1", "l1.txt", "--l2", "l2.txt"], {"l1.txt": "a_1.fq\r\n", "l2.txt": "a_2.fq\n"},
     "paired-end reads need --fpr 0"),
    (["sketch", "--gl", "missing.txt"], {}, "cannot open list file missing.txt"),
    (["query", "-S", "x", "r.fq", "g.fa"], {}, "unknown option -S"),
    (["profile", "--l1", "l1.txt", "g.fa"], {}, "unknown option --l1"),
]


@pytest.mark.parametrize("args,lists,msg", LIST_ERRORS)
def test_name_and_list_errors_before_the_device(exe, tmp_path, args, lists, msg):
    """Each is refused with exit code 1 and its message while the arguments are read: no GPU and no input file needed."""
    for name, text in lists.items():
        (tmp_path / name).write_text(text)
    out, err = run(exe, args, tmp_path, rc=1)
    assert msg in err and out == "", err


def test_names_that_fit_pass_argument_checks(exe, tmp_path):
    """With as many names as pairs plus reads the run gets past the checks: without a GPU it fails only at the device"""
    (tmp_path / "lst.txt").write_text("x.fq\n\ny.fa\n")
    (tmp_path / "rl.txt").write_text("z.fa\n\n")
    _, err = run(exe, ["sketch", "-l", "lst.txt", "--rl", "rl.txt", "p_1.fq", "-S", "a", "b", "c", "d", "e",
                       "-1", "p_1.fq", "-2", "p_2.fq", "--fpr", "0"], tmp_path, rc=1)
    assert "syl_ctx_create" in err and "Sample name length" not in err
