"""CPU: the rule syl_db_shards_create cuts a database by (sylph_b200/csrc/shard_cut.hpp, built on the host): contiguous
genome ranges of at most `cap` index entries, greedily in genome order; a genome above the cap alone; a genome above
2^32-3 entries refused; cap 0 and caps above 2^32-3 meaning 2^32-3."""
import itertools
import os
import subprocess

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "sylph_b200", "csrc")
MAX = 2**32 - 3


@pytest.fixture(scope="module")
def cut_exe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("shard_cut") / "shard_cut_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", CSRC, "-o", exe,
                           os.path.join(REPO, "tests", "cpp", "shard_cut_check.cpp")])
    return exe


def cut(exe, cases):
    """cases: [(cap, kmer counts per genome, tracked counts per genome or None)] -> ["ok ..." | "bad g"] per case"""
    lines = []
    for cap, nk, nt in cases:
        ko = " ".join(map(str, itertools.accumulate(nk, initial=0)))
        to = "-" if nt is None else " ".join(map(str, itertools.accumulate(nt, initial=0)))
        lines.append("%d %d %s %s" % (len(nk), cap, ko, to))
    out = subprocess.run([exe], input="\n".join(lines) + "\n", stdout=subprocess.PIPE, text=True, check=True).stdout
    return out.splitlines()


def expected(cap, nk, nt):
    """the rule, restated: first genome of every shard, then G"""
    cap = MAX if cap == 0 or cap > MAX else cap
    e = [a + (0 if nt is None else b) for a, b in zip(nk, nt if nt is not None else nk)]
    if any(x > MAX for x in e):
        return "bad %d" % next(g for g, x in enumerate(e) if x > MAX)
    first, n = [0], 0
    for g, x in enumerate(e):
        if g > first[-1] and n + x > cap:
            first.append(g)
            n = 0
        n += x
    if e:
        first.append(len(e))
    return "ok " + " ".join(map(str, first))


def test_ranges_of_uneven_genomes(cut_exe):
    rng = np.random.default_rng(3)
    cases = []
    for cap in (0, 1, 7, 100, 999, 5000, 10**6, MAX, MAX + 10, 2**64 - 1):
        for tracked in (False, True):
            nk = [int(x) for x in rng.choice([0, 0, 1, 30, 400, 2500], 60)]
            nt = [int(x) for x in rng.integers(0, 50, 60)] if tracked else None
            cases.append((cap, nk, nt))
    got = cut(cut_exe, cases)
    for (cap, nk, nt), g in zip(cases, got):
        assert g == expected(cap, nk, nt), (cap, g)
        first = [int(x) for x in g.split()[1:]]
        assert first[0] == 0 and first[-1] == len(nk) and all(b > a for a, b in zip(first, first[1:]))


def test_one_genome_per_shard_and_all_in_one(cut_exe):
    nk, nt = [5, 0, 9, 3], [1, 0, 0, 2]
    one, every, none = cut(cut_exe, [(1, nk, nt), (10**9, nk, nt), (0, [], None)])
    assert one == "ok 0 1 2 3 4"          # the empty genome 1 follows genome 0's full shard into its own
    assert every == "ok 0 4"
    assert none == "ok 0"                 # no genome, no shard


def test_single_large_genome(cut_exe):
    """a genome above the cap is a shard of its own; one above 2^32-3 entries cannot be indexed at all"""
    got = cut(cut_exe, [(10, [3, 4, 50, 2, 1], None),
                        (10, [3, MAX - 2, 2], [0, 2, 0]),          # exactly 2^32-3 entries: fits one index
                        (10, [3, MAX - 2, 2], [0, 3, 0]),          # one more: refused
                        (0, [2**31, 2**31, 5], None)])             # the default cap splits 2^32 entries in two
    assert got == ["ok 0 2 3 5", "ok 0 1 2 3", "bad 1", "ok 0 1 3"]
