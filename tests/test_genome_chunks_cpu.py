"""CPU: how a host-memory genome batch is cut into chunks for the host feeder (sylph_b200/csrc/genome_chunks.hpp, built
on the host).  Chunks hold whole genomes (whole contigs with `individual`), cover every genome exactly once and in
order, and keep to the chunk size in bases and the contig cap unless one genome alone exceeds them; such a genome is
a chunk of its own."""
import os
import subprocess

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "sylph_b200", "csrc")
MIB = 1 << 20
ING_CHUNK = 32 * MIB
ING_MAXREC = 1 << 19


@pytest.fixture(scope="module")
def plan_exe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("genome_chunks") / "genome_chunks_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", CSRC, "-o", exe,
                           os.path.join(REPO, "tests", "cpp", "genome_chunks_check.cpp")])
    return exe


def plan(exe, cases):
    """cases: [(max_bases, max_contigs, contig_off, genome_off or None)] -> per case [(g0, g1, c0, c1, own)]"""
    lines = []
    for max_bases, max_contigs, co, go in cases:
        f = [max_bases, max_contigs, int(go is None), len(co) - 1] + list(co)
        f += [len(co) - 1] if go is None else [len(go) - 1] + list(go)
        lines.append(" ".join(str(int(x)) for x in f))
    out = subprocess.run([exe], input="\n".join(lines) + "\n", stdout=subprocess.PIPE, text=True, check=True).stdout.split("\n")
    res, i = [], 0
    for _ in cases:
        n = int(out[i])
        res.append([tuple(map(int, out[i + 1 + j].split())) for j in range(n)])
        i += 1 + n
    return res


def check(chunks, max_bases, max_contigs, co, go):
    """The plan's invariants, from the offsets alone."""
    co = [int(x) for x in co]
    individual = go is None
    go = list(range(len(co))) if individual else [int(x) for x in go]
    G = len(go) - 1
    if G == 0:
        assert chunks == []
        return
    assert chunks[0][0] == 0 and chunks[-1][1] == G            # every genome, in order
    for (g0, g1, c0, c1, own), nxt in zip(chunks, chunks[1:] + [None]):
        assert g0 < g1                                           # at least one genome
        if nxt is not None:
            assert nxt[0] == g1                                  # contiguous, disjoint
        assert c0 == go[g0] and c1 == go[g1]                     # cut at genome (contig) boundaries only
        bases, contigs = co[c1] - co[c0], c1 - c0
        first_fits = co[go[g0 + 1]] - co[c0] <= max_bases and go[g0 + 1] - c0 <= max_contigs
        assert own == (not first_fits)
        if own:
            assert g1 == g0 + 1                                  # an oversized genome is alone
        else:
            assert bases <= max_bases and contigs <= max_contigs
            if nxt is not None and not nxt[4]:                   # greedy: the next genome did not fit
                g = g1
                assert co[go[g + 1]] - co[c0] > max_bases or go[g + 1] - c0 > max_contigs


def offsets(lengths):
    return np.concatenate([[0], np.cumsum(np.asarray(lengths, dtype=np.uint64))]).astype(np.uint64)


def run_check(exe, cases):
    for cs, chunks in zip(cases, plan(exe, cases)):
        check(chunks, *cs)
    return plan(exe, cases)


def test_genome_chunks_random(plan_exe):
    rng = np.random.default_rng(7)
    cases = []
    for t in range(60):
        n_genomes = int(rng.integers(1, 60))
        contigs = rng.integers(0, 6, n_genomes)               # zero-contig genomes included
        n_contigs = int(contigs.sum())
        lens = rng.integers(0, 5000, n_contigs)
        lens[rng.random(n_contigs) < 0.2] = 0                  # empty contigs
        lens[rng.random(n_contigs) < 0.2] = 30                 # shorter than 2k
        co, go = offsets(lens), offsets(contigs)
        max_bases = int(rng.choice([16, 1000, 4096, 20000, 10**9]))
        max_contigs = int(rng.choice([1, 3, 8, ING_MAXREC]))
        cases.append((max_bases, max_contigs, co, go))
        cases.append((max_bases, max_contigs, co, None))     # individual: every contig a genome
    run_check(plan_exe, cases)


def test_genome_chunks_edge_cases(plan_exe):
    cases = [
        (ING_CHUNK, ING_MAXREC, offsets([1000]), offsets([1])),                  # a single genome
        (ING_CHUNK, ING_MAXREC, offsets([]), offsets([0, 0, 0])),                # only empty genomes
        (ING_CHUNK, ING_MAXREC, offsets([0, 0]), offsets([0, 2, 0])),            # empty contigs
        (ING_CHUNK, ING_MAXREC, offsets([]), offsets([])),                       # no genome at all
        (1000, ING_MAXREC, offsets([400, 600, 1, 999]), offsets([2, 1, 1])),     # exactly one chunk, then one more
        (1000, ING_MAXREC, offsets([5000, 10, 10]), offsets([1, 0, 0, 2])),      # oversized first, empty ones behind it
        (1000, ING_MAXREC, offsets([10, 5000, 10]), offsets([1, 0, 1, 1])),      # oversized in the middle
        (1000, 2, offsets([1, 1, 1, 1, 1]), offsets([3, 2])),                    # too many contigs: own chunk
    ]
    res = run_check(plan_exe, cases)
    assert res[0] == [(0, 1, 0, 1, 0)]
    assert res[1] == [(0, 3, 0, 0, 0)]
    assert res[2] == [(0, 3, 0, 2, 0)]
    assert res[3] == []
    assert res[4] == [(0, 1, 0, 2, 0), (1, 3, 2, 4, 0)]
    assert res[5] == [(0, 1, 0, 1, 1), (1, 4, 1, 3, 0)]
    assert res[6] == [(0, 2, 0, 1, 0), (2, 3, 1, 2, 1), (3, 4, 2, 3, 0)]
    assert res[7] == [(0, 1, 0, 3, 1), (1, 2, 3, 5, 0)]


def test_genome_chunks_5gbp_genome(plan_exe):
    """Offsets of a 5 Gbp genome (no memory behind them): it is a chunk of its own, with u64 offsets, between small
    genomes that share chunks."""
    big = 5 * 10**9
    lens = [10**6] * 40 + [big // 2, big - big // 2] + [10**6] * 40
    co, go = offsets(lens), offsets([1] * 40 + [2] + [1] * 40)
    res = run_check(plan_exe, [(ING_CHUNK, ING_MAXREC, co, go)])[0]
    own = [c for c in res if c[4]]
    assert own == [(40, 41, 40, 42, 1)]
    assert sum(1 for c in res if not c[4]) == 4                  # 40 Mbp on either side: two 32 MiB chunks each
