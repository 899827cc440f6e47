"""CPU: how host-memory samples are cut into batches for syl_query_host_samples / syl_profile_host_samples
(sylph_b200/csrc/sample_batches.hpp, built on the host).  Batches are contiguous and cover every sample once; each is
the longest run from its first sample that keeps twice its device bytes within the budget, its pairs within the pair
cap, its k-mers within the k-mer cap and its samples within the sample cap.  A sample that alone does not fit is an
error naming the bytes it needs."""
import os
import random
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "sylph_b200", "csrc")
# per_kmer, per_sample, per_hit, per_pair, fixed
COST = (36, 200, 16, 1040, 1000)
BIG = 1 << 62


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("sample_batches") / "sample_batches_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I", CSRC, "-o", out,
                           os.path.join(REPO, "tests", "cpp", "sample_batches_check.cpp")])
    return out


def run(exe, cases):
    """cases: [(sizes, G, budget, max_pairs, max_kmers, max_samples, cost)] -> per case ("ok", first) / ("oom", i, bytes)
    / ("kmers", i, n)"""
    lines = []
    for sizes, G, budget, max_pairs, max_kmers, max_samples, cost in cases:
        off = [0]
        for n in sizes:
            off.append(off[-1] + n)
        lines.append(" ".join(str(x) for x in [len(sizes), G, budget, max_pairs, max_kmers, max_samples, *cost, *off]))
    out = subprocess.run([exe], input="\n".join(lines) + "\n", stdout=subprocess.PIPE, text=True, check=True).stdout
    res = []
    for ln in out.strip("\n").split("\n"):
        f = ln.split()
        res.append(("ok", [int(x) for x in f[1:]]) if f[0] == "ok" else (f[0], int(f[1]), int(f[2])))
    return res


def batch_bytes(cost, sizes, G):
    per_kmer, per_sample, per_hit, per_pair, fixed = cost
    return fixed + per_kmer * sum(sizes) + len(sizes) * (per_sample + per_hit * max(sizes) + per_pair * G)


def fits(sizes, G, budget, max_pairs, max_kmers, max_samples, cost):
    return (2 * batch_bytes(cost, sizes, G) <= budget and len(sizes) * G <= max_pairs and sum(sizes) <= max_kmers
            and (not max_samples or len(sizes) <= max_samples))


def model(sizes, G, budget, max_pairs, max_kmers, max_samples, cost):
    for i, n in enumerate(sizes):
        if n > max_kmers:
            return ("kmers", i, n)
        if 2 * batch_bytes(cost, [n], G) > budget:
            return ("oom", i, 2 * batch_bytes(cost, [n], G))
    first = [0]
    for i in range(len(sizes)):
        if i > first[-1] and not fits(sizes[first[-1]:i + 1], G, budget, max_pairs, max_kmers, max_samples, cost):
            first.append(i)
    if sizes:
        first.append(len(sizes))
    return ("ok", first)


def test_zero_samples(exe):
    assert run(exe, [([], 10, 1000, BIG, BIG, 0, COST)]) == [("ok", [0])]


def test_empty_samples(exe):
    """Samples without k-mers cost their per-sample bytes only and batch like any other."""
    need = 2 * batch_bytes(COST, [0, 0, 0], 5)
    assert run(exe, [([0, 0, 0], 5, need, BIG, BIG, 0, COST), ([0, 0, 0], 5, need - 1, BIG, BIG, 0, COST)]) == \
        [("ok", [0, 3]), ("ok", [0, 2, 3])]


def test_sample_exactly_at_budget(exe):
    need = 2 * batch_bytes(COST, [1000], 7)
    assert run(exe, [([1000], 7, need, BIG, BIG, 0, COST)]) == [("ok", [0, 1])]
    # two such samples never share a batch at that budget, and each fits alone
    assert run(exe, [([1000, 1000], 7, need, BIG, BIG, 0, COST)]) == [("ok", [0, 1, 2])]


def test_sample_over_budget_names_the_bytes(exe):
    need = 2 * batch_bytes(COST, [1000], 7)
    assert run(exe, [([10, 1000, 10], 7, need - 1, BIG, BIG, 0, COST)]) == [("oom", 1, need)]


def test_pair_cap(exe):
    """At most max_pairs (sample, genome) pairs per batch; a sample whose pairs alone pass the cap is a batch."""
    res = run(exe, [([5] * 10, 100, BIG, 300, BIG, 0, COST), ([5] * 3, 1000, BIG, 300, BIG, 0, COST)])
    assert res == [("ok", [0, 3, 6, 9, 10]), ("ok", [0, 1, 2, 3])]


def test_sample_and_kmer_caps(exe):
    res = run(exe, [([1] * 7, 1, BIG, BIG, BIG, 3, COST), ([4, 4, 4], 1, BIG, BIG, 8, 0, COST), ([4, 9], 1, BIG, BIG, 8, 0, COST)])
    assert res == [("ok", [0, 3, 6, 7]), ("ok", [0, 2, 3]), ("kmers", 1, 9)]


def test_random_plans_match_the_model(exe):
    rng = random.Random(7)
    cases = []
    for _ in range(300):
        S = rng.randrange(0, 40)
        sizes = [rng.choice([0, rng.randrange(1, 50), rng.randrange(1, 5000)]) for _ in range(S)]
        G = rng.randrange(0, 200)
        budget = rng.randrange(0, 4_000_000)
        cases.append((sizes, G, budget, rng.choice([BIG, rng.randrange(1, 5000)]), rng.choice([BIG, rng.randrange(1, 20000)]),
                      rng.choice([0, rng.randrange(1, 8)]), COST))
    for case, got in zip(cases, run(exe, cases)):
        assert got == model(*case), case
