"""CPU: the scan formulation's host rules (sylph_b200/csrc/scan_plan.hpp, built on the host): when a call on a
host-memory database scans instead of building (each side of the size floor, of the cost crossover and of the one-batch
condition), SYL_DB_SCAN's parsing, the scan chunks of whole genomes against a Python restatement, and the layout of a
sample's lookup table built from sorted keys."""
import itertools
import os
import re
import subprocess

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "sylph_b200", "csrc")
U64 = 2**64


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("scan_plan") / "scan_plan_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", CSRC, "-o", out,
                           os.path.join(REPO, "tests", "cpp", "scan_plan_check.cpp")])
    return out


def run(exe, lines):
    return subprocess.run([exe], input="\n".join(lines) + "\n", stdout=subprocess.PIPE, text=True,
                          check=True).stdout.splitlines()


def constants():
    """the rule's constants, as scan_plan.hpp states them"""
    src = open(os.path.join(CSRC, "scan_plan.hpp")).read()
    out = {}
    for m in re.finditer(r"constexpr (?:double|uint64_t) ([^;]+);", src):
        for part in m.group(1).split(","):
            name, v = (x.strip() for x in part.split("="))
            out[name] = float(eval(v.replace("ull", "")))
    return out


def rule(C, nk, nt, G, S, sk, one, pinned):
    """the rule, restated: the larger of link and probes against the build"""
    if not one or S == 0 or G == 0 or nk + nt < C["SCAN_MIN_ENTRIES"]:
        return 0
    probe = C["PROBE_NS_IN_L2"] if C["TABLE_BYTES_PER_KEY"] * sk <= C["L2_BYTES"] else C["PROBE_NS_BEYOND_L2"]
    link = (C["LINK_NS_PINNED"] if pinned else C["LINK_NS_PAGEABLE"]) * nk
    build = (C["BUILD_NS_PINNED"] if pinned else C["BUILD_NS_PAGEABLE"]) * (nk + nt)
    return int(max(link, probe * S * nk) < build)


def test_rule_at_each_boundary(exe):
    C = constants()
    floor = int(C["SCAN_MIN_ENTRIES"])
    assert run(exe, ["const"]) == ["%d %d" % (floor, 2**25)]
    small = 1000   # k-mers per sample: every table fits L2
    cases = []
    # the size floor: one entry below it builds, at it scans (one sample, tracked entries count towards it)
    cases += [(floor - 1, 0, 1000, 1, small, 1, 0), (floor, 0, 1000, 1, small, 1, 0), (floor - 10, 10, 1000, 1, small, 1, 0)]
    # the one-batch condition, no samples, no genomes
    cases += [(2 * floor, 0, 1000, 1, small, 0, 0), (2 * floor, 0, 1000, 0, 0, 1, 0), (2 * floor, 0, 0, 1, small, 1, 0)]
    # the L2 edge of the tables: a sample count that scans while all tables fit L2 and builds once they do not
    l2 = int(C["L2_BYTES"] / C["TABLE_BYTES_PER_KEY"])
    for pinned, S in ((0, 100), (1, 30)):
        cases += [(2 * floor, 0, 1000, S, l2, 1, pinned), (2 * floor, 0, 1000, S, l2 + 1, 1, pinned)]
    # the sample count where scanning stops paying, pageable and pinned, with and without tracked k-mers
    for nk, nt in ((2 * floor, 0), (1_970_000_000, 330_000_000)):
        for pinned in (0, 1):
            for per in (small, 1_100_000):
                pays = [S for S in range(1, 2000) if rule(C, nk, nt, 113_104, S, S * per, 1, pinned)]
                s_max = max(pays)
                assert s_max < 1999
                cases += [(nk, nt, 113_104, s, s * per, 1, pinned) for s in (1, s_max, s_max + 1, 4 * s_max)]
    got = run(exe, ["rule %d %d %d %d %d %d %d" % c for c in cases])
    want = [str(rule(C, *c)) for c in cases]
    assert got == want, list(zip(cases, got, want))
    assert want[:6] == ["0", "1", "1", "0", "0", "0"]
    assert want[6:10] == ["1", "0", "1", "0"]
    assert "1" in want[10:] and "0" in want[10:]


def test_forced_switch(exe):
    assert run(exe, ["forced 0", "forced 1", "forced -", "forced 2", "forced 10", "forced yes"]) == \
        ["0", "1", "-1", "-1", "-1", "-1"]


def chunks(nk, entries, genomes):
    """whole genomes greedily in genome order, at most `entries` genome k-mers and `genomes` genomes per chunk; a genome
    larger than a chunk alone; an empty genome joins the chunk in front of it unless that one is over the cap"""
    entries, genomes = max(entries, 1), max(genomes, 1)
    first, n = [0], 0
    for g, e in enumerate(nk):
        if g > first[-1] and (n + e > entries or g - first[-1] >= genomes):
            first.append(g)
            n = 0
        n += e
    if nk:
        first.append(len(nk))
    return first


def test_chunks_of_whole_genomes(exe):
    rng = np.random.default_rng(11)
    cases = [([], 5, 10), ([0, 0, 0], 1, 10), ([3, 0, 0, 4, 0], 1, 100),     # empty genomes at chunk starts and ends
             ([2, 50, 2, 0, 1], 10, 100),                                      # a genome larger than a chunk
             ([1] * 10, 100, 3), ([4, 4, 4], 12, 100), ([4, 4, 4], 11, 100)]  # genome cap; last chunk exact / one over
    for entries in (1, 7, 997, 5000):
        for genomes in (1, 5, 10**6):
            cases.append(([int(x) for x in rng.choice([0, 0, 1, 30, 400, 2500], 80)], entries, genomes))
    lines = ["cut %d %d %d %s" % (len(nk), e, gc, " ".join(map(str, itertools.accumulate(nk, initial=0))))
             for nk, e, gc in cases]
    for (nk, e, gc), got in zip(cases, run(exe, lines)):
        first = [int(x) for x in got.split()]
        assert first == chunks(nk, e, gc), (nk, e, gc)
        for a, b in zip(first, first[1:]):
            assert b > a and (b - a == 1 or sum(nk[a:b]) <= e) and b - a <= max(gc, 1)
    # empty genomes join the chunk in front of them, or start the next one after a chunk over the cap
    assert run(exe, lines[:3]) == ["0", "0 3", "0 1 3 4 5"]


def table(keys):
    """the lookup table restated: NB = max(n // 2, 1), M = NB * 2^64 // (maxkey + 1) (saturating), dir[b] = first key of
    bucket >= b, fp = the low 32 bits"""
    n = len(keys)
    NB = max(n // 2, 1)
    M = min((NB << 64) // ((keys[-1] if n else 0) + 1), U64 - 1)
    bucket = [min((k * M) >> 64, NB - 1) for k in keys]
    d = [next((i for i, b in enumerate(bucket) if b >= x), n) for x in range(NB + 1)]
    return NB, M, d, [k & 0xFFFFFFFF for k in keys]


def test_lookup_table_layout(exe):
    rng = np.random.default_rng(5)
    hi = U64 // 200
    samples = [[], [0], [U64 - 2], [0, U64 - 2], [5, 6, 7],
               sorted({int(x) for x in rng.integers(0, hi, 1000, dtype=np.uint64)}),
               sorted({int(x) for x in rng.integers(0, U64 - 1, 3001, dtype=np.uint64)}),
               # keys sharing one bucket and their low 32 bits
               sorted({(1 << 40) + (i << 32) + 77 for i in range(6)} | {int(x) for x in rng.integers(0, 1 << 50, 9, dtype=np.uint64)})]
    got = run(exe, ["table %d %s" % (len(k), " ".join(map(str, k))) for k in samples])
    for keys, line in zip(samples, got):
        v = [int(x) for x in line.split()]
        NB, M, d, fp = table(keys)
        assert v[:2] == [NB, M], keys[:5]
        assert v[2:3 + NB] == d and v[3 + NB:] == fp
        # every key is found in its bucket
        for k in keys:
            b = min((k * M) >> 64, NB - 1)
            assert k in keys[d[b]:d[b + 1]]
    crafted = table(samples[-1])
    fps = crafted[3]
    assert len(set(fps)) < len(fps)


def test_forced_decision_keeps_the_one_batch_condition(exe):
    """SYL_DB_SCAN=1 forces the scan only where the samples fit one batch (a scan stages them all at once); =0 always
    builds; unset leaves it to the rule.  No samples or no genomes never scan."""
    C = constants()
    big = int(2 * C["SCAN_MIN_ENTRIES"])
    cases = []
    for forced in (-1, 0, 1):
        for one in (0, 1):
            cases += [(forced, big, 0, 1000, 1, 1000, one, 0), (forced, 10, 0, 3, 1, 5, one, 0),
                      (forced, big, 0, 1000, 5000, 5000 * 10**6, one, 1), (forced, big, 0, 0, 1, 10, one, 0),
                      (forced, big, 0, 1000, 0, 0, one, 0)]
    got = run(exe, ["decide %d %d %d %d %d %d %d %d" % c for c in cases])
    for c, g in zip(cases, got):
        forced, nk, nt, G, S, sk, one, pinned = c
        if not one or S == 0 or G == 0:
            want = 0
        elif forced >= 0:
            want = forced
        else:
            want = rule(C, nk, nt, G, S, sk, one, pinned)
        assert g == str(want), c
    assert [g for c, g in zip(cases, got) if c[0] == 1 and c[6] == 1 and c[3] and c[4]] == ["1", "1", "1"]
    assert all(g == "0" for c, g in zip(cases, got) if c[6] == 0)
