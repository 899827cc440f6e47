"""ANI near-ties: a high-precision restatement of the reference's ANI expressions and pinned integer inputs whose ANIs
sit on a -m gate or one ulp from another genome's (a test helper module, not a conftest).

The reference computes (src/contain.rs:817-847, src/inference.rs:207-242, glibc pow / exp)
  naive     RN(pow(RN(n / gl), RN(1 / k)))
  adjusted  x1 = RN(exp(-lambda)), RN(pow(RN(RN(nz / RN(1 - x1)) / nfull), RN(1 / k))), lambda = RN(RN(cp1 / cm) * (mode + 1))
The cr_* functions evaluate the same expressions with every transcendental call correctly rounded (Python decimal at
50 digits, then the nearest double, oracle/pyref.py); the glibc_* functions with Python's float arithmetic, which calls
glibc.  The device (sylph_b200/csrc/crmath.cuh) is correctly rounded.

GATES, WINNER_PAIRS and TIE_PAIRS rest on inputs where glibc is correctly rounded too (checked by
tests/test_ani_ties_cpu.py); they were picked by scripts/find_ani_ties.py on an H100 among inputs where CUDA's own
pow / exp (torch float64) and glibc disagree, so a device that rounds like CUDA's pow fails them.  The MISROUNDED pins
are the other way round: glibc is one ulp off there (found by scripts/find_glibc_misroundings.py), and the device must
print the correctly rounded ANI and the rows and winners that follow from it, not the glibc reference's.
"""
import math

from oracle.pyref import cr_exp, cr_pow  # noqa: F401  (50-digit decimal, nearest double, a midpoint refused)


def ratio_lambda(hist):
    """src/inference.rs:207-242 on {value: multiplicity} (non-zero values, median <= 2 assumed); None if it fails"""
    if len(hist) == 1 or sum(hist.values()) < 25:
        return None
    mode = max(hist, key=lambda v: (hist[v], v))
    cp1, cm = float(hist.get(mode + 1, 0)), float(hist[mode])
    if cp1 == 0 or cp1 < 3.0 or cm < 3.0:
        return None
    return cp1 / cm * float(mode + 1)


def glibc_naive(n, gl, k):
    return (n / gl) ** (1.0 / k)


def cr_naive(n, gl, k):
    return cr_pow(n / gl, 1.0 / k)


def _adjusted(hist, z, k, exp_, pow_):
    lam = ratio_lambda(hist)
    nz = sum(hist.values())
    adj = nz / (1.0 - exp_(-lam)) / (nz + z)
    return pow_(adj, 1.0 / k)


def glibc_adjusted(hist, z, k):
    return _adjusted(hist, z, k, math.exp, lambda x, c: x ** c)


def cr_adjusted(hist, z, k):
    return _adjusted(hist, z, k, cr_exp, cr_pow)


def gate_percent(a):
    """a -m percent p with RN(p / 100) == a (src/contain.rs:746-749), or None when no double p maps there"""
    p = a * 100.0
    for q in (p, math.nextafter(p, math.inf), math.nextafter(p, -math.inf)):
        if q / 100.0 == a:
            return q
    return None


# ---- genomes and samples built from the tuples ---------------------------------------------------------------------
# A genome spec is ("naive", n, gl): n hit k-mers of count 5 (median 5: lambda status HIGH, the naive ANI is final) and
# gl - n unhit ones; or ("adj", h1, h2, z): h1 hits of count 1, h2 of count 2 (h1 > h2 >= 3, h1 + h2 >= 25: median 1,
# mode 1, lambda = RN(h2 / h1) * 2) and z unhit.  Every k-mer is a fresh key over [1, 2^64 - 2] (uploaded with c = 1).

def hist_of(spec):
    return {5: spec[1]} if spec[0] == "naive" else {1: spec[1], 2: spec[2]}


def unhit_of(spec):
    return spec[2] - spec[1] if spec[0] == "naive" else spec[3]


def glibc_ani(spec, k):
    return glibc_naive(spec[1], spec[2], k) if spec[0] == "naive" else glibc_adjusted(hist_of(spec), spec[3], k)


def cr_ani(spec, k):
    return cr_naive(spec[1], spec[2], k) if spec[0] == "naive" else cr_adjusted(hist_of(spec), spec[3], k)


def calls_of(spec, k):
    """the pow / exp calls (crmath_check eval form) the reference makes for spec's ANI"""
    if spec[0] == "naive":
        return [("pow", spec[1] / spec[2], 1.0 / k)]
    lam = ratio_lambda(hist_of(spec))
    nz = spec[1] + spec[2]
    return [("exp", -lam), ("pow", nz / (1.0 - cr_exp(-lam)) / (nz + spec[3]), 1.0 / k)]


class Case:
    """Genomes from specs; the first `shared` hit k-mers of the lowest count are common to every genome (a winner
    decision in profile's pass 2).  db: the CSR arrays (one unhit tracked k-mer per genome); sample: (hash, count)."""

    def __init__(self, specs, shared=0, seed=1):
        import numpy as np
        rng = np.random.default_rng(seed)
        n_keys = sum(sum(hist_of(s).values()) + unhit_of(s) + 1 for s in specs) + 64
        keys = iter(np.unique(rng.integers(1, 2**64 - 1, size=n_keys + 256, dtype=np.uint64))[rng.permutation(n_keys)].tolist())
        low = {min(hist_of(s)) for s in specs}
        assert not shared or len(low) == 1
        common = [next(keys) for _ in range(shared)]
        self.sample = {k: min(low) for k in common}
        kmers, offs, tracked = [], [0], []
        for s in specs:
            own = list(common)
            for v, m in sorted(hist_of(s).items()):
                for _ in range(m - (shared if v == min(low) else 0)):
                    x = next(keys)
                    self.sample[x] = v
                    own.append(x)
            own += [next(keys) for _ in range(unhit_of(s))]
            kmers += own
            offs.append(len(kmers))
            tracked.append(next(keys))
        self.db = dict(kmers=np.array(kmers, np.uint64), kmer_off=np.array(offs, np.uint64), tracked=np.array(tracked, np.uint64),
                       tracked_off=np.arange(len(specs) + 1, dtype=np.uint64),
                       gn_size=np.array([1_000_000 + 1000 * i for i in range(len(specs))], np.uint64))
        p = rng.permutation(len(self.sample))
        self.hash = np.array(list(self.sample), np.uint64)[p]
        self.count = np.array(list(self.sample.values()), np.uint32)[p]


# ---- pins ----------------------------------------------------------------------------------------------------------
# (k, spec, a, p, p_up, p_down): the genome's ANI a and -m percents with RN(p / 100) == a, RN(p_up / 100) == the next
# double up, RN(p_down / 100) == the next double down
GATES = [
    (21, ('naive', 47, 60), float.fromhex('0x1.fa14aa99820fbp-1'), float.fromhex('0x1.8b602547ed9c4p+6'), float.fromhex('0x1.8b602547ed9c5p+6'), float.fromhex('0x1.8b602547ed9c3p+6')),  # CUDA's pow / exp: 0x1.fa14aa99820fcp-1
    (21, ('naive', 23, 78), float.fromhex('0x1.e313276612edcp-1'), float.fromhex('0x1.7966f6c7bec9cp+6'), float.fromhex('0x1.7966f6c7bec9dp+6'), float.fromhex('0x1.7966f6c7bec9bp+6')),  # CUDA's pow / exp: 0x1.e313276612edbp-1
    (31, ('naive', 8, 63), float.fromhex('0x1.df0688969dfc9p-1'), float.fromhex('0x1.763d1ab5ab6d5p+6'), float.fromhex('0x1.763d1ab5ab6d6p+6'), float.fromhex('0x1.763d1ab5ab6d4p+6')),  # CUDA's pow / exp: 0x1.df0688969dfcap-1
    (31, ('naive', 2, 88), float.fromhex('0x1.c529f8f559689p-1'), float.fromhex('0x1.6208ca7fadd9bp+6'), float.fromhex('0x1.6208ca7fadd9cp+6'), float.fromhex('0x1.6208ca7fadd9ap+6')),  # CUDA's pow / exp: 0x1.c529f8f559688p-1
    (21, ('adj', 32, 29, 15), float.fromhex('0x1.fefc64682f153p-1'), float.fromhex('0x1.8f352e7164c89p+6'), float.fromhex('0x1.8f352e7164c8ap+6'), float.fromhex('0x1.8f352e7164c88p+6')),  # CUDA's pow / exp: 0x1.fefc64682f152p-1
    (21, ('adj', 20, 18, 19), float.fromhex('0x1.fa8c7d81b7793p-1'), float.fromhex('0x1.8bbdc20d5756bp+6'), float.fromhex('0x1.8bbdc20d5756cp+6'), float.fromhex('0x1.8bbdc20d5756ap+6')),  # CUDA's pow / exp: 0x1.fa8c7d81b7794p-1
    (31, ('adj', 15, 13, 32), float.fromhex('0x1.f6b57c415a3c0p-1'), float.fromhex('0x1.88bdc9130e7eep+6'), float.fromhex('0x1.88bdc9130e7efp+6'), float.fromhex('0x1.88bdc9130e7edp+6')),  # CUDA's pow / exp: 0x1.f6b57c415a3c1p-1
    (31, ('adj', 24, 21, 50), float.fromhex('0x1.f6e4c19b01445p-1'), float.fromhex('0x1.88e2b74118fd6p+6'), float.fromhex('0x1.88e2b74118fd7p+6'), float.fromhex('0x1.88e2b74118fd5p+6')),  # CUDA's pow / exp: 0x1.f6e4c19b01444p-1
    (31, ('adj', 36, 21, 0), float.fromhex('0x1.03198597c4c16p+0'), float.fromhex('0x1.94d7e0bd236e2p+6'), float.fromhex('0x1.94d7e0bd236e4p+6'), float.fromhex('0x1.94d7e0bd236e1p+6')),  # CUDA's pow / exp: 0x1.03198597c4c17p+0
]

# (k, spec A, spec B): glibc ANI(B) is the double just above glibc ANI(A)
WINNER_PAIRS = [
    (21, ("adj", 45, 9, 597), ("adj", 30, 6, 398)),        # CUDA: ANI(A) one ulp above ANI(B), the order reversed
    (21, ("adj", 216, 105, 411), ("adj", 288, 140, 548)),  # CUDA: reversed
    (31, ("adj", 645, 432, 531), ("adj", 215, 144, 177)),  # CUDA agrees with glibc
]

# (k, spec A, spec B): equal ANIs reached from different fractions (lambda 1 from 10/20 and 20/40, n / gl = 1/2)
TIE_PAIRS = [
    (31, ("adj", 20, 10, 40), ("adj", 40, 20, 80)),
    (21, ("naive", 50, 100), ("naive", 75, 150)),
]


# ---- pins where glibc misrounds (scripts/find_glibc_misroundings.py) ------------------------------------------------
# (k, spec, glibc's ANI, the correctly rounded ANI): one ulp apart either way, from the naive ANI's pow and from the
# adjusted ANI's exp / pow
MISROUNDED = [
    (21, ("naive", 78, 79), float.fromhex("0x1.ffb0835fb1302p-1"), float.fromhex("0x1.ffb0835fb1303p-1")),
    (21, ("naive", 71, 358), float.fromhex("0x1.da094e0e32ae4p-1"), float.fromhex("0x1.da094e0e32ae3p-1")),
    (21, ("adj", 17, 10, 169), float.fromhex("0x1.da21ff355a7d8p-1"), float.fromhex("0x1.da21ff355a7d7p-1")),
    (21, ("adj", 17, 15, 39), float.fromhex("0x1.f15cc12c4dbeep-1"), float.fromhex("0x1.f15cc12c4dbefp-1")),
    (31, ("naive", 120, 151), float.fromhex("0x1.fc3804b0174d2p-1"), float.fromhex("0x1.fc3804b0174d3p-1")),
    (31, ("naive", 246, 271), float.fromhex("0x1.fe6768b75ae50p-1"), float.fromhex("0x1.fe6768b75ae4fp-1")),
    (31, ("adj", 14, 13, 91), float.fromhex("0x1.eae46448b4ba6p-1"), float.fromhex("0x1.eae46448b4ba5p-1")),
    (31, ("adj", 19, 10, 91), float.fromhex("0x1.efe481cefeebap-1"), float.fromhex("0x1.efe481cefeebbp-1")),
]

# (k, spec, p): glibc's ANI is the double below the correctly rounded ANI a, and RN(p / 100) == a.  At -m p correct
# rounding keeps the row (a >= a) and the glibc reference drops it
MISROUNDED_GATES = [
    (21, ("naive", 78, 79), float.fromhex("0x1.8fc1e6a2c26dap+6")),
    (21, ("adj", 17, 15, 39), float.fromhex("0x1.849076ea9cbd3p+6")),
    (31, ("naive", 120, 151), float.fromhex("0x1.8d0bc3a992345p+6")),
    (31, ("adj", 19, 10, 91), float.fromhex("0x1.836a8569b7282p+6")),
]

# (k, spec A, spec B, winner under glibc, winner correctly rounded): genome 0 = A, genome 1 = B, B = A's counts scaled
# (the same rational ANI input rounded along another path), so the two ANIs are equal or adjacent doubles and one glibc
# misrounding reverses the pass-2 winner of the k-mers they share
MISROUNDED_WINNERS = [
    (21, ("adj", 65, 60, 1540), ("adj", 13, 12, 308), 0, 1),   # glibc: equal ANIs, A first; correct: B one ulp above
    (31, ("adj", 39, 36, 798), ("adj", 13, 12, 266), 1, 0),    # glibc: B one ulp above; correct: equal ANIs
]


def pinned_specs(misrounded=True):
    """(k, spec) of every pin; misrounded=False: only those glibc rounds correctly"""
    for k, spec, *_ in GATES + (MISROUNDED if misrounded else []):
        yield k, spec
    for k, a, b, *_ in WINNER_PAIRS + TIE_PAIRS + (MISROUNDED_WINNERS if misrounded else []):
        yield k, a
        yield k, b


def pinned_calls():
    return [c for k, spec in pinned_specs() for c in calls_of(spec, k)]
