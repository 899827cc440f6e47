"""Scripted count multisets turned into uploaded genome sketches and samples (a test helper module, not a conftest).

get_stats (src/contain.rs:601-814) is a function of one (sample, genome) pair's hit counts: their median, the Poisson
cut-off, the kept values' sum and histogram, ratio_lambda (src/inference.rs:207-242) and the bootstrap over them.  The
device reformulates each of these (sylph_b200/csrc/contain.cu: k_stats_hist / k_stats, ratio_lambda_hist, boot_one,
k_boot_final, k_boot_seq), and Poisson-like inputs almost never sit on their boundaries.  Here a script is one genome:
the multiset of sample counts of its hit k-mers and a number of unhit k-mers, each k-mer a fresh key drawn over
[1, 2^64 - 2] (uploaded with c = 1, so every such key is a legal hash; u64::MAX is the oracle's empty-slot marker).
Only the probe and winner families share keys between genomes, and only within their own sample.

Families (the scripts below), each a sample of its own:

  median  medians 1, 2, 3, 14, 15, 29, 30 with odd and even numbers of hits (the median is the hit of rank n/2)
  cut     every median 1..29 with the values cut[m] and cut[m] + 1 present and a far outlier, few hits
  ratio   every way ratio_lambda returns None, at its boundary; the mode tie (the larger value wins)
  boot    lambda rows whose mode lies in 1-3, 4-7 and 8-14, whose largest kept value is 3, 7, 8, 11 or 15, without
          zeros, with an empty class, and |genome_kmers| of 50, 255, 256, 257, 1023 and 1025
  huge    one lambda row of 2^20 + 1 genome k-mers
  suc     lambda rows whose bootstrap succeeds exactly 50 times, and 49 and 45 times (a seeded search, pinned)
  filter  |genome_kmers| of 49 / 50 against min_number_kmers = 50; ANI exactly 1 against minimum_ani = 100
  big     counts >= 256 in every byte position, wrapping sums (the CSR formulation)
  probe   keys 0, 1, 2^63 +- 1, 2^64 - 2 (the db's largest key); equal ranges of 1..9 and 33 genomes with kept and
          tracked entries mixed; 1000 consecutive keys in one directory bucket; repeated k-mers
  winner  tracked-only winners, with and without the tracked genome surviving pass 1; three-way ANI ties; derep at
          floor(t * glen) and one more reassigned k-mer, t = 0.99^31 and 0.95^31

Two boundaries of get_stats cannot be reached by any input: a mode of 11 at median 1 (a median of 1 needs more
than half of the hits at 1, so no other value can tie it), and ratio_lambda's `count < min_count_correct` on its own
(the mode's count is at least count_p1's, so count_p1's test fails first).  The ratio family therefore holds mode 11
and mode 15 at median 2, once with mode + 1 kept and once with mode + 1 only above the cut.
"""
import functools
import math
from collections import Counter

import numpy as np

from oracle import pyref as R

K = 31
MAX_KEY = 2**64 - 2       # largest legal key: u64::MAX is the oracle's empty-slot marker
COV_BINS = 256            # contain.hpp: a count >= 256 sends the call through the CSR formulation
BOOT_PYREF_MAX = 5000     # pyref bootstraps rows up to this many genome k-mers (100 * n Python draws)
REPLAY_MAX = 20000        # SYL_BOOT_REPLAY: one thread replays 100 * n draws per row
LOW, HIGH, LAMBDA = 0, 1, 2


def _cut(m):
    """src/contain.rs:664-675: largest v with PoissonCDF(v; m) < 0.9999999999 (statrs cdf, restated by pyref)."""
    v = m
    while R.poisson_cdf(float(m), v + 1) < 0.9999999999:
        v += 1
    return v


CUT = [0] + [_cut(m) for m in range(1, 30)]


class Script:
    """One genome: its k-mers (kept, tracked) and the sample counts of the keys it brings into its sample."""

    def __init__(self, tag, kmers, tracked=(), counts=None, gn_size=1_000_000):
        self.tag, self.kmers, self.tracked = tag, [int(x) for x in kmers], [int(x) for x in tracked]
        self.counts = dict(counts or {})
        self.gn_size = gn_size


class Keys:
    """Fresh keys over [1, 2^64 - 2], never handed out twice (explicit keys are reserved first)."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.used = set()

    def reserve(self, keys):
        keys = [int(x) for x in keys]
        assert not self.used.intersection(keys)
        self.used.update(keys)
        return keys

    def fresh(self, n):
        out = []
        while len(out) < n:
            for x in self.rng.integers(1, MAX_KEY + 1, size=n - len(out) + 16, dtype=np.uint64).tolist():
                if x not in self.used and len(out) < n:
                    self.used.add(x)
                    out.append(x)
        return out


def plain(keys, tag, hist, n_unhit, gn_size=1_000_000):
    """A genome whose hit counts are the multiset `hist` ({value: multiplicity}) plus n_unhit unhit k-mers."""
    counts = [v for v, m in sorted(hist.items()) for _ in range(m)]
    ks = keys.fresh(len(counts) + n_unhit)
    return Script(tag, ks, counts=dict(zip(ks, counts)), gn_size=gn_size)


# ---- families ------------------------------------------------------------------------------------------------------

def fam_median(keys):
    out = []
    for m in (1, 2, 3, 14, 15, 29, 30):
        for n in (30, 31):
            h = n // 2
            lo, up = max(m - 1, 1), (2 if m == 1 else m + 1 if m <= 2 else m + 4)
            counts = [lo] * h + [m] * (h // 2 + 1)
            counts += [up] * (n - 1 - len(counts)) + [200]     # 200: above every cut-off, kept at median 30
            out.append(plain(keys, "m%d_n%d" % (m, n), Counter(counts), 26))
    return out


def fam_cut(keys):
    return [plain(keys, "cut_m%d" % m, Counter([m] * 7 + [CUT[m], CUT[m] + 1, 200, 200]), 39) for m in range(1, 30)]


def fam_ratio(keys):
    S = [("distinct_1", {1: 30}, 30), ("distinct_2", {2: 30}, 30),
         ("nz24", {1: 14, 2: 10}, 26), ("nz25", {1: 14, 2: 11}, 25),
         ("p1_absent", {1: 20, 3: 10}, 30),
         ("mode15_m2", {1: 9, 2: 9, 15: 9, 14: 4}, 30),
         ("mode15_p1_above_cut", {1: 9, 2: 9, 15: 9, 16: 5}, 30),
         ("mode11_m2", {1: 9, 2: 9, 11: 9, 12: 4}, 30),
         ("cp1_2", {1: 20, 2: 2, 3: 5}, 30), ("cp1_3", {1: 20, 2: 3, 3: 5}, 30),
         ("cp1_1", {1: 20, 2: 1, 3: 5}, 30), ("cp1_0", {1: 20, 3: 5, 4: 2}, 30),
         ("tie_1_2", {1: 12, 2: 12, 3: 5}, 30), ("tie_1_2_11", {1: 10, 2: 10, 11: 10, 12: 3}, 30)]
    return [plain(keys, t, h, u) for t, h, u in S]


def _scaled(g):
    """A lambda row of g genome k-mers (median 1, mode 1, values up to 6, the rest unhit)."""
    h = {1: round(0.3 * g), 2: round(0.15 * g), 3: round(0.05 * g), 6: max(1, g // 100)}
    if g <= 60:
        h = {1: 15, 2: 8, 3: 3}
    return h, g - sum(h.values())


def fam_boot(keys):
    S = [("mode1_max3", {1: 30, 2: 20, 3: 10}, 40),
         ("mode2_max4", {1: 20, 2: 25, 3: 12, 4: 5}, 40),
         ("mode3_max4", {1: 20, 2: 20, 3: 25, 4: 10}, 40),
         ("mode4_max5", {1: 20, 2: 20, 4: 22, 5: 8}, 40),
         ("mode5_max7", {1: 21, 2: 21, 5: 25, 6: 10, 7: 6}, 40),
         ("mode6_max7", {1: 21, 2: 21, 3: 4, 6: 25, 7: 12}, 40),
         ("mode7_max8", {1: 21, 2: 21, 7: 25, 8: 10}, 40),
         ("mode8_max9", {1: 21, 2: 21, 8: 25, 9: 10}, 40),
         ("mode11_max12", {1: 21, 2: 21, 11: 25, 12: 10}, 40),
         ("mode14_max15", {1: 21, 2: 21, 14: 25, 15: 10}, 40),
         ("mode1_max11", {1: 30, 2: 20, 3: 5, 11: 2}, 40),
         ("mode2_max15", {1: 20, 2: 25, 3: 10, 15: 2}, 40),
         ("no_zero", {1: 40, 2: 30, 3: 10}, 0),
         ("no_zero_max7", {1: 21, 2: 21, 5: 25, 6: 10, 7: 6}, 0),
         ("gap_0125", {1: 30, 2: 20, 5: 5}, 40)]
    out = [plain(keys, t, h, u) for t, h, u in S]
    for g in (50, 255, 256, 257, 1023, 1025):
        h, u = _scaled(g)
        out.append(plain(keys, "glen%d" % g, h, u))
    return out


def fam_huge(keys):
    return [plain(keys, "glen%d" % (2**20 + 1), {1: 300000, 2: 150000, 3: 50000, 7: 1000}, 2**20 + 1 - 501000)]


# bootstrap success counts 50 (k_boot_final keeps the CI) and 49 / 45 (it drops it): found once by a seeded search over
# rows of 25-28 non-zero values with pyref's WyRand + ratio_lambda (boot_successes below), pinned here
SUC_ROWS = [
    ("suc50_a", {1: 19, 2: 5, 3: 1}, 32, 50),
    ("suc50_b", {1: 17, 2: 6, 4: 2}, 29, 50),
    ("suc49", {1: 15, 2: 7, 3: 1, 4: 2}, 27, 49),
    ("suc45", {1: 15, 2: 8, 4: 2}, 30, 45),
]


def fam_suc(keys):
    return [plain(keys, t, h, u) for t, h, u, _ in SUC_ROWS]


def fam_filter(keys):
    return [plain(keys, "glen49", {5: 49}, 0), plain(keys, "glen50", {5: 50}, 0),
            plain(keys, "ani_exactly_1", {5: 40, 6: 20}, 0), plain(keys, "miss_one", {5: 40, 6: 19}, 1)]


def fam_big(keys):
    B24, B31, TOP = 2**24 + 1, 2**31, 2**32 - 1
    S = [("every_byte", {256: 1, 65536: 1, B24: 1, B31: 1, TOP: 1, 40: 45}, 5),          # median 40, sum wraps
         ("median_2p24", {5: 10, B24: 30, TOP: 5}, 10),                                    # sum wraps
         ("median_2p31", {1: 10, 3: 10, B31: 20}, 10),
         ("median_top", {7: 5, TOP: 30}, 15),
         ("low_bytes_a", {5: 10, 0x01000005: 10, 0x02000005: 11}, 19),                  # median 0x01000005
         ("low_bytes_b", {5: 5, 0x00010005: 12, 0x01010005: 10}, 23),                   # median 0x00010005
         ("low_bytes_c", {0x05: 3, 0x0105: 10, 0x010105: 14}, 23),                       # median 0x010105
         ("c255_median", {3: 10, 255: 20, 256: 20}, 0),
         ("c256_median", {255: 10, 256: 30, 3: 5}, 5),
         ("median29_big_outlier", {29: 30, 65536: 5, TOP: 1}, 14),                        # cut removes both
         ("median2_big_outlier", {1: 20, 2: 20, 3: 5, TOP: 1}, 14)]                       # lambda row, CSR
    return [plain(keys, t, h, u) for t, h, u in S]


def fam_probe(keys):
    out = []
    edge = keys.reserve([0, 1, 2**63 - 1, 2**63, 2**63 + 1])
    own = keys.fresh(55)
    out.append(Script("edge_keys", edge + own, counts=dict(zip(edge + own[:40], [3] * 5 + [3, 4] * 20))))
    top = keys.reserve([MAX_KEY - 1, MAX_KEY])
    own = keys.fresh(50)
    out.append(Script("top_keys", top + own, counts=dict(zip(top + own[:30], [7, 7] + [6] * 30))))
    # k-mers shared by r genomes: genome j holds them kept when j % 3 != 1, tracked otherwise
    sizes = list(range(1, 10)) + [33]
    shared = {r: keys.fresh(3) for r in sizes}
    for j in range(33):
        own = keys.fresh(50)
        n_hit = 30 + (j * 7) % 20
        counts = dict(zip(own[:n_hit], [3 + (i + j) % 3 for i in range(n_hit)]))
        kept, tracked = list(own), []
        for r in sizes:
            if j < r:
                (tracked if j % 3 == 1 else kept).extend(shared[r])
                counts.update({x: 4 for x in shared[r]})
        out.append(Script("shared_g%d" % j, kept, tracked, counts))
    base = int(keys.rng.integers(2**40, 2**62))
    run = keys.reserve(range(base, base + 1000))
    out.append(Script("consecutive_1000", run, counts={x: 2 + i % 4 for i, x in enumerate(run[::3])}))
    own = keys.fresh(60)
    out.append(Script("repeated_kmer", own + [own[0], own[1], own[1]], counts={x: 5 for x in own[:40]}))
    own = keys.fresh(60)
    out.append(Script("kept_and_own_tracked", own, own[:5] + keys.fresh(5), counts={x: 6 for x in own[:45]}))
    return out


def fam_winner(keys):
    out = []
    x = keys.fresh(5)
    a = keys.fresh(50)
    out.append(Script("tracked_winner_A", a, x, counts={k: 5 for k in a}))             # ANI 1, wins x
    b = keys.fresh(60)
    out.append(Script("tracked_loser_B", b + x, counts={k: 5 for k in b[:55] + x}))
    x = keys.fresh(5)
    a = keys.fresh(60)
    out.append(Script("tracked_filtered_A", a, x, counts={k: 5 for k in a[:2]}))       # ANI 0.896: not a survivor
    b = keys.fresh(60)
    out.append(Script("tracked_keeper_B", b + x, counts={k: 5 for k in b[:55] + x}))
    sh = keys.fresh(10)
    for i in range(3):                                                                 # identical statistics
        own = keys.fresh(60)
        out.append(Script("tie3_%d" % i, own + sh, counts={**{k: 4 for k in own[:50]}, **{k: 4 for k in sh}}))
    for ra in (99.0, 95.0):
        d = math.floor((ra / 100.0) ** K * 100)
        for lost in (d, d + 1):
            s = keys.fresh(lost)
            a = keys.fresh(100 - lost)
            b = keys.fresh(100 - lost)
            out.append(Script("derep%d_A_%d" % (ra, lost), s + a, counts={k: 5 for k in s + a}))
            out.append(Script("derep%d_B_%d" % (ra, lost), s + b, counts={k: 5 for k in s + b}))
    return out


FAMILIES = {"median": fam_median, "cut": fam_cut, "ratio": fam_ratio, "boot": fam_boot, "huge": fam_huge,
            "suc": fam_suc, "filter": fam_filter, "big": fam_big, "probe": fam_probe, "winner": fam_winner}
SAMPLES = list(FAMILIES)
CSR_SAMPLES = ("big",)
REPLAY_SAMPLES = ("boot", "suc")

# parameter sets every sample runs with (contain_params / O.default_params keywords), and the extra ones per family
COMMON_PARAMS = [{}, {"minimum_ani": 0.0}]
EXTRA_PARAMS = {
    "median": [{"no_ci": 1, "minimum_ani": 0.0}, {"no_adj": 1, "minimum_ani": 0.0}, {"mean_coverage": 1},
               {"mean_coverage": 1, "minimum_ani": 0.0}],
    "ratio": [{"min_count_correct": 1.0, "minimum_ani": 0.0}],
    "filter": [{"minimum_ani": 100.0}],
    "winner": [{"redundant_ani": 95.0}],
}


def params_for(name):
    return COMMON_PARAMS + EXTRA_PARAMS.get(name, [])


class World:
    """All samples over one database: genomes in SAMPLES order; owner[g] = the sample genome g belongs to."""

    def __init__(self, seed=0x5C41):
        keys = Keys(seed)
        self.scripts, self.samples, self.owner, self.local = [], {}, [], {}
        for name in SAMPLES:
            sc = FAMILIES[name](keys)
            first = len(self.scripts)
            self.local[name] = list(range(first, first + len(sc)))
            self.scripts += sc
            self.owner += [name] * len(sc)
            cnt = {}
            for s in sc:
                for k, c in s.counts.items():
                    assert cnt.get(k, c) == c
                    cnt[k] = c
            self.samples[name] = cnt

    def db(self, sel=None):
        """CSR arrays of the genomes `sel` (all by default), in that order."""
        sel = range(len(self.scripts)) if sel is None else sel
        sc = [self.scripts[i] for i in sel]
        return dict(kmers=np.array([k for s in sc for k in s.kmers], dtype=np.uint64),
                    kmer_off=np.cumsum([0] + [len(s.kmers) for s in sc]).astype(np.uint64),
                    tracked=np.array([k for s in sc for k in s.tracked], dtype=np.uint64),
                    tracked_off=np.cumsum([0] + [len(s.tracked) for s in sc]).astype(np.uint64),
                    gn_size=np.array([s.gn_size + 1000 * i for i, s in enumerate(sc)], dtype=np.uint64))

    def sample_arrays(self, name):
        """(hash, count) in a seeded shuffled order: uploads sort them"""
        d = self.samples[name]
        h = np.array(list(d.keys()), dtype=np.uint64)
        c = np.array(list(d.values()), dtype=np.uint32)
        p = np.random.default_rng(len(h)).permutation(len(h))
        return h[p], c[p]

    def hits(self, name, g):
        """sample counts of genome g's hit k-mers (src/contain.rs:632-652, pass 1)"""
        smp = self.samples[name]
        return [smp[k] for k in self.scripts[g].kmers if smp.get(k, 0)]


@functools.lru_cache(maxsize=None)
def world():
    return World()


# ---- the classifier: what get_stats does with one pair, read off the count multiset ------------------------------

def ratio_reason(kept, mcc):
    """ratio_lambda on the kept non-zero values -> (lambda or None, reason, mode)"""
    cm = Counter(kept)
    if len(cm) == 1:
        return None, "distinct", None
    if len(kept) < 25:
        return None, "nz", None
    mode = max(cm, key=lambda v: (cm[v], v))
    if mode + 1 not in cm:
        return None, "p1_absent", mode
    if cm[mode + 1] < mcc:
        return None, "count_p1", mode
    if cm[mode] < mcc:
        return None, "count", mode
    return cm[mode + 1] / cm[mode] * (mode + 1), "ok", mode


def boot_successes(full, mcc=3.0, k=K):
    """bootstrap_interval (src/contain.rs:849-898) with pyref's WyRand: the number of successful iterations."""
    rng = R.WyRand(7)
    n, suc = len(full), 0
    for _ in range(100):
        rv = [full[rng.usize(n)] for _ in range(n)]
        lam = R.ratio_lambda(rv, mcc)
        suc += lam is not None and R.ani_from_lambda(lam, k, rv) is not None
    return suc


def classify_pair(hits, glen, P, with_boot=True):
    """hits: the pair's hit counts; P: O.default_params-like keywords.  -> dict, or None when there is no hit."""
    if not hits:
        return None
    mcc = P.get("min_count_correct", 3.0)
    cov = sorted(hits)
    n = len(cov)
    median = cov[n // 2]
    cut = CUT[median] if median < 30 else None
    kept = [v for v in cov if cut is None or v <= cut]
    full = [0] * (glen - n) + kept
    r = dict(median=median, n=n, glen=glen, csr=max(cov) >= COV_BINS, cut_removes=len(kept) < n,
             sum=sum(kept) % 2**32, sum_wraps=sum(kept) >= 2**32, nz=len(kept), status=HIGH, reason=None, mode=None, max_kept=max(kept),
             lam=None, boot=None)
    if median <= 2:
        lam, r["reason"], r["mode"] = ratio_reason(kept, mcc)
        r["status"], r["lam"] = (LAMBDA, lam) if lam is not None else (LOW, None)
    if r["status"] == LAMBDA:
        r["final"] = "lambda"
    elif median < 15:
        r["final"] = "mean"
    else:
        r["final"] = "mean_param" if P.get("mean_coverage") else "median"
    naive = (n / glen) ** (1.0 / K)
    ani = naive
    if r["status"] == LAMBDA and not P.get("no_adj"):
        est = R.ani_from_lambda(r["lam"], K, full)
        ani = naive if est is None else est
    ma = P.get("minimum_ani", -1.0)
    min_ani = ma / 100.0 if ma >= 0 else 0.90
    r["emitted"] = glen >= P.get("min_number_kmers", 50.0) and ani >= min_ani
    if r["status"] == LAMBDA:
        r["mode_class"] = "1-3" if r["mode"] <= 3 else "4-7" if r["mode"] <= 7 else "8-14"
        if with_boot and glen <= BOOT_PYREF_MAX:
            r["boot"] = boot_successes(full, mcc)
    return r


def classify(name, P=None, with_boot=True):
    """(genome, classification) of every genome of sample `name` (query, pass 1)."""
    w = world()
    P = P or {}
    return [(g, classify_pair(w.hits(name, g), len(w.scripts[g].kmers), P, with_boot)) for g in w.local[name]]


def tally(name, P=None, with_boot=True):
    t = Counter()
    for _, r in classify(name, P, with_boot):
        if r is None:
            continue
        t["status_%d" % r["status"]] += 1
        if r["reason"] and r["reason"] != "ok":
            t["low_" + r["reason"]] += 1
        t["final_" + r["final"]] += 1
        t["cut_removes"] += r["cut_removes"]
        t["emitted" if r["emitted"] else "filtered"] += 1
        t["csr"] += r["csr"]
        t["median_%d" % r["median"]] += 1
        t["n_%s" % ("even" if r["n"] % 2 == 0 else "odd")] += 1
        if r["status"] == LAMBDA:
            t["mode_" + r["mode_class"]] += 1
            t["max_kept_%d" % r["max_kept"]] += 1
            t["no_zero"] += r["glen"] == r["n"]
            if r["boot"] is not None:
                t["boot_%d" % r["boot"]] += 1
        t["sum_wraps"] += r["sum_wraps"]
    return t
