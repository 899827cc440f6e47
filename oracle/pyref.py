"""Independent pure-Python restatement of the reference's hot-path arithmetic (small inputs only).

TEST INFRASTRUCTURE ONLY.  Written from SURVEY.md §8 / the reference sources without looking at
oracle/sylph_oracle.c, so that the C oracle is cross-checked by a second implementation
(tests/test_oracle_cpu.py).  Every function cites the reference file:line it follows.
"""
import decimal
import math
from decimal import Decimal

MASK64 = (1 << 64) - 1

# src/types.rs:50-59
BYTE_TO_SEQ = [0] * 256
for _ch, _v in ((b"A", 0), (b"C", 1), (b"G", 2), (b"T", 3), (b"U", 3)):
    BYTE_TO_SEQ[_ch[0]] = _v
    BYTE_TO_SEQ[_ch.lower()[0]] = _v
BYTE_TO_SEQ[1], BYTE_TO_SEQ[2], BYTE_TO_SEQ[3] = 1, 2, 3


def mm_hash64(key):
    """src/seeding.rs:4-15 (line 7: NOT of the sum)."""
    key = (~(key + (key << 21))) & MASK64
    key ^= key >> 24
    key = (key + (key << 3) + (key << 8)) & MASK64
    key ^= key >> 14
    key = (key + (key << 2) + (key << 4)) & MASK64
    key ^= key >> 28
    key = (key + (key << 31)) & MASK64
    return key


def _windows(s, k):
    """yield (end_index, canonical kmer) for every window (src/seeding.rs:110-136)."""
    mask = (1 << (2 * k)) - 1
    for i in range(k - 1, len(s)):
        f = 0
        r = 0
        for j in range(k):
            c = BYTE_TO_SEQ[s[i - k + 1 + j]]
            f = (f << 2) | c
            r |= (3 - c) << (2 * j)
        f &= mask
        yield i, (f if f < r else r)


def seeds_scalar(s, k, c):
    """fmh_seeds_positions (src/seeding.rs:148-209) -> [(pos, hash)]"""
    if len(s) < k:
        return []
    thr = MASK64 // c
    return [(i, mm_hash64(km)) for i, km in _windows(s, k) if mm_hash64(km) < thr]


def seeds_avx2(s, k, c, with_pos):
    """extract_markers_avx2{,_positions} window set (src/avx2_seeding.rs:33-44, 152-162, 95, 213)."""
    L = len(s)
    if L < k:
        return []
    if L < (2 * k if with_pos else k + 1):
        return []
    assert k in (21, 31)
    lenq = (L - k + 1) // 4
    keep_end = 4 * lenq + k - 1  # windows with start < 4*lenq, i.e. end index < 4*lenq + k - 1
    return [(i, h) for i, h in seeds_scalar(s, k, c) if i < keep_end]


def sketch_genome(contigs, k, c, min_spacing, pseudotax, sem_avx2=True):
    """src/sketch.rs:550-622 -> (genome_kmers, tracked, gn_size)"""
    vec = []
    size = 0
    for ci, s in enumerate(contigs):
        size += len(s)
        sv = seeds_avx2(s, k, c, True) if sem_avx2 else seeds_scalar(s, k, c)
        vec += [(ci, p, h) for p, h in sv]
    vec.sort()
    seen, dup = set(), set()
    for _, _, h in vec:
        if h in seen:
            dup.add(h)
        seen.add(h)
    out, tracked = [], []
    last_pos, last_contig = 0, 0
    for ci, p, h in vec:
        if h in dup:
            continue
        if last_pos == 0 or last_contig != ci or p - last_pos > min_spacing:
            out.append(h)
            last_contig, last_pos = ci, p
        elif pseudotax:
            tracked.append(h)
    return out, tracked, size


def pair_kmer_single(s):
    """src/sketch.rs:624-656"""
    kk = 16
    if len(s) < 4 * kk + 2:
        return None
    half = len(s) // 2
    f = g = r = t = 0
    for i in range(kk):
        f = (f << 2) | BYTE_TO_SEQ[s[2 * i]]
        r = (r << 2) | BYTE_TO_SEQ[s[2 * i + half]]
        g = (g << 2) | BYTE_TO_SEQ[s[1 + 2 * i]]
        t = (t << 2) | BYTE_TO_SEQ[s[1 + 2 * i + half]]
    return (f, r), (g, t)


def sketch_reads(reads, k, c, no_dedup=False, sem_avx2=True):
    """src/sketch.rs:897-959 + :690-731 -> (dict hash->count, mean_read_length, num_dup_removed)"""
    counts, pairs = {}, set()
    mean = 0.0
    n = 0.0
    ndup = 0
    for s in reads:
        pair = None if len(s) > 400 else pair_kmer_single(s)
        sv = seeds_avx2(s, k, c, False) if sem_avx2 else seeds_scalar(s, k, c)
        for _, km in sv:
            cur = counts.setdefault(km, 0)
            if not no_dedup and cur < 4 and pair is not None:
                ret = False
                for pk in pair:
                    if (km, pk) in pairs:
                        if cur > 0:
                            ret = True
                    else:
                        pairs.add((km, pk))
                if ret:
                    ndup += 1
                    continue
            counts[km] = cur + 1
        n += 1.0
        mean = mean + (len(s) - mean) / n
    return counts, mean, ndup


def pair_kmer(s1, s2):
    """src/sketch.rs:658-688: 16 bases at even / odd offsets from the start of each mate; None if a mate < 33 bp"""
    if len(s1) < 33 or len(s2) < 33:
        return None
    f = g = r = t = 0
    for i in range(16):
        f = (f << 2) | BYTE_TO_SEQ[s1[2 * i]]
        r = (r << 2) | BYTE_TO_SEQ[s2[2 * i]]
        g = (g << 2) | BYTE_TO_SEQ[s1[2 * i + 1]]
        t = (t << 2) | BYTE_TO_SEQ[s2[2 * i + 1]]
    return ((f, r), (g, t))


def sketch_read_pairs(reads1, reads2, k, c, no_dedup=False, sem_avx2=True):
    """src/sketch.rs:771-895 with dedup_fpr == 0: the exact (k-mer, pair key) set, no count threshold
    -> (dict hash->count, mean_read_length, num_dup_removed)"""
    counts, pairs = {}, set()
    mean, n, ndup = 0.0, 0.0, 0

    def dedup(km, pair):
        nonlocal ndup
        cur = counts.setdefault(km, 0)
        if not no_dedup and pair is not None:      # threshold None: *c < u32::MAX always holds
            ret = False
            for pk in pair:
                if (km, pk) in pairs:
                    if cur > 0:
                        ret = True
                else:
                    pairs.add((km, pk))
            if ret:
                ndup += 1
                return
        counts[km] = cur + 1

    for s1, s2 in zip(reads1, reads2):
        v1 = [h for _, h in (seeds_avx2(s1, k, c, False) if sem_avx2 else seeds_scalar(s1, k, c))]
        v2 = [h for _, h in (seeds_avx2(s2, k, c, False) if sem_avx2 else seeds_scalar(s2, k, c))]
        pair = pair_kmer(s1, s2)
        n += 1.0
        mean = mean + (len(s1) - mean) / n
        for km in v1:
            dedup(km, pair)
        for km in v2:
            if km in v1:
                continue
            dedup(km, pair)
    return counts, mean, ndup


def poisson_cdf(lam, x):
    """statrs Poisson::cdf for integer x (Q(x+1, lam)) by direct summation."""
    term = math.exp(-lam)
    tot = 0.0
    for i in range(x + 1):
        if term == 0.0 and i > lam:  # every later term is 0 too (counts reach 2^32 - 1)
            break
        tot += term
        term *= lam / (i + 1)
    return tot


def ratio_lambda(full, min_count_correct):
    """src/inference.rs:207-242"""
    cm = {}
    nzero = 0
    for x in full:
        if x == 0:
            nzero += 1
        else:
            cm[x] = cm.get(x, 0) + 1
    if len(cm) == 1:
        return None
    if len(full) - nzero < 25:
        return None
    sv = sorted(((cnt, val) for val, cnt in cm.items()), reverse=True)
    most = sv[0][1]
    if most + 1 not in cm:
        return None
    cp1, cc = float(cm[most + 1]), float(cm[most])
    if cp1 < min_count_correct or cc < min_count_correct:
        return None
    return cp1 / cc * (most + 1)


# ---- the ANI's pow / exp, correctly rounded --------------------------------------------------------------------------
_CTX = decimal.Context(prec=50)
_EXACT = decimal.Context(prec=1200)   # a double and a midpoint between two doubles in decimal without rounding


def _nearest(v):
    """the double nearest the 50-digit Decimal v; refuses a v within 1e-40 (relative) of a midpoint between two
    doubles, where 50 digits cannot decide the rounding"""
    y = float(v)
    for nb in (math.nextafter(y, math.inf), math.nextafter(y, -math.inf)):
        mid = _EXACT.divide(_EXACT.add(Decimal(y), Decimal(nb)), 2)
        if _EXACT.abs(_EXACT.subtract(v, mid)) <= _EXACT.multiply(_EXACT.abs(v), Decimal("1e-40")):
            raise ValueError("too close to a rounding midpoint: %s" % v)
    return y


def cr_pow(x, c):
    """x ** c (doubles) correctly rounded"""
    return _nearest(_CTX.power(Decimal(x), Decimal(c)))


def cr_exp(z):
    """exp(z) correctly rounded"""
    return _nearest(_CTX.exp(Decimal(z)))


def ani_pow(x, c, cr_math):
    """the reference's ANI pow (src/contain.rs:657, :836): glibc's (Python's float power), or correctly rounded"""
    return cr_pow(x, c) if cr_math else x ** c


def ani_exp(z, cr_math):
    """the reference's ANI exp (src/contain.rs:833)"""
    return cr_exp(z) if cr_math else math.exp(z)


def ani_from_lambda(lam, k, full, cr_math=False):
    """src/contain.rs:817-847"""
    if lam is None:
        return None
    contain = sum(1 for x in full if x != 0)
    adj = contain / (1.0 - ani_exp(-lam, cr_math)) / len(full)
    ani = ani_pow(adj, 1.0 / k, cr_math)
    if ani < 0 or math.isnan(ani):
        return None
    return ani


class WyRand:
    """fastrand 2.1.1: WyRand with the wyhash v4.2 constants; usize(..n) = Lemire gen_mod_u64."""

    def __init__(self, seed):
        self.s = seed & MASK64

    def u64(self):
        self.s = (self.s + 0x2D358DCCAA6C78A5) & MASK64
        t = self.s * (self.s ^ 0x8BB84B93962EACC9)
        return (t & MASK64) ^ (t >> 64)

    def usize(self, n):
        r = self.u64()
        m = r * n
        hi, lo = m >> 64, m & MASK64
        if lo < n:
            t = ((1 << 64) - n) % n
            while lo < t:
                r = self.u64()
                m = r * n
                hi, lo = m >> 64, m & MASK64
        return hi


def bootstrap_interval(full, k, min_count_correct, cr_math=False):
    """src/contain.rs:849-898"""
    rng = WyRand(7)
    res_a, res_l = [], []
    n = len(full)
    for _ in range(100):
        rv = [full[rng.usize(n)] for _ in range(n)]
        lam = ratio_lambda(rv, min_count_correct)
        ani = ani_from_lambda(lam, k, rv, cr_math)
        if ani is not None and lam is not None:
            res_a.append(ani)
            res_l.append(lam)
    res_a.sort()
    res_l.sort()
    if len(res_a) < 50:
        return None
    suc = len(res_a)
    return res_a[suc * 5 // 100 - 1], res_a[suc * 95 // 100 - 1], res_l[suc * 5 // 100 - 1], res_l[suc * 95 // 100 - 1]


def get_stats(genome_kmers, sample, k=31, min_number_kmers=50.0, min_count_correct=3.0, min_ani=0.90, no_ci=False,
              winner=None, genome_id=None, mean_coverage=False, no_adj=False, cr_math=False):
    """src/contain.rs:601-814 (pass 1 when winner is None) -> dict or None.  mean_coverage: the final coverage of a
    median >= 15 is the mean too (:722); no_adj: the final ANI is the naive one (:740); cr_math: the ANI's pow / exp
    correctly rounded instead of glibc's."""
    if len(genome_kmers) < min_number_kmers:
        return None
    covs, lost = [], 0
    for km in genome_kmers:
        c = sample.get(km)
        if c is None or c == 0:
            continue
        if winner is not None and winner[km] != genome_id:
            lost += 1
            continue
        covs.append(c)
    if not covs:
        return None
    n = len(genome_kmers)
    naive = ani_pow(len(covs) / n, 1.0 / k, cr_math)
    covs.sort()
    median = covs[len(covs) // 2]
    max_cov = float("inf")
    if median < 30:
        for cv in covs[len(covs) // 2:]:
            if poisson_cdf(float(median), cv) < 0.9999999999:
                max_cov = cv
            else:
                break
    full = [0] * (n - len(covs)) + [c for c in covs if c <= max_cov]
    ssum = sum(full) & 0xFFFFFFFF
    geq1 = ssum / len(covs)
    lam = None
    if median > 2:
        status = "HIGH"
    else:
        lam = ratio_lambda(full, min_count_correct)
        status = "LOW" if lam is None else "LAMBDA"
    final_cov = lam if lam is not None else (geq1 if median < 15 or mean_coverage else float(median))
    est = ani_from_lambda(lam, k, full, cr_math)
    final_ani = naive if (lam is None or est is None or no_adj) else est
    if final_ani < min_ani:
        return None
    ci = None
    if not no_ci and lam is not None:
        ci = bootstrap_interval(full, k, min_count_correct, cr_math)
    return dict(naive_ani=naive, final_est_ani=final_ani, final_est_cov=final_cov, mean_cov=geq1, median_cov=float(median),
                contain=len(covs), glen=n, status=status, lam=lam, ci=ci, kmers_lost=lost if winner is not None else None)


def contain_sample(genomes, sample, k=31, pseudotax=False, min_number_kmers=50.0, min_count_correct=3.0,
                   minimum_ani=None, redundant_ani=99.0, no_ci=False, unknown=None, mean_coverage=False, no_adj=False,
                   cr_math=False):
    """Inner body of contain() for one sample (src/contain.rs:284-334), written from the reference
    source only.  genomes: list of dict(kmers=[..], tracked=[..], gn_size=int); sample: dict hash->count.
    Pass-1 results are taken in genome-index order (the reference's order is thread-timing dependent).
    unknown = (read_seq_id percent, mean_read_length, sample c): -u with --read-seq-id (:274-279, :377-408).
    cr_math: the ANI's pow / exp correctly rounded; the k-mer identity and the derep threshold stay on glibc.
    -> list of dicts (get_stats fields + genome, rel_abund, seq_abund) in output order."""
    min_ani = minimum_ani / 100.0 if minimum_ani is not None else (0.95 if pseudotax else 0.90)  # :746-748
    kw = dict(k=k, min_number_kmers=min_number_kmers, min_count_correct=min_count_correct, min_ani=min_ani, no_ci=no_ci,
              mean_coverage=mean_coverage, no_adj=no_adj, cr_math=cr_math)
    res = []
    for gi, g in enumerate(genomes):  # :286-292
        r = get_stats(g["kmers"], sample, **kw)
        if r is not None:
            r["genome"] = gi
            res.append(r)

    def true_cov(rows):  # estimate_true_cov :377-389
        if unknown is None:
            return
        seq_id, rl, _ = unknown
        kid = (seq_id / 100.0) ** k
        mult = rl / (rl - k + 1.0)
        for r in rows:
            r["final_est_cov"] = r["final_est_cov"] / kid * mult

    true_cov(res)
    if pseudotax:
        # winner_table (:410-430): first entry wins ties, a later genome needs a strictly larger ANI
        winner = {}
        for r in res:
            g = genomes[r["genome"]]
            for km in list(g["kmers"]) + list(g.get("tracked", [])):
                v = winner.get(km)
                if v is None or r["final_est_ani"] > v[0]:
                    winner[km] = (r["final_est_ani"], r["genome"])
        wmap = {km: v[1] for km, v in winner.items()}
        res2 = []
        for r in res:  # :302-307
            r2 = get_stats(genomes[r["genome"]]["kmers"], sample, winner=wmap, genome_id=r["genome"], **kw)
            if r2 is not None:
                r2["genome"] = r["genome"]
                res2.append(r2)
        # derep_if_reassign_threshold (:353-375)
        old = {r["genome"]: r for r in res}
        thr = (redundant_ani / 100.0) ** k
        res = [r for r in res2 if float(old[r["genome"]]["contain"] - r["contain"]) < thr * r["glen"]]
        true_cov(res)
        explained = 1.0
        if unknown is not None:  # estimate_covered_bases :391-408
            _, rl, sc = unknown
            mult = rl / (rl - k + 1.0)
            covered = sum(genomes[r["genome"]]["gn_size"] * r["final_est_cov"] for r in res)
            tentative = float(sc * sum(sample.values())) * mult
            explained = 0.0 if tentative == 0.0 else min(covered / tentative, 1.0)
        total_cov = sum(r["final_est_cov"] for r in res)  # :319-326
        total_seq = sum(r["final_est_cov"] * genomes[r["genome"]]["gn_size"] for r in res)
        for r in res:
            r["rel_abund"] = r["final_est_cov"] / total_cov * 100.0
            r["seq_abund"] = r["final_est_cov"] * genomes[r["genome"]]["gn_size"] / total_seq * 100.0 * explained
        res.sort(key=lambda r: -r["rel_abund"])  # stable, :329-331
    else:
        res.sort(key=lambda r: -r["final_est_ani"])  # :332-334
    return res
