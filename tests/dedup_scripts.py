"""Scripted duplicate-removal histories turned into reads (a test helper module, not a conftest).

A read sketch's counts come from dup_removal_lsh_full_exact (src/sketch.rs:690-731): for every survivor, the k-mer's
earlier events in read order and their two pair keys (src/sketch.rs:624-688) decide whether the read is a duplicate.
Random reads only ever match on both keys (exact duplicates) or on p0 == p1 (homopolymers).  Here a history is written
event by event instead: one target k-mer per script, every event one read that holds the target (or its reverse
complement, or the target twice) under chosen pair keys.  Keys come from a small pool per script, so matches on one key
only, matches across the two key slots (p0 of one read == p1 of another), A == B and keyless reads are all frequent.

The families are built to reach every device path of the single-end post-pass (sylph_b200/csrc/sample.cu):

  quick  k_group_dedup's four-event register replay: a k-mer with at most four events
  cut    the same replay with more than four events, four of them counted among the first four (c += len - 4)
  warp   the warp-cooperative replay: more than four events and a duplicate among the first four
  steps  generic k_dedup: the warp replay is still below MAX_DEDUP_COUNT after GRP_SELECT_STEPS events
  set    generic k_dedup: the warp replay's dedup set outgrows its 32 lanes
  slot   generic k_dedup: the k-mer alone has more events than a group's slot

Single-end layout with keys A = (A.x, A.y), B = (B.x, B.y), each part a 16-base word: bases [0, 32) interleave A.x (even
positions) and B.x (odd), bases [L//2, L//2 + 32) interleave A.y and B.y, so that pair_kmer_single gives
p0 = (A.x, A.y) and p1 = (B.x, B.y).  The target goes in a gap that overlaps neither window.  Keyless reads are
50-65 bp or 401-500 bp.  Read pairs: mate 1 interleaves (A.x, B.x) and mate 2 (A.y, B.y) in their first 32 bases.
"""
import functools
import zlib

import numpy as np

from oracle import oracle as O
from oracle import pyref as R

# sample.cu
SLOT = 1024          # GRP_CAP: events one k_group_dedup CTA holds (the slot of a post-pass group)
SELECT_STEPS = 64    # GRP_SELECT_STEPS: warp replay steps before a duplicate-heavy k-mer goes to the generic path
SET_LANES = 32       # the warp replay keeps dedup-set entry q in lane q
GRP_T = 640          # expected events per group
GRP_BPG = 32         # hash buckets per group (common.cuh)
MAX_DEDUP_COUNT = 4  # src/constants.rs:14

IN_KERNEL = ("quick", "cut", "warp")
FALLBACK = ("steps", "set", "slot")
MATCHES = ("one_key", "both_keys", "cross_slot", "a_eq_b")

_ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
_COMP = bytes.maketrans(b"ACGT", b"TGCA")


def revcomp(s):
    return s.translate(_COMP)[::-1]


def code16(w):
    """16 bases -> the 32-bit key word of pair_kmer_single (first base in the top bits)."""
    v = 0
    for b in w:
        v = (v << 2) | R.BYTE_TO_SEQ[b]
    return v


def _interleave(even, odd):
    out = bytearray(32)
    out[0::2] = even
    out[1::2] = odd
    return bytes(out)


class Gen:
    """Reads for scripted histories at one (k, c, sem).  A key is a pair of 16-base words (x, y)."""

    def __init__(self, seed, k=31, c=10, sem=O.SEM_AVX2):
        self.rng = np.random.default_rng(seed)
        self.k, self.c, self.sem = k, c, sem
        self._targets, self._used = [], set()

    def bases(self, n):
        return _ACGT[self.rng.integers(0, 4, size=n)].tobytes()

    def key(self):
        return (self.bases(16), self.bases(16))

    def target(self):
        """A fresh k-mer that survives FracMinHash at c: (bases, hash).  Targets are taken 2k apart: two overlapping
        survivors would let filler next to one target complete the other."""
        while not self._targets:
            s = self.bases(4000 * self.c)
            pos, h = O.extract_markers_positions(s, self.k, self.c, self.sem)
            last = -2 * self.k
            for p, x in zip(pos.tolist(), h.tolist()):
                if p - last >= 2 * self.k and x not in self._used:
                    last = p
                    self._used.add(x)
                    self._targets.append((s[p - self.k + 1:p + 1], x))
        return self._targets.pop()

    def keep_end(self, L):
        """Windows ending before this index are emitted (AVX2 semantics drop the tail windows, pyref.seeds_avx2)."""
        if self.sem == O.SEM_SCALAR:
            return L
        return 4 * ((L - self.k + 1) // 4) + self.k - 1

    def _starts(self, lo, hi, n):
        """n non-overlapping target starts in [lo, hi] (hi = last start allowed)."""
        k = self.k
        assert hi - lo >= (n - 1) * k, (lo, hi, n)
        s = [int(self.rng.integers(lo, hi - (n - 1) * k + 1))]
        for _ in range(n - 1):
            s.append(int(self.rng.integers(s[-1] + k, hi - (n - 1 - len(s)) * k + 1)))
        return s

    def _put(self, read, tgt, starts, rc):
        t = revcomp(tgt) if rc else tgt
        for s in starts:
            read[s:s + self.k] = t

    def single(self, tgt, keys, rc, twice):
        """One single-end read holding tgt once or twice; keys = (A, B) or None (keyless read)."""
        k, rng = self.k, self.rng
        n = 2 if twice else 1
        if keys is None:
            L = int(rng.integers(401, 501)) if twice or rng.random() < 0.5 else int(rng.integers(max(50, k + 1), 66))
            read = bytearray(self.bases(L))
            self._put(read, tgt, self._starts(0, self.keep_end(L) - k, n), rc)
            return bytes(read)
        L = int(rng.choice([150, 300, 400]))
        h = L // 2
        read = bytearray(self.bases(L))
        (a, b) = keys
        read[0:32] = _interleave(a[0], b[0])
        read[h:h + 32] = _interleave(a[1], b[1])
        gaps = [(32, h - k), (h + 32, self.keep_end(L) - k)]
        if twice:
            starts = [self._starts(*g, 1)[0] for g in gaps]
        else:
            starts = self._starts(*gaps[int(rng.integers(0, 2))], 1)
        self._put(read, tgt, starts, rc)
        return bytes(read)

    def mate(self, tgt, key_words, n_tgt, rc, short=False):
        """One mate: its first 32 bases interleave key_words (a pair's x or y words), then n_tgt copies of tgt."""
        k, rng = self.k, self.rng
        if short:                                  # < 33 bp: the pair has no keys (src/sketch.rs:661)
            return self.bases(int(rng.integers(20, 33)))
        L = int(rng.integers(100, 151))
        read = bytearray(self.bases(L))
        if key_words is not None:
            read[0:32] = _interleave(*key_words)
        if n_tgt:
            self._put(read, tgt, self._starts(32, self.keep_end(L) - k, n_tgt), rc)
        return bytes(read)


# ---- single-end families: an event is (key index a, key index b) into the script's key pool, or None (keyless) ------

def _fam_quick(rng):
    """1-4 events from a pool of three keys."""
    return 3, [None if rng.random() < 0.15 else (int(rng.integers(0, 3)), int(rng.integers(0, 3)))
               for _ in range(int(rng.integers(1, 5)))]


def _fam_cut(rng):
    """5-12 events, no duplicate among the first four: keyless or two unseen, distinct keys each; anything after."""
    ev, nxt = [], 0
    for i in range(4):
        if i > 0 and rng.random() < 0.2:
            ev.append(None)
        else:
            ev.append((nxt, nxt + 1) if rng.random() < 0.5 else (nxt + 1, nxt))
            nxt += 2
    for _ in range(int(rng.integers(1, 9))):
        ev.append(None if rng.random() < 0.1 else (int(rng.integers(0, nxt + 1)), int(rng.integers(0, nxt + 1))))
    return nxt + 1, ev


def _fam_warp(rng):
    """5-12 events from a pool of three keys with a duplicate among the first four."""
    while True:
        ev = [None if rng.random() < 0.1 else (int(rng.integers(0, 3)), int(rng.integers(0, 3)))
              for _ in range(int(rng.integers(5, 13)))]
        if replay(ev[:4])[0] < MAX_DEDUP_COUNT:
            return 3, ev


def _tail_past_the_cut(rng, ev, nxt, pool):
    """Events with unseen keys until four are counted, then events that share keys: with MAX_DEDUP_COUNT they count,
    without it they would be duplicates."""
    while replay(ev)[0] < MAX_DEDUP_COUNT:
        ev.append((nxt, nxt + 1))
        nxt += 2
    for _ in range(int(rng.integers(4, 9))):
        a = int(rng.integers(0, pool))
        ev.append((a, a) if rng.random() < 0.2 else (a, int(rng.integers(0, pool))))
    return nxt, ev


def _fam_steps(rng):
    """70 or more events, the count below four for the first GRP_SELECT_STEPS: every event after the first shares a key
    with an earlier one (at most two keyless); four keys, so the set stays small."""
    ev, seen, keyless = [(0, 1)], {0, 1}, 0
    while len(ev) < SELECT_STEPS + 1:
        if keyless < 2 and rng.random() < 0.04:
            ev.append(None)
            keyless += 1
            continue
        a = int(rng.choice(sorted(seen)))
        b = a if rng.random() < 0.15 else int(rng.integers(0, 4))
        ev.append((a, b) if rng.random() < 0.5 else (b, a))
        seen.add(b)
    nxt, ev = _tail_past_the_cut(rng, ev, 4, 4)
    while len(ev) < 70:
        ev.append((0, int(rng.integers(0, 4))))
    return nxt, ev


def _fam_set(rng):
    """(A0, B0), then about 40 events that share A0 (in either slot) with a fresh second key each: the set passes 32
    entries while the count stays at one."""
    ev, nxt = [(0, 1)], 2
    for _ in range(int(rng.integers(38, 44))):
        if rng.random() < 0.04:
            ev.append(None)
            continue
        ev.append((0, nxt) if rng.random() < 0.5 else (nxt, 0))
        nxt += 1
    return _tail_past_the_cut(rng, ev, nxt, nxt)


def _fam_slot(rng):
    """More than SLOT events of one k-mer from a pool of six keys."""
    ev = [None if rng.random() < 0.05 else (int(rng.integers(0, 6)), int(rng.integers(0, 6)))
          for _ in range(int(rng.integers(SLOT + 10, SLOT + 80)))]
    return 6, ev


FAMILIES = {"quick": _fam_quick, "cut": _fam_cut, "warp": _fam_warp, "steps": _fam_steps, "set": _fam_set,
            "slot": _fam_slot}

# scripts per family in each single-end sample
SAMPLES = {
    "in_kernel": {"quick": 300, "cut": 200, "warp": 200},
    "steps": {"steps": 24},
    "set": {"set": 30},
    "slot": {"slot": 4},
}
SMALL = {"quick": 60, "cut": 25, "warp": 40, "steps": 4, "set": 5}   # the pyref cross-check (slow)


class Sample:
    """reads in sample order; expect[i] = (pair keys or None, target hash, occurrences of the target in read i)"""

    def __init__(self, reads, expect, n_scripts):
        self.reads, self.expect, self.n_scripts = reads, expect, n_scripts

    def flat(self):
        return flatten(self.reads)


class PairSample:
    """expect[i] = (pair keys or None, target hash, occurrences in mate 1, occurrences in mate 2)"""

    def __init__(self, r1, r2, expect, n_scripts):
        self.r1, self.r2, self.expect, self.n_scripts = r1, r2, expect, n_scripts


def flatten(seqs):
    off = np.zeros(len(seqs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(s) for s in seqs], dtype=np.uint64)
    return np.frombuffer(b"".join(seqs), dtype=np.uint8).copy(), off


def _interleave_scripts(rng, scripts):
    """Merge the scripts' read lists in a seeded order that keeps every script's own order."""
    labels = np.repeat(np.arange(len(scripts)), [len(s) for s in scripts])
    rng.shuffle(labels)
    cur = [0] * len(scripts)
    out = []
    for s in labels.tolist():
        out.append(scripts[s][cur[s]])
        cur[s] += 1
    return out


def _pair_of(keys):
    (a, b) = keys
    return (code16(a[0]), code16(a[1])), (code16(b[0]), code16(b[1]))


@functools.lru_cache(maxsize=None)
def single_sample(name, k=31, c=10, sem=O.SEM_AVX2, seed=0):
    """A single-end sample of the scripts SAMPLES[name] (or SMALL for name == "small")."""
    plan = SMALL if name == "small" else SAMPLES[name]
    g = Gen(zlib.crc32(repr((name, k, c, sem, seed)).encode()), k, c, sem)
    rng = g.rng
    scripts = []
    for fam, n in plan.items():
        for _ in range(n):
            n_keys, events = FAMILIES[fam](rng)
            pool = [g.key() for _ in range(n_keys)]
            tgt, th = g.target()
            reads = []
            for e in events:
                keys = None if e is None else (pool[e[0]], pool[e[1]])
                # a keyless read with the target twice counts twice: not where the count has to stay below four
                twice = rng.random() < 0.1 and (e is not None or fam in ("quick", "cut", "warp", "slot"))
                read = g.single(tgt, keys, rng.random() < 0.5, twice)
                reads.append((read, (None if keys is None else _pair_of(keys), th, 2 if twice else 1)))
            scripts.append(reads)
    merged = _interleave_scripts(rng, scripts)
    return Sample([r for r, _ in merged], [e for _, e in merged], len(scripts))


# ---- read pairs: where the target sits, with keys from the script's pool ----------------------------------------------
PLACES = ("m1", "m2", "both", "m2_twice", "short_mate")


def _pair_events(rng, n, pool):
    return [(int(rng.integers(0, pool)), int(rng.integers(0, pool)), PLACES[int(rng.integers(0, len(PLACES)))])
            for _ in range(n)]


def _pair_big_set(rng):
    """(A0, B0), then 90 events that share A0 with a fresh key each: the dedup set passes 64 entries (more than two
    strides of k_dedup_paired's 32 lanes)."""
    ev = [(0, 1, "m1")]
    for i in range(90):
        place = PLACES[int(rng.integers(0, len(PLACES)))]
        ev.append((0, i + 2, place) if rng.random() < 0.5 else (i + 2, 0, place))
    return 92, ev


PAIR_SAMPLES = {"pairs": (400, 4), "small": (100, 1)}   # (scripts of 1-12 events, scripts with a set past 64)


@functools.lru_cache(maxsize=None)
def pair_sample(name="pairs", k=31, c=10, sem=O.SEM_AVX2, seed=0):
    n_short, n_big = PAIR_SAMPLES[name]
    g = Gen(zlib.crc32(repr(("pairs", name, k, c, sem, seed)).encode()), k, c, sem)
    rng = g.rng
    scripts = []
    for i in range(n_short + n_big):
        n_keys, events = (3, _pair_events(rng, int(rng.integers(1, 13)), 3)) if i < n_short else _pair_big_set(rng)
        pool = [g.key() for _ in range(n_keys)]
        tgt, th = g.target()
        reads = []
        for a, b, place in events:
            A, B = pool[a], pool[b]
            rc = rng.random() < 0.5
            if place == "short_mate":
                short1 = rng.random() < 0.5
                m1 = g.mate(tgt, (A[0], B[0]), 0 if short1 else 1, rc, short=short1)
                m2 = g.mate(tgt, (A[1], B[1]), 1 if short1 else 0, rc, short=not short1)
                reads.append((m1, m2, (None, th, 0 if short1 else 1, 1 if short1 else 0)))
                continue
            n1 = 1 if place in ("m1", "both") else 0
            n2 = {"m1": 0, "m2": 1, "both": 1, "m2_twice": 2}[place]
            m1 = g.mate(tgt, (A[0], B[0]), n1, rc)
            m2 = g.mate(tgt, (A[1], B[1]), n2, rc)
            reads.append((m1, m2, (_pair_of((A, B)), th, n1, n2)))
        scripts.append(reads)
    merged = _interleave_scripts(rng, scripts)
    return PairSample([a for a, _, _ in merged], [b for _, b, _ in merged], [e for _, _, e in merged], len(scripts))


# ---- the rule, transcribed, and the classifier ------------------------------------------------------------------------

def replay(events, threshold=MAX_DEDUP_COUNT, no_dedup=False, matches=None):
    """dup_removal_lsh_full_exact (src/sketch.rs:690-731) over ONE k-mer's events in read order: events = [pair keys or
    None] -> (count, duplicates removed).  threshold None = no MAX_DEDUP_COUNT (read pairs).  matches: a dict that
    tallies the key matches of the events whose duplicate test counts (c > 0)."""
    c, dups, slot_of = 0, 0, {}
    for pair in events:
        if not no_dedup and (threshold is None or c < threshold) and pair is not None:
            a, b = pair
            if matches is not None and c > 0:
                fa, fb = a in slot_of, b in slot_of
                if fa and fb:
                    matches["both_keys"] = matches.get("both_keys", 0) + 1
                elif fa or fb:
                    matches["one_key"] = matches.get("one_key", 0) + 1
                elif a == b:
                    matches["a_eq_b"] = matches.get("a_eq_b", 0) + 1
                if (fa and slot_of[a] == 1) or (fb and slot_of[b] == 0):
                    matches["cross_slot"] = matches.get("cross_slot", 0) + 1
            ret = False
            for slot, pk in enumerate(pair):
                if pk in slot_of:
                    ret = ret or c > 0
                else:
                    slot_of[pk] = slot
            if ret:
                dups += 1
                continue
        c += 1
    return c, dups


def device_path(events):
    """The single-end post-pass path a k-mer with these events (pair keys or None, in read order) takes in sample.cu,
    when its group fits its slot."""
    n = len(events)
    if n > SLOT:
        return "slot"
    if n <= 4:
        return "quick"
    if replay(events[:4])[0] >= MAX_DEDUP_COUNT:
        return "cut"
    c, nset, seen = 0, 0, set()     # the warp replay: GRP_SELECT_STEPS steps, one set entry per lane
    for done, pair in enumerate(events):
        if c >= MAX_DEDUP_COUNT:
            break
        if done >= SELECT_STEPS:
            return "steps"
        if pair is None:
            c += 1
            continue
        found = False
        for pk in pair:
            if pk in seen:
                found = True
            else:
                seen.add(pk)
        if len(seen) > SET_LANES:
            return "set"
        if not (found and c > 0):
            c += 1
    return "warp"


def kmer_events(reads, k, c, sem):
    """hash -> [pair keys or None] in read order, from the oracle's markers of every read (src/sketch.rs:917-939)."""
    ev = {}
    for s in reads:
        pair = R.pair_kmer_single(s) if len(s) <= 400 else None
        for h in O.extract_markers(s, k, c, sem).tolist():
            ev.setdefault(h, []).append(pair)
    return ev


def pair_kmer_events(r1, r2, k, c, sem):
    """hash -> [pair keys or None] in pair order; mate 2's k-mers that also occur in mate 1 are skipped
    (src/sketch.rs:840-865).  Also returns the number of skipped events per hash."""
    ev, skipped = {}, {}
    for s1, s2 in zip(r1, r2):
        pair = R.pair_kmer(s1, s2)
        v1 = O.extract_markers(s1, k, c, sem).tolist()
        for h in v1:
            ev.setdefault(h, []).append(pair)
        in1 = set(v1)
        for h in O.extract_markers(s2, k, c, sem).tolist():
            if h in in1:
                skipped[h] = skipped.get(h, 0) + 1
                continue
            ev.setdefault(h, []).append(pair)
    return ev, skipped


def group_sizes(ev, n_bases, n_reads, k, c):
    """Events per post-pass group, as SampleBuilder::begin() fixes the groups (sample.cu)."""
    win = n_bases - n_reads * (k - 1) if n_bases > n_reads * (k - 1) else 0
    ng = (win // c) // GRP_T + 1
    nbk = ng * GRP_BPG
    mb = min((nbk << 64) // ((2**64 - 1) // c + 1), 2**64 - 1)
    sizes = [0] * ng
    for h, e in ev.items():
        sizes[min((h * mb) >> 64, nbk - 1) // GRP_BPG] += len(e)
    return sizes


def classify(sample, k=31, c=10, sem=O.SEM_AVX2):
    """Per-class k-mer counts of a single-end sample (planned and unplanned k-mers alike), the key matches its
    duplicate tests see, and its largest post-pass group."""
    ev = kmer_events(sample.reads, k, c, sem)
    classes = dict.fromkeys(IN_KERNEL + FALLBACK, 0)
    matches = dict.fromkeys(MATCHES, 0)
    for e in ev.values():
        classes[device_path(e)] += 1
        replay(e, matches=matches)
    nb = sum(len(s) for s in sample.reads)
    return dict(classes=classes, matches=matches, max_group=max(group_sizes(ev, nb, len(sample.reads), k, c)))


def classify_pairs(sample, k=31, c=10, sem=O.SEM_AVX2):
    ev, skipped = pair_kmer_events(sample.r1, sample.r2, k, c, sem)
    matches = dict.fromkeys(MATCHES, 0)
    cases = dict(mate2_skip=len(skipped), keyless=0, set_over_64=0)
    for e in ev.values():
        replay(e, threshold=None, matches=matches)
        cases["keyless"] += any(p is None for p in e)
        cases["set_over_64"] += len({pk for p in e if p is not None for pk in p}) > 2 * SET_LANES
    return dict(cases=cases, matches=matches)
