"""Read and pair samples built k-mer by k-mer for the read-sketch grouping kernel (a test helper, not a conftest).

k_group_dedup (sylph_b200/csrc/sample.cu) takes one post-pass group per CTA: at most `slot` events (SYL_GROUP_CAP,
1024 by default) whose k-mers it groups in a 1024-slot open-addressing table, home slot (h ^ (h >> 23)) & 1023, and
whose uniques it orders by their rank within each of the group's 32 hash buckets.  Random reads fill a group to about
640 events, so the table never runs full.  The samples here are written hash by hash instead (genome_scripts' inverse
of mm_hash64): every k-mer is crafted to fall in a chosen group, bucket or home slot, or right at a bucket boundary, and
reads are laid out so that a group holds exactly the events a family claims.

Structural families use keyless reads (500 bp, longer than the 400 bp up to which pair_kmer_single gives keys), so
every event counts and the duplicate rule stays out of the way; read pairs use 500 bp mates, some k-mers in both mates
of one pair (mate 2's event is skipped by the rule but occupies the slot).  mixed_full writes dedup_scripts histories
into 150 bp keyed reads instead.  Filler is random, and every window that would survive at c without being scripted is
drawn again (genome_scripts._Builder._clean), so a record's survivors are exactly its scripted hashes.  Filler records
bring the sample's bases to the group count a family wants: the one-pass map (sample_parts.hpp sample_map) depends on
the bases and records only.

post_pass() is a CPU model of the structural decisions of the post-pass, computed from the oracle's survivors: events
per group, which groups stay in the kernel, the in-kernel uniques and the events handed to the generic path -- the
numbers the library prints as `[sample post-pass]` with SYL_DEBUG_TIMING=1.
"""
import functools
import zlib

import numpy as np

from oracle import oracle as O
from oracle import pyref as R
from tests import dedup_scripts as D
from tests import genome_scripts as GS

K = 31
C = 200
SEM = O.SEM_AVX2
U64 = 2**64 - 1
SLOT = 1024          # GRP_CAP: the default slot of a group
TABLE = 1024         # GRP_SLOTS: k_group_dedup's hash table
BPG = 32             # GRP_BPG: buckets per group
GRP_T = 640          # expected events per group of the map
READ_LEN = 500       # keyless reads and structural mates
SPACING = 50         # between scripted k-mers of a record (> k + genome_scripts.NEAR: no filler search)
PER_READ = 9         # scripted k-mers per 500 bp record
PAIR_START = 32      # structural mates keep their first 32 bases (the pair keys) free of scripted k-mers
FILL_LEN = 4000      # filler records
_ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)


# ---- the one-pass map (sample_parts.hpp), restated ------------------------------------------------------------------

def home(h):
    """k_group_dedup's home slot of hash h"""
    return (h ^ (h >> 23)) & (TABLE - 1)


class Map:
    """sample_map(bases, records, k, c): ng groups of 32 buckets, bucket = min(mulhi(h, Mb), nbk - 1)"""

    def __init__(self, bases, records, k=K, c=C):
        win = bases - records * (k - 1) if bases > records * (k - 1) else 0
        self.n_exp = win // c
        self.thr = U64 // c
        self.ng = self.n_exp // GRP_T + 1
        self.nbk = self.ng * BPG
        self.Mb = min((self.nbk << 64) // (self.thr + 1), U64)

    def bucket(self, h):
        return min((h * self.Mb) >> 64, self.nbk - 1)

    def group(self, h):
        return self.bucket(h) // BPG

    def first_hash(self, b):
        """bucket_first_hash: the smallest hash of bucket b (at most thr)"""
        return 0 if b == 0 else min(((b << 64) + self.Mb - 1) // self.Mb, self.thr)

    def bucket_range(self, b):
        return self.first_hash(b), (self.first_hash(b + 1) if b + 1 < self.nbk else self.thr)

    def group_range(self, g):
        return self.first_hash(g * BPG), (self.first_hash((g + 1) * BPG) if (g + 1) * BPG < self.nbk else self.thr)

    def parts(self, P):
        """cut_parts: P parts at the bucket boundaries nbk p / P -> [(lo, hi, g0, ng)]"""
        P = min(P, self.nbk)
        out = []
        for p in range(P):
            b0, b1 = self.nbk * p // P, self.nbk * (p + 1) // P
            lo = 0 if p == 0 else self.first_hash(b0)
            hi = self.thr if p == P - 1 else self.first_hash(b1)
            out.append((lo, hi, b0 // BPG, (b1 + BPG - 1) // BPG - b0 // BPG))
        return out


# ---- hashes with a canonical 31-mer ----------------------------------------------------------------------------------

class Crafter:
    """Unused hashes whose preimage under mm_hash64 is a canonical k-mer, in a chosen range and home slot."""

    def __init__(self, rng, k=K):
        self.rng, self.k, self.used = rng, k, set()

    def valid(self, h):
        h = np.array(h, dtype=np.uint64, ndmin=1)
        return GS.is_canonical(GS.unhash64(h), self.k)

    def hash_in(self, lo, hi, slot=None):
        """a hash in [lo, hi), with home slot `slot` if given"""
        for _ in range(2000):
            h = self.rng.integers(lo, hi, size=512, dtype=np.uint64, endpoint=False)
            if slot is not None:   # bits 23-32 stay, so the low ten bits fix the home slot
                h = (h & ~np.uint64(TABLE - 1)) | (((h >> np.uint64(23)) & np.uint64(TABLE - 1)) ^ np.uint64(slot))
                h = h[(h >= np.uint64(lo)) & (h < np.uint64(hi))]
            for x in h[self.valid(h)].tolist():
                if x not in self.used:
                    self.used.add(x)
                    return x
        raise RuntimeError("no hash in [%d, %d)" % (lo, hi))

    def nearest(self, h, step, lo, hi):
        """the first valid unused hash of h, h + step, h + 2 step, ... inside [lo, hi)"""
        for i0 in range(0, 1 << 20, 4096):
            x = [h + step * i for i in range(i0, i0 + 4096)]
            x = [v for v in x if lo <= v < hi]
            if not x:
                break
            ok = self.valid(np.array(x, dtype=np.uint64))
            for v, good in zip(x, ok.tolist()):
                if good and v not in self.used:
                    self.used.add(v)
                    return v
        raise RuntimeError("no valid hash near %d" % h)


# ---- records ---------------------------------------------------------------------------------------------------------

class _Writer:
    """Records whose survivors at c are exactly the placed hashes (genome_scripts._Builder orients and cleans)."""

    def __init__(self, seed, k, c):
        self.b = GS._Builder(seed, k, c, c)
        self.rng, self.k = self.b.rng, k

    def codes(self, n):
        return self.rng.integers(0, 4, size=n, dtype=np.uint8)

    def record(self, L, place, fixed_ranges=()):
        """place: [(start, hash)]; fixed_ranges: [(a, b)] bases kept as given (after codes are preset by the caller)"""
        return self.finish(self.codes(L), place, fixed_ranges)

    def finish(self, codes, place, fixed_ranges=()):
        k = self.k
        fixed = np.zeros(len(codes), dtype=bool)
        for a, b in fixed_ranges:
            fixed[a:b] = True
        keep = set()
        for s, h in place:
            codes[s:s + k] = self.b._orient(int(GS.unhash64(np.uint64(h))[0]))
            fixed[s:s + k] = True
            keep.add(s + k - 1)
        assert all(s + k <= GS.valid_starts(len(codes), k) + k - 1 for s, _ in place), "a k-mer past the AVX2 windows"
        self.b._clean(codes, fixed, keep)
        return _ACGT[codes].tobytes()

    def spread(self, hashes, L=READ_LEN, first=0):
        """a record of L bases holding hashes SPACING apart from a random start >= first"""
        n = len(hashes)
        last = GS.valid_starts(L, self.k) - 1 - (n - 1) * SPACING
        s0 = int(self.rng.integers(first, last + 1)) if n else 0
        return self.record(L, [(s0 + i * SPACING, h) for i, h in enumerate(hashes)])


class Sample:
    """reads (single-end) or r1 / r2 (pairs), and what each record was scripted to hold: script[i] = sorted hashes of
    record i (pairs: (mate 1's, mate 2's))."""

    def __init__(self, name, paired, k, c, slot, claims):
        self.name, self.paired, self.k, self.c, self.slot, self.claims = name, paired, k, c, slot, claims
        self.reads, self.r1, self.r2, self.script = [], [], [], []

    @property
    def records(self):
        return self.r1 if self.paired else self.reads

    def flat(self):
        """(bases, off) single-end, (b1, o1, b2, o2) pairs"""
        if self.paired:
            return D.flatten(self.r1) + D.flatten(self.r2)
        return D.flatten(self.reads)

    @property
    def n_bases(self):
        return sum(map(len, self.r1)) + sum(map(len, self.r2)) if self.paired else sum(map(len, self.reads))

    @property
    def n_records(self):
        return 2 * len(self.r1) if self.paired else len(self.reads)

    @functools.cached_property
    def map(self):
        return Map(self.n_bases, self.n_records, self.k, self.c)


def _plan_fill(ev_bases, ev_records, want_ng, k, c, mates):
    """number of filler records (pairs: of FILL_LEN / 2 bp mates) that put the map at want_ng groups"""
    target = (GRP_T * want_ng - GRP_T // 2) * c      # windows for the middle of the group count's range
    have = ev_bases - ev_records * (k - 1)
    assert have <= target, "the scripted records alone pass %d groups at c = %d" % (want_ng, c)
    per = FILL_LEN - mates * (k - 1)
    return (target - have) // per + 1


def _mix(rng, records, n_fill, filler):
    """the scripted records in their order, with n_fill filler records at random places"""
    slots = np.sort(rng.choice(len(records) + n_fill, size=n_fill, replace=False)).tolist() if n_fill else []
    out, it, f = [], iter(records), 0
    for i in range(len(records) + n_fill):
        if f < len(slots) and slots[f] == i:
            out.append(filler())
            f += 1
        else:
            out.append(next(it))
    return out


# ---- structural families: k-mers made from the map, laid out in keyless records ------------------------------------

def in_group(g, slot=None):
    return lambda m, cr: cr.hash_in(*m.group_range(g), slot)


def in_bucket(b, slot=None):
    return lambda m, cr: cr.hash_in(*m.bucket_range(b), slot)


def at_or_above(fh):
    """the smallest valid hash at or above fh(m)"""
    return lambda m, cr: cr.nearest(fh(m), 1, fh(m), m.thr)


def below(fh):
    """the largest valid hash below fh(m)"""
    return lambda m, cr: cr.nearest(fh(m) - 1, -1, 0, fh(m))


def structural(name, paired, want_ng, spec, slot=SLOT, claims=None, k=K, c=C, seed=0):
    """spec: [(maker, events, in_both)]: maker(map, crafter) -> hash; events in the k-mer's group; pairs: in_both of
    them are pairs holding the k-mer in both mates (2 events each, mate 2's skipped by the pair rule)."""
    w = _Writer(zlib.crc32(repr((name, paired, want_ng, slot, k, c, seed)).encode()), k, c)
    rng = w.rng
    items = []
    for i, (_, n, both) in enumerate(spec):
        assert 2 * both <= n
        items += [("one", i)] * (n - 2 * both) + [("both", i)] * both
    order = rng.permutation(len(items)).tolist()
    recs = []              # per record: [ids] (single-end) or ([ids mate 1], [ids mate 2])
    if not paired:
        ids = [items[j][1] for j in order]
        recs = [ids[i:i + PER_READ] for i in range(0, len(ids), PER_READ)]
    else:
        cur = ([], [])
        for j in order:
            kind, i = items[j]
            room = [PER_READ - len(cur[0]), PER_READ - len(cur[1])]
            if (kind == "both" and min(room) < 1) or max(room) < 1:
                recs.append(cur)
                cur = ([], [])
                room = [PER_READ, PER_READ]
            if kind == "both":
                cur[0].append(i)
                cur[1].append(i)
            else:
                mate = int(rng.integers(0, 2)) if min(room) > 0 else int(np.argmax(room))
                cur[mate].append(i)
        recs.append(cur)
    mates = 2 if paired else 1
    n_fill = _plan_fill(mates * READ_LEN * len(recs), mates * len(recs), want_ng, k, c, mates)
    s = Sample(name, paired, k, c, slot, dict(claims or {}))
    n_bases = mates * (READ_LEN * len(recs) + (FILL_LEN // mates) * n_fill)
    m = Map(n_bases, mates * (len(recs) + n_fill), k, c)
    assert m.ng == want_ng, (m.ng, want_ng)
    cr = Crafter(rng, k)
    hashes = [mk(m, cr) for mk, _, _ in spec]
    s.claims["hashes"] = hashes
    first = PAIR_START if paired else 0
    if not paired:
        made = [(w.spread([hashes[i] for i in r], first=first), sorted(hashes[i] for i in r)) for r in recs]
        made = _mix(rng, made, n_fill, lambda: (w.record(FILL_LEN, []), []))
        s.reads = [r for r, _ in made]
        s.script = [e for _, e in made]
    else:
        made = [((w.spread([hashes[i] for i in a], first=first), w.spread([hashes[i] for i in b], first=first)),
                 (sorted(hashes[i] for i in a), sorted(hashes[i] for i in b))) for a, b in recs]
        L = FILL_LEN // 2
        made = _mix(rng, made, n_fill, lambda: ((w.record(L, []), w.record(L, [])), ([], [])))
        s.r1 = [r[0] for r, _ in made]
        s.r2 = [r[1] for r, _ in made]
        s.script = [e for _, e in made]
    assert s.map.ng == want_ng and s.map.Mb == m.Mb
    return s


def _light(rng, g, n):
    """n events of k-mers with 1-3 events each in group g"""
    out = []
    while n > 0:
        e = min(n, int(rng.integers(1, 4)))
        out.append((in_group(g), e, 0))
        n -= e
    return out


def fam_full_distinct(paired):
    """group 0: exactly 1024 distinct k-mers of one event each (the table 100 % full); group 1: 300"""
    spec = [(in_group(0), 1, 0) for _ in range(TABLE)] + [(in_group(1), 1, 0) for _ in range(300)]
    return structural("full_distinct", paired, 2, spec, claims=dict(full=[0], sizes={0: TABLE, 1: 300}))


def fam_full_one_home(paired):
    """1024 distinct k-mers homed at slot 1023 (group 0: the chain wraps to slot 0 and covers the table) and at slot 0
    (group 1: the chain ends at slot 1023)"""
    spec = [(in_group(0, TABLE - 1), 1, 0) for _ in range(TABLE)] + [(in_group(1, 0), 1, 0) for _ in range(TABLE)]
    return structural("full_one_home", paired, 2, spec,
                      claims=dict(full=[0, 1], one_home={0: TABLE - 1, 1: 0}, sizes={0: TABLE, 1: TABLE}))


def fam_one_bucket(paired):
    """a full group (1024 distinct k-mers) in one bucket: bucket 0, bucket 63 (the middle group's local bucket 31) and
    the map's last bucket nbk - 1 = 95"""
    spec = []
    for b in (0, 63, 95):
        spec += [(in_bucket(b), 1, 0) for _ in range(TABLE)]
    return structural("one_bucket", paired, 3, spec,
                      claims=dict(full=[0, 1, 2], buckets={0: TABLE, 63: TABLE, 95: TABLE},
                                  sizes={0: TABLE, 1: TABLE, 2: TABLE}))


def fam_slot(paired, slot=SLOT, plus_one=False):
    """four groups: slot and slot + 1 events next to each other (groups 0, 1; slot_plus_one swaps them), a light group,
    and the last group: one k-mer of exactly `slot` events (slot_plus_one: and one more k-mer of one event).  Pairs:
    an eighth of the heavy k-mer's events are pairs holding it in both mates."""
    rng = np.random.default_rng(zlib.crc32(repr(("slot", paired, slot, plus_one)).encode()))
    a, b = (slot + 1, slot) if plus_one else (slot, slot + 1)
    light = min(200, slot // 2)
    spec = _light(rng, 0, a) + _light(rng, 1, b) + _light(rng, 2, light)
    spec.append((in_group(3), slot, slot // 16 if paired else 0))
    last = slot
    if plus_one:
        spec.append((in_group(3), 1, 0))
        last += 1
    name = "slot_plus_one" if plus_one else "slot_exact"
    return structural(name, paired, 4, spec, slot=slot, claims=dict(sizes={0: a, 1: b, 2: light, 3: last}, heavy=slot))


def fam_boundaries(paired):
    """a map of 8 groups: k-mers at and just below every bucket boundary first_hash(b), the smallest valid hash and the
    largest below thr; the odd groups hold a k-mer of 1100 events as well, so they leave the kernel and the generic
    path's uniques are slotted between in-kernel groups on both sides"""
    rng = np.random.default_rng(zlib.crc32(b"boundaries%d" % paired))
    spec = [(at_or_above(lambda m: 0), 2, 0), (below(lambda m: m.thr), 2, 0)]
    for b in range(1, 8 * BPG):
        fh = (lambda b: lambda m: m.first_hash(b))(b)
        spec.append((at_or_above(fh), int(rng.integers(1, 3)), 0))
        spec.append((below(fh), int(rng.integers(1, 3)), 0))
    for g in (1, 3, 5, 7):
        spec.append((in_group(g), 1100, 100 if paired else 0))
    return structural("boundaries", paired, 8, spec, claims=dict(boundaries=8 * BPG, fallback=[1, 3, 5, 7]))


PARTS = 3


def fam_parts(paired):
    """a map of 8 groups cut into 3 parts at buckets 85 and 170: group 2 (buckets 64-95) holds 1500 events split 750 /
    750 across the bound at bucket 85, each part's share within its slot; group 3, inside the middle part (g0 = 2),
    1024 distinct k-mers; group 4 slot + 1 events"""
    rng = np.random.default_rng(zlib.crc32(b"parts%d" % paired))
    spec = []
    for _ in range(750):
        spec.append((in_bucket(int(rng.integers(64, 85))), 1, 0))
        spec.append((in_bucket(int(rng.integers(85, 96))), 1, 0))
    spec += [(in_group(3), 1, 0) for _ in range(TABLE)]
    spec += _light(rng, 4, SLOT + 1) + _light(rng, 0, 300) + _light(rng, 6, 300)
    return structural("parts", paired, 8, spec,
                      claims=dict(parts=PARTS, split=(2, 85), full=[3], sizes={2: 1500, 3: TABLE, 4: SLOT + 1}))


# ---- mixed_full: dedup_scripts histories filling whole groups --------------------------------------------------------

def _key(rng):
    return rng.integers(0, 4, size=16, dtype=np.uint8), rng.integers(0, 4, size=16, dtype=np.uint8)


def _key_pool(rng, n, used, k=K, c=C):
    """n keys such that no 32-base key window a read interleaves from two of them (the pairs `used`) holds a survivor:
    those windows are fixed, so the clean-up could not draw them again"""
    pool = [_key(rng) for _ in range(n)]
    thr = GS.threshold(c)
    for _ in range(1000):
        bad = None
        for a, b in used:
            for t in (0, 1):
                cod = np.empty(32, dtype=np.uint8)
                cod[0::2], cod[1::2] = pool[a][t], pool[b][t]
                if bool((GS.hash64(GS.window_values(cod, k)) < np.uint64(thr)).any()):
                    bad = (a, b)
        if bad is None:
            return pool
        pool[bad[int(rng.integers(0, 2))]] = _key(rng)
    raise RuntimeError("no clean key pool")


def _retry(make):
    """make() again, at other random places, when a window fixed but for a base or two cannot be cleaned"""
    for _ in range(50):
        try:
            return make()
        except (AssertionError, RuntimeError):
            continue
    raise RuntimeError("no clean record")


def _single_keyed(w, h, A, B):
    """150 bp: A.x / B.x interleaved at bases 0-31, A.y / B.y at 75-106 (pair_kmer_single: p0 = A, p1 = B), the
    k-mer between or after them, a free base on each side"""
    def make():
        codes = w.codes(150)
        codes[0:32:2], codes[1:32:2], codes[75:107:2], codes[76:107:2] = A[0], B[0], A[1], B[1]
        s = int(w.rng.integers(33, 44)) if w.rng.random() < 0.5 else int(w.rng.integers(108, 120))
        return w.finish(codes, [(s, h)], [(0, 32), (75, 107)])
    return _retry(make)


def _mate_keyed(w, hs, x, y, short=False):
    """a mate whose first 32 bases interleave x and y, then the k-mers hs; short: 32 bp, no keys and no window"""
    if short:
        return w.record(32, [])

    def make():
        codes = w.codes(150)
        codes[0:32:2], codes[1:32:2] = x, y
        s0 = int(w.rng.integers(33, 70))
        return w.finish(codes, [(s0 + i * SPACING, h) for i, h in enumerate(hs)], [(0, 32)])
    return _retry(make)


def _fill_group(rng, total, draw, size):
    """scripts from draw() until they hold exactly `total` events (size(script) events each)"""
    out, n = [], 0
    while n < total:
        sc = draw(total - n)
        out.append(sc)
        n += size(sc)
    assert n == total
    return out


def _single_script(rng, left):
    fam = ("quick", "cut", "warp")[int(rng.integers(0, 3))]
    nk, ev = D.FAMILIES[fam](rng)
    if len(ev) > left:
        nk, ev = 3, [None if rng.random() < 0.15 else (int(rng.integers(0, 3)), int(rng.integers(0, 3)))
                     for _ in range(min(left, 4))]
    return nk, ev


def _script_on(rng, path):
    """a dedup_scripts history of the family `path` that takes that path (key indices stand for distinct keys)"""
    while True:
        nk, ev = D.FAMILIES[path](rng)
        if D.device_path(ev) == path:
            return nk, ev


_PAIR_SLOTS = {"m1": 1, "m2": 1, "both": 2, "m2_twice": 2, "short_mate": 1}


def _pair_script(rng, left):
    n = int(rng.integers(1, 9)) if rng.random() < 0.8 else int(rng.integers(9, 41))
    pool = 3 if n <= 8 else 5
    ev, used = [], 0
    while used < min(n, left):
        place = D.PLACES[int(rng.integers(0, len(D.PLACES)))]
        if used + _PAIR_SLOTS[place] > left:
            place = "m1"
        a = int(rng.integers(0, pool))
        ev.append((a, a if rng.random() < 1 / 6 else int(rng.integers(0, pool)), place))
        used += _PAIR_SLOTS[place]
    return pool, ev


def fam_mixed_full(paired):
    """single-end: groups 0 and 1 of exactly 1024 events from quick / cut / warp histories (150 bp keyed reads, keyless
    ones 450 bp), group 2 the same kind plus one 64-step and one 32-entry history (it leaves the kernel by the replay);
    pairs: groups 0 and 1 of exactly 1024 events from histories of 1-8 and 9-40 events in every mate placement"""
    name = "mixed_full"
    w = _Writer(zlib.crc32(repr((name, paired)).encode()), K, C)
    rng = w.rng
    if not paired:
        draw, size = (lambda left: _single_script(rng, left)), (lambda sc: len(sc[1]))
        groups = {g: _fill_group(rng, TABLE, draw, size) for g in (0, 1)}
        groups[2] = [_script_on(rng, "steps"), _script_on(rng, "set")] + _fill_group(rng, 300, draw, size)
        n_rec = sum(len(sc[1]) for v in groups.values() for sc in v)
        n_bases = sum(150 if e is not None else 450 for v in groups.values() for sc in v for e in sc[1])
        mates = 1
    else:
        groups = {g: _fill_group(rng, TABLE, lambda left: _pair_script(rng, left),
                                 lambda sc: sum(_PAIR_SLOTS[p] for _, _, p in sc[1])) for g in (0, 1)}
        n_rec = sum(len(sc[1]) for v in groups.values() for sc in v)
        n_bases = sum(150 + (32 if p == "short_mate" else 150)
                      for v in groups.values() for sc in v for _, _, p in sc[1])
        mates = 2
    want = 4
    n_fill = _plan_fill(n_bases, mates * n_rec, want, K, C, mates)
    m = Map(n_bases + FILL_LEN * n_fill, mates * (n_rec + n_fill), K, C)
    assert m.ng == want
    cr = Crafter(rng)
    scripts = []
    for g, v in groups.items():
        for nk, ev in v:
            h = cr.hash_in(*m.group_range(g))
            pool = _key_pool(rng, nk, {e[:2] for e in ev if e is not None})
            recs = []
            for e in ev:
                if not paired:
                    if e is None:
                        recs.append((w.spread([h], L=450), [h]))
                    else:
                        recs.append((_single_keyed(w, h, pool[e[0]], pool[e[1]]), [h]))
                    continue
                a, b, place = e
                A, B = pool[a], pool[b]
                if place == "short_mate":
                    s1 = rng.random() < 0.5
                    m1 = _mate_keyed(w, [] if s1 else [h], A[0], B[0], short=s1)
                    m2 = _mate_keyed(w, [h] if s1 else [], A[1], B[1], short=not s1)
                    recs.append(((m1, m2), ([] if s1 else [h], [h] if s1 else [])))
                    continue
                n1 = 1 if place in ("m1", "both") else 0
                n2 = {"m1": 0, "m2": 1, "both": 1, "m2_twice": 2}[place]
                recs.append(((_mate_keyed(w, [h] * n1, A[0], B[0]), _mate_keyed(w, [h] * n2, A[1], B[1])),
                             ([h] * n1, [h] * n2)))
            scripts.append(recs)
    merged = D._interleave_scripts(rng, scripts)
    s = Sample(name, paired, K, C, SLOT, dict(full=[0, 1], sizes={0: TABLE, 1: TABLE}))
    if not paired:
        merged = _mix(rng, merged, n_fill, lambda: (w.record(FILL_LEN, []), []))
        s.reads = [r for r, _ in merged]
    else:
        L = FILL_LEN // 2
        merged = _mix(rng, merged, n_fill, lambda: ((w.record(L, []), w.record(L, [])), ([], [])))
        s.r1 = [r[0] for r, _ in merged]
        s.r2 = [r[1] for r, _ in merged]
    s.script = [e for _, e in merged]
    assert s.map.ng == want and s.map.Mb == m.Mb
    return s


FAMILIES = ("full_distinct", "full_one_home", "one_bucket", "slot_exact", "slot_plus_one", "mixed_full", "boundaries",
            "parts")
FULL = ("full_distinct", "full_one_home", "one_bucket", "mixed_full")
SMALL_CAPS = (32, 255, 256, 257, 700)


@functools.lru_cache(maxsize=None)
def sample(name, paired, slot=SLOT):
    if name in ("slot_exact", "slot_plus_one"):
        return fam_slot(paired, slot, name == "slot_plus_one")
    assert slot == SLOT
    return {"full_distinct": fam_full_distinct, "full_one_home": fam_full_one_home, "one_bucket": fam_one_bucket,
            "mixed_full": fam_mixed_full, "boundaries": fam_boundaries, "parts": fam_parts}[name](paired)


# ---- what the oracle finds, and the model of the post-pass -----------------------------------------------------------

def oracle_survivors(s):
    """per record the sorted survivors the C oracle finds (pairs: (mate 1's, mate 2's))"""
    mk = lambda r: sorted(O.extract_markers(r, s.k, s.c, SEM).tolist())  # noqa: E731
    if s.paired:
        return [(mk(a), mk(b)) for a, b in zip(s.r1, s.r2)]
    return [mk(r) for r in s.reads]


@functools.lru_cache(maxsize=None)
def _events(s):
    """single-end: hash -> [pair keys or None] in read order; pairs: hash -> events in the slots (mate 2's events of a
    k-mer that mate 1 of the same pair holds included)"""
    if not s.paired:
        return D.kmer_events(s.reads, s.k, s.c, SEM)
    ev, skipped = D.pair_kmer_events(s.r1, s.r2, s.k, s.c, SEM)
    return {h: len(e) + skipped.get(h, 0) for h, e in ev.items()}


def group_events(s, lo=0, hi=None):
    """group of the map -> {hash: events} over the hashes in [lo, hi)"""
    hi = s.map.thr if hi is None else hi
    out = {}
    for h, e in _events(s).items():
        if lo <= h < hi:
            out.setdefault(s.map.group(h), {})[h] = e if isinstance(e, int) else len(e)
    return out


def stays(s, g_events, slot, no_dedup=False):
    """does a group with these {hash: events} stay in k_group_dedup?"""
    n = sum(g_events.values())
    if n == 0 or n > slot:
        return False
    if s.paired or no_dedup:
        return True
    ev = _events(s)
    return all(D.device_path(ev[h]) in D.IN_KERNEL for h in g_events)


def post_pass(s, slot=None, no_dedup=False, parts=1):
    """The `[sample post-pass]` line of every part: [(groups, slot, overflow list, in-kernel uniques, events handed to
    the generic path)]."""
    slot = slot or s.slot
    m = s.map
    bounds = m.parts(parts) if parts > 1 else [(0, m.thr, 0, m.ng)]
    out = []
    for lo, hi, g0, ng in bounds:
        if parts > 1 and lo == hi:
            continue
        ge = group_events(s, lo, hi)
        u1 = nf = ovf = 0
        for g in range(g0, g0 + ng):
            e = ge.get(g, {})
            n = sum(e.values())
            ovf += max(0, n - slot)
            if stays(s, e, slot, no_dedup):
                u1 += len(e)
            else:
                nf += n
        assert set(ge) <= set(range(g0, g0 + ng))
        out.append((ng, slot, ovf, u1, nf))
    return out


def probe(hashes, order):
    """k_group_dedup's table filled in this order: (slot of every hash, longest probe, a probe passed slot 1023)"""
    ht = [None] * TABLE
    at, longest, wrapped = {}, 0, False
    for i in order:
        h = hashes[i]
        sl, d = home(h), 0
        while ht[sl] is not None and ht[sl] != h:
            sl = (sl + 1) % TABLE
            d += 1
        ht[sl] = h
        at[h] = sl
        longest = max(longest, d)
        wrapped = wrapped or sl < home(h)
    return at, longest, wrapped


def pyref_counts(s):
    """oracle/pyref.py's sketch of the sample: {hash: count}"""
    if s.paired:
        return R.sketch_read_pairs(s.r1, s.r2, s.k, s.c)[0]
    return R.sketch_reads(s.reads, s.k, s.c)[0]
