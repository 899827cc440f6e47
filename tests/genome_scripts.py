"""Scripted genome batches for the genome post-pass (a test helper module, not a conftest).

A genome sketch (src/sketch.rs:550-622) depends only on the (contig, pos, hash) list of a genome's FracMinHash
survivors: hashes seen twice are dropped, the rest go through the greedy min-spacing walk.  Random genomes reach the
common cases only.  Here a batch is written survivor by survivor instead: genomes -> contigs -> events, every event
a survivor at a chosen gap from the previous one, with a chosen identity:

  F()               a fresh hash
  SLOT_(s)          a fresh hash whose home slot in the duplicate table (dup_slot(h, 2 n_g), genome.cu) is s;
                    s = -1 is the genome's last slot
  LOW38(name)       a fresh hash equal to the named event's hash in bits 0-37 (so the same home slot too)
  HASH(h)           exactly the hash h (threshold edges; h >= thr(c) is no survivor)
  KMER(v)           exactly the canonical k-mer v (k = 21 threshold edges, see K21_EDGES)
  COPY(name, rc)    the named event's k-mer again, in the other orientation when rc

mm_hash64 (src/seeding.rs:4-15) is a bijection on u64 and every step inverts (unhash64), so a k-mer with a chosen
hash exists whenever the preimage is a canonical k-mer: below 4^k and below its reverse complement (1 in 8 for
k = 31).  Where the script leaves hash bits free they are drawn again until it is.  Filler between the events is
random and drawn again wherever the C oracle would see a survivor the script does not have, so a batch realises its
script exactly (Batch.scripted_survivors() == the oracle's list).  Gaps up to k overlap the previous k-mer: there, and
up to k + NEAR, the new bases are searched (about c tries for a fresh survivor) so that the new window survives and
the windows between do not.

The classifier (classify) reads the oracle's survivor list, not the script, and reports what a batch reaches: per
survivor duplicate / head / chain-kept / tracked, per genome its count, home slots, wraps and collisions, per batch
the tile counts, N, the slotted front half's capacity and the launches the post-pass must make.
"""
import functools
import zlib

import numpy as np

from oracle import oracle as O

MASK = (1 << 64) - 1
TILE = 32768            # window starts per k_seed tile (seed_kernel.cuh SEED_TILE)
SLOT = 512              # survivors per tile slot of the slotted front half (genome.cu GEN_SLOT = SEED_STAGE)
DUP_BLOCK = 256         # survivors per k_dups block (genome.cu)
SCAN_BLOCK = 1024       # survivors per k_flag_counts / k_scatter_flagged_blocks block (genome.cu)
REC_CHUNK = 256         # records per k_seed record chunk (SEED_THREADS)
SLOTTED_MIN_C = 96      # sketch_genomes_device takes the slotted front half for c >= 96
SEM = O.SEM_AVX2
K = 31
NEAR = 16               # gaps up to k + NEAR are searched whole (every window between the two survivors is checked)

# k = 21 threshold edges.  A 21-mer is below 2^42, so only rare hashes have one: a numpy search over every
# c < 2^25 of unhash64(thr(c)) and unhash64(thr(c) - 1) (about 3 s) finds 20 preimages below 2^42, seven of them
# canonical.  (c, canonical 21-mer, its hash - thr(c)): -1 survives, 0 is the first hash that does not.
K21_EDGES = ((3971953, 2064928168833, -1), (20948030, 429553872180, -1),
             (9875655, 954612156537, 0), (22580163, 984489468301, 0))

_ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
_U = np.uint64
_INV = {m: pow(m, -1, 1 << 64) for m in (1 + (1 << 31), 21, 265, 1 + (1 << 21))}


def threshold(c):
    return MASK // c   # src/seeding.rs:108: a window survives when hash < threshold


def hash64(x):
    """mm_hash64 on a uint64 array (wrapping arithmetic)."""
    x = np.array(x, dtype=np.uint64, ndmin=1)
    x = ~(x + (x << _U(21)))
    x ^= x >> _U(24)
    x = x + (x << _U(3)) + (x << _U(8))
    x ^= x >> _U(14)
    x = x + (x << _U(2)) + (x << _U(4))
    x ^= x >> _U(28)
    return x + (x << _U(31))


def unhash64(h):
    """The inverse of mm_hash64, step by step: odd multipliers invert mod 2^64, x ^= x >> s inverts by xoring every
    further shift by s."""
    x = np.array(h, dtype=np.uint64, ndmin=1)
    x = x * _U(_INV[1 + (1 << 31)])
    x ^= (x >> _U(28)) ^ (x >> _U(56))
    x = x * _U(_INV[21])
    x ^= (x >> _U(14)) ^ (x >> _U(28)) ^ (x >> _U(42)) ^ (x >> _U(56))
    x = x * _U(_INV[265])
    x ^= (x >> _U(24)) ^ (x >> _U(48))
    return ~x * _U(_INV[1 + (1 << 21)])


def revcomp_value(v, k):
    v = np.array(v, dtype=np.uint64, ndmin=1)
    r = np.zeros_like(v)
    for j in range(k):
        r = (r << _U(2)) | (_U(3) - ((v >> _U(2 * j)) & _U(3)))
    return r


def is_canonical(v, k):
    v = np.array(v, dtype=np.uint64, ndmin=1)
    return (v < _U(1 << (2 * k))) & (v < revcomp_value(v, k))


def codes_of(v, k):
    """Canonical k-mer value -> its 2-bit codes, first base first."""
    return np.array([(int(v) >> (2 * (k - 1 - j))) & 3 for j in range(k)], dtype=np.uint8)


def window_values(codes, k):
    """Canonical k-mer of every window of a 2-bit code array (last axis)."""
    n = codes.shape[-1] - k + 1
    f = np.zeros(codes.shape[:-1] + (max(n, 0),), dtype=np.uint64)
    r = np.zeros_like(f)
    if n <= 0:
        return f
    for t in range(k):
        c = codes[..., t:t + n].astype(np.uint64)
        f = (f << _U(2)) | c
        r |= (_U(3) - c) << _U(2 * t)
    return np.minimum(f, r)


def dup_slot(h, size):
    """genome.cu dup_slot: bits 6-37 of the hash scaled to [0, size)."""
    return (((int(h) >> 6) & 0xFFFFFFFF) * size) >> 32


def valid_starts(L, k):
    """Window starts the AVX2 positions variant emits (src/avx2_seeding.rs: L >= 2k, start < 4 floor((L-k+1)/4))."""
    return 0 if L < 2 * k else 4 * ((L - k + 1) // 4)


def lost_cap(n_bases, c):
    """Survivors the compact arrays of the slotted front half hold (genome.cu genomes_slotted)."""
    return min(((n_bases + TILE - 1) // TILE) * SLOT, n_bases // c + n_bases // (4 * c) + 65536)


def sorted_cap(n_bases, c):
    """First survivor buffer of the sorted front half (genome.cu genomes_sorted)."""
    s = n_bases // c + n_bases // (4 * c) + 65536
    return n_bases + 16 if s > n_bases else s


# ---- events --------------------------------------------------------------------------------------------------------

def F(name=None):
    return ("fresh", None, name)


def SLOT_(s, name=None):
    return ("slot", s, name)


def LOW38(src, name=None):
    return ("low38", src, name)


def HASH(h, name=None):
    return ("hash", int(h), name)


def KMER(v, name=None):
    return ("kmer", int(v), name)


def COPY(src, rc=False):
    return ("copy", (src, rc), None)


def contig(events, tail=0):
    """events: [(gap, ident)]; the first gap is the first survivor's position (end index, >= k-1)."""
    return dict(ev=list(events), tail=int(tail))


def filler(L):
    """A contig without survivors."""
    return dict(ev=[], tail=int(L))


class Batch:
    """contigs (bytes), contig_off, genome_off, and the scripted survivors of every contig [(pos, hash)]."""

    def __init__(self, name, k, c, contigs, genome_off, expect, c_hash):
        self.name, self.k, self.c, self.c_hash = name, k, c, c_hash
        self.contigs = contigs
        self.genome_off = np.asarray(genome_off, dtype=np.uint64)
        self.expect = expect
        self.contig_off = np.zeros(len(contigs) + 1, dtype=np.uint64)
        self.contig_off[1:] = np.cumsum([len(s) for s in contigs])
        self.buf = np.frombuffer(b"".join(contigs), dtype=np.uint8).copy()

    @property
    def n_bases(self):
        return len(self.buf)

    def genome_contigs(self, g):
        return range(int(self.genome_off[g]), int(self.genome_off[g + 1]))

    def oracle_survivors(self, c=None):
        """[(contig, pos, hash)] of the whole batch from the C oracle, in (contig, pos) order."""
        out = []
        for ci, s in enumerate(self.contigs):
            pos, h = O.extract_markers_positions(s, self.k, c or self.c, SEM)
            out += [(ci, int(p), int(x)) for p, x in sorted(zip(pos.tolist(), h.tolist()))]
        return out

    def scripted_survivors(self):
        return [(ci, p, h) for ci, e in enumerate(self.expect) for p, h in e]


class _Builder:
    def __init__(self, seed, k, c, c_hash):
        self.rng = np.random.default_rng(seed)
        self.k, self.c = k, c
        self.thr = threshold(c)              # stray-free at c
        self.thr_hash = threshold(c_hash)    # crafted and fresh hashes are below this one
        self.named = {}                      # name -> (canonical value, placed codes, hash)
        self.used = set()
        self._pool = []

    def _draw_hashes(self, n, fixed_mask=0, fixed_bits=0):
        """n hashes below thr_hash with fixed_bits on fixed_mask (low bits only), the rest uniform."""
        h = self.rng.integers(0, self.thr_hash, size=n, dtype=np.uint64, endpoint=False)
        h = (h & ~_U(fixed_mask)) | _U(fixed_bits)
        return h[h < _U(self.thr_hash)]

    def _craft(self, fixed_mask=0, fixed_bits=0):
        """A canonical k-mer whose hash is below thr_hash, matches fixed_bits on fixed_mask and is unused."""
        if fixed_mask == 0:   # fresh hashes come from a pool, drawn and inverted 65536 at a time
            while True:
                while not self._pool:
                    h = self._draw_hashes(1 << 16)
                    v = unhash64(h)
                    ok = is_canonical(v, self.k)
                    self._pool = list(zip(v[ok].tolist(), h[ok].tolist()))[::-1]
                v, h = self._pool.pop()
                if h not in self.used:
                    return v, h
        for _ in range(10000):
            h = self._draw_hashes(256, fixed_mask, fixed_bits)
            v = unhash64(h)
            ok = is_canonical(v, self.k)
            for hv, vv in zip(h[ok].tolist(), v[ok].tolist()):
                if hv not in self.used:
                    return vv, hv
        raise RuntimeError("no canonical preimage found")

    def _orient(self, v, rc=None):
        cod = codes_of(v, self.k)
        if rc is None:
            rc = self.rng.random() < 0.5
        return (3 - cod[::-1]) if rc else cod

    def _search(self, codes, p, gap):
        """A fresh survivor ending at p, the gap bases after the previous survivor all new: the window at p survives and
        the windows between the two do not.  gap None: a k-mer of k new bases (the first of a contig, k = 21)."""
        k = self.k
        nf = k if gap is None else gap
        pre = codes[p - gap - k + 2:p - gap + 1] if gap is not None else np.zeros(0, dtype=np.uint8)
        n = 2048
        for _ in range(4000):
            cand = self.rng.integers(0, 4, size=(n, nf), dtype=np.uint8)
            full = np.concatenate([np.broadcast_to(pre, (n, len(pre))), cand], axis=1)
            h = hash64(window_values(full, k).ravel()).reshape(n, -1)
            ok = (h[:, -1] < _U(self.thr_hash)) & np.all(h[:, :-1] >= _U(self.thr), axis=1)
            for i in np.nonzero(ok)[0].tolist():
                if int(h[i, -1]) not in self.used:
                    return cand[i], int(h[i, -1])
        raise RuntimeError("no survivor found for gap %s" % gap)

    def _fill(self, codes, prev, p):
        """Filler between the survivor at prev and the k-mer just placed at p such that no window between survives."""
        k = self.k
        f = p - k - prev
        pre, post = codes[prev - k + 2:prev + 1], codes[p - k + 1:p + 1]
        n = 256 if f else 1
        for _ in range(2000):
            cand = self.rng.integers(0, 4, size=(n, f), dtype=np.uint8)
            full = np.concatenate([np.broadcast_to(pre, (n, k - 1)), cand, np.broadcast_to(post, (n, k))], axis=1)
            h = hash64(window_values(full, k).ravel()).reshape(n, -1)
            ok = np.nonzero(np.all(h[:, :-1] >= _U(self.thr), axis=1))[0]
            if len(ok):
                codes[prev + 1:p - k + 1] = cand[ok[0]]
                return
        raise RuntimeError("no stray-free filler of %d bases before position %d" % (f, p))

    def genome(self, contigs):
        """-> [(contig bytes, [(pos, hash)])] for one genome."""
        k = self.k
        n_g = sum(1 for ct in contigs for _, e in ct["ev"] if not (e[0] == "hash" and e[1] >= self.thr))
        size = 2 * n_g
        out = []
        for ct in contigs:
            ev = ct["ev"]
            pos = np.cumsum([g for g, _ in ev]).tolist() if ev else []
            L = (pos[-1] + 1 + ct["tail"]) if ev else ct["tail"]
            if ev:
                assert pos[0] >= k - 1
                L = max(L, 2 * k)
                while pos[-1] - k + 1 >= valid_starts(L, k):
                    L += 1
            codes = self.rng.integers(0, 4, size=L, dtype=np.uint8)
            fixed = np.zeros(L, dtype=bool)
            expect = []
            for i, ((gap, (kind, arg, name)), p) in enumerate(zip(ev, pos)):
                near = i > 0 and gap <= k + NEAR
                if kind == "fresh" and (near or k != 31):
                    new, h = self._search(codes, p, gap if near else None)
                    codes[p - len(new) + 1:p + 1] = new
                    fixed[p - len(new) + 1:p + 1] = True
                    v = int(window_values(codes[p - k + 1:p + 1], k)[0])
                else:
                    assert i == 0 or gap >= k, "a fixed k-mer cannot overlap the previous one"
                    if kind == "fresh":
                        v, h = self._craft()
                    elif kind == "slot":
                        s = arg % size   # bits 6-37 in [ceil(s 2^32 / size), ceil((s + 1) 2^32 / size))
                        m = int(self.rng.integers(-(-(s << 32) // size), -(-((s + 1) << 32) // size)))
                        v, h = self._craft(((1 << 32) - 1) << 6, m << 6)
                        assert dup_slot(h, size) == s
                    elif kind == "low38":
                        src = self.named[arg][2]
                        v, h = self._craft((1 << 38) - 1, src & ((1 << 38) - 1))
                    elif kind == "hash":
                        h = arg
                        v = int(unhash64(h)[0])
                        assert bool(is_canonical(v, k)[0]), "hash %x has no canonical %d-mer" % (h, k)
                    elif kind == "kmer":
                        v, h = arg, int(hash64(arg)[0])
                        assert bool(is_canonical(v, k)[0])
                    else:
                        sv, scodes, h = self.named[arg[0]]
                        v = sv
                    if kind == "copy":
                        cod = (3 - scodes[::-1]) if arg[1] else scodes
                    else:
                        cod = self._orient(v)
                    codes[p - k + 1:p + 1] = cod
                    fixed[p - k + 1:p + 1] = True
                    if near:
                        self._fill(codes, pos[i - 1], p)
                        fixed[pos[i - 1] + 1:p + 1] = True
                self.used.add(h)
                if name is not None:
                    self.named[name] = (v, codes[p - k + 1:p + 1].copy(), h)
                if h < self.thr:
                    expect.append((p, h))
            self._clean(codes, fixed, {p for p, _ in expect})
            s = _ACGT[codes].tobytes()
            out.append((s, expect))
        return out

    def _clean(self, codes, fixed, keep):
        """Draw the free bases of every window that survives at c without being scripted again, until none is left."""
        k = self.k
        nv = valid_starts(len(codes), k)
        for _ in range(200):
            if nv == 0:
                return
            h = hash64(window_values(codes[:nv + k - 1], k))
            surv = (np.nonzero(h < _U(self.thr))[0] + (k - 1)).tolist()
            stray = [p for p in surv if p not in keep]
            assert keep <= set(surv), "a scripted survivor is gone"
            if not stray:
                return
            for p in stray:
                free = ~fixed[p - k + 1:p + 1]
                assert free.any(), "stray window at %d has no free base" % p
                seg = codes[p - k + 1:p + 1]
                seg[free] = self.rng.integers(0, 4, size=int(free.sum()), dtype=np.uint8)
        raise RuntimeError("filler did not converge")


def build(name, genomes, k=K, c=200, c_hash=None, seed=0):
    """genomes: [[contig(...) | filler(L)]] -> Batch, stray-free at c, every crafted hash below thr(c_hash)."""
    b = _Builder(zlib.crc32(repr((name, k, c, seed)).encode()), k, c, c_hash or c)
    contigs, expect, goff = [], [], [0]
    for g in genomes:
        for s, e in b.genome(g):
            contigs.append(s)
            expect.append(e)
        goff.append(len(contigs))
    return Batch(name, k, c, contigs, goff, expect, c_hash or c)


# ---- families ------------------------------------------------------------------------------------------------------
GAPS = (7, 8, 10, 12, 15, 20, 25, 29, 30, 31, 32, 35, 40, 45, 60, 64, 69, 70, 71, 72, 90)
SPACINGS = (0, 30, 70, 1 << 20)   # min_spacing values the spacing family runs at; the last exceeds every contig


def _chain(rng, n, lead, tail):
    ev = [(int(lead), F())] + [(int(rng.choice(GAPS)), F()) for _ in range(n)]
    return contig(ev, tail)


def fam_spacing(rng):
    """Chains of closely spaced survivors (gaps of ms and ms + 1 for ms = 30 and 70, kept / tracked / chain-kept
    runs), sparse enough that no tile passes its slot; one cluster of 1201 survivors 64-70 bases apart (a single
    cluster at ms = 70) across two seeding tiles, several k_dups blocks and two scan blocks."""
    big = contig([(40, F())] + [(int(rng.integers(64, 71)), F()) for _ in range(1200)], 60)
    g0 = [big] + [_chain(rng, int(rng.integers(8, 20)), rng.integers(31, 400), rng.integers(900, 1400)) for _ in range(20)]
    g1 = [_chain(rng, int(rng.integers(8, 20)), rng.integers(31, 400), rng.integers(900, 1400)) for _ in range(12)]
    return [g0, g1]


def fam_dups(rng):
    """Duplicates around the spacing walk (ms = 30): between a head and its follower, the only survivor within ms
    before a k-mer (which is then a head), reverse-complement copies, 2 / 3 / 5 occurrences, copies in two contigs of
    one genome, the same hash once in each of two adjacent genomes, a genome made only of duplicates.  The whole batch
    is one k_dups block, most of it in the first genome."""
    g0 = [
        contig([(100, F()), (15, F("d1")), (10, F()), (40, F()), (36, F("d2")), (20, F()), (60, COPY("d1", True)),
                (45, F()), (40, COPY("d2")), (12, F()), (50, F("t3")), (40, F("f5")), (70, COPY("t3", True)), (8, F())],
               300),
        contig([(200, COPY("t3")), (40, COPY("f5", True)), (20, F()), (50, COPY("f5")), (33, F()), (40, F()),
                (36, COPY("f5", True)), (15, F()), (70, COPY("f5"))], 200),
    ]
    g0 += [_chain(rng, 12, rng.integers(31, 300), 800) for _ in range(7)]
    g1 = [contig([(90, F()), (50, F()), (60, F("y"))], 100)]
    g2 = [contig([(80, COPY("y", True)), (40, F()), (35, F())], 100)]
    g3 = [contig([(100, F("p")), (40, F("q")), (40, COPY("p", True)), (40, F("r")), (40, COPY("q"))], 50),
          contig([(60, COPY("r", True)), (45, COPY("p"))], 80)]
    g4 = [contig([(70, F()), (20, F())], 100)]
    return [g0, g1, g2, g3, g4]


def fam_table(rng):
    """The duplicate table: genomes of 1, 2 and 3 survivors; two distinct hashes homed at a genome's last slot (the
    second one's probe wraps to slot 0), in genomes of 1-3 survivors and of 40; distinct hashes sharing a home slot,
    one of them duplicated; distinct hashes equal in bits 0-37."""
    gs = []
    for n in (1, 2, 3):
        gs.append([contig([(50, F())] + [(int(rng.integers(40, 90)), F()) for _ in range(n - 1)], 60)])
    gs.append([contig([(50, SLOT_(-1)), (60, SLOT_(-1))], 60)])
    gs.append([contig([(50, SLOT_(-1)), (60, F()), (45, SLOT_(-1))], 60)])
    gs.append([contig([(40, SLOT_(-1))] + [(int(rng.integers(35, 90)), F()) for _ in range(38)] + [(50, SLOT_(-1))], 80)])
    gs.append([contig([(40, SLOT_(7, "s7")), (50, SLOT_(7)), (50, F()), (60, COPY("s7", True)), (40, SLOT_(7)),
                       (45, SLOT_(8)), (50, SLOT_(6))] + [(int(rng.integers(35, 90)), F()) for _ in range(5)], 80)])
    gs.append([contig([(40, F("a")), (50, LOW38("a")), (45, F("b")), (50, LOW38("b")), (60, LOW38("b"))]
                      + [(int(rng.integers(35, 90)), F()) for _ in range(6)], 80),
               contig([(35, LOW38("a")), (50, F())], 40)])
    return gs


def fam_bounds(rng):
    """Contig and genome boundaries (ms = 30): a contig whose first survivor lies 0-30 above the previous contig's
    last one; empty contigs and contigs shorter than 2k between survivors; genomes starting at survivor index 255,
    256, 257 and 1023, 1024, 1025; leading, middle and trailing empty genomes, and genomes without contigs; more
    than 256 records in one seeding tile.  Stray-free at c = 95 with every hash below thr(96), so that c = 95 and c = 96 (one
    on each side of the slotted front half) see the same survivors."""
    gs = [[filler(300)], []]

    def body(n, lead=60):   # about 60-110 bases apart: no tile past its slot at c = 96
        return contig([(lead, F())] + [(int(rng.choice(GAPS[8:])) if rng.random() < 0.2 else int(rng.integers(60, 111)), F())
                                       for _ in range(n - 1)], 200)
    # genome starts 255, 256, 257: 255 survivors, then one, then one
    gs.append([body(100), filler(40), body(80), filler(10), filler(0), body(75)])
    gs.append([body(1)])
    gs.append([body(1), filler(61)])
    # contig boundaries: next contig's first survivor 0, 10, 30 and 31 above the previous contig's last one
    close = []
    last = 0
    for d in (0, 10, 30, 31, -5, 1):
        ev = [(last + d if last else 200, F())] + [(int(rng.choice(GAPS[8:])), F()) for _ in range(3)]
        close.append(contig(ev, 100))
        last = sum(g for g, _ in ev)
    gs.append(close + [filler(50)])
    gs.append([filler(20), filler(100)])   # middle empty genome
    # up to index 1023: the survivors so far are counted in classify; pad with one genome, then 1, 1
    gs.append(["pad1023"])
    gs.append([body(1)])
    gs.append([body(1)])
    # 700 short records (at most two tiles, so one tile holds more than 256: several k_seed record chunks)
    many = []
    for i in range(700):
        if i % 3 == 0:
            many.append(contig([(int(rng.integers(30, 40)), F())], int(rng.integers(0, 10))))
        else:
            many.append(filler(int(rng.integers(1, 70))))
    gs.append(many)
    gs.append([filler(10)])                # trailing empty genomes
    gs.append([])
    return gs


def fam_slot(rng, n):
    """One tile (window starts 0 .. 32767) with exactly n survivors, the next tile with 300 (c = 200)."""
    gap = TILE // n
    a = contig([(30 + 10, F())] + [(gap, F()) for _ in range(n - 1)], 0)
    # pad the contig to the tile edge, then the next tile's survivors in a second genome
    last_start = 10 + (n - 1) * gap
    a["tail"] = TILE - last_start - 1
    b = contig([(40, F())] + [(100, F()) for _ in range(299)], 500)
    return [[a], [b]]


CAP_TILES = 160          # 5.24 Mbp
CAP_C = 1000


def fam_cap(rng, extra):
    """N == cap (extra = 0) or cap + 1 (extra = 1) survivors at c = 1000 in 160 contigs of one tile each, no tile
    over its slot: about 451 survivors per tile, 60-72 bases apart."""
    cap = lost_cap(CAP_TILES * TILE, CAP_C)
    n = cap + extra
    per = [n // CAP_TILES + (1 if t < n % CAP_TILES else 0) for t in range(CAP_TILES)]
    gs = []
    for t in range(CAP_TILES):
        gaps = rng.integers(60, 73, size=per[t] - 1)
        while 40 + int(gaps.sum()) > TILE - 64:
            gaps = np.maximum(gaps - 1, 60)
        ev = [(40, F())] + [(int(x), F()) for x in gaps]
        ct = contig(ev, 0)
        ct["tail"] = TILE - 1 - (40 + int(gaps.sum()))
        gs.append(ct)
    return [gs[:80], gs[80:]]


# ---- threshold edges -----------------------------------------------------------------------------------------------
EDGE_W = (24, 30, 32)    # k_seed run lengths
EDGE_C31 = 200


def edge_hashes(c, rng):
    """(hash, survives, label) for k = 31 at c: thr - 1, thr, high word == thr_hi with the low word below / above
    thr_lo, and a high word of thr_hi + 1 (never a candidate)."""
    thr = threshold(c)
    hi, lo = thr >> 32, thr & 0xFFFFFFFF

    def with_canonical(make):
        for _ in range(100000):
            h = make()
            if bool(is_canonical(unhash64(h)[0], 31)[0]):
                return h
        raise RuntimeError
    return [(thr - 1, True, "thr-1"), (thr, False, "thr"),
            (with_canonical(lambda: (hi << 32) | int(rng.integers(0, lo))), True, "hi=thr_hi,lo<thr_lo"),
            (with_canonical(lambda: (hi << 32) | int(rng.integers(lo + 1, 1 << 32))), False, "hi=thr_hi,lo>thr_lo"),
            (with_canonical(lambda: ((hi + 1) << 32) | int(rng.integers(0, 1 << 32))), False, "hi=thr_hi+1")]


def record_length(k, W):
    """Record length whose valid window count makes k_seed pick run length W (seed.cu pick_run_length): 48, 60 and
    64 windows for W = 24, 30, 32."""
    return {24: 48, 30: 60, 32: 64}[W] + k - 1


def edge_batch(k, W, c=None, seed=0):
    """One record per (edge k-mer, window start 0 .. W-1), every record its own genome; records of equal length so
    that k_seed runs at W and each record's first run starts at its first window (records inside a tile).  k = 31:
    the five edge_hashes at c = 200; k = 21: the pinned K21_EDGES k-mer of c."""
    rng = np.random.default_rng(zlib.crc32(repr(("edge", k, W, c, seed)).encode()))
    if k == 31:
        c = EDGE_C31
        edges = [(HASH(h), ok, lab) for h, ok, lab in edge_hashes(c, rng)]
    else:
        e = [x for x in K21_EDGES if x[0] == c][0]
        edges = [(KMER(e[1]), e[2] == -1, "thr%d" % e[2])]
    L = record_length(k, W)
    genomes, labels = [], []
    for ident, ok, lab in edges:
        for o in range(W):
            ct = contig([(o + k - 1, ident)], 0)
            ct["tail"] = L - (o + k)
            genomes.append([ct])
            labels.append((lab, ok, o))
    b = build("edge%d_%d" % (k, W), genomes, k=k, c=c, seed=seed)
    b.labels = labels
    assert all(len(s) == L for s in b.contigs)
    return b


# ---- the batches ---------------------------------------------------------------------------------------------------

def _pad_bounds(genomes, rng):
    """Replace the "pad1023" genome of the bounds family by one whose survivors bring the next genome's start to 1023."""
    before = 0
    for g in genomes:
        if g == ["pad1023"]:
            break
        before += sum(1 for ct in g for _, e in ct["ev"])
    need = 1023 - before
    assert need > 0
    ev = [(60, F())] + [(int(rng.integers(60, 111)), F()) for _ in range(need - 1)]
    return [g if g != ["pad1023"] else [contig(ev, 100)] for g in genomes]


FAMILIES = ("spacing", "dups", "table", "bounds", "slot512", "slot513", "cap", "cap1")
SMALL = ("spacing", "dups", "table", "bounds", "slot512", "slot513")   # pyref is fast enough for these
MS = {"spacing": SPACINGS, "dups": (30,), "table": (30,), "bounds": (30,), "slot512": (30,), "slot513": (30,),
      "cap": (30,), "cap1": (30,)}


@functools.lru_cache(maxsize=None)
def batch(name, seed=0):
    rng = np.random.default_rng(zlib.crc32(repr(("family", name, seed)).encode()))
    if name == "spacing":
        return build(name, fam_spacing(rng), seed=seed)
    if name == "dups":
        return build(name, fam_dups(rng), seed=seed)
    if name == "table":
        return build(name, fam_table(rng), seed=seed)
    if name == "bounds":
        return build(name, _pad_bounds(fam_bounds(rng), rng), c=95, c_hash=96, seed=seed)
    if name in ("slot512", "slot513"):
        return build(name, fam_slot(rng, int(name[4:])), seed=seed)
    if name in ("cap", "cap1"):
        return build(name, fam_cap(rng, 1 if name == "cap1" else 0), c=CAP_C, seed=seed)
    raise KeyError(name)


# ---- the rule, transcribed, and the classifier ---------------------------------------------------------------------

def sketch_from_survivors(sv, min_spacing, pseudotax=True):
    """src/sketch.rs:590-614 over one genome's (contig, pos, hash) survivors -> (kept, tracked)."""
    vec = sorted(sv)
    seen, dup = set(), set()
    for _, _, h in vec:
        if h in seen:
            dup.add(h)
        seen.add(h)
    kept, tracked = [], []
    last_pos, last_contig = 0, 0
    for ci, p, h in vec:
        if h in dup:
            continue
        if last_pos == 0 or last_contig != ci or p - last_pos > min_spacing:
            kept.append(h)
            last_contig, last_pos = ci, p
        elif pseudotax:
            tracked.append(h)
    return kept, tracked


def launches(n_bases, c, N, max_tile, force_sort, n_contigs=1, n_genomes=1):
    """(seed launches, genome_post launches) of one sketch_genomes call (genome.cu sketch_genomes_device)."""
    retry = N > sorted_cap(n_bases, c)
    if not force_sort and c >= SLOTTED_MIN_C and n_bases and n_contigs and n_genomes:
        if max_tile <= SLOT and N <= lost_cap(n_bases, c):
            return 1, 1
        return 2 + retry, 2
    return 1 + retry, 1


def classify(b, min_spacing, c=None, individual=False):
    """What batch b reaches at min_spacing, from the oracle's survivor list (at c, default b.c)."""
    c = c or b.c
    k = b.k
    sv = b.oracle_survivors(c)
    goff = np.arange(len(b.contigs) + 1) if individual else b.genome_off
    n_genomes = len(goff) - 1
    g_of_contig = np.repeat(np.arange(n_genomes), np.diff(goff.astype(np.int64)))
    per_genome = [[] for _ in range(n_genomes)]
    for ci, p, h in sv:
        per_genome[int(g_of_contig[ci])].append((ci, p, h))
    cls = dict.fromkeys(("survivors", "dup", "dup_rc", "dup_2", "dup_3", "dup_5", "dup_two_contigs", "head", "chain_kept",
                         "tracked", "gap_eq_ms", "gap_eq_ms1", "head_past_dup", "dup_inside_chain", "contig_close",
                         "adjacent_genome_pair", "all_dup_genome", "empty_genome", "zero_contig_genome", "wrap",
                         "slot_collision", "slot_collision_dup", "low38_pair"), 0)
    kept, tracked, counts, starts = [], [], [], []
    idx = 0
    prev_hashes = set()
    for g, gsv in enumerate(per_genome):
        starts.append(idx)
        idx += len(gsv)
        counts.append(len(gsv))
        cls["survivors"] += len(gsv)
        if not gsv:
            cls["empty_genome"] += 1
            cls["zero_contig_genome"] += int(goff[g] == goff[g + 1])
        occ = {}
        for ci, p, h in gsv:
            occ.setdefault(h, []).append((ci, p))
        hashes = {h for _, _, h in gsv}
        cls["adjacent_genome_pair"] += sum(1 for h in hashes & prev_hashes if len(occ[h]) == 1)
        prev_hashes = {h for h in hashes if len(occ[h]) == 1}
        if gsv and all(len(v) > 1 for v in occ.values()):
            cls["all_dup_genome"] += 1
        for h, o in occ.items():
            if len(o) > 1:
                cls["dup"] += len(o)
                if len(o) in (2, 3, 5):
                    cls["dup_%d" % len(o)] += 1
                cls["dup_two_contigs"] += len({ci for ci, _ in o}) > 1
                fw = set()
                for ci, p in o:
                    s = b.contigs[ci]
                    cod = np.frombuffer(s[p - k + 1:p + 1], dtype=np.uint8)
                    cod = np.searchsorted(_ACGT, cod).astype(np.uint8)
                    fv = 0
                    for x in cod.tolist():
                        fv = (fv << 2) | x
                    fw.add(int(window_values(cod, k)[0]) == fv)
                cls["dup_rc"] += len(fw) == 2
        # the walk, with the reason for every state
        last_p = None          # last kept survivor's position (the walk restarts at every head)
        prev = None            # previous non-duplicate survivor (ci, p) of the genome
        prev_any = None        # previous survivor, duplicate or not
        for ci, p, h in gsv:
            dup = len(occ[h]) > 1
            if dup:
                if prev is not None and prev[0] == ci and p - prev[1] <= min_spacing:
                    cls["dup_inside_chain"] += 1
                prev_any = (ci, p, True)
                continue
            if prev is not None and prev[0] != ci and 0 <= p - prev[1] <= min_spacing:
                cls["contig_close"] += 1
            same = prev is not None and prev[0] == ci
            gap = p - prev[1] if same else None
            if gap == min_spacing:
                cls["gap_eq_ms"] += 1
            if gap == min_spacing + 1:
                cls["gap_eq_ms1"] += 1
            head = not same or gap > min_spacing
            if head and prev_any is not None and prev_any[2] and prev_any[0] == ci and p - prev_any[1] <= min_spacing:
                cls["head_past_dup"] += 1
            if head:
                cls["head"] += 1
                last_p = p
            elif p - last_p > min_spacing:
                cls["chain_kept"] += 1
                last_p = p
            else:
                cls["tracked"] += 1
            prev = (ci, p)
            prev_any = (ci, p, False)
        km, tr = sketch_from_survivors(gsv, min_spacing)
        kept.append(km)
        tracked.append(tr)
        # the duplicate table of this genome
        size = 2 * len(gsv)
        homes = {}
        for h in hashes:
            homes.setdefault(dup_slot(h, size), []).append(h)
        cls["wrap"] += len(homes.get(size - 1, [])) >= 2
        for s, hs in homes.items():
            if len(hs) >= 2:
                cls["slot_collision"] += 1
                cls["slot_collision_dup"] += any(len(occ[h]) > 1 for h in hs)
                lows = [h & ((1 << 38) - 1) for h in hs]
                cls["low38_pair"] += len(lows) - len(set(lows))
    # tiles, in flat window-start coordinates
    n_tiles = (b.n_bases + TILE - 1) // TILE
    tiles = np.zeros(max(n_tiles, 1), dtype=np.int64)
    for ci, p, _ in sv:
        tiles[(int(b.contig_off[ci]) + p - (k - 1)) // TILE] += 1
    recs = np.zeros(max(n_tiles, 1), dtype=np.int64)
    for ci in range(len(b.contigs)):
        a, e = int(b.contig_off[ci]), int(b.contig_off[ci + 1])
        if e > a:
            recs[a // TILE:(e - 1) // TILE + 1] += 1
    N, mt = len(sv), int(tiles.max())
    return dict(classes=cls, kept=kept, tracked=tracked, counts=counts, genome_starts=starts, tiles=tiles,
                max_tile=mt, records_per_tile=int(recs.max()), N=N, cap=lost_cap(b.n_bases, c),
                launches={fs: launches(b.n_bases, c, N, mt, fs, len(b.contigs), n_genomes) for fs in (False, True)})


def oracle_sketch(b, min_spacing, pseudotax=True, individual=False, c=None):
    """The C oracle's sketch_genome of every genome of b, in the CSR form Genomes.download() returns."""
    goff = np.arange(len(b.contigs) + 1, dtype=np.uint64) if individual else b.genome_off
    km, tr, ko, to, gs = [], [], [0], [0], []
    for g in range(len(goff) - 1):
        c0, c1 = int(goff[g]), int(goff[g + 1])
        sub = (b.contig_off[c0:c1 + 1] - b.contig_off[c0]).astype(np.uint64)
        k_, t_, n = O.sketch_genome(b.buf[int(b.contig_off[c0]):int(b.contig_off[c1])], sub, k=b.k, c=c or b.c,
                                    min_spacing=min_spacing, pseudotax=pseudotax, sem=SEM)
        km.append(k_)
        tr.append(t_)
        ko.append(ko[-1] + len(k_))
        to.append(to[-1] + len(t_))
        gs.append(n)
    cat = lambda xs: np.concatenate(xs).astype(np.uint64) if xs else np.zeros(0, np.uint64)
    return dict(kmers=cat(km), kmer_off=np.array(ko, np.uint64), tracked=cat(tr), tracked_off=np.array(to, np.uint64),
                gn_size=np.array(gs, np.uint64))
