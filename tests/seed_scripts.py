"""Scripted seeding batches for k_seed (a test helper module, not a conftest).

k_seed (sylph_b200/csrc/seed_kernel.cuh) has capacity edges that random reads reach only in bulk: survivors staged per
tile (SEED_STAGE) before global atomics, candidates listed per record chunk (SEED_CAND) before inline resolves, record
chunks of SEED_THREADS records, runs of W windows with a masked last run, the TMA body against the tail loads of the
last tile, and the pair-key rule that flags an event pending.  Each batch here puts one of them exactly at N - 1, N or
N + 1, by cutting random sequence where the model below says the count reaches N.

The constants come from the kernel: tests/cpp/seed_constants.cu includes seed_kernel.cuh and prints them, so the
edges follow the kernel if its geometry changes.

The model restates k_seed's bookkeeping per tile (k_tile_first_rec's record range, the record chunks, each record's
windows inside the tile, the runs, the candidates whose hash's high word passes thr_hi, the survivors staged, the
pending flags).  It only decides which branch a batch reaches; expected outputs always come from the C oracle.
Hashes and windows are genome_scripts' (hash64, unhash64, window_values, threshold, is_canonical).
"""
import functools
import os
import subprocess
import tempfile
import zlib

import numpy as np

from tests.genome_scripts import _ACGT, hash64, is_canonical, threshold, unhash64, window_values
from tests.util import flatten

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "sylph_b200", "csrc")
U64 = 2**64 - 1
SEM_SCALAR, SEM_AVX2 = 0, 1
PAIR_MIN, PAIR_MAX = 66, 400   # reads with pair keys (src/sketch.rs:923, :627)


@functools.lru_cache(maxsize=None)
def constants():
    """seed_kernel.cuh's geometry, printed by a host program built with nvcc (and any SYL_BUILD_DEFS of the library)."""
    from sylph_b200 import build as B
    d = tempfile.mkdtemp(prefix="seed_constants_")
    exe = os.path.join(d, "seed_constants")
    subprocess.check_call([B._nvcc(), "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC]
                          + B.EXTRA_NVCC + ["-o", exe, os.path.join(REPO, "tests", "cpp", "seed_constants.cu")])
    out = subprocess.run([exe], stdout=subprocess.PIPE, text=True, check=True).stdout
    return {a: int(b) for a, b in (ln.split() for ln in out.splitlines())}


def run_lengths():
    """The run lengths k_seed is instantiated for (SEED_DEFINE_KERNELS): W_MIN, 30, W_MAX."""
    C = constants()
    return (C["SEED_W_MIN"], 30, C["SEED_W_MAX"])


def valid_windows(L, k, sem, with_pos):
    """common.cuh valid_windows: window starts the reference visits in a record of length L."""
    if L < k:
        return 0
    if sem == SEM_SCALAR:
        return L - k + 1
    if L < (2 * k if with_pos else k + 1):
        return 0
    return 4 * ((L - k + 1) // 4)


def _byte_to_seq():
    t = np.zeros(256, dtype=np.uint8)
    for chars, v in ((b"Aa", 0), (b"Cc", 1), (b"Gg", 2), (b"TtUu", 3)):
        for ch in chars:
            t[ch] = v
    t[1], t[2], t[3] = 1, 2, 3
    return t


BYTE_TO_SEQ = _byte_to_seq()   # src/types.rs:50-59


# ---- batches -------------------------------------------------------------------------------------------------------
class Batch:
    """Records (flat ASCII buffer + offsets) at k and c, the edges it claims, and the outputs it runs through.

    claims: [(label, filter(inst) -> bool, value(model, inst) -> int, expected)]; expected None: reported only.
    outputs: subset of ("emit0", "reads", "sort", "pairs", "no_dedup", "parts")."""

    def __init__(self, family, name, k, c, seqs, claims, outputs, parts=None):
        self.family, self.name, self.k, self.c = family, name, k, c
        self.buf, self.off = flatten([bytes(s) for s in seqs])
        self.claims, self.outputs, self.parts = claims, outputs, parts

    @property
    def n_bases(self):
        return len(self.buf)

    @property
    def n_rec(self):
        return len(self.off) - 1

    def __repr__(self):
        return "Batch(%s, k=%d, c=%d, %d bases, %d records)" % (self.name, self.k, self.c, self.n_bases, self.n_rec)


def insts(b):
    """Every (emit, sem, with_pos, no_dedup, paired, part) the batch runs under; the part is (lo, hi) or None."""
    out = []
    if "emit0" in b.outputs:
        out += [dict(emit=0, sem=s, with_pos=p, no_dedup=0, paired=False, part=None) for s in (0, 1) for p in (0, 1)]
    for s in (0, 1):
        if {"reads", "sort"} & set(b.outputs):
            out.append(dict(emit=1, sem=s, with_pos=0, no_dedup=0, paired=False, part=None))
        if "no_dedup" in b.outputs:
            out.append(dict(emit=1, sem=s, with_pos=0, no_dedup=1, paired=False, part=None))
        if "pairs" in b.outputs:
            out.append(dict(emit=1, sem=s, with_pos=0, no_dedup=0, paired=True, part=None))
        if "parts" in b.outputs:
            for part in part_bounds(b.n_bases, b.n_rec, b.k, b.c, b.parts):
                out.append(dict(emit=1, sem=s, with_pos=0, no_dedup=0, paired=False, part=part))
    return out


def part_bounds(n_bases, n_records, k, c, P):
    """sample_parts.hpp restated: the one-pass map and the hash bounds [lo, hi) of P parts."""
    n_exp = max(n_bases - n_records * (k - 1), 0) // c
    nbk = 32 * (n_exp // 640 + 1)
    thr = U64 // c
    mb = min((nbk << 64) // (thr + 1), U64)
    first = lambda b: 0 if b == 0 else min((((b << 64) + mb - 1) // mb), thr)  # noqa: E731
    P = min(P, nbk)
    cuts = [nbk * p // P for p in range(P + 1)]
    return [(0 if p == 0 else first(cuts[p]), thr if p == P - 1 else first(cuts[p + 1])) for p in range(P)]


# ---- the model -----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=256)
def _flat_hashes(b, k):
    """mm_hash64 of the canonical k-mer of every window start of the flat buffer (windows across records included;
    the model keeps only each record's valid ones)."""
    codes = BYTE_TO_SEQ[b.buf]
    if len(codes) < k:
        return np.zeros(0, dtype=np.uint64)
    return hash64(window_values(codes, k))


def windows(b, sem, with_pos):
    """-> (start, rec, hash) of every valid window of the batch, flat starts in record order."""
    k = b.k
    h = _flat_hashes(b, k)
    off = b.off.astype(np.int64)
    L = np.diff(off)
    nv = np.array([valid_windows(int(x), k, sem, with_pos) for x in L], dtype=np.int64)
    rec = np.repeat(np.arange(b.n_rec), nv)
    start = np.repeat(off[:-1], nv) + (np.arange(int(nv.sum())) - np.repeat(np.cumsum(nv) - nv, nv))
    return start, rec, h[start] if len(start) else np.zeros(0, np.uint64)


def survivors(b, sem, with_pos, c=None):
    """The model's survivors [(rec, pos, hash)] (pos: end index of the window, as the reference reports it)."""
    start, rec, h = windows(b, sem, with_pos)
    ok = h < np.uint64(threshold(c or b.c))
    pos = start[ok] - b.off.astype(np.int64)[rec[ok]] + (b.k - 1)
    return sorted(zip(rec[ok].tolist(), pos.tolist(), h[ok].tolist()))


def tile_rec(off, n_bases, T):
    """k_tile_first_rec: tile t starts at the last record whose offset is <= t T (upper bound - 1); tile n_tiles is
    the last record."""
    n_rec = len(off) - 1
    n_tiles = (n_bases + T - 1) // T
    pos = np.arange(n_tiles, dtype=np.uint64) * np.uint64(T)
    r = np.searchsorted(off, pos, side="right").astype(np.int64) - 1
    r = np.clip(r, 0, n_rec - 1)
    return np.concatenate([r, [n_rec - 1]])


def staging(n_bases, T):
    """Per tile (avail, nbulk) of the staging phase, ASCII bytes and 2-bit words."""
    C = constants()
    out = []
    for t in range((n_bases + T - 1) // T):
        a = min(n_bases - t * T, C["SEED_TILE"] + C["SEED_HALO"])
        w = min((n_bases + 15) // 16 - t * T // 16, C["SEED_PK_WORDS"])
        out.append(dict(ascii=(a, a & ~15), packed=(w, w & ~3)))
    return out


def model(b, W, inst):
    """What k_seed<K, EMIT, W, PACKED> does with batch b under inst, tile by tile."""
    C = constants()
    T, NT, lim = C["SEED_TILE"], C["SEED_THREADS"], C["SEED_NCHUNK16"] * 16
    k = b.k
    thr = threshold(b.c)
    lo = 0
    if inst["part"] is not None:
        lo, hi = inst["part"]
        thr = min(hi, thr)
    thr_hi = thr >> 32
    start, rec, h = windows(b, inst["sem"], inst["with_pos"])
    hh = (h >> np.uint64(32)).astype(np.uint64)
    cand = hh <= np.uint64(thr_hi)
    surv = (h < np.uint64(thr)) & (h >= np.uint64(lo))
    false = cand & (h >= np.uint64(thr))
    off = b.off.astype(np.int64)
    L = np.diff(off)
    tr = tile_rec(b.off, b.n_bases, T)
    tiles = []
    for t in range(len(tr) - 1):
        T0, T1 = t * T, (t + 1) * T
        r_lo, r_hi = int(tr[t]), int(tr[t + 1])
        in_tile = (start >= T0) & (start < T1)
        chunks = []
        for rc in range(r_lo, r_hi + 1, NT):
            re = min(rc + NT - 1, r_hi)
            m = in_tile & (rec >= rc) & (rec <= re)
            cnt = np.bincount(rec[m] - rc, minlength=re - rc + 1)
            runs = (cnt + W - 1) // W
            last = np.where(runs > 0, cnt - (runs - 1) * W, 0)
            cm = m & cand
            slots = (rec[cm] - rc).tolist()
            chunks.append(dict(records=re - rc + 1, runs=int(runs.sum()), masked=int(((last > 0) & (last < W)).sum()),
                               masked_n=sorted(set(last[(last > 0) & (last < W)].tolist())), cnt=cnt,
                               cand=int(cm.sum()), false=int((m & false).sum()), surv=int((m & surv).sum()),
                               top_slot=max(slots) if slots else -1))
        ts = in_tile & surv
        ev = dict(pend_st=0, pend_mid=0, inplace_lim=0, inplace_st0=0, no_pair=0, pend=0)
        if inst["emit"] == 1:
            for r in rec[ts].tolist():
                Lr, st = int(L[r]), int(off[r]) - T0
                has_pair = not inst["no_dedup"] and PAIR_MIN <= Lr <= PAIR_MAX
                mid = st + (Lr >> 1)
                if inst["paired"]:
                    ev["pend"] += 1
                elif not has_pair:
                    ev["no_pair"] += 1
                elif st < 0:
                    ev["pend_st"] += 1
                    ev["pend"] += 1
                elif mid + 32 > lim:
                    ev["pend_mid"] += mid + 32 == lim + 1
                    ev["pend"] += 1
                else:
                    ev["inplace_lim"] += mid + 32 == lim
                    ev["inplace_st0"] += st == 0
        tiles.append(dict(tile=t, r_lo=r_lo, r_hi=r_hi, records=r_hi - r_lo + 1, chunks=chunks, staged=int(ts.sum()),
                          cand=int((in_tile & cand).sum()), events=ev))
    return tiles


# ---- builders ------------------------------------------------------------------------------------------------------
def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def _ascii(codes):
    return _ACGT[np.asarray(codes, dtype=np.uint8)].tobytes()


def _flags(codes, k, thr, what):
    h = hash64(window_values(np.asarray(codes, dtype=np.uint8), k))
    return ((h >> np.uint64(32)) <= np.uint64(thr >> 32)) if what == "cand" else (h < np.uint64(thr))


def cut_record(rng, k, thr, n, what):
    """Random codes of a record with exactly n windows flagged `what` ("cand": high word <= thr_hi, "surv": hash < thr),
    the n-th in its last window group, and a window count that is a multiple of 4 with length >= 2k, so that every
    window rule (scalar, AVX2, with and without positions) sees the same windows."""
    c = max(1, U64 // thr)
    codes = rng.integers(0, 4, size=int(n * c * 1.4) + 4 * k + 64, dtype=np.uint8)
    f = _flags(codes, k, thr, what)
    while f.sum() < n:
        codes = np.concatenate([codes, rng.integers(0, 4, size=len(codes) // 2, dtype=np.uint8)])
        f = _flags(codes, k, thr, what)
    i = int(np.nonzero(f)[0][n - 1])
    m = max(-(-(i + 1) // 4) * 4, k + 4)
    for _ in range(10000):
        if m <= len(f) and not f[i + 1:m].any():
            return codes[:m + k - 1]
        codes[i + k:] = rng.integers(0, 4, size=len(codes) - i - k, dtype=np.uint8)
        f = _flags(codes, k, thr, what)
        assert f[:i + 1].sum() == n
    raise RuntimeError("no cut")


def short_records(n, k):
    """Records of n bases in all, none long enough for a window (k - 1 bases each, the last shorter)."""
    return [b"A" * min(k - 1, n - i) for i in range(0, n, k - 1)]


def craft_false(rng, k, thr, n):
    """n distinct canonical k-mers (codes) whose hash has high word thr_hi and is >= thr: false candidates."""
    hi, lo = thr >> 32, thr & 0xFFFFFFFF
    assert lo < 0xFFFFFFFF - 2**20
    out, seen = [], set()
    while len(out) < n:
        h = (np.uint64(hi) << np.uint64(32)) | rng.integers(lo + 1, 1 << 32, size=1 << 16, dtype=np.uint64)
        v = unhash64(h)
        for vv, x in zip(v[is_canonical(v, k)].tolist(), h[is_canonical(v, k)].tolist()):
            if x not in seen:
                seen.add(x)
                out.append(np.array([(vv >> (2 * (k - 1 - j))) & 3 for j in range(k)], dtype=np.uint8))
    return out[:n]


def _stage(k, d):
    """Tile 0 holds exactly SEED_STAGE + d survivors, all in one record; the rest of the tile is records too short
    for a window; tile 1 a few hundred survivors."""
    C = constants()
    T, N = C["SEED_TILE"], C["SEED_STAGE"] + d
    rng = _rng("stage", k, d)
    c = 50
    a = cut_record(rng, k, threshold(c), N, "surv")
    assert len(a) < T - 64
    seqs = [_ascii(a)] + short_records(T - len(a), k) + [_ascii(rng.integers(0, 4, size=6000, dtype=np.uint8))]
    claims = [("tile 0 survivors", lambda i: True, lambda m, i: m[0]["staged"], N),
              ("tile 0 candidates < SEED_CAND", lambda i: True, lambda m, i: int(m[0]["cand"] < C["SEED_CAND"]), 1),
              ("tile 1 survivors < SEED_STAGE", lambda i: True, lambda m, i: int(m[1]["staged"] < C["SEED_STAGE"]), 1)]
    return Batch("stage", "stage%d_k%d" % (N, k), k, c, seqs, claims, ("emit0", "reads", "sort", "pairs"))


def _cand(k, d):
    """Record chunk 0 of tile 0 lists exactly SEED_CAND + d candidates.  k = 31: its last two candidates (in window
    order) are false candidates, high word thr_hi and full hash >= thr, so that with d = +1 one candidate is always
    resolved inline and false ones are rejected on the list and (whichever the atomics pick) the inline path."""
    C = constants()
    T, N = C["SEED_TILE"], C["SEED_CAND"] + d
    rng = _rng("cand", k, d)
    c = 25
    thr = threshold(c)
    n_false = 2 if k == 31 else 0
    a = cut_record(rng, k, thr, N - n_false, "cand")
    if n_false:
        fk = craft_false(rng, k, thr, n_false)
        for _ in range(100000):
            f1, f2 = (rng.integers(0, 4, size=int(rng.integers(1, 6)), dtype=np.uint8) for _ in range(2))
            tail = rng.integers(0, 4, size=8, dtype=np.uint8)
            rec = np.concatenate([a, f1, fk[0], f2, fk[1], tail])
            nw = (len(rec) - k + 1) // 4 * 4
            rec = rec[:nw + k - 1]
            if int(_flags(rec, k, thr, "cand").sum()) == N:
                a = rec
                break
        else:
            raise RuntimeError("no stray-free false candidates")
    assert len(a) < T - 64
    seqs = [_ascii(a)] + short_records(T - len(a), k) + [_ascii(rng.integers(0, 4, size=3000, dtype=np.uint8))]
    claims = [("chunk 0 candidates", lambda i: i["part"] is None, lambda m, i: m[0]["chunks"][0]["cand"], N),
              ("chunk 0 false candidates", lambda i: i["part"] is None, lambda m, i: m[0]["chunks"][0]["false"], n_false)]
    return Batch("cand", "cand%d_k%d" % (N, k), k, c, seqs, claims, ("emit0", "reads", "pairs"))


def _cand_nosurv():
    """SEED_CAND + 1 false candidates back to back in one record at c = 10^6 and no survivor: the list fills, one
    candidate goes inline, every one is rejected."""
    C = constants()
    k, c, N = 31, 10**6, C["SEED_CAND"] + 1
    thr = threshold(c)
    rng = _rng("cand_nosurv")
    for _ in range(100):
        fk = craft_false(rng, k, thr, N)
        rec = np.concatenate(fk + [rng.integers(0, 4, size=4, dtype=np.uint8)])
        rec = rec[:(len(rec) - k + 1) // 4 * 4 + k - 1]
        h = hash64(window_values(rec, k))
        if int(((h >> np.uint64(32)) <= np.uint64(thr >> 32)).sum()) == N and not (h < np.uint64(thr)).any():
            break
    else:
        raise RuntimeError("stray candidates")
    seqs = [_ascii(rec), _ascii(rng.integers(0, 4, size=3000, dtype=np.uint8))]
    claims = [("chunk 0 candidates", lambda i: True, lambda m, i: m[0]["chunks"][0]["cand"], N),
              ("chunk 0 false candidates", lambda i: True, lambda m, i: m[0]["chunks"][0]["false"], N),
              ("tile 0 survivors", lambda i: True, lambda m, i: m[0]["staged"], 0)]
    return Batch("cand", "cand_nosurv", k, c, seqs, claims, ("emit0", "reads", "pairs"))


def _chunks(k, n):
    """Tile 0 overlapped by exactly n records: n - 1 inside it, the last across its end.  c = 20, so that the
    records in the last slots of a chunk have candidates (the 8-bit record slot of a list entry)."""
    C = constants()
    T = C["SEED_TILE"]
    rng = _rng("chunks", k, n)
    avg = (T - 400) / (n - 1)
    ln = rng.integers(int(avg * 0.6), int(avg * 1.4) + 1, size=n - 1)
    ln = np.maximum((ln * (T - 400) / ln.sum()).astype(np.int64), 1)
    ln = np.maximum(ln, k + 8)
    assert ln.sum() < T - 100, ln.sum()
    seqs = [_ascii(rng.integers(0, 4, size=int(x), dtype=np.uint8)) for x in ln]
    seqs.append(_ascii(rng.integers(0, 4, size=T - int(ln.sum()) + 2000, dtype=np.uint8)))
    seqs += [_ascii(rng.integers(0, 4, size=int(x), dtype=np.uint8)) for x in rng.integers(50, 400, size=40)]
    NT = C["SEED_THREADS"]
    claims = [("tile 0 records", lambda i: True, lambda m, i: m[0]["records"], n),
              ("tile 0 chunks", lambda i: True, lambda m, i: len(m[0]["chunks"]), -(-n // NT)),
              ("top record slot with a candidate", lambda i: i["part"] is None,
               lambda m, i: max(ch["top_slot"] for ch in m[0]["chunks"]), min(n, NT) - 1)]
    return Batch("chunks", "chunks%d_k%d" % (n, k), k, 20, seqs, claims, ("emit0", "reads", "pairs"))


def _mod4_len(L, k):
    """A length near L (>= 2k) whose window count L - k + 1 is a multiple of 4."""
    L = max(L, 2 * k)
    return L + (-(L - k + 1)) % 4


def _chunk_bounds(k):
    """Record ranges at tile starts: a record starting exactly at T1 (tile 0 iterates it with no window); a record
    whose last valid window starts at 2T - 1 (its bases end in tile 1's halo); empty records on 3T (tile 3 starts at
    the last of the equal offsets); a record starting mid tile 3 and spanning tiles 4 and 5."""
    C = constants()
    T = C["SEED_TILE"]
    rng = _rng("chunk_bounds", k)
    rnd = lambda n: _ascii(rng.integers(0, 4, size=int(n), dtype=np.uint8))  # noqa: E731
    seqs, pos = [], 0

    def fill_to(p):
        nonlocal pos
        while p - pos > 700:
            seqs.append(rnd(rng.integers(100, 600)))
            pos += len(seqs[-1])
        seqs.append(rnd(p - pos))
        pos = p

    fill_to(T)                                  # the previous record ends exactly at T1
    at_t1 = len(seqs)
    seqs.append(rnd(500))
    pos += 500
    Lh = _mod4_len(300, k)                # last window start 2T - 1: starts at 2T - (Lh - k + 1)
    fill_to(2 * T - (Lh - k + 1))
    halo = len(seqs)
    seqs.append(rnd(Lh))
    pos += Lh
    fill_to(3 * T)
    seqs += [b""] * 5
    first3 = len(seqs)
    seqs.append(rnd(400))
    pos += 400
    fill_to(3 * T + 5000)
    span = len(seqs)
    seqs.append(rnd(2 * T + 3000))
    pos += 2 * T + 3000
    seqs += [rnd(x) for x in rng.integers(50, 400, size=20)]
    off = np.cumsum([0] + [len(s) for s in seqs])
    assert off[at_t1] == T and off[halo + 1] - k == 2 * T - 1 and off[first3] == 3 * T
    claims = [("tile 0 ends at the record starting at T1", lambda i: True, lambda m, i: m[0]["r_hi"], at_t1),
              ("tile 1 starts at the record starting at T1", lambda i: True, lambda m, i: m[1]["r_lo"], at_t1),
              ("tile 2 starts at the record whose last window is 2T - 1", lambda i: True, lambda m, i: m[2]["r_lo"], halo),
              ("last window of that record", lambda i: True, lambda m, i: last_start(i, halo), 2 * T - 1),
              ("tile 3 starts after the empty records", lambda i: True, lambda m, i: m[3]["r_lo"], first3),
              ("tile 2 iterates the empty records", lambda i: True, lambda m, i: m[2]["r_hi"], first3),
              ("tile 4 is one record", lambda i: True, lambda m, i: m[4]["records"], 1),
              ("tile 5 starts in the spanning record", lambda i: True, lambda m, i: m[5]["r_lo"], span)]
    return Batch("chunks", "chunk_bounds_k%d" % k, k, 20, seqs, claims, ("emit0", "reads", "pairs"))


def _runs(k, W):
    """Records of (scalar) window counts mW - 1, mW and mW + 1 for m = 1, 2, 3, shuffled, at c = 8: with the kernel at
    run length W the masked last run has W - 1 and 1 windows, and full runs end exactly on record ends."""
    rng = _rng("runs", k, W)
    counts = [m * W + d for m in (1, 2, 3) for d in (-1, 0, 1)] * 40
    counts = [counts[i] for i in rng.permutation(len(counts))]
    seqs = [_ascii(rng.integers(0, 4, size=n + k - 1, dtype=np.uint8)) for n in counts]
    sc = lambda i: i["sem"] == SEM_SCALAR  # noqa: E731
    claims = [("masked runs of W-1 windows", lambda i: sc(i) and i["_W"] == W,
               lambda m, i: int(any(W - 1 in ch["masked_n"] for t in m for ch in t["chunks"])), 1),
              ("masked runs of 1 window", lambda i: sc(i) and i["_W"] == W,
               lambda m, i: int(any(1 in ch["masked_n"] for t in m for ch in t["chunks"])), 1),
              ("masked runs (any)", lambda i: True, lambda m, i: sum(ch["masked"] for t in m for ch in t["chunks"]), None)]
    return Batch("runs", "runs%d_k%d" % (W, k), k, 8, seqs, claims, ("emit0", "reads"))


def fullest_runs(k, W):
    """Most runs one record chunk can hold at W: SEED_THREADS records back to back, each costing k - 1 bases past its
    windows, the last clipped at the tile end; window counts 1 mod W."""
    C = constants()
    NT, T = C["SEED_THREADS"], C["SEED_TILE"]
    return NT + (T - (NT - 1) * k - 1) // W


def _runs_full(k, W):
    """SEED_THREADS records that fill tile 0 with window counts 1 mod W (scalar): the fullest run table at W."""
    C = constants()
    NT, T = C["SEED_THREADS"], C["SEED_TILE"]
    rng = _rng("runs_full", k, W)
    Q = (T - (NT - 1) * k - 1) // W
    q = [Q // NT + (1 if i < Q % NT else 0) for i in range(NT)]
    slack = (T - (NT - 1) * k - 1) - Q * W          # extra windows for record 0, fewer than W - 1
    cnt = [q[i] * W + 1 + (slack if i == 0 else 0) for i in range(NT)]
    seqs = [_ascii(rng.integers(0, 4, size=cnt[i] + k - 1, dtype=np.uint8)) for i in range(NT - 1)]
    a_last = sum(len(s) for s in seqs)
    assert T - a_last == cnt[-1]
    seqs.append(_ascii(rng.integers(0, 4, size=cnt[-1] + k - 1 + 3000, dtype=np.uint8)))
    want = fullest_runs(k, W)
    claims = [("tile 0 runs at W", lambda i: i["sem"] == SEM_SCALAR and i["_W"] == W,
               lambda m, i: m[0]["chunks"][0]["runs"], want),
              ("tile 0 records", lambda i: True, lambda m, i: m[0]["records"], NT)]
    return Batch("runs", "runs_full%d_k%d" % (W, k), k, 8, seqs, claims, ("emit0", "reads"))


STAGING_R = (0, 1, 15, 16, 17, 47, 48, 49, 63, 64, 65)   # ASCII: 0-49 around 16-byte groups and the halo; 2-bit: 0-65


def _staging(k, r):
    """n_bases = TILE + r; the last record ends at n_bases with a window count that is a multiple of 4, so its last
    window starts at n_bases - k under every window rule.  c = 3: most windows survive, so a wrong staged base shows.
    r = k - 1: that last window starts at T1 - 1 and its bases lie in tile 0's halo."""
    C = constants()
    T = C["SEED_TILE"]
    rng = _rng("staging", k, r)
    n = T + r
    last = _mod4_len(200, k)
    seqs, pos = [], 0
    while n - last - pos > 3500:
        seqs.append(_ascii(rng.integers(0, 4, size=int(rng.integers(100, 3000)), dtype=np.uint8)))
        pos += len(seqs[-1])
    seqs.append(_ascii(rng.integers(0, 4, size=n - last - pos, dtype=np.uint8)))
    seqs.append(_ascii(rng.integers(0, 4, size=last, dtype=np.uint8)))
    last_tile = (n - 1) // T
    st = staging(n, T)
    claims = [("tile %d ASCII bytes staged" % t, lambda i: True, lambda m, i, t=t: st[t]["ascii"][0],
               min(n - t * T, T + C["SEED_HALO"])) for t in range(last_tile + 1)]
    claims += [("tile %d ASCII bulk bytes" % t, lambda i: True, lambda m, i, t=t: st[t]["ascii"][1], None)
               for t in range(last_tile + 1)]
    claims += [("tile %d 2-bit words staged / bulk" % t, lambda i: True, lambda m, i, t=t: st[t]["packed"], None)
               for t in range(last_tile + 1)]
    if r == k - 1:
        claims.append(("last window starts at T1 - 1", lambda i: True, lambda m, i: last_start(i, len(seqs) - 1), T - 1))
    return Batch("staging", "staging%d_k%d" % (r, k), k, 3, seqs, claims, ("emit0", "reads"))


def last_start(inst, r):
    """Flat start of record r's last valid window under inst's window rule."""
    start, rec, _ = windows(inst["_b"], inst["sem"], inst["with_pos"])
    return int(start[rec == r].max())


def _staging_tiny(k):
    """A whole batch under 16 bases: no bulk copy, no window."""
    seqs = [b"ACGTACG", b"", b"TTAC"]
    claims = [("ASCII bulk bytes", lambda i: True, lambda m, i: staging(11, constants()["SEED_TILE"])[0]["ascii"][1], 0),
              ("tile 0 candidates", lambda i: True, lambda m, i: m[0]["cand"], 0)]
    return Batch("staging", "staging_tiny_k%d" % k, k, 3, seqs, claims, ("emit0", "reads"))


EVENT_L = (65, 66, 400, 401)


def _events(k, L):
    """Reads of length L across tile edges (c = 4): at edge 1 the read's middle 32 bases end exactly at the staged
    limit (SEED_NCHUNK16 * 16, keys taken in place), at edge 2 one base past it (pending), at edge 3 the read starts one
    base before the tile (st < 0 in the next tile: pending), at edge 4 exactly on it (st = 0).  The edge reads are
    copies of reads in the middle of tiles, so deduplication compares keys from the tile with keys from memory."""
    C = constants()
    T, lim = C["SEED_TILE"], C["SEED_NCHUNK16"] * 16
    for attempt in range(50):
        rng = _rng("events", k, L, attempt)
        proto = [_ascii(rng.integers(0, 4, size=L, dtype=np.uint8)) for _ in range(2)]
        starts = [lim - 32 - L // 2, T + lim - 31 - L // 2, 3 * T - 1, 4 * T]
        seqs, pos = [], 0
        for e, st in enumerate(starts):
            while st - pos > 900:
                x = proto[int(rng.integers(0, 2))] if rng.random() < 0.05 else \
                    _ascii(rng.integers(0, 4, size=int(rng.integers(60, 420)), dtype=np.uint8))
                seqs.append(x)
                pos += len(x)
            seqs.append(_ascii(rng.integers(0, 4, size=st - pos, dtype=np.uint8)))
            seqs.append(proto[e % 2])
            pos = st + L
        seqs += proto + [_ascii(rng.integers(0, 4, size=300, dtype=np.uint8))]
        b = Batch("events", "events%d_k%d" % (L, k), k, 4, seqs, [], ("reads", "no_dedup", "pairs"))
        pair = PAIR_MIN <= L <= PAIR_MAX
        single = lambda i: i["emit"] == 1 and not i["paired"] and not i["no_dedup"]  # noqa: E731
        claims = [("edge 1: keys in place at the staged limit", single, lambda m, i: m[0]["events"]["inplace_lim"],
                   ">0" if pair else 0),
                  ("edge 2: pending one base past the limit", single, lambda m, i: m[1]["events"]["pend_mid"],
                   ">0" if pair else 0),
                  ("edge 3: pending, read starts before the tile", single, lambda m, i: m[3]["events"]["pend_st"],
                   ">0" if pair else 0),
                  ("edge 4: keys in place, read starts on the tile", single, lambda m, i: m[4]["events"]["inplace_st0"],
                   ">0" if pair else 0),
                  ("no pending events without dedup", lambda i: i["no_dedup"] == 1,
                   lambda m, i: sum(t["events"]["pend"] for t in m), 0),
                  ("read pairs: every event pending", lambda i: i["paired"],
                   lambda m, i: int(sum(t["events"]["pend"] for t in m) == sum(t["staged"] for t in m)), 1)]
        b.claims = claims
        if all(ok for _, _, _, ok, _ in claim_cases(b)):
            return b
    raise RuntimeError("no event batch reaches its edges")


def _parts(k):
    """150 bp reads with duplicates at c = 10 sketched in 2 parts: tile 0 holds more than SEED_STAGE survivors of
    each part, so events below a part's lower bound are dropped in front of the inline path too."""
    C = constants()
    rng = _rng("parts", k)
    base = [_ascii(rng.integers(0, 4, size=150, dtype=np.uint8)) for _ in range(500)]
    reads = base + [base[i] for i in rng.integers(0, 500, 250)]
    reads = [reads[i] for i in rng.permutation(len(reads))]
    b = Batch("parts", "parts_k%d" % k, k, 10, reads, [], ("parts",), parts=2)
    b.claims = [("tile 0 survivors of the part > SEED_STAGE", lambda i: i["part"] is not None,
                 lambda m, i: int(m[0]["staged"] > C["SEED_STAGE"]), 1)]
    return b


def oracle_survivors(b, sem, with_pos):
    """The C oracle's survivors of every record [(rec, pos, hash)], sorted; pos 0 without positions."""
    from oracle import oracle as O
    out = []
    for r in range(b.n_rec):
        s = b.buf[int(b.off[r]):int(b.off[r + 1])]
        if with_pos:
            pos, h = O.extract_markers_positions(s, b.k, b.c, sem)
            out += [(r, int(p), int(x)) for p, x in zip(pos.tolist(), h.tolist())]
        else:
            out += [(r, 0, int(x)) for x in O.extract_markers(s, b.k, b.c, sem).tolist()]
    return sorted(out)


# ---- the batches ---------------------------------------------------------------------------------------------------
def names():
    C = constants()
    out = []
    for k in (31, 21):
        out += [("stage", k, d) for d in (-1, 0, 1)]
        out += [("cand", k, d) for d in (-1, 0, 1)]
        out += [("chunks", k, n) for n in (C["SEED_THREADS"] - 1, C["SEED_THREADS"], C["SEED_THREADS"] + 1,
                                           2 * C["SEED_THREADS"] + 1)]
        out += [("chunk_bounds", k, None)]
        out += [("runs", k, W) for W in run_lengths()] + [("runs_full", k, W) for W in run_lengths()]
        out += [("staging", k, r) for r in STAGING_R + (k - 1,)] + [("staging_tiny", k, None)]
        out += [("events", k, L) for L in EVENT_L]
        out += [("parts", k, None)]
    out.append(("cand_nosurv", 31, None))
    return out


FAMILIES = ("stage", "cand", "chunks", "runs", "staging", "events", "parts")


@functools.lru_cache(maxsize=None)
def batch(kind, k, arg):
    f = {"stage": _stage, "cand": _cand, "chunks": _chunks, "runs": _runs, "runs_full": _runs_full,
         "staging": _staging, "events": _events}
    if kind in f:
        return f[kind](k, arg)
    return {"chunk_bounds": _chunk_bounds, "staging_tiny": _staging_tiny, "parts": _parts}[kind](k) \
        if kind != "cand_nosurv" else _cand_nosurv()


def family_batches(family):
    return [batch(*n) for n in names() if batch(*n).family == family]


def claim_cases(b):
    """-> [(W, inst, label, ok, value)] for every claim of b under every instantiation and run length it holds for.
    The model of each (W, inst) is computed once."""
    out = []
    for W in run_lengths():
        for inst in insts(b):
            inst = dict(inst, _W=W, _b=b)
            cls = [cl for cl in b.claims if cl[1](inst)]
            if not cls:
                continue
            m = model(b, W, inst)
            for label, _, fn, want in cls:
                v = fn(m, inst)
                ok = True if want is None else (v > 0 if want == ">0" else v == want)
                out.append((W, inst, label, ok, v))
    return out
