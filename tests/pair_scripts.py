"""Scripted duplicate-removal histories for read pairs (a test helper module, not a conftest), in the manner of
tests/dedup_scripts.py and built from its generator: one target k-mer per script, every event one pair that holds the
target in mate 1, mate 2 or both under chosen pair keys (mate 1 interleaves (A.x, B.x), mate 2 (A.y, B.y)).

Pairs have no MAX_DEDUP_COUNT (src/sketch.rs:829-865), so the device path of a k-mer in k_group_dedup<PAIRED>
(sylph_b200/csrc/sample.cu) depends on its number of events only, counted with the mate-2 events the rule skips:

  thread         1-8 events: one thread compares every event with every other
  keyless_first  the same path; the first pair has a mate under 33 bp (no keys, but it counts), the second has
                 A == B, then key hits: a first event with A == B counts, behind a keyless one it is a duplicate
  warp           9-60 events: a warp, one event per lane
  warp_big       100-250 events that share one key with a fresh second key each: a dedup set far past any fixed size
  slot           more than 1024 events: the k-mer's group is past its slot and takes the generic path
"""
import functools
import zlib

from oracle import oracle as O
from tests import dedup_scripts as D

THREAD_MAX = 8       # GRP_PAIR_THREAD
PLACES = {"m1": (1, 0), "m2": (0, 1), "both": (1, 1), "m1_twice": (2, 0), "m1_twice_m2": (2, 1), "m2_twice": (0, 2)}
# events a script of the family holds
EVENTS = {"thread": (1, THREAD_MAX), "keyless_first": (3, THREAD_MAX), "warp": (THREAD_MAX + 1, 60),
          "warp_big": (100, 250), "slot": (D.SLOT + 1, D.SLOT + 200)}
IN_KERNEL = ("thread", "keyless_first", "warp", "warp_big")


def _draw(rng, pool, keyless=0.12):
    """(key a, key b, place) from a pool of keys: A == B one time in six, a keyless pair now and then"""
    place = "short_mate" if rng.random() < keyless else list(PLACES)[int(rng.integers(0, len(PLACES)))]
    a = int(rng.integers(0, pool))
    return (a, a if rng.random() < 1 / 6 else int(rng.integers(0, pool)), place)


def _n_events(ev):
    return sum(1 if p == "short_mate" else sum(PLACES[p]) for _, _, p in ev)


def _fill(rng, lo, hi, ev, draw):
    """events from draw() until the script holds a number of events drawn from [lo, hi]"""
    want = int(rng.integers(max(lo, _n_events(ev)), hi + 1))
    while _n_events(ev) < want:
        e = draw()
        if _n_events(ev + [e]) <= hi:
            ev.append(e)
    return ev


def _fam_thread(rng):
    return 3, _fill(rng, *EVENTS["thread"], [], lambda: _draw(rng, 3))


def _fam_keyless_first(rng):
    ev = [(0, 1, "short_mate"), (0, 0, "m1" if rng.random() < 0.5 else "m2"), (0, 2, "m1")]
    return 3, _fill(rng, *EVENTS["keyless_first"], ev, lambda: _draw(rng, 3))


def _fam_warp(rng):
    return 5, _fill(rng, *EVENTS["warp"], [], lambda: _draw(rng, 5))


def _fam_warp_big(rng):
    nxt = [2]

    def draw():
        if rng.random() < 0.1:
            return _draw(rng, nxt[0])
        nxt[0] += 1
        place = list(PLACES)[int(rng.integers(0, len(PLACES)))]
        return (0, nxt[0] - 1, place) if rng.random() < 0.5 else (nxt[0] - 1, 0, place)
    ev = _fill(rng, *EVENTS["warp_big"], [(0, 1, "m1")], draw)
    return nxt[0], ev


def _fam_slot(rng):
    return 6, _fill(rng, *EVENTS["slot"], [], lambda: _draw(rng, 6, keyless=0.05))


FAMILIES = {"thread": _fam_thread, "keyless_first": _fam_keyless_first, "warp": _fam_warp, "warp_big": _fam_warp_big,
            "slot": _fam_slot}
# scripts per family; "small" is the sample the slow pyref cross-check runs on
SAMPLES = {
    "in_kernel": {"thread": 250, "keyless_first": 60, "warp": 40, "warp_big": 4},
    "slot": {"thread": 40, "slot": 2},
    "small": {"thread": 60, "keyless_first": 20, "warp": 10, "warp_big": 1},
}


class PairScripts(D.PairSample):
    """scripts[i] = (family, target hash, events scripted)"""

    def __init__(self, r1, r2, expect, scripts):
        super().__init__(r1, r2, expect, len(scripts))
        self.scripts = scripts

    def flat(self):
        return D.flatten(self.r1) + D.flatten(self.r2)


@functools.lru_cache(maxsize=None)
def sample(name, k=31, c=10, sem=O.SEM_AVX2, seed=0):
    g = D.Gen(zlib.crc32(repr(("pair_scripts", name, k, c, sem, seed)).encode()), k, c, sem)
    rng = g.rng
    reads, scripts = [], []
    for fam, n in SAMPLES[name].items():
        for _ in range(n):
            n_keys, events = FAMILIES[fam](rng)
            pool = [g.key() for _ in range(n_keys)]
            tgt, th = g.target()
            script = []
            for a, b, place in events:
                A, B = pool[a], pool[b]
                rc = rng.random() < 0.5
                if place == "short_mate":
                    short1 = rng.random() < 0.5
                    m1 = g.mate(tgt, (A[0], B[0]), 0 if short1 else 1, rc, short=short1)
                    m2 = g.mate(tgt, (A[1], B[1]), 1 if short1 else 0, rc, short=not short1)
                    script.append((m1, m2, (None, th, 0 if short1 else 1, 1 if short1 else 0)))
                    continue
                n1, n2 = PLACES[place]
                script.append((g.mate(tgt, (A[0], B[0]), n1, rc), g.mate(tgt, (A[1], B[1]), n2, rc),
                               (D._pair_of((A, B)), th, n1, n2)))
            reads.append(script)
            scripts.append((fam, th, _n_events(events)))
    merged = D._interleave_scripts(rng, reads)
    return PairScripts([a for a, _, _ in merged], [b for _, b, _ in merged], [e for _, _, e in merged], scripts)


def events_per_kmer(s, k=31, c=10, sem=O.SEM_AVX2):
    """hash -> events the seeding finds for it (the ones the mate-2 rule skips included), and the rule's view of them"""
    ev, skipped = D.pair_kmer_events(s.r1, s.r2, k, c, sem)
    return {h: len(e) + skipped.get(h, 0) for h, e in ev.items()}, ev, skipped
