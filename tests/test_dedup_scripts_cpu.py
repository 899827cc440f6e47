"""CPU suite: scripted duplicate-removal histories (tests/dedup_scripts.py).

Every generated read realises its script; every sample reaches the device paths it is built for; and the C oracle, the
pure-Python restatement (oracle/pyref.py) and a per-k-mer transcription of dup_removal_lsh_full_exact
(src/sketch.rs:690-731) agree on the scripted samples, single-end and paired."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import pyref as R
from tests import dedup_scripts as D

CONFIGS = [(31, O.SEM_AVX2), (21, O.SEM_SCALAR)]
C = 10


@pytest.mark.parametrize("k,sem", CONFIGS)
@pytest.mark.parametrize("name", list(D.SAMPLES) + ["small"])
def test_single_end_reads_realise_their_scripts(name, k, sem):
    s = D.single_sample(name, k=k, c=C, sem=sem)
    for read, (pair, th, occ) in zip(s.reads, s.expect):
        assert (R.pair_kmer_single(read) if len(read) <= 400 else None) == pair
        assert O.extract_markers(read, k, C, sem).tolist().count(th) == occ


@pytest.mark.parametrize("k,sem", CONFIGS)
@pytest.mark.parametrize("name", list(D.PAIR_SAMPLES))
def test_read_pairs_realise_their_scripts(name, k, sem):
    s = D.pair_sample(name, k=k, c=C, sem=sem)
    places = set()
    for m1, m2, (pair, th, n1, n2) in zip(s.r1, s.r2, s.expect):
        assert R.pair_kmer(m1, m2) == pair
        assert O.extract_markers(m1, k, C, sem).tolist().count(th) == n1
        assert O.extract_markers(m2, k, C, sem).tolist().count(th) == n2
        places.add((pair is None, n1, n2))
    # mate 1 only, mate 2 only, both mates, twice in mate 2, a mate shorter than 33 bp
    assert {(False, 1, 0), (False, 0, 1), (False, 1, 1), (False, 0, 2), (True, 1, 0), (True, 0, 1)} <= places


# fewest k-mers per class each sample must hold; a sample of in-kernel families must hold none of the fallback classes
MIN_IN_KERNEL, MIN_FALLBACK, MIN_MATCHES = 20, 3, 20
BUILT_FOR = {"in_kernel": D.IN_KERNEL, "steps": ("steps",), "set": ("set",), "slot": ("slot",),
             "small": ("quick", "cut", "warp", "steps", "set")}


@pytest.mark.parametrize("k,sem", CONFIGS)
@pytest.mark.parametrize("name", list(BUILT_FOR))
def test_samples_reach_every_class_they_are_built_for(name, k, sem):
    r = D.classify(D.single_sample(name, k=k, c=C, sem=sem), k=k, c=C, sem=sem)
    for cls in BUILT_FOR[name]:
        assert r["classes"][cls] >= (MIN_IN_KERNEL if cls in D.IN_KERNEL else MIN_FALLBACK), (cls, r)
    for m in D.MATCHES:
        assert r["matches"][m] >= MIN_MATCHES, (m, r)
    if name == "in_kernel":   # no k-mer and no group leaves k_group_dedup
        assert all(r["classes"][cls] == 0 for cls in D.FALLBACK), r
        assert r["max_group"] <= D.SLOT, r
    if name == "slot":
        assert r["max_group"] > D.SLOT, r


@pytest.mark.parametrize("name", list(D.PAIR_SAMPLES))
def test_pair_samples_reach_every_case(name):
    r = D.classify_pairs(D.pair_sample(name, c=C))
    assert r["cases"]["mate2_skip"] >= MIN_IN_KERNEL and r["cases"]["keyless"] >= MIN_IN_KERNEL, r
    assert r["cases"]["set_over_64"] >= 1, r
    for m in D.MATCHES:
        assert r["matches"][m] >= MIN_MATCHES, (m, r)


def _direct(ev, **kw):
    out = {h: D.replay(e, **kw) for h, e in ev.items()}
    return ({h: c for h, (c, _) in out.items()}, sum(d for _, d in out.values()))


@pytest.mark.parametrize("no_dedup", [False, True])
@pytest.mark.parametrize("k,sem", CONFIGS)
@pytest.mark.parametrize("name", list(D.SAMPLES))
def test_single_end_oracle_equals_the_direct_transcription(name, k, sem, no_dedup):
    s = D.single_sample(name, k=k, c=C, sem=sem)
    h, cnt, _, nd = O.sketch_reads(*s.flat(), k=k, c=C, no_dedup=no_dedup, sem=sem)
    counts, dups = _direct(D.kmer_events(s.reads, k, C, sem), no_dedup=no_dedup)
    assert dict(zip(h.tolist(), cnt.tolist())) == counts
    assert nd == dups and (nd > 1000) != no_dedup


@pytest.mark.parametrize("no_dedup", [False, True])
@pytest.mark.parametrize("name", list(D.PAIR_SAMPLES))
def test_pair_oracle_equals_the_direct_transcription(name, no_dedup):
    s = D.pair_sample(name, c=C)
    b1, o1 = D.flatten(s.r1)
    b2, o2 = D.flatten(s.r2)
    h, cnt, _, nd = O.sketch_read_pairs(b1, o1, b2, o2, k=31, c=C, no_dedup=no_dedup)
    counts, dups = _direct(D.pair_kmer_events(s.r1, s.r2, 31, C, O.SEM_AVX2)[0], threshold=None, no_dedup=no_dedup)
    assert dict(zip(h.tolist(), cnt.tolist())) == counts
    assert nd == dups and (nd > 500) != no_dedup


def test_oracle_equals_pyref_on_scripted_reads():
    """pyref is slow: one sample of every single-end family but the slot one (about 1900 reads), one of read pairs."""
    s = D.single_sample("small", c=C)
    assert len(s.reads) <= 3000
    h, cnt, mean, nd = O.sketch_reads(*s.flat(), k=31, c=C)
    ec, emean, end = R.sketch_reads(s.reads, 31, C)
    assert dict(zip(h.tolist(), cnt.tolist())) == ec
    assert nd == end and abs(mean - emean) < 1e-9
    p = D.pair_sample("small", c=C)
    assert len(p.r1) <= 3000
    b1, o1 = D.flatten(p.r1)
    b2, o2 = D.flatten(p.r2)
    h, cnt, mean, nd = O.sketch_read_pairs(b1, o1, b2, o2, k=31, c=C)
    ec, emean, end = R.sketch_read_pairs(p.r1, p.r2, 31, C)
    assert dict(zip(h.tolist(), cnt.tolist())) == ec
    assert nd == end and abs(mean - emean) < 1e-9
