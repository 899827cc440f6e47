"""CPU suite: scripted read-pair histories (tests/pair_scripts.py) are proven before a GPU sees them.

Every pair realises its script; every script has the number of events its family promises, so each k-mer lands in
the device path it is built for; and the C oracle, the pure-Python restatement (oracle/pyref.py) and the per-k-mer
transcription of dup_removal_lsh_full_exact without a threshold (tests/dedup_scripts.py replay) agree on them."""
import pytest

from oracle import oracle as O
from oracle import pyref as R
from tests import dedup_scripts as D
from tests import pair_scripts as P

C = 10


@pytest.mark.parametrize("name", list(P.SAMPLES))
def test_pairs_realise_their_scripts(name):
    s = P.sample(name, c=C)
    places = set()
    for m1, m2, (pair, th, n1, n2) in zip(s.r1, s.r2, s.expect):
        assert R.pair_kmer(m1, m2) == pair
        assert O.extract_markers(m1, 31, C, O.SEM_AVX2).tolist().count(th) == n1
        assert O.extract_markers(m2, 31, C, O.SEM_AVX2).tolist().count(th) == n2
        places.add((pair is None, n1, n2))
    # mate 1 only, mate 2 only, both mates, twice in mate 1 (with and without mate 2), twice in mate 2, keyless mates
    assert {(False, 1, 0), (False, 0, 1), (False, 1, 1), (False, 2, 0), (False, 2, 1), (False, 0, 2), (True, 1, 0),
            (True, 0, 1)} <= places


@pytest.mark.parametrize("name", list(P.SAMPLES))
def test_every_script_has_the_event_count_of_its_family(name):
    s = P.sample(name, c=C)
    n_ev, ev, skipped = P.events_per_kmer(s, c=C)
    seen = dict.fromkeys(P.SAMPLES[name], 0)
    for fam, th, scripted in s.scripts:
        lo, hi = P.EVENTS[fam]
        assert lo <= scripted <= hi and n_ev[th] == scripted, (fam, scripted, n_ev[th])
        seen[fam] += 1
    assert seen == P.SAMPLES[name]
    matches = dict.fromkeys(D.MATCHES, 0)
    for e in ev.values():
        D.replay(e, threshold=None, matches=matches)
    assert all(matches[m] >= 20 for m in D.MATCHES), matches
    assert len(skipped) >= 20
    # a keyless first event, then A == B: the second event is a duplicate only because the first one counted
    for fam, th, _ in s.scripts:
        if fam == "keyless_first":
            e = ev[th]
            assert e[0] is None and e[1][0] == e[1][1] and D.replay(e[:2], threshold=None) == (1, 1)
            assert D.replay(e[1:2], threshold=None) == (1, 0)
    sizes = D.group_sizes({h: [0] * n for h, n in n_ev.items()}, sum(map(len, s.r1)) + sum(map(len, s.r2)),
                          2 * len(s.r1), 31, C)
    assert (max(sizes) > D.SLOT) == (name == "slot"), max(sizes)   # groups leave the kernel in the slot sample only


@pytest.mark.parametrize("no_dedup", [False, True])
@pytest.mark.parametrize("name", list(P.SAMPLES))
def test_oracle_equals_the_direct_transcription(name, no_dedup):
    s = P.sample(name, c=C)
    h, cnt, _, nd = O.sketch_read_pairs(*s.flat(), k=31, c=C, no_dedup=no_dedup)
    out = {x: D.replay(e, threshold=None, no_dedup=no_dedup) for x, e in P.events_per_kmer(s, c=C)[1].items()}
    assert dict(zip(h.tolist(), cnt.tolist())) == {x: c for x, (c, _) in out.items()}
    assert nd == sum(d for _, d in out.values()) and (nd > 100) != no_dedup


def test_oracle_equals_pyref_on_the_small_sample():
    s = P.sample("small", c=C)
    assert len(s.r1) <= 1500
    h, cnt, mean, nd = O.sketch_read_pairs(*s.flat(), k=31, c=C)
    ec, emean, end = R.sketch_read_pairs(s.r1, s.r2, 31, C)
    assert dict(zip(h.tolist(), cnt.tolist())) == ec
    assert nd == end and abs(mean - emean) < 1e-9
