"""CPU: the read and pair samples of tests/read_group_scripts.py hold what they claim.  Every record's survivors are
exactly the scripted hashes (C oracle); the restated one-pass map and part bounds are the planner's
(sample_parts.hpp, built on the host); each family reaches its structural edge of k_group_dedup whatever the order the
events are inserted in -- a full table, a probe chain past slot 1023, one bucket holding a whole group, groups of
exactly slot and slot + 1 events, k-mers at every bucket boundary, a group split across a part bound; and on two
families the post-pass model's k-mers and counts are oracle/pyref.py's."""
import numpy as np
import pytest

from tests import dedup_scripts as D
from tests import read_group_scripts as G
from tests.test_sample_parts_cpu import plan, plan_exe  # noqa: F401 (plan_exe: the fixture that builds the planner)

U64 = 2**64 - 1
CASES = [(name, paired) for name in G.FAMILIES for paired in (False, True)]
IDS = ["%s-%s" % (n, "pairs" if p else "single") for n, p in CASES]
ORDERS = 4      # random insertion orders the table claims are checked in


@pytest.mark.parametrize("name,paired", CASES, ids=IDS)
def test_records_hold_exactly_the_scripted_survivors(name, paired):
    s = G.sample(name, paired)
    got = G.oracle_survivors(s)
    assert len(got) == len(s.script)
    for i, (a, b) in enumerate(zip(got, s.script)):
        assert (tuple(a) if paired else a) == (tuple(b) if paired else b), (name, i)
    assert sum(len(x) for r in s.script for x in (r if paired else [r])) > G.SLOT


@pytest.mark.parametrize("slot", G.SMALL_CAPS)
def test_small_cap_records_hold_exactly_the_scripted_survivors(slot):
    for name in ("slot_exact", "slot_plus_one"):
        for paired in (False, True):
            s = G.sample(name, paired, slot)
            got = G.oracle_survivors(s)
            assert [tuple(x) for x in got] == [tuple(x) for x in s.script] if paired else got == s.script
            sizes = {g: sum(e.values()) for g, e in G.group_events(s).items()}
            assert sizes == s.claims["sizes"], (name, paired, slot, sizes)


def test_restated_map_and_parts_equal_the_planner(plan_exe):  # noqa: F811
    cases, samples = [], []
    for name, paired in CASES:
        s = G.sample(name, paired)
        mates = 2 if paired else 1
        for P in (0, 2, 3, 7):
            cases.append((s.n_bases, s.n_records // mates, mates, s.k, s.c, 1, U64, 0, P))
            samples.append((s, P))
    for (s, P), r in zip(samples, plan(plan_exe, cases)):
        assert r[0] == "ok"
        head, parts = r[1], r[2]
        m = s.map
        assert (head["thr"], head["nbk"], head["Mb"]) == (m.thr, m.nbk, m.Mb), s.name
        want = m.parts(P) if P else [(0, m.thr, 0, m.ng)]
        assert [p[:4] for p in parts] == want, (s.name, P)


def _groups(s):
    return G.group_events(s)


@pytest.mark.parametrize("name,paired", [c for c in CASES if c[0] in G.FULL + ("parts",)],
                         ids=[i for c, i in zip(CASES, IDS) if c[0] in G.FULL + ("parts",)])
def test_full_groups_fill_the_table_in_any_order(name, paired):
    s = G.sample(name, paired)
    ge = _groups(s)
    rng = np.random.default_rng(1)
    for g in s.claims["full"]:
        assert sum(ge[g].values()) == G.SLOT
        hs = list(ge[g])
        distinct = name != "mixed_full"
        assert len(hs) == (G.TABLE if distinct else len(hs))
        for _ in range(ORDERS):
            at, longest, wrapped = G.probe(hs, rng.permutation(len(hs)).tolist())
            assert len(set(at.values())) == len(hs)
            if distinct:                                   # every slot taken
                assert sorted(at.values()) == list(range(G.TABLE))
                if name != "full_one_home":            # random homes: some chain passes slot 1023
                    assert wrapped and longest > 100
        if name == "full_one_home":
            slot = s.claims["one_home"][g]
            assert {G.home(h) for h in hs} == {slot}
            at, longest, wrapped = G.probe(hs, rng.permutation(len(hs)).tolist())
            assert longest == G.TABLE - 1                  # one chain over the whole table
            assert wrapped == (slot == G.TABLE - 1)        # from 1023 it wraps to 0; from 0 it ends at 1023
            assert at[max(hs, key=lambda h: at[h])] == G.TABLE - 1
        if name == "full_distinct":
            assert len({G.home(h) for h in hs}) > 500      # random homes


@pytest.mark.parametrize("paired", [False, True])
def test_one_bucket_groups(paired):
    s = G.sample("one_bucket", paired)
    m = s.map
    pop = {}
    for g, e in _groups(s).items():
        for h in e:
            pop[m.bucket(h)] = pop.get(m.bucket(h), 0) + 1
    assert pop == s.claims["buckets"] == {0: G.TABLE, 63: G.TABLE, m.nbk - 1: G.TABLE}
    assert 63 % G.BPG == G.BPG - 1


@pytest.mark.parametrize("name", ["slot_exact", "slot_plus_one"])
@pytest.mark.parametrize("paired", [False, True])
@pytest.mark.parametrize("slot", (G.SLOT,) + G.SMALL_CAPS)
def test_slot_groups_stay_or_leave_by_one_event(name, paired, slot):
    s = G.sample(name, paired, slot)
    ge = _groups(s)
    sizes = {g: sum(e.values()) for g, e in ge.items()}
    assert sizes == s.claims["sizes"] and s.map.ng == 4
    first, last = (slot + 1, slot + 1) if name == "slot_plus_one" else (slot, slot)
    assert sizes[0] == first and sizes[3] == last and {sizes[0], sizes[1]} == {slot, slot + 1}
    heavy = max(ge[3], key=ge[3].get)
    assert ge[3][heavy] == slot                            # one k-mer of exactly `slot` events
    if paired:                                             # some of them mate-2 events the pair rule skips
        _, skipped = D.pair_kmer_events(s.r1, s.r2, s.k, s.c, G.SEM)
        assert skipped.get(heavy, 0) >= slot // 16
    elif slot > 4:
        assert D.device_path(G._events(s)[heavy]) == "cut"
    for g, n in sizes.items():
        assert G.stays(s, ge[g], slot) == (n <= slot), (g, n)
    (ng, sl, ovf, u1, nf), = G.post_pass(s)
    assert (ng, sl, ovf) == (4, slot, sum(max(0, n - slot) for n in sizes.values()))
    assert nf == sum(n for n in sizes.values() if n > slot) > 0


@pytest.mark.parametrize("paired", [False, True])
def test_boundaries_sit_at_every_bucket_boundary(paired):
    s = G.sample("boundaries", paired)
    m = s.map
    cr = G.Crafter(np.random.default_rng(0))
    hashes = set(G._events(s))
    assert m.ng == 8
    ordered = sorted(hashes)
    for b in range(1, m.nbk):
        f = m.first_hash(b)
        i = np.searchsorted(ordered, f)
        at, under = ordered[i], ordered[i - 1]
        assert m.bucket(at) == b and m.bucket(under) == b - 1 and m.bucket(f - 1) == b - 1
        assert not cr.valid(list(range(f, at))).any() if at > f else True       # the nearest valid at or above
        assert not cr.valid(list(range(under + 1, f))).any() if f > under + 1 else True  # and just below
    lo, hi = ordered[0], ordered[-1]
    assert not cr.valid(list(range(0, lo))).any() and not cr.valid(list(range(hi + 1, m.thr))).any()
    ge = _groups(s)
    for g in range(m.ng):                                  # in-kernel and fallback groups alternate
        assert G.stays(s, ge[g], G.SLOT) == (g % 2 == 0), g
        assert len({m.bucket(h) for h in ge[g]}) == G.BPG


@pytest.mark.parametrize("paired", [False, True])
def test_parts_split_a_group_and_keep_a_full_one_in_the_middle(paired):
    s = G.sample("parts", paired)
    m = s.map
    bounds = m.parts(G.PARTS)
    assert [(g0, ng) for _, _, g0, ng in bounds] == [(0, 3), (2, 4), (5, 3)]
    g, b = s.claims["split"]
    assert bounds[1][0] == m.first_hash(b) and b // G.BPG == g
    one = {g: sum(e.values()) for g, e in _groups(s).items()}
    assert one[g] == 1500 and one[3] == G.SLOT and one[4] == G.SLOT + 1
    shares = [sum(G.group_events(s, lo, hi).get(g, {}).values()) for lo, hi, _, _ in bounds[:2]]
    assert shares == [750, 750]
    lines = G.post_pass(s, parts=G.PARTS)
    whole, = G.post_pass(s)
    assert whole[4] == sum(one[x] for x in (g, 4))         # one pass: the split group and group 4 leave
    assert lines[0][4] == 0 and lines[1][4] == one[4]      # in parts: only group 4 leaves
    assert sum(x[3] for x in lines) == whole[3] + len(G.group_events(s)[g])


@pytest.mark.parametrize("paired", [False, True])
def test_mixed_groups_reach_every_in_kernel_path_at_full_occupancy(paired):
    s = G.sample("mixed_full", paired)
    ge = _groups(s)
    ev = G._events(s)
    for g in (0, 1):
        assert sum(ge[g].values()) == G.SLOT and G.stays(s, ge[g], G.SLOT)
        if not paired:
            paths = [D.device_path(ev[h]) for h in ge[g]]
            assert all(paths.count(p) > 5 for p in D.IN_KERNEL), paths
        else:
            sizes = list(ge[g].values())
            assert sum(n <= 8 for n in sizes) > 20 and sum(n > 8 for n in sizes) > 5
    if not paired:
        paths = {D.device_path(ev[h]) for h in ge[2]}
        assert {"steps", "set"} <= paths and not G.stays(s, ge[2], G.SLOT)
    else:
        _, skipped = D.pair_kmer_events(s.r1, s.r2, s.k, s.c, G.SEM)
        assert len(skipped) > 20


@pytest.mark.parametrize("paired", [False, True])
def test_model_agrees_with_pyref(paired):
    """the model's k-mers and events are oracle/pyref.py's sketch: keyless reads, and pairs whose k-mers occur once,
    count every event"""
    name = "full_distinct"
    from oracle import oracle as O
    s = G.sample(name, paired)
    pc = G.pyref_counts(s)
    if paired:
        eh, ec, _, nd = O.sketch_read_pairs(*s.flat(), k=s.k, c=s.c)
        ev, _ = D.pair_kmer_events(s.r1, s.r2, s.k, s.c, G.SEM)
        model = {h: len(e) for h, e in ev.items()}
    else:
        eh, ec, _, nd = O.sketch_reads(*s.flat(), k=s.k, c=s.c)
        model = {h: len(e) for h, e in G._events(s).items()}
    assert dict(zip(eh.tolist(), ec.tolist())) == pc == model and nd == 0
    (ng, _, _, u1, nf), = G.post_pass(s)
    ge = _groups(s)
    assert u1 + sum(len(ge[g]) for g in ge if not G.stays(s, ge[g], s.slot)) == len(pc)
    assert nf == sum(sum(ge[g].values()) for g in ge if not G.stays(s, ge[g], s.slot))
