"""CPU suite: scripted genome batches (tests/genome_scripts.py).

The inverse of mm_hash64 is exact and crafted k-mers are canonical with the wanted hash; every batch realises its
script exactly (the oracle's survivors are the scripted ones, no stray); every family reaches the cases it is built
for; and the C oracle's sketch_genome equals the pure-Python restatement (oracle/pyref.py) on the small families and a
transcription of src/sketch.rs:590-614 over the oracle's own survivor list on all of them."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import pyref as R
from tests import genome_scripts as G


def test_inverse_hash_is_exact():
    rng = np.random.default_rng(5)
    x = np.concatenate([rng.integers(0, 1 << 63, size=20000, dtype=np.uint64) * np.uint64(2) + np.uint64(1),
                        np.array([0, 1, (1 << 64) - 1, 1 << 63, (1 << 62) - 1], dtype=np.uint64)])
    assert np.array_equal(G.unhash64(G.hash64(x)), x)
    assert np.array_equal(G.hash64(G.unhash64(x)), x)
    for v in x[:200].tolist() + x[-5:].tolist():
        assert int(G.hash64(v)[0]) == R.mm_hash64(v) == O.mm_hash64(v)


def test_crafted_kmers_are_canonical_with_the_wanted_hash():
    c = G.EDGE_C31      # thr - 1 and thr both have canonical 31-mers at c = 200
    for h, survives, _ in G.edge_hashes(c, np.random.default_rng(6)):
        v = int(G.unhash64(h)[0])
        assert v < 1 << 62 and v < int(G.revcomp_value(v, 31)[0])
        s = bytes(G._ACGT[G.codes_of(v, 31)])
        rc = s.translate(bytes.maketrans(b"ACGT", b"TGCA"))[::-1]
        for seq in (s, rc):   # both orientations hash to h
            assert list(R._windows(seq, 31))[0][1] == v and R.mm_hash64(v) == h
        assert (h < G.threshold(c)) == survives
    for c, v, d in G.K21_EDGES:
        assert v < 1 << 42 and v < int(G.revcomp_value(v, 21)[0])
        assert R.mm_hash64(v) == G.threshold(c) + d


def test_dup_slot_crafting():
    b = G.batch("table")
    r = G.classify(b, 30)
    assert r["classes"]["wrap"] >= 3 and r["classes"]["low38_pair"] >= 3 and r["classes"]["slot_collision_dup"] >= 1


@pytest.mark.parametrize("name", G.FAMILIES)
def test_batches_realise_their_scripts(name):
    b = G.batch(name)
    assert b.oracle_survivors() == b.scripted_survivors()
    if b.c_hash != b.c:      # bounds: the same survivors one step up the threshold
        assert b.oracle_survivors(b.c_hash) == b.scripted_survivors()


EDGES = [(31, W, None) for W in G.EDGE_W] + [(21, W, c) for W in G.EDGE_W for c, _, _ in G.K21_EDGES]


@pytest.mark.parametrize("k,W,c", EDGES)
def test_edge_batches_realise_their_scripts(k, W, c):
    b = G.edge_batch(k, W, c)
    assert b.oracle_survivors() == b.scripted_survivors()
    kept = {lab for lab, ok, _ in b.labels if ok}
    assert len(b.scripted_survivors()) == W * len(kept)
    assert sorted({o for _, _, o in b.labels}) == list(range(W))
    # every record has W or more windows and k_seed picks W for records of this length
    assert all(G.valid_starts(len(s), k) == G.record_length(k, W) - k + 1 for s in b.contigs)


def _walk_classes(name):
    b = G.batch(name)
    return {ms: G.classify(b, ms) for ms in G.MS[name]}


def test_spacing_family_reaches_its_classes():
    r = _walk_classes("spacing")
    for ms in (30, 70):
        c = r[ms]["classes"]
        assert c["gap_eq_ms"] >= 10 and c["gap_eq_ms1"] >= 10, (ms, c)
        assert c["chain_kept"] >= 20 and c["tracked"] >= 100 and c["head"] >= 30, (ms, c)
    assert r[0]["classes"]["tracked"] == 0
    assert r[1 << 20]["classes"]["head"] == sum(1 for ct in G.batch("spacing").expect if ct)   # one head per contig
    x = r[70]
    assert x["N"] > G.SCAN_BLOCK + G.DUP_BLOCK and x["max_tile"] <= G.SLOT
    # the 1201-survivor cluster is one chain at ms = 70 that crosses a tile edge
    b = G.batch("spacing")
    big = b.expect[0]
    assert len(big) == 1201 and max(q - p for (p, _), (q, _) in zip(big, big[1:])) <= 70
    assert (int(b.contig_off[0]) + big[-1][0]) // G.TILE >= 2


def test_dups_family_reaches_its_classes():
    r = G.classify(G.batch("dups"), 30)
    c = r["classes"]
    for cls in ("dup_rc", "dup_2", "dup_3", "dup_5", "dup_two_contigs", "head_past_dup", "dup_inside_chain",
                "adjacent_genome_pair", "all_dup_genome"):
        assert c[cls] >= 1, (cls, c)
    assert r["N"] <= G.DUP_BLOCK and len(r["counts"]) >= 5      # one k_dups block over every genome
    # the first genome's table holds every survivor of the block (see the dup_genome_of note in the GPU suite)
    assert 2 * r["counts"][0] >= r["N"]


def test_table_family_reaches_its_classes():
    r = G.classify(G.batch("table"), 30)
    assert r["counts"][:3] == [1, 2, 3]
    assert r["classes"]["wrap"] >= 3 and r["classes"]["slot_collision_dup"] >= 1 and r["classes"]["low38_pair"] >= 3


def test_bounds_family_reaches_its_classes():
    b = G.batch("bounds")
    for c in (95, 96):
        r = G.classify(b, 30, c=c)
        starts = r["genome_starts"]
        for i in (255, 256, 257, 1023, 1024, 1025):
            assert i in starts, (i, starts)
        cls = r["classes"]
        assert cls["contig_close"] >= 3 and cls["zero_contig_genome"] >= 2 and cls["empty_genome"] >= 5
        assert r["counts"][0] == 0 and r["counts"][-1] == 0
        assert r["records_per_tile"] > G.REC_CHUNK and r["max_tile"] <= G.SLOT
        assert any(len(s) < 2 * b.k for s in b.contigs)
        # c = 95 takes the sorted front half, c = 96 the slotted one, without fallback
        assert r["launches"][False] == (1, 1)


@pytest.mark.parametrize("name,n", [("slot512", 512), ("slot513", 513)])
def test_slot_families(name, n):
    r = G.classify(G.batch(name), 30)
    assert r["max_tile"] == n and sorted(r["tiles"].tolist())[-2] < G.SLOT
    assert r["launches"] == ({False: (1, 1), True: (1, 1)} if n == G.SLOT else {False: (2, 2), True: (1, 1)})


@pytest.mark.parametrize("name,extra", [("cap", 0), ("cap1", 1)])
def test_cap_families(name, extra):
    b = G.batch(name)
    r = G.classify(b, 30)
    assert b.n_bases == G.CAP_TILES * G.TILE
    assert r["cap"] == b.n_bases // G.CAP_C + b.n_bases // (4 * G.CAP_C) + 65536 == 72088
    assert r["N"] == r["cap"] + extra and r["max_tile"] <= G.SLOT
    assert r["launches"] == ({False: (1, 1), True: (1, 1)} if extra == 0 else {False: (3, 2), True: (2, 1)})


@pytest.mark.parametrize("pseudotax", [True, False])
@pytest.mark.parametrize("name", G.FAMILIES)
def test_oracle_rows_follow_the_transcription(name, pseudotax):
    """sketch_genome of every genome == src/sketch.rs:590-614 over the oracle's own survivor list, at every min_spacing
    of the family (bounds also one contig per genome)."""
    b = G.batch(name)
    for ms in G.MS[name]:
        for individual in ((False, True) if name == "bounds" else (False,)):
            d = G.oracle_sketch(b, ms, pseudotax, individual)
            r = G.classify(b, ms, individual=individual)
            for g, (km, tr) in enumerate(zip(r["kept"], r["tracked"])):
                assert d["kmers"][d["kmer_off"][g]:d["kmer_off"][g + 1]].tolist() == km, (ms, g)
                assert d["tracked"][d["tracked_off"][g]:d["tracked_off"][g + 1]].tolist() == (tr if pseudotax else []), (ms, g)
                if r["counts"][g] == 0:   # empty genomes (no survivor, or no contig) have empty rows
                    assert not km and d["kmer_off"][g] == d["kmer_off"][g + 1]


@pytest.mark.parametrize("name", G.SMALL)
def test_oracle_equals_pyref(name):
    b = G.batch(name)
    for ms in G.MS[name]:
        d = G.oracle_sketch(b, ms)
        for g in range(len(b.genome_off) - 1):
            km, tr, gs = R.sketch_genome([b.contigs[ci] for ci in b.genome_contigs(g)], b.k, b.c, ms, True)
            assert d["kmers"][d["kmer_off"][g]:d["kmer_off"][g + 1]].tolist() == km
            assert d["tracked"][d["tracked_off"][g]:d["tracked_off"][g + 1]].tolist() == tr
            assert int(d["gn_size"][g]) == gs


def test_edge_oracle_rows():
    """Every edge record is its own genome: the kept hashes are its only k-mer, the dropped ones leave it empty."""
    for k, W, c in EDGES[:3] + EDGES[3:5]:
        b = G.edge_batch(k, W, c)
        d = G.oracle_sketch(b, 30, individual=True)
        for g, (lab, ok, o) in enumerate(b.labels):
            assert d["kmer_off"][g + 1] - d["kmer_off"][g] == (1 if ok else 0), (k, W, lab, o)
