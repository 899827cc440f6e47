"""CPU suite: scripted seeding batches (tests/seed_scripts.py).

The kernel's geometry comes from seed_kernel.cuh (built with nvcc, run on the host); every named batch reaches the
edge it is named for under every instantiation and run length it claims (the realised counts are printed against the
constants); no input can fill more runs than SEED_MAXRUNS; and the model's survivors are the C oracle's on every batch,
which pins the model's window and hash rules."""
import pytest

from tests import seed_scripts as S

NAMES = S.names()


def _id(n):
    return "%s-k%d-%s" % n


def test_constants_come_from_the_kernel():
    C = S.constants()
    for key in ("SEED_TILE", "SEED_THREADS", "SEED_HALO", "SEED_STAGE", "SEED_CAND", "SEED_W_MIN", "SEED_MAXRUNS",
                "SEED_NCHUNK16"):
        assert key in C
    assert C["SEED_NCHUNK16"] * 16 == C["SEED_TILE"] + C["SEED_HALO"]
    assert C["SEED_THREADS"] <= 256      # cand entries keep the record slot in 8 bits
    print("\n" + " ".join("%s=%d" % kv for kv in sorted(C.items())))


def test_no_input_exceeds_the_run_table():
    """A chunk of SEED_THREADS records with n_i >= 1 windows inside the tile (sum <= SEED_TILE) has
    sum ceil(n_i / W) <= SEED_THREADS + (SEED_TILE - SEED_THREADS) // W runs, at most SEED_MAXRUNS at every W; the
    fullest table a real chunk can hold (each record but the last costs k - 1 bases past its windows) is below that."""
    C = S.constants()
    for W in S.run_lengths():
        bound = C["SEED_THREADS"] + (C["SEED_TILE"] - C["SEED_THREADS"]) // W
        assert bound <= C["SEED_MAXRUNS"], (W, bound)
        for k in (21, 31):
            assert S.fullest_runs(k, W) <= bound


@pytest.mark.parametrize("name", NAMES, ids=_id)
def test_batch_reaches_its_edge(name, capsys):
    b = S.batch(*name)
    cases = S.claim_cases(b)
    assert cases, b
    seen = {}
    bad = []
    for W, inst, label, ok, v in cases:
        key = (label, v)
        seen.setdefault(key, set()).add("W%d/e%d/s%d/p%d%s%s" % (W, inst["emit"], inst["sem"], inst["with_pos"],
                                                              "/pairs" if inst["paired"] else "",
                                                              "/nodedup" if inst["no_dedup"] else ""))
        if not ok:
            bad.append((W, {k: v for k, v in inst.items() if not k.startswith("_")}, label, v))
    with capsys.disabled():
        print("\n%r" % b)
        for (label, v), where in sorted(seen.items(), key=lambda x: x[0][0]):
            print("    %-48s %-14s in %d instantiations" % (label, v, len(where)))
    assert not bad, bad[:5]
    labels = {cl[0] for cl in b.claims if cl[3] is not None}
    assert labels <= {c[2] for c in cases if c[3]}, labels - {c[2] for c in cases}


@pytest.mark.parametrize("name", NAMES, ids=_id)
def test_model_survivors_are_the_oracles(name):
    b = S.batch(*name)
    for sem in (0, 1):
        for with_pos in (0, 1):
            m = S.survivors(b, sem, with_pos)
            if not with_pos:
                m = sorted((r, 0, h) for r, _, h in m)
            assert m == S.oracle_survivors(b, sem, with_pos), (sem, with_pos)
    if b.family == "parts":
        C = S.constants()
        assert sum(t["staged"] for t in S.model(b, 32, dict(emit=1, sem=1, with_pos=0, no_dedup=0, paired=False,
                                                                 part=None))) > C["SEED_STAGE"]
