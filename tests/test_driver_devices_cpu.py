"""CPU suite: `sylph-b200 --devices` argument errors, reported before any device is touched, and the split of samples
into one contiguous block per context (the hidden `sample-blocks` subcommand)."""
import subprocess

import numpy as np
import pytest

from tests.test_driver_cpu import exe  # noqa: F401  (fixture)


@pytest.mark.parametrize("args,msg", [
    (["query", "--device", "0", "--devices", "0,1", "r.fq", "g.fa"], "--device and --devices exclude each other"),
    (["profile", "--devices", "0,1", "--device", "1", "r.fq", "g.fa"], "--device and --devices exclude each other"),
    (["sketch", "--devices", "", "g.fa"], "--devices: empty device list"),
    (["query", "--devices", "0,x", "r.fq", "g.fa"], "`x` is not a device ordinal"),
    (["query", "--devices", "0,,1", "r.fq", "g.fa"], "`` is not a device ordinal"),
    (["sketch", "--devices", "1,", "g.fa"], "`` is not a device ordinal"),
    (["profile", "--devices", "-1", "r.fq", "g.fa"], "`-1` is not a device ordinal"),
    (["profile", "--devices", "0, 1", "r.fq", "g.fa"], "` 1` is not a device ordinal"),
    (["sketch", "g.fa", "--devices"], "missing value for --devices"),
])
def test_device_list_errors_before_the_device(exe, tmp_path, args, msg):  # noqa: F811
    r = subprocess.run([exe] + args, cwd=tmp_path, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 1 and msg in r.stderr and r.stdout == "", r.stderr


def blocks(exe, weights, n):  # noqa: F811
    out = subprocess.run([exe, "sample-blocks", "--devices", ",".join(["0"] * n)] + [str(w) for w in weights],
                         stdout=subprocess.PIPE, text=True, check=True, timeout=60).stdout
    return [tuple(int(x) for x in ln.split("\t")) for ln in out.splitlines()]


def check_blocks(b, weights, n):
    assert len(b) == n
    pos = 0
    for first, count, total in b:            # contiguous, in order, every sample once
        assert first == pos or count == 0
        assert total == sum(weights[first:first + count])
        pos = first + count if count else pos
    assert sum(c for _, c, _ in b) == len(weights) and pos == len(weights)
    if sum(weights):                         # balanced by weight: no block more than its share plus one sample
        assert max(t for _, _, t in b) <= sum(weights) / n + max(weights)
    else:                                    # no weights at all: balanced by count
        assert max(c for _, c, _ in b) - min(c for _, c, _ in b) <= 1


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_sample_blocks_random_weights(exe, n):  # noqa: F811
    rng = np.random.default_rng(n)
    for trial in range(20):
        m = int(rng.integers(0, 40))
        w = [int(x) for x in rng.integers(0, 10 ** int(rng.integers(1, 9)), m)]
        if trial % 5 == 0 and m:
            w[int(rng.integers(0, m))] *= 1000        # one sample far larger than the rest
        check_blocks(blocks(exe, w, n), w, n)


def test_sample_blocks_by_weight_not_count(exe):  # noqa: F811
    w = [1000, 1, 1, 1, 1, 1, 1, 1000]
    assert blocks(exe, w, 2) == [(0, 4, 1003), (4, 4, 1003)]
    w = [5000, 10, 10, 10, 10, 10]                   # the big sample alone, the rest together
    assert blocks(exe, w, 2) == [(0, 1, 5000), (1, 5, 50)]
    assert blocks(exe, [7], 1) == [(0, 1, 7)]


def test_sample_blocks_more_contexts_than_samples(exe):  # noqa: F811
    b = blocks(exe, [3, 3], 4)
    check_blocks(b, [3, 3], 4)
    assert sorted(c for _, c, _ in b) == [0, 0, 1, 1]
    assert blocks(exe, [], 3) == [(0, 0, 0)] * 3
    check_blocks(blocks(exe, [0, 0, 0, 0, 0], 2), [0] * 5, 2)
