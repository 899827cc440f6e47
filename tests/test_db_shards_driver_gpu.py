"""GPU: `sylph-b200 query | profile` through db shards (SYL_DRIVER_SHARD_ENTRIES, --max-db-entries) prints what the
one-index run prints, byte for byte: pre-sketched and raw inputs, -u, and two .syldb files given together."""
import os

import pytest

from tests.test_driver_gpu import GENOMES, SAMPLES, SK_PAIRS, SK_SAMPLES, d, exe, run, sk  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

CAPS = ["1", "3000", "12000", "4000000000"]   # db: 41 genomes, about 40 000 entries


def _shard_lines(stderr):
    return [ln for ln in stderr.splitlines() if "Database shard " in ln]


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_shard_hook_output_identical(exe, d, sk, cmd):  # noqa: F811
    args = [cmd] + SK_SAMPLES + SK_PAIRS + ["sk/db.syldb"]
    one = run(exe, args, d)
    assert not _shard_lines(one.stderr)
    assert len(one.stdout.splitlines()) > 10
    counts = []
    for cap in CAPS:
        r = run(exe, args, d, env={"SYL_DRIVER_SHARD_ENTRIES": cap})
        assert r.stdout == one.stdout, cap
        counts.append(len(_shard_lines(r.stderr)))
    assert counts[0] == len(GENOMES) and counts[0] > counts[1] > counts[2] > 1 and counts[3] == 1, counts


@pytest.mark.parametrize("cmd", ["query", "profile"])
def test_max_db_entries_option(exe, d, sk, cmd):  # noqa: F811
    """the option, on raw reads and genomes, and with -u -I on sketches"""
    for args in ([cmd] + SAMPLES + GENOMES, [cmd, "-u", "-I", "98.5"] + SK_SAMPLES + ["sk/db.syldb"]):
        one = run(exe, args, d).stdout
        r = run(exe, args[:1] + ["--max-db-entries", "10000"] + args[1:], d)
        assert r.stdout == one
        assert len(_shard_lines(r.stderr)) >= 3


def test_two_syldb_files(exe, d, sk):  # noqa: F811
    """two databases profiled together: the same rows through shards as through one index"""
    os.makedirs(os.path.join(d, "two"), exist_ok=True)
    run(exe, ["sketch", "-o", "two/a"] + GENOMES[:17], d)
    run(exe, ["sketch", "-o", "two/b"] + GENOMES[17:], d)
    for cmd in ("query", "profile"):
        args = [cmd] + SK_SAMPLES + SK_PAIRS + ["two/a.syldb", "two/b.syldb"]
        one = run(exe, args, d).stdout
        assert len(one.splitlines()) > 10
        for env in ({"SYL_DRIVER_SHARD_ENTRIES": "1"}, {"SYL_DRIVER_SHARD_ENTRIES": "5000"}):
            assert run(exe, args, d, env=env).stdout == one, env
        assert run(exe, [cmd, "--max-db-entries", "8000"] + args[1:], d).stdout == one
