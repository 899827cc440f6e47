"""CPU: `--max-sample-bytes` of `sylph-b200 query | profile` takes a positive number of bytes; anything else is refused
with exit code 1 while parsing, before a device or an input file is needed."""
import subprocess

import pytest

from tests.test_driver_cpu import exe  # noqa: F401  (fixture)


@pytest.mark.parametrize("cmd", ["query", "profile"])
@pytest.mark.parametrize("value", ["0", "abc", "-5", "12k", "1.5", "", "99999999999999999999"])
def test_bad_values_exit_1(exe, tmp_path, cmd, value):  # noqa: F811
    r = subprocess.run([exe, cmd, "--max-sample-bytes", value, "r.fq", "g.fa"], cwd=tmp_path, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 1 and "--max-sample-bytes" in r.stderr and r.stdout == "", r.stderr


def test_missing_value_exits_1(exe, tmp_path):  # noqa: F811
    r = subprocess.run([exe, "query", "--max-sample-bytes"], cwd=tmp_path, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=60)
    assert r.returncode == 1 and "missing value for --max-sample-bytes" in r.stderr


def test_good_value_passes_parsing(exe, tmp_path):  # noqa: F811
    """a valid value gets past the parser: whatever stops the run afterwards (no device here, or no genome files) is not
    an objection to the option"""
    r = subprocess.run([exe, "query", "--max-sample-bytes", "1", "r.fq"], cwd=tmp_path, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=60)
    assert "--max-sample-bytes" not in r.stderr, r.stderr
