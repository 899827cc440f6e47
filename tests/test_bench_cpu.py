"""CPU suite: the parts of bench.py that need no GPU — the reference arm's JSON line (bench contract)
and the helpers around it."""
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_contract_line():
    r = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1",
                        "--reads", "40000"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600, cwd=REPO)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "bases/s sketched" and d["unit"] == "bases/s"
    assert d["higher_is_better"] is True and d["vs_baseline"] is None and d["n_gpus"] == 1
    assert d["value"] > 0 and d["steps"] == 1 and d["warmup"] == 1 and d["ms_per_step"] > 0
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"]


def test_reference_arm_profile_workload():
    r = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference", "--workload", "profile", "--steps", "1",
                        "--warmup", "1", "--reads", "20000", "--genomes", "3"], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=600, cwd=REPO)
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads([l for l in r.stdout.splitlines() if l.strip()][-1])
    assert d["impl"] == "reference" and d["unit"] == "pairs/s" and d["value"] > 0
    assert d["config"]["genomes_per_gpu"] == 3 and d["cpu_baseline"]["value"] == d["value"]


def test_both_arms_share_the_config_object():
    sys.path.insert(0, REPO)
    import bench

    class A:
        reads, genomes, samples = 1000, 7, None
    assert bench.sketch_config(A) == bench.sketch_config(A) and set(bench.sketch_config(A)) >= {"workload", "reads_per_gpu", "k", "c"}
    assert bench.profile_config(A, 1)["samples"] == 1 and bench.profile_config(A, 8)["samples"] == 16


def test_output_dump_is_exact_seeded_and_bounded(tmp_path):
    """--dump-outputs: u64 hashes survive as float64 halves, long arrays are sampled at the same rows every time."""
    import numpy as np
    sys.path.insert(0, REPO)
    import bench
    h = np.sort(np.random.default_rng(7).integers(0, 2**63, bench.DUMP_MAX_ROWS + 5, dtype=np.uint64))
    for d in (tmp_path / "a", tmp_path / "b"):
        dump = bench.OutputDump(str(d))
        dump.add("hash", h)
        dump.add("count", np.arange(10, dtype=np.uint32))
    a = {p.name: np.load(p) for p in (tmp_path / "a").iterdir()}
    assert set(a) == {"hash_hi.npy", "hash_lo.npy", "count.npy"} and all(x.dtype == np.float64 for x in a.values())
    back = (a["hash_hi.npy"].astype(np.uint64) << np.uint64(32)) | a["hash_lo.npy"].astype(np.uint64)
    assert len(back) == bench.DUMP_MAX_ROWS and np.all(np.isin(back, h)) and np.all(back[1:] > back[:-1])
    assert all(np.array_equal(x, np.load(tmp_path / "b" / n)) for n, x in a.items())
    assert a["count.npy"].tolist() == list(range(10))
    big = bench.OutputDump(str(tmp_path / "c"))
    try:
        for i in range(9):
            big.add("x%d" % i, np.zeros(bench.DUMP_MAX_ROWS, np.uint32))
        raise AssertionError("the 64 MB bound was not enforced")
    except SystemExit:
        pass
    assert not bench.OutputDump(None)


def test_clock_sampler_degrades_without_a_gpu():
    sys.path.insert(0, REPO)
    import bench
    c = bench.ClockSampler(0)   # no NVML device and no nvidia-smi in this container: both fallbacks are taken
    c.start()
    out = c.stop()
    assert set(out) >= {"sm_mhz", "sm_max_mhz", "reasons"}
    assert out["sm_mhz"] is None or out["sm_mhz"] > 0
    off = bench.ClockSampler(None)
    off.start()
    assert off.stop() == {}
