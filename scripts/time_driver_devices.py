"""Wall time of `sylph-b200 sketch` over N generated read files and of `profile` of N samples against a generated
database, at one context and with --devices LIST (default 0,0: two contexts on one GPU, where the gain can only be the
overlap of host parsing with GPU work).  Runs are alternated (one-context, LIST, one-context, ...) and every run's time
is printed, so the spread is visible next to the difference.  Outputs of both settings are compared byte for byte.

  python scripts/time_driver_devices.py [--files 16] [--reads 200000] [--genomes 200] [--devices 0,0] [--reps 3]

Reads the GPU name and power limit (nvidia-smi, query only) so that the numbers can be stated with them."""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def write_inputs(d, n_files, n_reads, n_genomes):
    import torch
    from sylph_b200 import synth
    lut = np.frombuffer(b"ACGT", np.uint8)
    glen = 200_000
    genomes = []
    for g in range(n_genomes):
        s = lut[synth.genome_codes(g, torch.arange(glen, dtype=torch.int64)).numpy()].tobytes()
        name = os.path.join(d, "g%04d.fa" % g)
        with open(name, "wb") as f:
            f.write(b">g%d\n" % g + b"\n".join(s[i:i + 80] for i in range(0, len(s), 80)) + b"\n")
        genomes.append(name)
    samples = []
    for i in range(n_files):
        b, o = synth.reads(n_reads, 150, n_comm=min(n_genomes, 64), genome_len=glen, seed=1000 + i)
        b, o = b.numpy(), o.numpy()
        name = os.path.join(d, "s%03d.fq" % i)
        with open(name, "wb") as f:
            for r in range(n_reads):
                seq = b[o[r]:o[r + 1]].tobytes()
                f.write(b"@r%d\n%s\n+\n%s\n" % (r, seq, b"I" * len(seq)))
        samples.append(name)
    return genomes, samples


def timed(cmd, cwd):
    t0 = time.perf_counter()
    r = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=3600)
    dt = time.perf_counter() - t0
    if r.returncode != 0:
        raise SystemExit("failed: %s\n%s" % (" ".join(cmd), r.stderr.decode()[-2000:]))
    return dt, r.stdout


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=16)
    ap.add_argument("--reads", type=int, default=200_000)
    ap.add_argument("--genomes", type=int, default=200)
    ap.add_argument("--devices", default="0,0")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", default="3")
    a = ap.parse_args()
    exe = os.path.join(ROOT, "host", "sylph-b200")
    print("GPUs:", gpu_info().replace("\n", "; "))
    d = tempfile.mkdtemp(prefix="time_driver_devices_")
    try:
        genomes, samples = write_inputs(d, a.files, a.reads, a.genomes)
        subprocess.run([exe, "sketch", "-o", "db"] + genomes, cwd=d, check=True, stderr=subprocess.DEVNULL, timeout=3600)
        settings = [("1 context", []), ("--devices " + a.devices, ["--devices", a.devices])]
        times = {n: {"sketch": [], "profile": []} for n, _ in settings}
        outs = {}
        for rep in range(a.reps + 1):              # rep 0 warms the page cache and the driver; not reported
            for name, extra in settings:
                out_dir = os.path.join(d, "sk_%d" % len(outs))
                dt_s, _ = timed([exe, "sketch", "-t", a.threads, "-d", out_dir] + extra + samples, d)
                dt_p, tsv = timed([exe, "profile", "-t", a.threads] + extra + samples + ["db.syldb"], d)
                files = {f: open(os.path.join(out_dir, f), "rb").read() for f in sorted(os.listdir(out_dir))}
                outs[(rep, name)] = (files, tsv)
                shutil.rmtree(out_dir)
                if rep:
                    times[name]["sketch"].append(dt_s)
                    times[name]["profile"].append(dt_p)
        ref = outs[(0, settings[0][0])]
        assert all(v == ref for v in outs.values()), "outputs differ between settings"
        for name, _ in settings:
            for what in ("sketch", "profile"):
                t = times[name][what]
                print("%-22s %-8s %d files: %s s (min %.2f, max %.2f)" % (name, what, a.files, " ".join("%.2f" % x for x in t),
                                                                        min(t), max(t)))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
