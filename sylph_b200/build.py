"""Build the sm_90a shared library in-tree (sylph_b200/libsylph_b200.so).

nvcc cross-compiles without a GPU; the .so is a build product and is git-ignored.
Each .cu is compiled to build/<name>.o (in parallel, only when stale) and the
objects are linked into the .so.  `python -m sylph_b200.build [-v] [-f]`.
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
SO = os.path.join(HERE, "libsylph_b200.so")
HEADER = os.path.join(HERE, "..", "include", "sylph_b200.h")
SOURCES = ["api.cu", "seed.cu", "seed_k31_sv.cu", "seed_k31_ev.cu", "seed_k21_sv.cu", "seed_k21_ev.cu",
           "sample.cu", "genome.cu", "contain.cu", "host_pack.cpp"]
CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC", "-pthread"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


# tuning experiments: extra -D flags and an alternative output name (SYL_BUILD_DEFS="-DSEED_MINB_CFG=3"
# SYL_BUILD_TAG=minb3 -> libsylph_b200_minb3.so, objects under build_minb3/), loaded with SYLPH_B200_LIB
EXTRA_NVCC = os.environ.get("SYL_BUILD_DEFS", "").split()
_TAG = os.environ.get("SYL_BUILD_TAG", "")
if _TAG:
    OBJ = os.path.join(HERE, "build_" + _TAG)
    SO = os.path.join(HERE, "libsylph_b200_%s.so" % _TAG)


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _sources():
    return [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def _headers_mtime():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h", ".hpp"))] + [HEADER]
    return max(os.path.getmtime(h) for h in hs)


def _stale(src, obj, hm):
    return (not os.path.exists(obj)) or os.path.getmtime(obj) < max(os.path.getmtime(src), hm)


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    if os.path.getmtime(os.path.abspath(__file__)) > t:  # source list / flags changed
        return True
    if any(not os.path.exists(os.path.join(OBJ, os.path.splitext(s)[0] + ".o")) for s in _sources()):
        return True
    return _headers_mtime() > t or any(os.path.getmtime(os.path.join(CSRC, s)) > t for s in _sources())


def _run(cmd, verbose):
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout)
    if r.returncode != 0:
        raise RuntimeError("command failed: " + " ".join(cmd))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    os.makedirs(OBJ, exist_ok=True)
    # one builder at a time (torchrun starts N ranks that all import the package): the others wait
    # on the lock and then find the library up to date
    import fcntl
    with open(os.path.join(OBJ, ".lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not needs_build():
                return SO
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(force, verbose):
    nvcc = _nvcc()
    hm = _headers_mtime()
    jobs, objs = [], []
    for s in _sources():
        src, obj = os.path.join(CSRC, s), os.path.join(OBJ, os.path.splitext(s)[0] + ".o")
        objs.append(obj)
        if force or _stale(src, obj, hm):
            if s.endswith(".cpp"):  # host-only code (thread pool, AVX2 packer): plain g++
                jobs.append([os.environ.get("SYL_CXX", "g++")] + CXX_FLAGS + ["-c", src, "-o", obj])
            else:
                jobs.append([nvcc] + NVCC_FLAGS + EXTRA_NVCC + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj])
    with ThreadPoolExecutor(max_workers=8) as ex:
        list(ex.map(lambda c: _run(c, verbose), jobs))
    tmp = SO + ".tmp.%d" % os.getpid()
    _run([nvcc, "-shared", "-o", tmp] + objs + ["-lpthread"], verbose)
    os.replace(tmp, SO)  # atomic: a process that already mapped the old file keeps it
    return SO


if __name__ == "__main__":
    build(force="-f" in sys.argv, verbose="-v" in sys.argv)
    print(SO)
