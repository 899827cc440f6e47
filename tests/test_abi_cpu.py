"""CPU suite: the C-ABI library builds for sm_90a, loads, exports every symbol the header
declares, and refuses to work without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

from tests.util import REPO


def declared_symbols():
    hdr = open(os.path.join(REPO, "include", "sylph_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(syl_[a-z0-9_]+)\s*\(", hdr)))


def test_header_symbols_all_exported_and_bound():
    from sylph_b200 import _lib
    lib = _lib.lib()
    names = declared_symbols()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), "library does not export " + n
        assert n in _lib.SIGNATURES, "python binding misses " + n
    assert lib.syl_abi_version() == 2


def test_struct_layouts_match_header():
    from sylph_b200 import _lib
    from sylph_b200.api import ANI_ROW_DTYPE, SURVIVOR_DTYPE
    assert C.sizeof(_lib.Survivor) == SURVIVOR_DTYPE.itemsize == 16
    assert C.sizeof(_lib.AniRow) == ANI_ROW_DTYPE.itemsize == 144
    for (name, _), f in zip(_lib.AniRow._fields_, ANI_ROW_DTYPE.names):
        assert name.rstrip("_") == f
        assert getattr(_lib.AniRow, name).offset == ANI_ROW_DTYPE.fields[f][1]
    p = _lib.ContainParams()
    _lib.lib().syl_contain_params_default(C.byref(p), 31, 1)
    assert (p.k, p.pseudotax, p.min_number_kmers, p.min_count_correct, p.minimum_ani, p.redundant_ani) == (31, 1, 50.0, 3.0, -1.0, 99.0)
    assert (p.estimate_unknown, p.read_seq_id) == (0, -1.0) and C.sizeof(_lib.ContainParams) == 64


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import sylph_b200
    with pytest.raises(sylph_b200.SylphError) as e:
        sylph_b200.Context(0)
    assert e.value.code == 2  # SYL_ERR_CUDA
    assert "no CPU fallback" in str(e.value) or "CUDA" in str(e.value)


def test_product_never_imports_oracle():
    for root, _, files in os.walk(os.path.join(REPO, "sylph_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(root, f)).read()
                code = "\n".join(l for l in src.splitlines() if not l.strip().startswith(("#", "//", '"""', "*")))
                assert not re.search(r"(from|import)\s+oracle\b|#include\s+[\"<].*oracle|liboracle", code), os.path.join(root, f)


def test_sass_is_hopper_native():
    """cuobjdump evidence: sm_90a cubin, TMA bulk copy (UBLKCP) + mbarrier (SYNCS) in the seeding kernel."""
    import shutil
    import subprocess
    from sylph_b200 import build
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("no cuobjdump")
    build.build()
    obj = os.path.join(build.OBJ, "seed_k31_ev.o")  # k_seed<31, events> for the three run lengths
    out = subprocess.run([cuobjdump, "-sass", obj], stdout=subprocess.PIPE, text=True).stdout
    assert "sm_90a" in out or "SM90A" in out.upper()
    assert "UBLKCP" in out and "SYNCS" in out
