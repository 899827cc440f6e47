"""ctypes binding of include/sylph_b200.h.  Fails loudly if the CUDA library is missing: there
is no CPU fallback anywhere in this package."""
import ctypes as C
import os

from . import build as _build

_LIB = None


class Survivor(C.Structure):
    _fields_ = [("hash", C.c_uint64), ("rec", C.c_uint32), ("pos", C.c_uint32)]


class ContainParams(C.Structure):
    _fields_ = [
        ("k", C.c_int32), ("pseudotax", C.c_int32), ("no_ci", C.c_int32), ("no_adj", C.c_int32),
        ("mean_coverage", C.c_int32), ("estimate_unknown", C.c_int32),
        ("min_number_kmers", C.c_double), ("min_count_correct", C.c_double),
        ("minimum_ani", C.c_double), ("redundant_ani", C.c_double), ("read_seq_id", C.c_double),
    ]


class AniRow(C.Structure):
    _fields_ = [
        ("sample", C.c_uint32), ("genome", C.c_uint32), ("lambda_status", C.c_uint32),
        ("ci_valid", C.c_uint32), ("contain", C.c_uint64), ("glen", C.c_uint64),
        ("kmers_lost", C.c_int64), ("naive_ani", C.c_double), ("final_est_ani", C.c_double),
        ("final_est_cov", C.c_double), ("mean_cov", C.c_double), ("median_cov", C.c_double),
        ("lambda_", C.c_double), ("ci", C.c_double * 4), ("rel_abund", C.c_double),
        ("seq_abund", C.c_double), ("reserved", C.c_double),
    ]


class HostSamples(C.Structure):
    _fields_ = [
        ("hash", C.c_void_p), ("count", C.c_void_p), ("off", C.c_void_p), ("c", C.c_void_p),
        ("mean_read_length", C.c_void_p), ("n_samples", C.c_uint32), ("k", C.c_int),
    ]


assert C.sizeof(Survivor) == 16
assert C.sizeof(AniRow) == 144

SYL_OK, SYL_ERR_ARG, SYL_ERR_CUDA, SYL_ERR_OOM, SYL_ERR_CAPACITY, SYL_ERR_UNSUPPORTED = range(6)
MEM_HOST, MEM_DEVICE = 0, 1
SEM_SCALAR, SEM_AVX2 = 0, 1

# name -> (restype, argtypes); must list every symbol include/sylph_b200.h declares
_vp, _u64, _u32, _i, _d = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_double
_pp = C.POINTER(C.c_void_p)
_pu64 = C.POINTER(C.c_uint64)
SIGNATURES = {
    "syl_last_error": (C.c_char_p, []),
    "syl_abi_version": (_i, []),
    "syl_ctx_create": (_i, [_i, _vp, _pp]),
    "syl_ctx_destroy": (None, [_vp]),
    "syl_ctx_sync": (_i, [_vp]),
    "syl_ctx_launch_count": (_u64, [_vp]),
    "syl_ctx_enable_timing": (_i, [_vp, _i]),
    "syl_ctx_seed_kernel_time": (_i, [_vp, C.POINTER(C.c_double), _pu64, _pu64, _i]),
    "syl_ctx_kernel_time": (_i, [_vp, _i, C.POINTER(C.c_double), _pu64, _i]),
    "syl_ctx_device_bytes": (_i, [_vp, _pu64, _pu64, _i]),
    "syl_seed_batch": (_i, [_vp, _i, _vp, _u64, _vp, _u64, _i, _u64, _i, _i, _vp, _u64, _pu64]),
    "syl_seed_batch_packed2": (_i, [_vp, _i, _vp, _u64, _vp, _u64, _i, _u64, _i, _i, _vp, _u64, _pu64]),
    "syl_sketch_reads": (_i, [_vp, _i, _vp, _u64, _vp, _u64, _i, _u64, _i, _i, _pp]),
    "syl_sketch_reads_packed2": (_i, [_vp, _i, _vp, _u64, _vp, _u64, _i, _u64, _i, _i, _pp]),
    "syl_sketch_read_pairs": (_i, [_vp, _i, _vp, _u64, _vp, _vp, _u64, _vp, _u64, _i, _u64, _i, _i, _pp]),
    "syl_sketch_read_pairs_packed2": (_i, [_vp, _i, _vp, _u64, _vp, _vp, _u64, _vp, _u64, _i, _u64, _i, _i, _pp]),
    "syl_pack2": (_i, [_vp, _u64, _vp, _i]),
    "syl_pack_threads": (_i, []),
    "syl_ctx_ingest_stats": (_i, [_vp, _vp, _vp, _vp]),
    "syl_ctx_ingest_ring_bytes": (_i, [_vp, _pu64, _pu64]),
    "syl_ctx_set_sample_memory": (_i, [_vp, _u64]),
    "syl_ctx_sample_memory": (_i, [_vp, _pu64, _pu64]),
    "syl_ctx_sample_parts": (_i, [_vp, C.POINTER(C.c_uint32)]),
    "syl_sample_upload": (_i, [_vp, _i, _vp, _vp, _u64, _i, _u64, _pp]),
    "syl_sample_size": (_u64, [_vp]),
    "syl_sample_mean_read_length": (_d, [_vp]),
    "syl_sample_num_dup_removed": (_u64, [_vp]),
    "syl_sample_set_mean_read_length": (None, [_vp, _d]),
    "syl_sample_download": (_i, [_vp, _vp, _vp, _vp]),
    "syl_sample_device_ptrs": (_i, [_vp, _pp, _pp]),
    "syl_sample_free": (None, [_vp]),
    "syl_sketch_genomes": (_i, [_vp, _i, _vp, _u64, _vp, _u64, _vp, _u64, _i, _u64, _u64, _i, _i, _i, _pp]),
    "syl_sketch_genomes_packed2": (_i, [_vp, _i, _vp, _u64, _vp, _u64, _vp, _u64, _i, _u64, _u64, _i, _i, _i, _pp]),
    "syl_genomes_upload": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _u64, _i, _u64, _pp]),
    "syl_genomes_concat": (_i, [_vp, _pp, _u32, _pp]),
    "syl_genomes_count": (_u64, [_vp]),
    "syl_genomes_total_kmers": (_u64, [_vp]),
    "syl_genomes_total_tracked": (_u64, [_vp]),
    "syl_genomes_has_tracked": (_i, [_vp]),
    "syl_genomes_k": (_i, [_vp]),
    "syl_genomes_c": (_u64, [_vp]),
    "syl_genomes_download": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "syl_genomes_device_ptrs": (_i, [_vp, _pp, _pp, _pp, _pp, _pp]),
    "syl_genomes_free": (None, [_vp]),
    "syl_db_build": (_i, [_vp, _vp, _u32, _pp]),
    "syl_db_build_arrays": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _u64, _i, _u64, _u32, _pp]),
    "syl_db_download": (_i, [_vp, _vp, _vp, _vp, _vp, _pu64, _pu64]),
    "syl_db_num_genomes": (_u64, [_vp]),
    "syl_db_free": (None, [_vp]),
    "syl_contain_params_default": (None, [C.POINTER(ContainParams), _i, _i]),
    "syl_query": (_i, [_vp, _vp, _pp, _u32, C.POINTER(ContainParams), _vp, _u64, _pu64]),
    "syl_profile": (_i, [_vp, _vp, _pp, _u32, C.POINTER(ContainParams), _vp, _u64, _pu64]),
    "syl_profile_shard_begin": (_i, [_vp, _vp, _pp, _u32, C.POINTER(ContainParams), _u32, _u32, _u64, _i, _pp]),
    "syl_profile_job_buffers": (_i, [_vp, _pp, _pp, _pu64, _pp, _pu64, _pp, _pp]),
    "syl_profile_shard_rank": (_i, [_vp]),
    "syl_profile_shard_pass2": (_i, [_vp]),
    "syl_profile_shard_finish": (_i, [_vp, _vp, _u64, _pu64, _pu64]),
    "syl_profile_job_free": (None, [_vp]),
    "syl_db_shards_create": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _u64, _i, _u64, _u64, _pp]),
    "syl_db_shards_count": (_u64, [_vp]),
    "syl_db_shards_range": (_i, [_vp, _u64, _pu64, _pu64, _pu64]),
    "syl_query_shards": (_i, [_vp, _vp, _pp, _u32, C.POINTER(ContainParams), _vp, _u64, _pu64]),
    "syl_profile_shards": (_i, [_vp, _vp, _pp, _u32, C.POINTER(ContainParams), _vp, _u64, _pu64]),
    "syl_db_shards_free": (None, [_vp]),
    "syl_db_scan_plan": (_i, [_vp, _u64, _u64, _u64, _u32, _u64, C.POINTER(C.c_int)]),
    "syl_query_host_samples": (_i, [_vp, _vp, _vp, C.POINTER(HostSamples), C.POINTER(ContainParams), _vp, _u64, _pu64]),
    "syl_profile_host_samples": (_i, [_vp, _vp, _vp, C.POINTER(HostSamples), C.POINTER(ContainParams), _vp, _u64, _pu64]),
}


class SylphError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("sylph_b200 error %d: %s" % (code, msg))
        self.code = code


def lib():
    """Load (building first if the sources are newer) sylph_b200/libsylph_b200.so."""
    global _LIB
    if _LIB is not None:
        return _LIB
    so = os.environ.get("SYLPH_B200_LIB")  # tuning experiments only: an alternative build of the same sources
    if not so:
        so = _build.SO
        if _build.needs_build():
            so = _build.build()
    L = C.CDLL(so)  # raises OSError if missing: no fallback
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(L, name)  # AttributeError if the library lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    _LIB = L
    return L


def check(code):
    if code != SYL_OK:
        raise SylphError(code, lib().syl_last_error().decode(errors="replace"))
