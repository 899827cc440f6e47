"""ctypes binding of the CPU oracle (oracle/sylph_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs. The product package (sylph_b200/) never imports this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

SEM_SCALAR = 0
SEM_AVX2 = 1
SEM_AVX2_INTRIN = 2


class Params(C.Structure):
    _fields_ = [
        ("k", C.c_int),
        ("min_number_kmers", C.c_double),
        ("min_count_correct", C.c_double),
        ("minimum_ani", C.c_double),
        ("pseudotax", C.c_int),
        ("no_ci", C.c_int),
        ("no_adj", C.c_int),
        ("mean_coverage", C.c_int),
        ("redundant_ani", C.c_double),
        ("cr_math", C.c_int),                        # 1: the ANI's pow / exp correctly rounded (sylph_oracle.h)
        ("cr_undecided", C.POINTER(C.c_uint64)),     # set per call by _decided
    ]


class AniResult(C.Structure):
    _fields_ = [
        ("genome", C.c_uint32),
        ("lambda_status", C.c_uint32),
        ("contain", C.c_uint64),
        ("glen", C.c_uint64),
        ("kmers_lost", C.c_int64),
        ("naive_ani", C.c_double),
        ("final_est_ani", C.c_double),
        ("final_est_cov", C.c_double),
        ("mean_cov", C.c_double),
        ("median_cov", C.c_double),
        ("lambda_", C.c_double),
        ("ci", C.c_double * 4),
        ("ci_valid", C.c_uint32),
        ("pad", C.c_uint32),
        ("rel_abund", C.c_double),
        ("seq_abund", C.c_double),
    ]

    def as_dict(self):
        d = {f: getattr(self, f) for f, _ in self._fields_ if f not in ("ci", "pad")}
        d["ci"] = list(self.ci)
        return d


def default_params(k=31, pseudotax=False, **kw):
    """the reference's defaults; cr_math=1 rounds the ANI's pow / exp correctly (as the device does) instead of
    calling glibc"""
    p = Params(k=k, min_number_kmers=50.0, min_count_correct=3.0, minimum_ani=-1.0,
               pseudotax=int(pseudotax), no_ci=0, no_adj=0, mean_coverage=0, redundant_ani=99.0, cr_math=0)
    for a, b in kw.items():
        setattr(p, a, b)
    return p


def build(force=False):
    """Compile oracle/liboracle.so with the committed Makefile (gcc, -O3 -fopenmp)."""
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "sylph_oracle.c")
    hdr = os.path.join(_HERE, "sylph_oracle.h")
    if force or not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        env = dict(os.environ)
        env.pop("CC", None)
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], env=env,
                              stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    so = build()
    L = C.CDLL(so)
    u8p, u64p, u32p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)
    L.syo_mm_hash64.restype = C.c_uint64
    L.syo_mm_hash64.argtypes = [C.c_uint64]
    L.syo_byte_to_seq.restype = C.c_uint8
    L.syo_byte_to_seq.argtypes = [C.c_uint8]
    L.syo_extract_markers.restype = C.c_size_t
    L.syo_extract_markers.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_uint64, C.c_int, C.c_void_p, C.c_size_t]
    L.syo_extract_markers_positions.restype = C.c_size_t
    L.syo_extract_markers_positions.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_uint64, C.c_int,
                                                C.c_void_p, C.c_void_p, C.c_size_t]
    L.syo_extract_markers_avx2_intrin.restype = C.c_size_t
    L.syo_extract_markers_avx2_intrin.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_uint64, C.c_void_p, C.c_size_t]
    L.syo_sketch_genome.restype = C.c_int
    L.syo_sketch_genome.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_uint64, C.c_uint64, C.c_int,
                                    C.c_int, C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p,
                                    C.POINTER(C.c_size_t), C.c_size_t, C.POINTER(C.c_uint64)]
    L.syo_sketch_reads.restype = C.c_int
    L.syo_sketch_reads.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_uint64, C.c_int, C.c_int,
                                   C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t), C.c_size_t,
                                   C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
    L.syo_sketch_read_pairs.restype = C.c_int
    L.syo_sketch_read_pairs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_uint64, C.c_int,
                                        C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t), C.c_size_t,
                                        C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
    L.syo_sample_new.restype = C.c_void_p
    L.syo_sample_new.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.syo_sample_free.restype = None
    L.syo_sample_free.argtypes = [C.c_void_p]
    L.syo_get_stats.restype = C.c_int
    L.syo_get_stats.argtypes = [C.POINTER(Params), C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32,
                                C.POINTER(AniResult)]
    L.syo_contain_sample.restype = C.c_int64
    L.syo_contain_sample.argtypes = [C.POINTER(Params), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
    L.syo_contain_sample_unknown.restype = C.c_int64
    L.syo_contain_sample_unknown.argtypes = [C.POINTER(Params), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
    L.syo_poisson_cutoff.restype = C.c_uint32
    L.syo_poisson_cutoff.argtypes = [C.c_uint32]
    L.syo_fastrand_usize.restype = C.c_uint64
    L.syo_fastrand_usize.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64]
    L.syo_format_row.restype = C.c_int
    L.syo_format_row.argtypes = [C.POINTER(AniResult), C.c_int, C.c_char_p, C.c_char_p, C.c_char_p,
                                 C.c_char_p, C.c_size_t]
    _LIB = L
    return L


def _u8(a):
    a = np.ascontiguousarray(np.frombuffer(a, dtype=np.uint8) if isinstance(a, (bytes, bytearray)) else a,
                             dtype=np.uint8)
    return a


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def mm_hash64(x):
    return int(lib().syo_mm_hash64(C.c_uint64(int(x) & (2**64 - 1))))


def extract_markers(seq, k=31, c=200, sem=SEM_AVX2):
    s = _u8(seq)
    cap = max(64, len(s) // 16 + 64)
    while True:
        out = np.empty(cap, dtype=np.uint64)
        n = lib().syo_extract_markers(_ptr(s), len(s), k, c, sem, _ptr(out), cap)
        if n == 2**64 - 1:
            raise ValueError("unsupported k for AVX2 semantics")
        if n <= cap:
            return out[:n].copy()
        cap = n


def extract_markers_positions(seq, k=31, c=200, sem=SEM_AVX2):
    s = _u8(seq)
    cap = max(64, len(s) // 16 + 64)
    while True:
        pos = np.empty(cap, dtype=np.uint64)
        out = np.empty(cap, dtype=np.uint64)
        n = lib().syo_extract_markers_positions(_ptr(s), len(s), k, c, sem, _ptr(pos), _ptr(out), cap)
        if n == 2**64 - 1:
            raise ValueError("unsupported k for AVX2 semantics")
        if n <= cap:
            return pos[:n].copy(), out[:n].copy()
        cap = n


def extract_markers_avx2_intrin(seq, k=31, c=200):
    s = _u8(seq)
    cap = max(64, len(s) // 16 + 64)
    while True:
        out = np.empty(cap, dtype=np.uint64)
        n = lib().syo_extract_markers_avx2_intrin(_ptr(s), len(s), k, c, _ptr(out), cap)
        if n == 2**64 - 1:
            raise RuntimeError("AVX2 unavailable")
        if n <= cap:
            return out[:n].copy()
        cap = n


def sketch_genome(bases, contig_off, k=31, c=200, min_spacing=30, pseudotax=True, sem=SEM_AVX2):
    """-> (genome_kmers, tracked, gn_size)"""
    b = _u8(bases)
    off = np.ascontiguousarray(contig_off, dtype=np.uint64)
    cap = max(1024, len(b) // 16 + 1024)
    while True:
        km = np.empty(cap, dtype=np.uint64)
        tr = np.empty(cap, dtype=np.uint64)
        nk, nt, gs = C.c_size_t(0), C.c_size_t(0), C.c_uint64(0)
        rc = lib().syo_sketch_genome(_ptr(b), _ptr(off), len(off) - 1, k, c, min_spacing, int(pseudotax), sem,
                                     _ptr(km), C.byref(nk), _ptr(tr), C.byref(nt), cap, C.byref(gs))
        if rc == 2:
            raise ValueError("unsupported k")
        if rc == 0:
            return km[:nk.value].copy(), tr[:nt.value].copy(), gs.value
        cap = max(nk.value, nt.value) + 16


def sketch_reads(bases, rec_off, k=31, c=200, no_dedup=False, sem=SEM_AVX2, nthreads=1):
    """-> (hash sorted, count, mean_read_length, num_dup_removed)"""
    b = _u8(bases)
    off = np.ascontiguousarray(rec_off, dtype=np.uint64)
    cap = max(1024, len(b) // 16 + 1024)
    while True:
        h = np.empty(cap, dtype=np.uint64)
        ct = np.empty(cap, dtype=np.uint32)
        n, mean, nd = C.c_size_t(0), C.c_double(0), C.c_uint64(0)
        rc = lib().syo_sketch_reads(_ptr(b), _ptr(off), len(off) - 1, k, c, int(no_dedup), sem, nthreads,
                                    _ptr(h), _ptr(ct), C.byref(n), cap, C.byref(mean), C.byref(nd))
        if rc == 2:
            raise ValueError("unsupported k")
        if rc == 0:
            return h[:n.value].copy(), ct[:n.value].copy(), mean.value, nd.value
        cap = n.value + 16


def sketch_read_pairs(bases1, off1, bases2, off2, k=31, c=200, no_dedup=False, sem=SEM_AVX2):
    """sketch_pair_sequences with --fpr 0 (src/sketch.rs:771-895) -> (hash sorted, count, mean_read_length, num_dup_removed)"""
    b1, b2 = _u8(bases1), _u8(bases2)
    o1 = np.ascontiguousarray(off1, dtype=np.uint64)
    o2 = np.ascontiguousarray(off2, dtype=np.uint64)
    n_pairs = min(len(o1), len(o2)) - 1
    cap = max(1024, (len(b1) + len(b2)) // 16 + 1024)
    while True:
        h = np.empty(cap, dtype=np.uint64)
        ct = np.empty(cap, dtype=np.uint32)
        n, mean, nd = C.c_size_t(0), C.c_double(0), C.c_uint64(0)
        rc = lib().syo_sketch_read_pairs(_ptr(b1), _ptr(o1), _ptr(b2), _ptr(o2), n_pairs, k, c, int(no_dedup), sem,
                                         _ptr(h), _ptr(ct), C.byref(n), cap, C.byref(mean), C.byref(nd))
        if rc == 2:
            raise ValueError("unsupported k")
        if rc == 0:
            return h[:n.value].copy(), ct[:n.value].copy(), mean.value, nd.value
        cap = n.value + 16


class Sample:
    def __init__(self, hashes, counts):
        h = np.ascontiguousarray(hashes, dtype=np.uint64)
        c = np.ascontiguousarray(counts, dtype=np.uint32)
        self._h = lib().syo_sample_new(_ptr(h), _ptr(c), len(h))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().syo_sample_free(self._h)
            self._h = None


def _decided(params, call):
    """call(params) with a private undecided-call counter under cr_math; raises if any ANI call fell within 2^-100 of
    a rounding midpoint, where the correctly rounded value is not known from the quad result"""
    if not params.cr_math:
        return call(params)
    n = C.c_uint64(0)
    p = Params.from_buffer_copy(params)
    p.cr_undecided = C.pointer(n)
    out = call(p)
    if n.value:
        raise ValueError("%d ANI pow / exp calls lie too close to a rounding midpoint to be rounded correctly" % n.value)
    return out


def get_stats(params, genome_kmers, sample, genome_index=0):
    g = np.ascontiguousarray(genome_kmers, dtype=np.uint64)
    r = AniResult()
    ok = _decided(params, lambda p: lib().syo_get_stats(C.byref(p), _ptr(g), len(g), sample._h, genome_index, C.byref(r)))
    return r if ok else None


class Unknown(C.Structure):
    """-u with --read-seq-id: (read identity %, the sample's mean read length, the sample's c)"""
    _fields_ = [("read_seq_id", C.c_double), ("mean_read_length", C.c_double), ("sample_c", C.c_uint64)]


def contain_sample(params, kmers, kmer_off, tracked, tracked_off, gn_size, sample, nthreads=1, unknown=None):
    kmers = np.ascontiguousarray(kmers, dtype=np.uint64)
    kmer_off = np.ascontiguousarray(kmer_off, dtype=np.uint64)
    tr = np.ascontiguousarray(tracked, dtype=np.uint64) if tracked is not None else None
    tro = np.ascontiguousarray(tracked_off, dtype=np.uint64) if tracked_off is not None else None
    gs = np.ascontiguousarray(gn_size, dtype=np.uint64)
    n = len(kmer_off) - 1
    out = (AniResult * max(n, 1))()
    if unknown is not None:
        m = _decided(params, lambda p: lib().syo_contain_sample_unknown(
            C.byref(p), _ptr(kmers), _ptr(kmer_off), _ptr(tr), _ptr(tro), _ptr(gs), n, sample._h, nthreads, out, max(n, 1),
            C.byref(unknown)))
    else:
        m = _decided(params, lambda p: lib().syo_contain_sample(
            C.byref(p), _ptr(kmers), _ptr(kmer_off), _ptr(tr), _ptr(tro), _ptr(gs), n, sample._h, nthreads, out, max(n, 1)))
    assert m >= 0
    return [out[i] for i in range(m)]


def poisson_cutoff(median):
    return int(lib().syo_poisson_cutoff(median))


def fastrand_usize(seed, n_draw, rng):
    return int(lib().syo_fastrand_usize(seed, n_draw, rng))


def format_row(r, pseudotax, seq_name, gn_name, contig_name):
    buf = C.create_string_buffer(4096)
    lib().syo_format_row(C.byref(r), int(pseudotax), seq_name.encode(), gn_name.encode(), contig_name.encode(),
                         buf, 4096)
    return buf.value.decode()
