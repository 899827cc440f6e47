"""Host-side mirror of the reference's operator interface for the two hot paths, over the C ABI.

Names follow the reference (extract_markers, sketch_genome, sketch_sequences, get_stats/query/
profile); the only change is granularity: every call takes a *batch* (flat base buffer + record
offsets) because a GPU call per record / per pair would be pure launch overhead.

Inputs may be numpy arrays (host memory, copied inside the call) or torch CUDA tensors (device
memory, zero-copy).  torch is plumbing only (device buffers / streams); it is imported lazily.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import SEM_AVX2, SEM_SCALAR, AniRow, ContainParams, Survivor, SylphError  # noqa: F401

SURVIVOR_DTYPE = np.dtype([("hash", "<u8"), ("rec", "<u4"), ("pos", "<u4")])
ANI_ROW_DTYPE = np.dtype([
    ("sample", "<u4"), ("genome", "<u4"), ("lambda_status", "<u4"), ("ci_valid", "<u4"),
    ("contain", "<u8"), ("glen", "<u8"), ("kmers_lost", "<i8"), ("naive_ani", "<f8"),
    ("final_est_ani", "<f8"), ("final_est_cov", "<f8"), ("mean_cov", "<f8"), ("median_cov", "<f8"),
    ("lambda", "<f8"), ("ci", "<f8", (4,)), ("rel_abund", "<f8"), ("seq_abund", "<f8"), ("reserved", "<f8")])
assert ANI_ROW_DTYPE.itemsize == 144


def _is_torch(x):
    return type(x).__module__.startswith("torch")


_CTX_STREAM = [0]  # stream of the Context currently issuing a call (set by Context._enter)


def _arg(x, dtype):
    """-> (mem, pointer, n, keepalive)"""
    if x is None:
        return None, None, 0, None
    if _is_torch(x):
        if not x.is_cuda:
            x = x.numpy()
        else:
            import torch
            # a producer on torch's current stream must be finished before the library's stream reads
            # the tensor, unless the Context was created on that very stream
            cur = torch.cuda.current_stream(x.device)
            if cur.cuda_stream != _CTX_STREAM[0]:
                cur.synchronize()
            want = {np.uint8: torch.uint8, np.uint64: torch.int64, np.uint32: torch.int32}[dtype]
            if x.dtype not in (want, getattr(torch, np.dtype(dtype).name, want)):
                raise TypeError("expected tensor of %s-compatible dtype, got %s" % (np.dtype(dtype).name, x.dtype))
            if not x.is_contiguous():
                x = x.contiguous()
            return _lib.MEM_DEVICE, C.c_void_p(x.data_ptr()), x.numel(), x
    a = np.ascontiguousarray(x, dtype=dtype)
    return _lib.MEM_HOST, a.ctypes.data_as(C.c_void_p), a.size, a


class Context:
    """One CUDA device + one stream (syl_ctx)."""

    def __init__(self, device=0, stream=None):
        self._h = C.c_void_p()
        L = _lib.lib()
        _lib.check(L.syl_ctx_create(int(device), C.c_void_p(stream) if stream else None, C.byref(self._h)))
        self.device = device
        self._stream = int(stream) if stream else -1

    def close(self):
        if self._h:
            _lib.lib().syl_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        _lib.check(_lib.lib().syl_ctx_sync(self._h))

    @property
    def launches(self):
        return int(_lib.lib().syl_ctx_launch_count(self._h))

    def enable_timing(self, on=True):
        _lib.check(_lib.lib().syl_ctx_enable_timing(self._h, int(on)))

    def seed_kernel_time(self, reset=True):
        """-> (total_ms, launches, bases) of the seeding kernel since the last reset (CUDA events
        on the ctx stream, recorded inside the library around each launch)."""
        ms, n, b = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
        _lib.check(_lib.lib().syl_ctx_seed_kernel_time(self._h, C.byref(ms), C.byref(n), C.byref(b), int(reset)))
        return ms.value, n.value, b.value

    KERNELS = {"seed": 0, "group_dedup": 1, "join": 2, "join2": 3, "stats": 4, "boot": 5, "genome_post": 6, "pack": 7}

    def ingest_stats(self):
        """-> (h2d_bytes, chunks_packed, chunks_ascii) of the last host-memory sketch_sequences call."""
        a, b, c = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        _lib.check(_lib.lib().syl_ctx_ingest_stats(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def kernel_time(self, which, reset=True):
        """-> (total_ms, launches) of kernel class `which` (name in Context.KERNELS) since the last reset."""
        ms, n = C.c_double(0), C.c_uint64(0)
        _lib.check(_lib.lib().syl_ctx_kernel_time(self._h, self.KERNELS[which], C.byref(ms), C.byref(n), int(reset)))
        return ms.value, n.value

    # ---- (1) seeding -------------------------------------------------------------------------
    def extract_markers_batch(self, bases, rec_off, k=31, c=200, sem=SEM_AVX2, with_pos=False, cap=None,
                              out=None, packed_bases=None):
        """Batched extract_markers / extract_markers_positions (src/sketch.rs:53-93).
        Returns a numpy structured array (hash, rec, pos) in unspecified order, or — when `out`
        is a torch CUDA tensor of >= cap*16 bytes — the survivor count (survivors stay on device)."""
        _CTX_STREAM[0] = self._stream
        L = _lib.lib()
        fn = L.syl_seed_batch
        if packed_bases is not None:   # `bases` = 2-bit words (see pack2)
            mem_b, pb, nw, kb = _arg(bases, np.uint32)
            nb, fn = int(packed_bases), L.syl_seed_batch_packed2
        else:
            mem_b, pb, nb, kb = _arg(bases, np.uint8)
        mem_o, po, no, ko = _arg(rec_off, np.uint64)
        if mem_b != mem_o:
            raise ValueError("bases and rec_off must live in the same memory space")
        n_rec = no - 1
        n_out = C.c_uint64(0)
        if out is not None:
            assert mem_b == _lib.MEM_DEVICE and _is_torch(out)
            cap = out.numel() * out.element_size() // 16
            _lib.check(fn(self._h, mem_b, pb, nb, po, n_rec, k, c, sem, int(with_pos),
                          C.c_void_p(out.data_ptr()), cap, C.byref(n_out)))
            return n_out.value
        if cap is None:
            cap = max(1024, int(nb / c * 1.3) + 4096)
        while True:
            if mem_b == _lib.MEM_DEVICE:
                import torch
                dbuf = torch.empty(cap * 2, dtype=torch.int64, device=bases.device)
                pout = C.c_void_p(dbuf.data_ptr())
            else:
                hbuf = np.empty(cap, dtype=SURVIVOR_DTYPE)
                pout = hbuf.ctypes.data_as(C.c_void_p)
            rc = fn(self._h, mem_b, pb, nb, po, n_rec, k, c, sem, int(with_pos), pout, cap, C.byref(n_out))
            if rc == _lib.SYL_ERR_CAPACITY:
                cap = n_out.value + 16
                continue
            _lib.check(rc)
            n = n_out.value
            if mem_b == _lib.MEM_DEVICE:
                return dbuf[: 2 * n].cpu().numpy().view(SURVIVOR_DTYPE).copy()
            return hbuf[:n].copy()

    # ---- (2) sample sketch -------------------------------------------------------------------
    def sketch_sequences(self, bases, rec_off, k=31, c=200, no_dedup=False, sem=SEM_AVX2, packed_bases=None):
        """Batched body of sketch_sequences_needle (src/sketch.rs:897-959) -> Sample.
        packed_bases: `bases` holds 2-bit words (see pack2) for this many bases (syl_sketch_reads_packed2)."""
        _CTX_STREAM[0] = self._stream
        L = _lib.lib()
        mem_o, po, no, ko = _arg(rec_off, np.uint64)
        h = C.c_void_p()
        if packed_bases is not None:
            mem_b, pb, nw, kb = _arg(bases, np.uint32)
            if nw < (packed_bases + 15) // 16:
                raise ValueError("packed buffer too short")
            if mem_b != mem_o:
                raise ValueError("bases and rec_off must live in the same memory space")
            _lib.check(L.syl_sketch_reads_packed2(self._h, mem_b, pb, int(packed_bases), po, no - 1, k, c, int(no_dedup), sem, C.byref(h)))
            return Sample(self, h)
        mem_b, pb, nb, kb = _arg(bases, np.uint8)
        if mem_b != mem_o:
            raise ValueError("bases and rec_off must live in the same memory space")
        _lib.check(L.syl_sketch_reads(self._h, mem_b, pb, nb, po, no - 1, k, c, int(no_dedup), sem, C.byref(h)))
        return Sample(self, h)

    def sketch_pair_sequences(self, bases1, rec_off1, bases2, rec_off2, k=31, c=200, no_dedup=False, sem=SEM_AVX2,
                              packed=False):
        """Batched body of sketch_pair_sequences with --fpr 0 (src/sketch.rs:771-895): mate i of pair p is record p of
        buffer i; pairs = min(records) of the two buffers -> Sample.
        packed: `bases1` / `bases2` hold 2-bit words (see pack2) (syl_sketch_read_pairs_packed2)."""
        _CTX_STREAM[0] = self._stream
        L = _lib.lib()
        dt, fn = (np.uint32, L.syl_sketch_read_pairs_packed2) if packed else (np.uint8, L.syl_sketch_read_pairs)
        m1, p1, n1, k1 = _arg(bases1, dt)
        mo1, po1, no1, k2 = _arg(rec_off1, np.uint64)
        m2, p2, n2, k3 = _arg(bases2, dt)
        mo2, po2, no2, k4 = _arg(rec_off2, np.uint64)
        if len({m1, mo1, m2, mo2}) != 1:
            raise ValueError("all four buffers must live in the same memory space")
        n_pairs = min(no1, no2) - 1
        nb1, nb2 = int(k2[n_pairs]), int(k4[n_pairs])   # bases of the zipped records only (a longer file's tail is ignored)
        if packed and (n1 < (nb1 + 15) // 16 or n2 < (nb2 + 15) // 16):
            raise ValueError("packed buffer too short")
        h = C.c_void_p()
        _lib.check(fn(self._h, m1, p1, nb1, po1, p2, nb2, po2, n_pairs, k, c, int(no_dedup), sem, C.byref(h)))
        return Sample(self, h)

    def upload_sample(self, hashes, counts, k=31, c=200):
        _CTX_STREAM[0] = self._stream
        L = _lib.lib()
        mem_h, ph, nh, kh = _arg(hashes, np.uint64)
        mem_c, pc, nc, kc = _arg(counts, np.uint32)
        assert mem_h == mem_c and nh == nc
        h = C.c_void_p()
        _lib.check(L.syl_sample_upload(self._h, mem_h, ph, pc, nh, k, c, C.byref(h)))
        return Sample(self, h)

    # ---- (3) genome sketches -----------------------------------------------------------------
    def sketch_genomes(self, bases, contig_off, genome_off=None, k=31, c=200, min_spacing=30, pseudotax=True,
                       individual=False, sem=SEM_AVX2, packed_bases=None):
        """Batched sketch_genome / sketch_genome_individual (src/sketch.rs:550-622, 481-548).
        packed_bases: `bases` holds 2-bit words (see pack2) for this many bases (syl_sketch_genomes_packed2)."""
        _CTX_STREAM[0] = self._stream
        L = _lib.lib()
        mem_o, po, no, ko = _arg(contig_off, np.uint64)
        fn = L.syl_sketch_genomes
        if packed_bases is not None:
            mem_b, pb, nw, kb = _arg(bases, np.uint32)
            if nw < (packed_bases + 15) // 16:
                raise ValueError("packed buffer too short")
            if mem_b != mem_o:
                raise ValueError("bases and contig_off must live in the same memory space")
            nb, fn = int(packed_bases), L.syl_sketch_genomes_packed2
        else:
            mem_b, pb, nb, kb = _arg(bases, np.uint8)
        n_genomes = 0
        pg = None
        if not individual:
            mem_g, pg, ng, kg = _arg(genome_off, np.uint64)
            assert mem_g == mem_b
            n_genomes = ng - 1
        h = C.c_void_p()
        _lib.check(fn(self._h, mem_b, pb, nb, po, no - 1, pg, n_genomes, k, c, min_spacing,
                      int(pseudotax), int(individual), sem, C.byref(h)))
        return Genomes(self, h)

    def upload_genomes(self, kmers, kmer_off, tracked=None, tracked_off=None, gn_size=None, k=31, c=200):
        _CTX_STREAM[0] = self._stream
        L = _lib.lib()
        mem, pk, nk, k1 = _arg(kmers, np.uint64)
        _, pko, nko, k2 = _arg(kmer_off, np.uint64)
        _, pt, nt, k3 = _arg(tracked, np.uint64)
        _, pto, nto, k4 = _arg(tracked_off, np.uint64)
        _, pg, ngs, k5 = _arg(gn_size, np.uint64)
        h = C.c_void_p()
        _lib.check(L.syl_genomes_upload(self._h, mem, pk, pko, pt, pto, pg, nko - 1, k, c, C.byref(h)))
        return Genomes(self, h)

    def concat_genomes(self, parts):
        arr = (C.c_void_p * max(len(parts), 1))(*[p._h for p in parts])
        h = C.c_void_p()
        _lib.check(_lib.lib().syl_genomes_concat(self._h, arr, len(parts), C.byref(h)))
        return Genomes(self, h)

    def select_genomes(self, genomes, idx):
        a = np.ascontiguousarray(idx, dtype=np.uint32)
        h = C.c_void_p()
        _lib.check(_lib.lib().syl_genomes_select(self._h, genomes._h, a.ctypes.data_as(C.c_void_p), len(a), C.byref(h)))
        return Genomes(self, h)

    # ---- (4) containment ---------------------------------------------------------------------
    def build_db(self, genomes, genome_base=0):
        """Index a batch of genome sketches for probing (syl_db_build)."""
        h = C.c_void_p()
        _lib.check(_lib.lib().syl_db_build(self._h, genomes._h, int(genome_base), C.byref(h)))
        return Db(self, h)

    def _pairs(self, fn, db, samples, params, cap):
        L = _lib.lib()
        n = len(samples)
        arr = (C.c_void_p * max(n, 1))(*[s._h for s in samples])
        if cap is None:
            cap = max(4096, 1024 * max(n, 1))  # rows are the pairs that pass the ANI gate: far fewer than pairs
        while True:
            rows = np.empty(cap, dtype=ANI_ROW_DTYPE)
            n_rows = C.c_uint64(0)
            rc = fn(self._h, db._h, arr, n, C.byref(params), rows.ctypes.data_as(C.c_void_p), cap, C.byref(n_rows))
            if rc == _lib.SYL_ERR_CAPACITY:
                cap = n_rows.value
                continue
            _lib.check(rc)
            return rows[: n_rows.value].copy()

    def query(self, db, samples, params=None, cap=None):
        """Pass-1 get_stats over samples x db (`sylph query`); rows ordered by (sample, genome)."""
        params = params or contain_params(pseudotax=False)
        return self._pairs(_lib.lib().syl_query, db, samples, params, cap)

    def profile_shard_begin(self, db, samples, params=None, world=1, rank=0, rows_per_rank=0):
        """Stage 1 of `profile` over a genome-sharded db (pass 1 on this rank's shard) -> ProfileJob."""
        _CTX_STREAM[0] = self._stream
        params = params or contain_params(pseudotax=True)
        arr = (C.c_void_p * max(len(samples), 1))(*[s._h for s in samples])
        h = C.c_void_p()
        _lib.check(_lib.lib().syl_profile_shard_begin(self._h, db._h, arr, len(samples), C.byref(params), int(world), int(rank),
                                                      int(rows_per_rank), C.byref(h)))
        return ProfileJob(self, h, int(world))

    def profile(self, db, samples, params=None, cap=None):
        """`sylph profile`: pass 1, winner table, pass 2, derep, abundances; per sample sorted by rel_abund."""
        params = params or contain_params(pseudotax=True)
        return self._pairs(_lib.lib().syl_profile, db, samples, params, cap)


class ProfileJob:
    """One in-flight `profile` over a genome-sharded db (syl_profile_job): see include/sylph_b200.h section (5).
    The torch tensors returned by tables() / winner() alias the job's device buffers for the collectives."""

    def __init__(self, ctx, handle, world):
        self.ctx, self._h, self.world = ctx, handle, world

    def _tensor(self, ptr, n, typestr):
        import torch
        if not ptr or n == 0:
            return None
        return torch.as_tensor(_CudaArray(ptr, n, self, typestr), device="cuda")

    def buffers(self):
        """-> dict(table1, gathered1, winner, table2, gathered2) of torch CUDA tensors (uint8 / int32)."""
        L = _lib.lib()
        p = [C.c_void_p() for _ in range(5)]
        tb, wn = C.c_uint64(0), C.c_uint64(0)
        _lib.check(L.syl_profile_job_buffers(self._h, C.byref(p[0]), C.byref(p[1]), C.byref(tb), C.byref(p[2]), C.byref(wn),
                                             C.byref(p[3]), C.byref(p[4])))
        w = self.world
        return dict(table1=self._tensor(p[0].value, tb.value, "|u1"),
                    gathered1=self._tensor(p[1].value, tb.value * w, "|u1") if w > 1 else None,
                    winner=self._tensor(p[2].value, wn.value, "<i4") if w > 1 else None,
                    table2=self._tensor(p[3].value, tb.value, "|u1"),
                    gathered2=self._tensor(p[4].value, tb.value * w, "|u1") if w > 1 else None)

    def rank(self):
        _lib.check(_lib.lib().syl_profile_shard_rank(self._h))

    def pass2(self):
        _lib.check(_lib.lib().syl_profile_shard_pass2(self._h))

    def finish(self, cap=4096):
        """-> (rows or None, return code, rows_per_rank needed)"""
        L = _lib.lib()
        while True:
            rows = np.empty(cap, dtype=ANI_ROW_DTYPE)
            n, need = C.c_uint64(0), C.c_uint64(0)
            rc = L.syl_profile_shard_finish(self._h, rows.ctypes.data_as(C.c_void_p), cap, C.byref(n), C.byref(need))
            if rc == _lib.SYL_ERR_CAPACITY and need.value == 0:   # the caller's buffer, not the row table
                cap = max(n.value, 2 * cap)
                continue
            if rc == _lib.SYL_OK:
                return rows[: n.value].copy(), rc, 0
            if rc in (_lib.SYL_ERR_CAPACITY, _lib.SYL_ERR_UNSUPPORTED):
                return None, rc, need.value
            _lib.check(rc)

    def free(self):
        if self._h:
            _lib.lib().syl_profile_job_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def pack2(bases, threads=0):
    """Host packer (syl_pack2): ASCII bases (numpy uint8) -> uint32 words, 16 bases per word, base 16w+j in
    bits [30-2j, 31-2j], exact BYTE_TO_SEQ codes (src/types.rs:50-59)."""
    a = np.ascontiguousarray(bases, dtype=np.uint8)
    out = np.zeros((a.size + 15) // 16, dtype=np.uint32)
    _lib.check(_lib.lib().syl_pack2(a.ctypes.data_as(C.c_void_p), a.size, out.ctypes.data_as(C.c_void_p), int(threads)))
    return out


def contain_params(k=31, pseudotax=False, **kw):
    p = ContainParams()
    _lib.lib().syl_contain_params_default(C.byref(p), k, int(pseudotax))
    for a, b in kw.items():
        setattr(p, a, b)
    return p


class Db:
    """Probe index over a batch of genome sketches (syl_db)."""

    def __init__(self, ctx, handle):
        self.ctx, self._h = ctx, handle

    def __len__(self):
        return int(_lib.lib().syl_db_num_genomes(self._h))

    def free(self):
        if self._h:
            _lib.lib().syl_db_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class _CudaArray:
    """Minimal __cuda_array_interface__ carrier (default: int64 view of a device u64 array)."""

    def __init__(self, ptr, n, owner, typestr="<i8"):
        self.owner = owner
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


class Sample:
    """Device-resident SequencesSketch.kmer_counts (src/types.rs:145-155), sorted by hash."""

    def __init__(self, ctx, handle):
        self.ctx, self._h = ctx, handle

    def __len__(self):
        return int(_lib.lib().syl_sample_size(self._h))

    @property
    def mean_read_length(self):
        return float(_lib.lib().syl_sample_mean_read_length(self._h))

    @mean_read_length.setter
    def mean_read_length(self, v):
        """for uploaded sketches (.sylsp files carry the value; -u reads it)"""
        _lib.lib().syl_sample_set_mean_read_length(self._h, float(v))

    @property
    def num_dup_removed(self):
        return int(_lib.lib().syl_sample_num_dup_removed(self._h))

    def download(self, hash_out=None, count_out=None):
        """-> (hash u64[n] ascending, count u32[n]).  hash_out / count_out: optional caller buffers
        (e.g. views of pinned memory, reused across calls) with room for n entries; the returned
        arrays are then views of them."""
        n = len(self)
        if hash_out is None:
            hash_out = np.empty(n, dtype=np.uint64)
        if count_out is None:
            count_out = np.empty(n, dtype=np.uint32)
        if hash_out.dtype != np.uint64 or count_out.dtype != np.uint32 or hash_out.size < n or count_out.size < n \
                or not hash_out.flags.c_contiguous or not count_out.flags.c_contiguous:
            raise ValueError("download buffers must be contiguous uint64 / uint32 arrays with >= %d entries" % n)
        _lib.check(_lib.lib().syl_sample_download(self.ctx._h, self._h, hash_out.ctypes.data_as(C.c_void_p),
                                                  count_out.ctypes.data_as(C.c_void_p)))
        return hash_out[:n], count_out[:n]

    def free(self):
        if self._h:
            _lib.lib().syl_sample_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Genomes:
    """Device-resident batch of GenomeSketch (src/types.rs:163-173) in CSR form."""

    def __init__(self, ctx, handle):
        self.ctx, self._h = ctx, handle

    def __len__(self):
        return int(_lib.lib().syl_genomes_count(self._h))

    @property
    def has_tracked(self):
        return bool(_lib.lib().syl_genomes_has_tracked(self._h))

    @property
    def k(self):
        return int(_lib.lib().syl_genomes_k(self._h))

    @property
    def c(self):
        return int(_lib.lib().syl_genomes_c(self._h))

    def download(self):
        """-> dict(kmers, kmer_off, tracked, tracked_off, gn_size)"""
        L = _lib.lib()
        n = len(self)
        nk, nt = int(L.syl_genomes_total_kmers(self._h)), int(L.syl_genomes_total_tracked(self._h))
        d = dict(kmers=np.empty(nk, np.uint64), kmer_off=np.empty(n + 1, np.uint64), tracked=np.empty(nt, np.uint64),
                 tracked_off=np.empty(n + 1, np.uint64), gn_size=np.empty(n, np.uint64))
        _lib.check(L.syl_genomes_download(self.ctx._h, self._h, *[d[x].ctypes.data_as(C.c_void_p) for x in
                                                                   ("kmers", "kmer_off", "tracked", "tracked_off",
                                                                    "gn_size")]))
        return d

    def device_tensors(self):
        """Zero-copy torch views (int64) of the device CSR arrays: dict(kmers, kmer_off, tracked, tracked_off,
        gn_size). Valid while this object is alive."""
        import torch
        L = _lib.lib()
        ptrs = [C.c_void_p() for _ in range(5)]
        _lib.check(L.syl_genomes_device_ptrs(self._h, *[C.byref(p) for p in ptrs]))
        n = len(self)
        sizes = (int(L.syl_genomes_total_kmers(self._h)), n + 1, int(L.syl_genomes_total_tracked(self._h)), n + 1, n)
        out = {}
        for name, p, sz in zip(("kmers", "kmer_off", "tracked", "tracked_off", "gn_size"), ptrs, sizes):
            if sz == 0 or not p.value:
                out[name] = torch.empty(0, dtype=torch.int64, device="cuda")
            else:
                out[name] = torch.as_tensor(_CudaArray(p.value, sz, self), device="cuda")
        return out

    def free(self):
        if self._h:
            _lib.lib().syl_genomes_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
