"""kallisto_b200 -- host-side Python mirror of the C ABI (include/kallisto_b200.h).

The product is the shared library ``libkallisto_b200.so`` (hand-written sm_90a CUDA behind an
``extern "C"`` boundary) and the ``kallisto_b200`` command-line binary; this module is the thin
ctypes binding used by the tests and ``bench.py``.  Class and method names follow the reference
objects they stand in for: ``KmerIndex`` (src/KmerIndex.h), ``MinCollector``/``MasterProcessor``
(src/MinCollector.h, src/ProcessReads.h) and ``EMAlgorithm`` (src/EMAlgorithm.h).

There is no CPU fallback: if the library is missing, or no CUDA device is present, every call
that would compute something raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KB_LIB_PATH") or os.path.join(_HERE, "libkallisto_b200.so")   # KB_LIB_PATH: experiments only

KB_OK = 0
KB_ERR_INVALID = -1
KB_ERR_NO_DEVICE = -3


class KallistoB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("kallisto_b200 error %d: %s" % (code, msg))
        self.code = code


class kb_index_info(C.Structure):
    _fields_ = [("k", C.c_int32), ("n_targets", C.c_uint32), ("n_unitigs", C.c_uint32), ("n_ec_blocks", C.c_uint32),
                ("n_ec_sets", C.c_uint32), ("n_kmers", C.c_uint64), ("table_slots", C.c_uint64),
                ("load_seconds", C.c_double), ("build_seconds", C.c_double)]


class kb_quant_opts(C.Structure):
    _fields_ = [("paired", C.c_int32), ("strand_mode", C.c_int32), ("collect_fld", C.c_int32),
                ("max_batch_reads", C.c_uint32), ("max_batch_bases", C.c_uint64), ("single_overhang", C.c_int32),
                ("fld_mean", C.c_double)]


class kb_kernel_timings(C.Structure):
    _fields_ = [("match_ms", C.c_double), ("resolve_ms", C.c_double), ("em_ms", C.c_double), ("em_prep_ms", C.c_double),
                ("match_launches", C.c_uint64), ("resolve_launches", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("bs_resample_ms", C.c_double), ("bs_em_ms", C.c_double), ("pack_ms", C.c_double),
                ("em_comp_blocks", C.c_uint64), ("em_comp_resident", C.c_uint64)]


class kb_bus_substr(C.Structure):
    _fields_ = [("fileno", C.c_int32), ("start", C.c_int32), ("stop", C.c_int32)]


class kb_bus_opts(C.Structure):
    _fields_ = [("nfiles", C.c_int32), ("n_bc", C.c_int32), ("bc", kb_bus_substr * 4), ("n_umi", C.c_int32),
                ("umi", kb_bus_substr * 4), ("seq", kb_bus_substr), ("strand_mode", C.c_int32), ("num", C.c_int32),
                ("max_batch_sets", C.c_uint32), ("max_batch_bases", C.c_uint64), ("paired", C.c_int32),
                ("seq2", kb_bus_substr), ("tag", C.c_char_p)]


BUS_RECORD_DTYPE = np.dtype([("barcode", "<u8"), ("umi", "<u8"), ("ec", "<i4"), ("count", "<u4"), ("flags", "<u4"),
                             ("pad", "<u4")])

# technology table of `kallisto bus -x` (src/main.cpp:1283-1437): (nfiles, bc pieces, umi pieces, seq, default strand)
TECHNOLOGIES = {
    "10XV1": (3, [(0, 0, 14)], [(1, 0, 10)], (2, 0, 0), 1),
    "10XV2": (2, [(0, 0, 16)], [(0, 16, 26)], (1, 0, 0), 1),
    "10XV3": (2, [(0, 0, 16)], [(0, 16, 28)], (1, 0, 0), 1),
    "VISIUM": (2, [(0, 0, 16)], [(0, 16, 28)], (1, 0, 0), 1),
    "SURECELL": (2, [(0, 0, 6), (0, 21, 27), (0, 42, 48)], [(0, 51, 59)], (1, 0, 0), 1),
    "DROPSEQ": (2, [(0, 0, 12)], [(0, 12, 20)], (1, 0, 0), 0),
    "INDROPSV1": (2, [(0, 0, 11), (0, 30, 38)], [(0, 42, 48)], (1, 0, 0), 0),
    "INDROPSV2": (2, [(1, 0, 11), (1, 30, 38)], [(1, 42, 48)], (0, 0, 0), 0),
    "INDROPSV3": (3, [(0, 0, 8), (1, 0, 8)], [(1, 8, 14)], (2, 0, 0), 0),
    "CELSEQ": (2, [(0, 0, 8)], [(0, 8, 12)], (1, 0, 0), 1),
    "CELSEQ2": (2, [(0, 6, 12)], [(0, 0, 6)], (1, 0, 0), 1),
    "SPLIT-SEQ": (2, [(1, 10, 18), (1, 48, 56), (1, 78, 86)], [(1, 0, 10)], (0, 0, 0), 1),
    "SCRBSEQ": (2, [(0, 0, 6)], [(0, 6, 16)], (1, 0, 0), 0),
    # technologies without a UMI read ("bulk_like") and / or with two sequence reads (busopt.paired); a sixth entry
    # is the second sequence read
    "BULK": (1, [], [(-1, -1, -1)], (0, 0, 0), 0),                                # `bus -x BULK`: one sample per file
    "BULK-PAIRED": (2, [], [(-1, -1, -1)], (0, 0, 0), 0, (1, 0, 0)),              # `bus -x BULK --paired`
    "SMARTSEQ2": (3, [(0, 0, 0), (1, 0, 0)], [(-1, -1, -1)], (2, 0, 0), 0),
    "SMARTSEQ2-PAIRED": (4, [(0, 0, 0), (1, 0, 0)], [(-1, -1, -1)], (2, 0, 0), 0, (3, 0, 0)),
    "STORM-SEQ": (2, [], [(1, 0, 8)], (0, 0, 0), 2, (1, 14, 0)),
    "SMARTSEQ3": (4, [(0, 0, 0), (1, 0, 0)], [(2, 0, 19)], (2, 22, 0), 1, (3, 0, 0)),   # with tag="ATTGCGCAATG"
}


class kb_run_stats(C.Structure):
    _fields_ = [("n_processed", C.c_uint64), ("n_pseudoaligned", C.c_uint64), ("n_unique", C.c_uint64),
                ("n_ecs", C.c_uint64), ("n_ec_entries", C.c_uint64), ("n_probes", C.c_uint64),
                ("n_slot_visits", C.c_uint64), ("n_resolved", C.c_uint64), ("n_memo_hits", C.c_uint64)]


# every symbol declared in include/kallisto_b200.h
EXPORTED_SYMBOLS = [
    "kb_last_error", "kb_version", "kb_index_load", "kb_index_free", "kb_index_get_info", "kb_index_target_name",
    "kb_index_target_lens", "kb_index_inspect", "kb_quant_create", "kb_quant_free", "kb_pseudoalign_batch",
    "kb_pseudoalign_batch_pe", "kb_host_alloc", "kb_host_free", "kb_pseudoalign_batch_device", "kb_quant_sync", "kb_quant_set_stream", "kb_quant_enable_timing",
    "kb_quant_get_timings", "kb_quant_finalize", "kb_quant_ec_table", "kb_quant_get_flens",
    "kb_quant_set_flens", "kb_em_run", "kb_em_run_table", "kb_read_priors", "kb_em_set_priors", "kb_bootstrap_run", "kb_quant_export_prepare", "kb_quant_export_device", "kb_quant_import_device",
    "kb_comm_unique_id", "kb_comm_create", "kb_comm_create_from_nccl", "kb_comm_create_all", "kb_comm_reserve", "kb_comm_free",
    "kb_quant_merge_nccl", "kb_quant_merge_local", "kb_quant_set_frag_base", "kb_quant_reserve", "kb_tcc_run", "kb_tcc_bootstrap_run", "kb_tcc_run_genes", "kb_tcc_run_priors", "kb_tcc_bootstrap_run_genes", "kb_eff_lens", "kb_bus_create", "kb_bus_batch", "kb_bus_batch_device", "kb_bus_begin_sample", "kb_bus_set_batch_barcodes", "kb_bus_lengths", "kb_bus_set_aa", "kb_bus_frame_clashes", "kb_bus_group_create", "kb_bus_group_free", "kb_bus_group_submit", "kb_bus_group_complete", "kb_bus_group_begin_sample", "kb_bus_group_finalize", "kb_bus_group_ec_table", "kb_bus_group_lengths", "kb_bus_group_frame_clashes", "kb_fastx_summary", "kb_fastx_summary_mt", "kb_gz_summary", "kb_counts_to_tpm",
]

# kb_tcc_bootstrap_cb: (user, first problem, count, est_counts, rounds, resampled counts or NULL) -> 0 to go on
TCC_BOOTSTRAP_CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.c_uint32, C.POINTER(C.c_double), C.POINTER(C.c_int32),
                               C.POINTER(C.c_uint32))
# kb_tcc_bootstrap_genes_cb: the same, then gene counts and gene TPM (count x n_genes) or NULL
TCC_BOOTSTRAP_GENES_CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.c_uint32, C.POINTER(C.c_double),
                                     C.POINTER(C.c_int32), C.POINTER(C.c_uint32), C.POINTER(C.c_double),
                                     C.POINTER(C.c_double))

_lib = None


def lib():
    """Load libkallisto_b200.so (built in-tree by __graft_entry__.build() / make)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise KallistoB200Error(-5, "%s not found: build it with `make -C kallisto_b200/csrc` "
                                    "(there is no Python/CPU fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, u32, i32, u64, dbl = C.c_void_p, C.c_uint32, C.c_int32, C.c_uint64, C.c_double
    L.kb_last_error.restype = C.c_char_p
    L.kb_version.restype = C.c_char_p
    L.kb_index_load.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.kb_index_free.argtypes = [vp]
    L.kb_index_get_info.argtypes = [vp, C.POINTER(kb_index_info)]
    L.kb_index_inspect.argtypes = [C.c_char_p, C.POINTER(kb_index_info)]
    L.kb_index_target_name.argtypes = [vp, u32]
    L.kb_index_target_name.restype = C.c_char_p
    L.kb_index_target_lens.argtypes = [vp, vp]
    L.kb_quant_create.argtypes = [vp, C.POINTER(kb_quant_opts), C.POINTER(vp)]
    L.kb_quant_free.argtypes = [vp]
    L.kb_pseudoalign_batch.argtypes = [vp, vp, vp, u32, u32, vp]
    L.kb_pseudoalign_batch_pe.argtypes = [vp, vp, vp, vp, vp, u32, u32, vp]
    L.kb_host_alloc.argtypes = [C.c_size_t]
    L.kb_host_alloc.restype = vp
    L.kb_host_free.argtypes = [vp]
    L.kb_pseudoalign_batch_device.argtypes = [vp, vp, vp, u32, u32, u32]
    L.kb_quant_sync.argtypes = [vp]
    L.kb_quant_set_stream.argtypes = [vp, vp]
    L.kb_quant_enable_timing.argtypes = [vp, C.c_int]
    L.kb_quant_get_timings.argtypes = [vp, C.POINTER(kb_kernel_timings)]
    L.kb_quant_finalize.argtypes = [vp, C.POINTER(kb_run_stats)]
    L.kb_quant_ec_table.argtypes = [vp, vp, vp, vp, vp]
    L.kb_quant_get_flens.argtypes = [vp, vp]
    L.kb_quant_set_flens.argtypes = [vp, vp]
    L.kb_em_run.argtypes = [vp, dbl, dbl, vp, vp, C.POINTER(i32), C.POINTER(dbl)]
    L.kb_em_run_table.argtypes = [vp, u32, vp, vp, vp, dbl, dbl, vp, vp, C.POINTER(i32), C.POINTER(dbl)]
    L.kb_read_priors.argtypes = [C.c_char_p, vp, u64, C.POINTER(u64)]
    L.kb_em_set_priors.argtypes = [vp, vp, u32]
    L.kb_bootstrap_run.argtypes = [vp, dbl, dbl, u64, i32, vp, vp, vp]
    L.kb_counts_to_tpm.argtypes = [vp, vp, u32, vp]
    L.kb_quant_export_prepare.argtypes = [vp, C.POINTER(u32), C.POINTER(u32)]
    L.kb_quant_export_device.argtypes = [vp, vp, vp, vp, vp]
    L.kb_quant_import_device.argtypes = [vp, u32, vp, vp, vp, vp, u64, u64]
    L.kb_comm_unique_id.argtypes = [vp]
    L.kb_comm_create.argtypes = [C.c_int, C.c_int, vp, C.c_int, C.POINTER(vp)]
    L.kb_comm_create_from_nccl.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.kb_comm_create_all.argtypes = [vp, C.c_int, vp]
    L.kb_comm_reserve.argtypes = [vp, u64, u64]
    L.kb_comm_free.argtypes = [vp]
    L.kb_quant_merge_nccl.argtypes = [vp, vp, u64, C.POINTER(u64)]
    L.kb_quant_merge_local.argtypes = [vp, vp, i32, C.POINTER(u64)]
    L.kb_quant_set_frag_base.argtypes = [vp, u64]
    L.kb_quant_reserve.argtypes = [vp, u64, u64]
    L.kb_tcc_run.argtypes = [vp, u32, vp, vp, u32, vp, vp, vp, vp, i32, vp, vp]
    L.kb_tcc_bootstrap_run.argtypes = [vp, u32, vp, vp, u32, vp, vp, vp, vp, i32, u64, i32, i32, TCC_BOOTSTRAP_CB, vp]
    L.kb_tcc_run_genes.argtypes = [vp, u32, vp, vp, u32, vp, vp, vp, vp, i32, vp, u32, vp, vp, vp, vp]
    L.kb_tcc_run_priors.argtypes = [vp, u32, vp, vp, u32, vp, vp, vp, vp, i32, vp, u32, vp, vp, vp, vp, vp]
    L.kb_tcc_bootstrap_run_genes.argtypes = [vp, u32, vp, vp, u32, vp, vp, vp, vp, i32, vp, u32, u64, i32, i32,
                                             TCC_BOOTSTRAP_GENES_CB, vp]
    L.kb_eff_lens.argtypes = [vp, vp, dbl, dbl, vp, C.POINTER(dbl), C.POINTER(dbl)]
    L.kb_bus_create.argtypes = [vp, C.POINTER(kb_bus_opts), C.POINTER(vp)]
    L.kb_bus_batch.argtypes = [vp, vp, vp, u32, vp, C.POINTER(u32)]
    L.kb_bus_batch_device.argtypes = [vp, vp, vp, u32, u32, C.POINTER(u32), C.POINTER(vp)]
    L.kb_bus_lengths.argtypes = [vp, vp, vp]
    L.kb_bus_begin_sample.argtypes = [vp, C.c_uint64]
    L.kb_bus_set_batch_barcodes.argtypes = [vp, C.c_int32]
    L.kb_bus_set_aa.argtypes = [vp, C.c_int32]
    L.kb_bus_frame_clashes.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.kb_bus_group_create.argtypes = [vp, i32, C.POINTER(vp)]
    L.kb_bus_group_free.argtypes = [vp]
    L.kb_bus_group_submit.argtypes = [vp, i32, vp, vp, u32, C.POINTER(u64)]
    L.kb_bus_group_complete.argtypes = [vp, u64, vp, C.POINTER(u32)]
    L.kb_bus_group_begin_sample.argtypes = [vp, u64]
    L.kb_bus_group_finalize.argtypes = [vp, C.POINTER(kb_run_stats)]
    L.kb_bus_group_ec_table.argtypes = [vp, vp, vp, vp]
    L.kb_bus_group_lengths.argtypes = [vp, vp, vp]
    L.kb_bus_group_frame_clashes.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.kb_fastx_summary.argtypes = [C.c_char_p, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.kb_gz_summary.argtypes = [C.c_char_p, C.POINTER(u64), C.POINTER(C.c_uint32)]
    L.kb_fastx_summary_mt.argtypes = [C.c_char_p, C.c_int, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    _lib = L
    return L


def _ck(rc):
    if rc != KB_OK:
        raise KallistoB200Error(rc, lib().kb_last_error().decode(errors="replace"))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def inspect_index(path):
    """Parse an index file on the host only (no device needed): sizes for tooling and tests."""
    info = kb_index_info()
    _ck(lib().kb_index_inspect(os.fsencode(path), C.byref(info)))
    return {f: getattr(info, f) for f, _ in kb_index_info._fields_}


def read_priors(path):
    """EMAlgorithm::read_priors (kb_read_priors, host only): the priors of a --priors file as the EM would start from
    them (raw counts get a pseudocount and are normalised) -> float64 array."""
    n = C.c_uint64(0)
    _ck(lib().kb_read_priors(os.fsencode(path), None, 0, C.byref(n)))
    out = np.zeros(n.value, np.float64)
    if n.value:
        _ck(lib().kb_read_priors(os.fsencode(path), _p(out), n.value, C.byref(n)))
    return out


class KmerIndex:
    """KmerIndex::load (src/KmerIndex.cpp:1330-1559) -> flat tables resident in HBM."""

    def __init__(self, path, device=0, load_positions=False, threads=4):
        self._h = C.c_void_p()
        _ck(lib().kb_index_load(os.fsencode(path), device, int(load_positions), threads, C.byref(self._h)))
        info = kb_index_info()
        _ck(lib().kb_index_get_info(self._h, C.byref(info)))
        self.info = {f: getattr(info, f) for f, _ in kb_index_info._fields_}
        self.k = info.k
        self.num_trans = info.n_targets
        self.target_lens_ = np.zeros(self.num_trans, np.uint32)
        _ck(lib().kb_index_target_lens(self._h, _p(self.target_lens_)))
        self.target_names_ = [lib().kb_index_target_name(self._h, i).decode() for i in range(self.num_trans)]
        self.device = device

    def close(self):
        if self._h:
            lib().kb_index_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MinCollector:
    """One quantification run: per-batch pseudoalignment, EC bookkeeping, EM, bootstrap.

    Stands in for MinCollector + MasterProcessor/ReadProcessor (src/ProcessReads.cpp) followed by
    EMAlgorithm / Bootstrap."""

    def __init__(self, index, paired=True, strand=None, collect_fld=True, max_batch_reads=0, max_batch_bases=0,
                 single_overhang=True, fld_mean=0.0):
        self.index = index
        self.paired = bool(paired)
        o = kb_quant_opts()
        o.paired = int(self.paired)
        o.strand_mode = {None: 0, "unstranded": 0, "fr": 1, "rf": 2, 0: 0, 1: 1, 2: 2}[strand]
        o.collect_fld = int(collect_fld)
        o.max_batch_reads = max_batch_reads
        o.max_batch_bases = max_batch_bases
        o.single_overhang = int(single_overhang)
        o.fld_mean = fld_mean
        self._h = C.c_void_p()
        _ck(lib().kb_quant_create(index._h, C.byref(o), C.byref(self._h)))
        self._stats = None

    def close(self):
        if self._h:
            lib().kb_quant_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- ReadProcessor::processBuffer ------------------------------------------------------
    def process_buffer(self, bases, offsets=None, fixed_len=0, want_handles=True):
        """Host arrays in, one set handle per fragment out (or None)."""
        bases = np.ascontiguousarray(bases, dtype=np.uint8)
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
            n_reads = len(offsets) - 1
        else:
            n_reads = len(bases) // fixed_len if fixed_len else 0
        n_frag = n_reads // 2 if self.paired else n_reads
        out = np.full(n_frag, -1, np.int32) if want_handles else None
        _ck(lib().kb_pseudoalign_batch(self._h, _p(bases), _p(offsets), n_reads, fixed_len, _p(out)))
        self._stats = None
        return out

    def process_buffer_pe(self, bases1, offsets1, bases2, offsets2, want_handles=True):
        """Paired batch, one buffer per mate (numpy arrays)."""
        b1 = np.ascontiguousarray(bases1, np.uint8); b2 = np.ascontiguousarray(bases2, np.uint8)
        o1 = np.ascontiguousarray(offsets1, np.uint32); o2 = np.ascontiguousarray(offsets2, np.uint32)
        n = len(o1) - 1
        out = np.full(n, -1, np.int32) if want_handles else None
        _ck(lib().kb_pseudoalign_batch_pe(self._h, _p(b1), _p(o1), _p(b2), _p(o2), n, 0, _p(out)))
        self._stats = None
        return out

    def process_buffer_ptr(self, bases_ptr, offsets_ptr, n_reads, fixed_len, out_ptr=None):
        """Same, raw host pointers (e.g. pinned torch tensors)."""
        _ck(lib().kb_pseudoalign_batch(self._h, bases_ptr, offsets_ptr, n_reads, fixed_len, out_ptr))
        self._stats = None

    def process_buffer_device(self, d_bases_ptr, d_offsets_ptr, n_reads, fixed_len, max_read_len=0):
        _ck(lib().kb_pseudoalign_batch_device(self._h, d_bases_ptr, d_offsets_ptr, n_reads, fixed_len, max_read_len))
        self._stats = None

    def sync(self):
        _ck(lib().kb_quant_sync(self._h))

    def set_stream(self, cuda_stream_ptr):
        _ck(lib().kb_quant_set_stream(self._h, C.c_void_p(cuda_stream_ptr)))

    def enable_timing(self, on=True):
        _ck(lib().kb_quant_enable_timing(self._h, int(on)))

    def timings(self):
        t = kb_kernel_timings()
        _ck(lib().kb_quant_get_timings(self._h, C.byref(t)))
        return {f: getattr(t, f) for f, _ in kb_kernel_timings._fields_}

    # -- MasterProcessor::update / increaseCount --------------------------------------------
    def finalize(self):
        s = kb_run_stats()
        _ck(lib().kb_quant_finalize(self._h, C.byref(s)))
        self._stats = {f: getattr(s, f) for f, _ in kb_run_stats._fields_}
        return self._stats

    def ec_table(self):
        """-> (offsets uint64[n+1], tids uint32, counts uint32[n], handles int32[n]); ids in order of
        first occurrence."""
        st = self._stats or self.finalize()
        n, m = st["n_ecs"], st["n_ec_entries"]
        off = np.zeros(n + 1, np.uint64)
        tids = np.zeros(max(1, m), np.uint32)
        counts = np.zeros(max(1, n), np.uint32)
        handles = np.zeros(max(1, n), np.int32)
        _ck(lib().kb_quant_ec_table(self._h, _p(off), _p(tids), _p(counts), _p(handles)))
        return off, tids[:m], counts[:n], handles[:n]

    @property
    def flens(self):
        f = np.zeros(1000, np.uint32)
        _ck(lib().kb_quant_get_flens(self._h, _p(f)))
        return f

    def set_flens(self, f):
        f = np.ascontiguousarray(f, np.uint32)
        assert len(f) == 1000
        _ck(lib().kb_quant_set_flens(self._h, _p(f)))

    # -- multi-GPU exchange (device pointers; see kallisto_b200/multigpu.py) -----------------------
    def export_prepare(self):
        n, m = C.c_uint32(0), C.c_uint32(0)
        _ck(lib().kb_quant_export_prepare(self._h, C.byref(n), C.byref(m)))
        return n.value, m.value

    def export_device(self, off_ptr, tids_ptr, counts_ptr, first_ptr):
        _ck(lib().kb_quant_export_device(self._h, off_ptr, tids_ptr, counts_ptr, first_ptr))

    def import_device(self, n_sets, off_ptr, tids_ptr, counts_ptr, first_ptr, first_offset, n_processed):
        _ck(lib().kb_quant_import_device(self._h, n_sets, off_ptr, tids_ptr, counts_ptr, first_ptr, first_offset,
                                         n_processed))
        self._stats = None

    def merge_nccl(self, comm, first_stride=1 << 40):
        """Collective: fold every rank's equivalence classes into rank 0's run (csrc/comm.cu); returns the
        number of fragments processed by all ranks."""
        tot = C.c_uint64(0)
        _ck(lib().kb_quant_merge_nccl(self._h, comm._h, first_stride, C.byref(tot)))
        self._stats = None
        return tot.value

    def merge_local(self, others):
        """Fold the equivalence classes of other runs of THIS process (any devices) into this one by content."""
        arr = (C.c_void_p * len(others))(*[o._h for o in others])
        tot = C.c_uint64(0)
        _ck(lib().kb_quant_merge_local(self._h, arr, len(others), C.byref(tot)))
        self._stats = None
        return tot.value

    def set_frag_base(self, base):
        _ck(lib().kb_quant_set_frag_base(self._h, base))

    def reserve(self, n_ecs, n_entries):
        _ck(lib().kb_quant_reserve(self._h, n_ecs, n_entries))

    # -- EMAlgorithm::run / Bootstrap::run_em --------------------------------------------------
    def set_priors(self, priors):
        """EMAlgorithm::set_priors: every later run_em starts from `priors` (n_targets values); None goes back to the
        uniform start.  run_bootstrap always starts uniform."""
        if priors is None:
            _ck(lib().kb_em_set_priors(self._h, None, 0))
            return
        a = np.ascontiguousarray(priors, np.float64)
        _ck(lib().kb_em_set_priors(self._h, _p(a), a.size))

    def run_em(self, fld_mean=0.0, fld_sd=0.0, table=None):
        T = self.index.num_trans
        est = np.zeros(T, np.float64)
        eff = np.zeros(T, np.float64)
        rounds = C.c_int32(0)
        secs = C.c_double(0)
        if table is None:
            _ck(lib().kb_em_run(self._h, fld_mean, fld_sd, _p(est), _p(eff), C.byref(rounds), C.byref(secs)))
        else:
            off, tids, counts = (np.ascontiguousarray(table[0], np.uint64), np.ascontiguousarray(table[1], np.uint32),
                                 np.ascontiguousarray(table[2], np.uint32))
            _ck(lib().kb_em_run_table(self._h, len(counts), _p(off), _p(tids), _p(counts), fld_mean, fld_sd, _p(est),
                                      _p(eff), C.byref(rounds), C.byref(secs)))
        return dict(est_counts=est, eff_lens=eff, rounds=rounds.value, seconds=secs.value)

    def run_bootstrap(self, n_bootstrap, seed=42, fld_mean=0.0, fld_sd=0.0, want_samples=False):
        T = self.index.num_trans
        st = self._stats or self.finalize()
        est = np.zeros((n_bootstrap, T), np.float64)
        samples = np.zeros((n_bootstrap, max(1, st["n_ecs"])), np.uint32) if want_samples else None
        rounds = np.zeros(max(1, n_bootstrap), np.int32)
        _ck(lib().kb_bootstrap_run(self._h, fld_mean, fld_sd, seed, n_bootstrap, _p(est), _p(samples), _p(rounds)))
        return dict(est_counts=est, samples=samples, rounds=rounds[:n_bootstrap])


class Comm:
    """NCCL communicator of the multi-GPU merge (kb_comm_*).  `unique_id()` on rank 0, broadcast the 128 bytes
    to the other ranks (torch.distributed, a file, ...), then every rank constructs Comm(n_ranks, rank, id, device)."""

    @staticmethod
    def unique_id():
        buf = (C.c_ubyte * 128)()
        _ck(lib().kb_comm_unique_id(buf))
        return bytes(buf)

    def __init__(self, n_ranks, rank, uid, device):
        self._h = C.c_void_p()
        b = (C.c_ubyte * 128).from_buffer_copy(uid)
        _ck(lib().kb_comm_create(n_ranks, rank, b, device, C.byref(self._h)))
        self.n_ranks, self.rank = n_ranks, rank

    def reserve(self, n_sets, n_entries):
        _ck(lib().kb_comm_reserve(self._h, n_sets, n_entries))

    def close(self):
        if self._h:
            lib().kb_comm_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BUSProcessor(MinCollector):
    """`kallisto bus` run (BUSProcessor::processBuffer + the BUS part of MasterProcessor::update)."""

    def __init__(self, index, technology, strand="default", num=False, max_batch_sets=0, tag=None, aa=False,
                 batch_barcodes=False):
        """aa: `bus --aa`, the reads translated in six frames against an index built with `kallisto index --aa`.
        batch_barcodes: `bus --batch --batch-barcodes`, the sample of begin_sample in front of every barcode."""
        self.index = index
        self.paired = False
        tech = TECHNOLOGIES[technology.upper()] if isinstance(technology, str) else technology
        nfiles, bc, umi, seq, dstrand = tech[:5]
        o = kb_bus_opts()
        if len(tech) > 5:
            o.paired = 1
            o.seq2 = kb_bus_substr(*tech[5])
            self.paired = True
        o.nfiles = nfiles
        o.n_bc = len(bc)
        for i, t in enumerate(bc):
            o.bc[i] = kb_bus_substr(*t)
        o.n_umi = len(umi)
        for i, t in enumerate(umi):
            o.umi[i] = kb_bus_substr(*t)
        o.seq = kb_bus_substr(*seq)
        o.strand_mode = dstrand if strand == "default" else {None: 0, "unstranded": 0, "fr": 1, "rf": 2}[strand]
        o.num = int(num)
        o.max_batch_sets = max_batch_sets
        if tag:
            o.tag = tag if isinstance(tag, bytes) else tag.encode()      # --tag / SMARTSEQ3: umi[0] covers tag + UMI
        self.nfiles = nfiles
        self._h = C.c_void_p()
        _ck(lib().kb_bus_create(index._h, C.byref(o), C.byref(self._h)))
        self._stats = None
        if aa:
            _ck(lib().kb_bus_set_aa(self._h, 1))
        if batch_barcodes:
            _ck(lib().kb_bus_set_batch_barcodes(self._h, 1))

    def process_sets(self, files):
        """files: list of (bases uint8, offsets uint32) per file of the technology -> structured record array."""
        assert len(files) == self.nfiles
        bs = [np.ascontiguousarray(b, np.uint8) for b, _ in files]
        os_ = [np.ascontiguousarray(o, np.uint32) for _, o in files]
        n = len(os_[0]) - 1
        bp = (C.c_void_p * self.nfiles)(*[b.ctypes.data for b in bs])
        op = (C.c_void_p * self.nfiles)(*[o.ctypes.data for o in os_])
        rec = np.zeros(max(1, n), BUS_RECORD_DTYPE)
        nrec = C.c_uint32(0)
        _ck(lib().kb_bus_batch(self._h, bp, op, n, _p(rec), C.byref(nrec)))
        self._stats = None
        return rec[: nrec.value]

    def process_sets_device(self, base_ptrs, offset_ptrs, n_sets, max_seq_len):
        """Device pointers in (one per file of the technology), records stay on the device: -> (n_records, device pointer)."""
        bp = (C.c_void_p * self.nfiles)(*base_ptrs)
        op = (C.c_void_p * self.nfiles)(*offset_ptrs)
        nrec = C.c_uint32(0)
        drec = C.c_void_p()
        _ck(lib().kb_bus_batch_device(self._h, bp, op, n_sets, max_seq_len, C.byref(nrec), C.byref(drec)))
        self._stats = None
        return nrec.value, drec.value

    def begin_sample(self, barcode):
        """Batch mode (`bus -x BULK` / `--batch`): the following read sets belong to this sample: the fake barcode without
        a barcode read, the prefix of batch_barcodes with one; fragment lengths and --num read numbers start again."""
        _ck(lib().kb_bus_begin_sample(self._h, C.c_uint64(barcode)))

    def lengths(self):
        b, u = np.zeros(33, np.uint32), np.zeros(33, np.uint32)
        _ck(lib().kb_bus_lengths(self._h, _p(b), _p(u)))
        return b, u

    def frame_clashes(self):
        """--aa: the run's frame clashes ("n_frame_clashes" of run_info.json)."""
        n = C.c_uint64(0)
        _ck(lib().kb_bus_frame_clashes(self._h, C.byref(n)))
        return n.value


class BUSGroup:
    """`bus --devices` (kb_bus_group_*): batches of one read stream dealt to several fresh BUSProcessor runs with the same
    options (one index replica each), records and EC table numbered as one run fed the whole stream would number them.
    Batches complete in submission order; fragment lengths are member 0's."""

    def __init__(self, members):
        self.members = list(members)
        arr = (C.c_void_p * len(self.members))(*[m._h.value for m in self.members])
        self._h = C.c_void_p()
        _ck(lib().kb_bus_group_create(arr, len(self.members), C.byref(self._h)))
        self._pending = {}          # ticket -> number of read sets (the capacity of its records)
        self._stats = None

    def close(self):
        if self._h:
            lib().kb_bus_group_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def submit(self, member, files):
        """files: (bases uint8, offsets uint32) per file of the technology, as BUSProcessor.process_sets -> ticket"""
        nf = self.members[member].nfiles if 0 <= member < len(self.members) else len(files)
        bs = [np.ascontiguousarray(b, np.uint8) for b, _ in files]
        os_ = [np.ascontiguousarray(o, np.uint32) for _, o in files]
        n = len(os_[0]) - 1
        bp = (C.c_void_p * nf)(*[b.ctypes.data for b in bs])
        op = (C.c_void_p * nf)(*[o.ctypes.data for o in os_])
        t = C.c_uint64(0)
        _ck(lib().kb_bus_group_submit(self._h, member, bp, op, n, C.byref(t)))
        self._pending[t.value] = n
        self._stats = None
        return t.value

    def complete(self, ticket):
        """-> the batch's records (structured array), run-wide EC ids"""
        rec = np.zeros(max(1, self._pending.get(ticket, 0)), BUS_RECORD_DTYPE)
        nrec = C.c_uint32(0)
        _ck(lib().kb_bus_group_complete(self._h, C.c_uint64(ticket), _p(rec), C.byref(nrec)))
        self._pending.pop(ticket, None)
        return rec[: nrec.value]

    def begin_sample(self, barcode):
        _ck(lib().kb_bus_group_begin_sample(self._h, C.c_uint64(barcode)))

    def finalize(self):
        s = kb_run_stats()
        _ck(lib().kb_bus_group_finalize(self._h, C.byref(s)))
        self._stats = {f: getattr(s, f) for f, _ in kb_run_stats._fields_}
        return self._stats

    def ec_table(self):
        """-> (offsets uint64[n+1], tids uint32, counts uint32[n]), ids in run-wide order"""
        st = self._stats or self.finalize()
        n, m = st["n_ecs"], st["n_ec_entries"]
        off = np.zeros(n + 1, np.uint64)
        tids = np.zeros(max(1, m), np.uint32)
        counts = np.zeros(max(1, n), np.uint32)
        _ck(lib().kb_bus_group_ec_table(self._h, _p(off), _p(tids), _p(counts)))
        return off, tids[:m], counts[:n]

    @property
    def flens(self):
        return self.members[0].flens

    def lengths(self):
        b, u = np.zeros(33, np.uint32), np.zeros(33, np.uint32)
        _ck(lib().kb_bus_group_lengths(self._h, _p(b), _p(u)))
        return b, u

    def frame_clashes(self):
        n = C.c_uint64(0)
        _ck(lib().kb_bus_group_frame_clashes(self._h, C.byref(n)))
        return n.value


def eff_lens(index, flens=None, fld_mean=0.0, fld_sd=0.0):
    """Effective lengths as the reference forms them (kb_eff_lens) -> (eff_lens, mean_fl, sd_fl)."""
    out = np.zeros(index.num_trans, np.float64)
    m, s = C.c_double(0), C.c_double(0)
    fl = None if flens is None else np.ascontiguousarray(flens, np.uint32)
    _ck(lib().kb_eff_lens(index._h, _p(fl), fld_mean, fld_sd, _p(out), C.byref(m), C.byref(s)))
    return out, m.value, s.value


def _genes_arg(index, genes):
    """genes = (gene of every target, -1 for none; number of genes) -> (int32 array, n_genes)."""
    gene_of, n_genes = genes
    gene_of = np.ascontiguousarray(gene_of, np.int32)
    if gene_of.shape != (index.num_trans,):
        raise ValueError("genes: one gene id per target (%d), got shape %s" % (index.num_trans, gene_of.shape))
    return gene_of, int(n_genes)


def tcc_run(index, ec_sets, rows, eff, genes=None, priors=None):
    """`kallisto quant-tcc` on the device: ec_sets = list of sorted transcript-id tuples (EC id = position), rows = per sample
    a list of (ec id, count); eff = effective lengths (n_targets, or n_samples x n_targets) -> (est_counts (S, T), rounds (S)).
    genes = (gene of every target, -1 for none; number of genes): gene-level output summed on the device
    (kb_tcc_run_genes) -> (est_counts, rounds, gene_counts (S, G), gene_tpm (S, G)).  priors (n_targets values): the start of
    every sample's EM instead of the uniform one (kb_tcc_run_priors)."""
    T = index.num_trans
    eo = np.zeros(len(ec_sets) + 1, np.uint64)
    tids = []
    for i, s_ in enumerate(ec_sets):
        tids.extend(s_)
        eo[i + 1] = len(tids)
    tids = np.asarray(tids, np.uint32) if tids else np.zeros(1, np.uint32)
    ro = np.zeros(len(rows) + 1, np.uint64)
    ids, vals = [], []
    for i, r in enumerate(rows):
        for e, c in r:
            ids.append(e); vals.append(c)
        ro[i + 1] = len(ids)
    ids = np.asarray(ids, np.uint32) if ids else np.zeros(1, np.uint32)
    vals = np.asarray(vals, np.uint32) if vals else np.zeros(1, np.uint32)
    eff = np.ascontiguousarray(eff, np.float64)
    per_sample = int(eff.ndim == 2)
    est = np.zeros((len(rows), T), np.float64)
    rounds = np.zeros(max(1, len(rows)), np.int32)
    if priors is not None:
        priors = np.ascontiguousarray(priors, np.float64)
        if priors.shape != (T,):
            raise ValueError("priors: one value per target (%d), got shape %s" % (T, priors.shape))
        gene_of, G = _genes_arg(index, genes) if genes is not None else (None, 0)
        gc = np.zeros((len(rows), max(1, G)), np.float64)
        gt = np.zeros((len(rows), max(1, G)), np.float64)
        _ck(lib().kb_tcc_run_priors(index._h, len(ec_sets), _p(eo), _p(tids), len(rows), _p(ro), _p(ids), _p(vals),
                                    _p(eff), per_sample, _p(gene_of), G, _p(priors), _p(est), _p(rounds),
                                    _p(gc) if G else None, _p(gt) if G else None))
        if genes is None:
            return est, rounds[: len(rows)]
        return est, rounds[: len(rows)], gc[:, :G], gt[:, :G]
    if genes is None:
        _ck(lib().kb_tcc_run(index._h, len(ec_sets), _p(eo), _p(tids), len(rows), _p(ro), _p(ids), _p(vals), _p(eff),
                             per_sample, _p(est), _p(rounds)))
        return est, rounds[: len(rows)]
    gene_of, G = _genes_arg(index, genes)
    gc = np.zeros((len(rows), max(1, G)), np.float64)
    gt = np.zeros((len(rows), max(1, G)), np.float64)
    _ck(lib().kb_tcc_run_genes(index._h, len(ec_sets), _p(eo), _p(tids), len(rows), _p(ro), _p(ids), _p(vals), _p(eff),
                               per_sample, _p(gene_of), G, _p(est), _p(rounds), _p(gc), _p(gt)))
    return est, rounds[: len(rows)], gc[:, :G], gt[:, :G]


def tcc_bootstrap(index, ec_off, ec_tids, row_off, ec_ids, counts, eff, seed, n_bootstrap, on_chunk, want_samples=False,
                  genes=None):
    """kb_tcc_bootstrap_run on CSR arrays (EC table ec_off / ec_tids, TCC rows row_off / ec_ids / counts, EC ids strictly
    increasing within a row).  on_chunk(first, est (count, T), rounds (count,), samples (count, n_ecs) or None) receives
    the problems g = row * n_bootstrap + b in order; the arrays are copies.  genes = (gene of every target, -1 for none;
    number of genes): kb_tcc_bootstrap_run_genes, and on_chunk also receives gene_counts and gene_tpm (count, G)."""
    T = index.num_trans
    n_ecs = len(ec_off) - 1
    ec_off, ro = np.ascontiguousarray(ec_off, np.uint64), np.ascontiguousarray(row_off, np.uint64)
    ec_tids = np.ascontiguousarray(ec_tids if len(ec_tids) else np.zeros(1), np.uint32)
    ec_ids = np.ascontiguousarray(ec_ids if len(ec_ids) else np.zeros(1), np.uint32)
    counts = np.ascontiguousarray(counts if len(counts) else np.zeros(1), np.uint32)
    eff = np.ascontiguousarray(eff, np.float64)
    err = []

    def arrays(count, est, rounds, samples):
        return (np.ctypeslib.as_array(est, (count, T)).copy(), np.ctypeslib.as_array(rounds, (count,)).copy(),
                np.ctypeslib.as_array(samples, (count, n_ecs)).copy() if samples and n_ecs else None)

    def cb(_user, first, count, est, rounds, samples):
        try:
            on_chunk(first, *arrays(count, est, rounds, samples))
            return 0
        except BaseException as e:      # stops the run; raised again below
            err.append(e)
            return 1

    def cb_genes(_user, first, count, est, rounds, samples, gc, gt):
        try:
            g = [np.ctypeslib.as_array(x, (count, G)).copy() if G else np.zeros((count, 0)) for x in (gc, gt)]
            on_chunk(first, *arrays(count, est, rounds, samples), *g)
            return 0
        except BaseException as e:
            err.append(e)
            return 1
    if genes is None:
        rc = lib().kb_tcc_bootstrap_run(index._h, n_ecs, _p(ec_off), _p(ec_tids), len(ro) - 1, _p(ro), _p(ec_ids),
                                        _p(counts), _p(eff), int(eff.ndim == 2), int(seed), int(n_bootstrap),
                                        int(want_samples), TCC_BOOTSTRAP_CB(cb), None)
    else:
        gene_of, G = _genes_arg(index, genes)
        rc = lib().kb_tcc_bootstrap_run_genes(index._h, n_ecs, _p(ec_off), _p(ec_tids), len(ro) - 1, _p(ro), _p(ec_ids),
                                              _p(counts), _p(eff), int(eff.ndim == 2), _p(gene_of), G, int(seed),
                                              int(n_bootstrap), int(want_samples), TCC_BOOTSTRAP_GENES_CB(cb_genes), None)
    if err:
        raise err[0]
    _ck(rc)


def fastx_summary(path, threads=1):
    """(reads, bases, FNV-1a of the sequences) through the CLI's reader; threads > 1 = the parallel ingest path."""
    n, b, h = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    _ck(lib().kb_fastx_summary_mt(os.fsencode(path), int(threads), C.byref(n), C.byref(b), C.byref(h)))
    return n.value, b.value, h.value


def gz_summary(path):
    """(bytes, crc32) of a gzip file's content through the CLI's own inflate (csrc/fast_inflate.hpp)."""
    n, c = C.c_uint64(0), C.c_uint32(0)
    _ck(lib().kb_gz_summary(os.fsencode(path), C.byref(n), C.byref(c)))
    return n.value, c.value


def counts_to_tpm(est_counts, eff_lens):
    est_counts = np.ascontiguousarray(est_counts, np.float64)
    eff_lens = np.ascontiguousarray(eff_lens, np.float64)
    out = np.zeros(len(est_counts), np.float64)
    _ck(lib().kb_counts_to_tpm(_p(est_counts), _p(eff_lens), len(est_counts), _p(out)))
    return out
