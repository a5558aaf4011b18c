"""ctypes binding of the C-ABI declared in include/fastp_b200.h.

This is the thin Python mirror used by tests/ and bench.py; the product is libfastp_b200.so
(hand-written CUDA for sm_90a + a C++ host side).  Loading fails loudly when the shared library is
missing: there is no CPU fallback.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfastp_b200.so")

# verdict codes (reference src/common.h:43-51)
PASS_FILTER, FAIL_POLY_X, FAIL_OVERLAP, FAIL_N_BASE = 0, 4, 8, 12
FAIL_LENGTH, FAIL_TOO_LONG, FAIL_QUALITY, FAIL_COMPLEXITY, FAIL_ADAPTER_DIMER = 16, 17, 20, 24, 28

F_DROPPED, F_ADAPTER_TRIMMED, F_POLYX_TRIMMED, F_CORRECTED, F_POLYG_TRIMMED, F_ADAPTER_DIMER = 1, 2, 4, 8, 16, 32

FR_READSTATS, FR_ADAPTER_READS, FR_ADAPTER_BASES, FR_POLYX_READS, FR_POLYX_BASES = 0, 32, 33, 34, 38
FR_CORRECTION, FR_CORRECTED_READS, FR_MERGED_PAIRS, FR_WORDS = 42, 106, 107, 108

STATS_PRE1, STATS_POST1, STATS_PRE2, STATS_POST2 = 0, 1, 2, 3
KMER_BINS, QUAL_BINS, CYCLE_KINDS = 1024, 128, 34


class Params(C.Structure):
    """fp_params: POD mirror of the reference Options fields the chain reads (src/options.h)."""
    _fields_ = [
        ("paired", C.c_int32), ("thread0_semantics", C.c_int32),
        ("trim_front1", C.c_int32), ("trim_tail1", C.c_int32), ("trim_front2", C.c_int32),
        ("trim_tail2", C.c_int32), ("max_len1", C.c_int32), ("max_len2", C.c_int32),
        ("cut_front", C.c_int32), ("cut_tail", C.c_int32), ("cut_right", C.c_int32),
        ("cut_front_window", C.c_int32), ("cut_front_quality", C.c_int32),
        ("cut_tail_window", C.c_int32), ("cut_tail_quality", C.c_int32),
        ("cut_right_window", C.c_int32), ("cut_right_quality", C.c_int32),
        ("polyg_enabled", C.c_int32), ("polyg_min_len", C.c_int32),
        ("polyx_enabled", C.c_int32), ("polyx_min_len", C.c_int32),
        ("adapter_enabled", C.c_int32), ("has_seq_r1", C.c_int32), ("has_seq_r2", C.c_int32),
        ("adapter_seq_r1", C.c_char_p), ("adapter_seq_r2", C.c_char_p),
        ("n_fasta_adapters", C.c_int32), ("fasta_adapters", C.POINTER(C.c_char_p)),
        ("allow_gap_overlap_trimming", C.c_int32), ("dimer_max_len", C.c_int32),
        ("correction_enabled", C.c_int32),
        ("overlap_require", C.c_int32), ("overlap_diff_limit", C.c_int32), ("overlap_diff_percent_limit", C.c_int32),
        ("qual_filter_enabled", C.c_int32), ("qualified_qual", C.c_int32),
        ("unqualified_percent_limit", C.c_int32), ("n_base_limit", C.c_int32), ("avg_qual_req", C.c_int32),
        ("length_filter_enabled", C.c_int32), ("length_required", C.c_int32), ("length_limit", C.c_int32),
        ("complexity_filter_enabled", C.c_int32), ("complexity_threshold", C.c_double),
        ("insert_size_max", C.c_int32), ("seq_len1", C.c_int32), ("seq_len2", C.c_int32),
        ("overrep_enabled", C.c_int32), ("overrep_sampling", C.c_int32),
        ("n_overrep1", C.c_int32), ("overrep_seqs1", C.POINTER(C.c_char_p)),
        ("n_overrep2", C.c_int32), ("overrep_seqs2", C.POINTER(C.c_char_p)),
        ("merge_enabled", C.c_int32), ("merge_include_unmerged", C.c_int32),
    ]


class Batch(C.Structure):
    _fields_ = [
        ("n", C.c_int64), ("stride", C.c_int32), ("flags", C.c_int32),
        ("seq1", C.c_void_p), ("qual1", C.c_void_p), ("len1", C.c_void_p),
        ("seq2", C.c_void_p), ("qual2", C.c_void_p), ("len2", C.c_void_p),
        ("first_read_index", C.c_int64),
    ]


class PackedBatch(C.Structure):
    _fields_ = [
        ("n", C.c_int64), ("pitch_b", C.c_int32), ("pitch_q", C.c_int32),
        ("bases1", C.c_void_p), ("qual1", C.c_void_p), ("len1", C.c_void_p),
        ("bases2", C.c_void_p), ("qual2", C.c_void_p), ("len2", C.c_void_p),
        ("npos", C.c_void_p), ("n_npos", C.c_int64), ("npos_cap", C.c_int64),
        ("flags", C.c_int32), ("_pad", C.c_int32), ("first_read_index", C.c_int64),
    ]


class CounterLayout(C.Structure):
    _fields_ = [
        ("cycles", C.c_int32), ("n_stats", C.c_int32), ("isize_bins", C.c_int32), ("_pad", C.c_int32),
        ("stats_stride", C.c_int64), ("off_kmer", C.c_int64), ("off_qualhist", C.c_int64),
        ("off_reads", C.c_int64), ("off_length_sum", C.c_int64),
        ("off_filter", C.c_int64), ("off_isize", C.c_int64),
        ("n_overrep", C.c_int32 * 2), ("overrep_len", C.c_int32 * 2), ("off_overrep", C.c_int64 * 4),
        ("total", C.c_int64),
    ]


# numpy views of the record structs
READ_RESULT_DTYPE = np.dtype([
    ("front", "<u2"), ("len", "<u2"), ("verdict", "u1"), ("flags", "u1"), ("adapter_pos", "<i2"),
    ("adapter_len", "<u2"), ("polyx_base", "u1"), ("pair_verdict", "u1"), ("polyx_len", "<u2"),
    ("reserved", "<u2"),      # flags2 of the C struct (FP_F2_*): 0 unless the index filter is on, so it keeps its old column name here
])
OV_RESULT_DTYPE = np.dtype([
    ("overlapped", "u1"), ("has_gap", "u1"), ("offset", "<i2"), ("overlap_len", "<i2"), ("diff", "<i2"),
])
PATCH_DTYPE = np.dtype([
    ("pair", "<u4"), ("pos", "<u2"), ("which", "u1"), ("base", "u1"), ("qual", "u1"), ("old_base", "u1"), ("old_qual", "u1"), ("_pad", "u1"),
])
assert READ_RESULT_DTYPE.itemsize == 16 and OV_RESULT_DTYPE.itemsize == 8 and PATCH_DTYPE.itemsize == 12

EVENT_DTYPE = np.dtype([("unit", "<u4"), ("start", "<u2"), ("len", "<u2"), ("key", "<u2"), ("which", "u1"), ("kind", "u1"),
                        ("adapter", "<u2"), ("_pad", "<u2")])
assert EVENT_DTYPE.itemsize == 16

FASTQ_REC_DTYPE = np.dtype([("name_off", "<u4"), ("name_len", "<u4"), ("strand_off", "<u4"), ("strand_len", "<u4")])


class FastqInfo(C.Structure):
    _fields_ = [("n_records", C.c_int64), ("consumed", C.c_int64), ("n_lines", C.c_int64), ("error", C.c_int32), ("more", C.c_int32),
                ("error_record", C.c_int64)]


# name -> (restype, argtypes): every symbol include/fastp_b200.h declares
FP_B_INDEXED = 0x1          # fp_batch.flags
FP_B_PACK2BIT = 0x2
FP_FQ_OUT_MERGED, FP_FQ_OUT_R1, FP_FQ_OUT_R2 = 0, 1, 2   # fp_fastq_encode_merge `which`
FP_FQ_OUT_UNPAIRED1, FP_FQ_OUT_UNPAIRED2, FP_FQ_OUT_FAILED = 3, 4, 5   # fp_fastq_encode_rejects `which`
FP_FQ_OUTS = 6                                           # fp_fastq_process_host_outs: buffers indexed by FP_FQ_OUT_*
FP_FQ_W_UNPAIRED1, FP_FQ_W_UNPAIRED2 = 0x1, 0x2          # fp_fastq_encode_rejects `writers`

SYMBOLS = {
    "fp_params_default": (None, [C.POINTER(Params), C.c_int]),
    "fp_counter_layout_make": (None, [C.POINTER(CounterLayout), C.c_int, C.c_int, C.c_int]),
    "fp_counter_layout_make_overrep": (None, [C.POINTER(CounterLayout), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "fp_abi_sizeof": (C.c_size_t, [C.c_int]),
    "fp_ctx_create": (C.c_int, [C.POINTER(Params), C.c_int, C.c_int64, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
    "fp_ctx_destroy": (None, [C.c_void_p]),
    "fp_last_error": (C.c_char_p, []),
    "fp_ctx_layout": (C.c_int, [C.c_void_p, C.POINTER(CounterLayout)]),
    "fp_process_se": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p]),
    "fp_process_pe": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_uint32, C.c_void_p, C.c_void_p]),
    "fp_process_se_host": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p]),
    "fp_process_pe_host": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_void_p]),
    "fp_process_pe_host_patches": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                             C.POINTER(C.c_uint64)]),
    "fp_set_event_sink": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]),
    "fp_set_host_event_sink": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "fp_set_host_threads": (C.c_int, [C.c_void_p, C.c_int]),
    "fp_host_pack_rows": (C.c_int, [C.POINTER(Batch), C.c_int, C.POINTER(PackedBatch), C.c_int]),
    "fp_process_se_host_packed": (C.c_int, [C.c_void_p, C.POINTER(PackedBatch), C.c_void_p]),
    "fp_process_pe_host_packed": (C.c_int, [C.c_void_p, C.POINTER(PackedBatch), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                            C.POINTER(C.c_uint64)]),
    "fp_counters_reset": (C.c_int, [C.c_void_p]),
    "fp_counters_fetch": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fp_counters_device_ptr": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "fp_counters_allreduce": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "fp_patches_undo": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]),
    "fp_overrep_defer_post": (C.c_int, [C.c_void_p, C.c_int32]),
    "fp_pass_count": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p]),
    "fp_overrep_post": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "fp_host_overrep_candidates": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64,
                                             C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "fp_gz_is_bgzf": (C.c_int, [C.c_void_p, C.c_int64]),
    "fp_gz_inflate": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_int]),
    "fp_gz_deflate_bound": (C.c_int64, [C.c_int64, C.c_int64]),
    "fp_gz_deflate": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_int64, C.c_int, C.c_int]),
    "fp_gz_open": (C.c_void_p, [C.c_char_p]),
    "fp_gz_read": (C.c_int64, [C.c_void_p, C.c_void_p, C.c_int64]),
    "fp_gz_close": (None, [C.c_void_p]),
    "fp_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_size_t]),
    "fp_host_free": (C.c_int, [C.c_void_p]),
    "fp_synth_fill": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_int64, C.c_uint64, C.c_int32, C.c_int32, C.c_void_p]),
    "fp_kernel_time_ms": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.c_int]),
    "fp_version": (C.c_int, []),
    "fp_dup_check": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_int32, C.c_void_p, C.c_void_p]),
    "fp_dup_totals": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "fp_dup_reset": (C.c_int, [C.c_void_p]),
    "fp_set_dup_flags": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fp_fastq_set_dedup": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "fp_fastq_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                  C.c_void_p, C.POINTER(FastqInfo)]),
    "fp_fastq_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                  C.POINTER(C.c_int64)]),
    "fp_fastq_process_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p, C.c_int64, C.POINTER(C.c_int64),
                                        C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                        C.POINTER(FastqInfo), C.POINTER(FastqInfo)]),
    "fp_fastq_encode_merge": (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 11 + [C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]),
    "fp_fastq_process_host_merge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                              C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p, C.c_int64, C.POINTER(C.c_int64),
                                              C.c_void_p, C.c_int64, C.POINTER(C.c_int64),
                                              C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                              C.POINTER(FastqInfo), C.POINTER(FastqInfo)]),
    "fp_fastq_encode_rejects": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [C.c_void_p] * 12 + [C.c_int64, C.c_void_p, C.c_int64,
                                                                                                   C.POINTER(C.c_int64)]),
    "fp_fastq_process_host_outs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                             C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                             C.POINTER(FastqInfo), C.POINTER(FastqInfo)]),
    "fp_fastq_decode_interleaved": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32] + [C.c_void_p] * 8
                                    + [C.c_int64, C.POINTER(FastqInfo)]),
    "fp_fastq_encode_interleaved": (C.c_int, [C.c_void_p] + [C.c_void_p] * 10 + [C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]),
    "fp_fastq_set_interleaved": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "fp_set_overlapped_sink": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fp_fastq_encode_overlapped": (C.c_int, [C.c_void_p] + [C.c_void_p] * 7 + [C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]),
    "fp_fastq_set_overlapped_out": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]),
    "fp_set_index_flags": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fp_fastq_set_index_filter": (C.c_int, [C.c_void_p, C.POINTER(C.c_char_p), C.c_int64, C.POINTER(C.c_char_p), C.c_int64, C.c_int32]),
    "fp_fastq_index_flags": (C.c_int, [C.c_void_p] + [C.c_void_p] * 4 + [C.c_int64, C.c_void_p]),
}


def bind(lib, names=None):
    for name in (names or SYMBOLS):
        res, args = SYMBOLS[name]
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


_lib = None


def load():
    """Load libfastp_b200.so (built in-tree by __graft_entry__.build()).  No fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
                "fastp_b200 has no CPU fallback.")
        _lib = bind(C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL))
        assert _lib.fp_abi_sizeof(0) == C.sizeof(Params), "fp_params ABI mismatch"
        assert _lib.fp_abi_sizeof(1) == C.sizeof(Batch)
        assert _lib.fp_abi_sizeof(5) == C.sizeof(CounterLayout)
    return _lib


def default_params(paired, lib=None, **overrides):
    """fp_params_default + keyword overrides.  Adapter strings are kept alive on the object."""
    lib = lib or load()
    p = Params()
    lib.fp_params_default(C.byref(p), 1 if paired else 0)
    set_params(p, **overrides)
    return p


def set_params(p, **kw):
    for k, v in kw.items():
        if k in ("adapter_seq_r1", "adapter_seq_r2"):
            b = v.encode() if isinstance(v, str) else v
            setattr(p, k, b)
            setattr(p, "has_seq_" + k[-2:], 1 if b else 0)
        elif k in ("overrep_seqs1", "overrep_seqs2"):
            items = [a.encode() if isinstance(a, str) else a for a in v]
            arr = (C.c_char_p * max(len(items), 1))(*items)
            keep = getattr(p, "_overrep_keepalive", {})
            keep[k] = (arr, items)
            p._overrep_keepalive = keep
            setattr(p, k, C.cast(arr, C.POINTER(C.c_char_p)))
            setattr(p, "n_overrep" + k[-1], len(items))
        elif k == "fasta_adapters":
            items = [a.encode() if isinstance(a, str) else a for a in v]
            arr = (C.c_char_p * len(items))(*items)
            p._fasta_keepalive = (arr, items)
            p.fasta_adapters = C.cast(arr, C.POINTER(C.c_char_p))
            p.n_fasta_adapters = len(items)
        else:
            if not hasattr(p, k):
                raise AttributeError(k)
            setattr(p, k, v)
    return p


def make_layout(lib, paired, cycles, insert_size_max=512, params=None):
    """Counter layout; with `params` the over-representation regions follow its candidate lists."""
    L = CounterLayout()
    if params is not None and params.overrep_enabled:
        lib.fp_counter_layout_make_overrep(C.byref(L), 1 if paired else 0, cycles, insert_size_max,
                                           params.n_overrep1, params.seq_len1, params.n_overrep2, params.seq_len2)
    else:
        lib.fp_counter_layout_make(C.byref(L), 1 if paired else 0, cycles, insert_size_max)
    return L


class CounterView:
    """Named views into the packed int64 counter block (layout in include/fastp_b200.h)."""

    def __init__(self, layout, data):
        self.L = layout
        self.data = np.asarray(data, dtype=np.int64)
        assert self.data.size == layout.total

    def stats(self, s):
        L = self.L
        base = s * L.stats_stride
        d = self.data
        return {
            "cycle": d[base: base + CYCLE_KINDS * L.cycles].reshape(CYCLE_KINDS, L.cycles),
            "kmer": d[base + L.off_kmer: base + L.off_kmer + KMER_BINS],
            "qualhist": d[base + L.off_qualhist: base + L.off_qualhist + QUAL_BINS],
            "reads": int(d[base + L.off_reads]),
            "length_sum": int(d[base + L.off_length_sum]),
        }

    def overrep(self, s):
        """(count[K], dist[K][seqLen]) of Stats s (stats.cpp:270-288)."""
        L = self.L
        side = s >> 1
        k, ln = L.n_overrep[side], L.overrep_len[side]
        base = L.off_overrep[s]
        return self.data[base: base + k], self.data[base + k: base + k + k * ln].reshape(k, ln) if k else self.data[base:base].reshape(0, max(ln, 1))

    @property
    def filter(self):
        return self.data[self.L.off_filter: self.L.off_filter + FR_WORDS]

    @property
    def isize(self):
        return self.data[self.L.off_isize: self.L.off_isize + self.L.isize_bins]

    def summary(self, s):
        """What Stats::summarize derives (src/stats.cpp:102-182): cycles, bases, q20, q30."""
        st = self.stats(s)
        tb = st["cycle"][32]
        nz = np.nonzero(tb == 0)[0]
        cycles = int(nz[0]) if nz.size else tb.size
        return {
            "reads": st["reads"], "bases": int(tb[:cycles].sum()),
            "q20": int(st["cycle"][8:16, :cycles].sum()), "q30": int(st["cycle"][0:8, :cycles].sum()),
            "cycles": cycles,
        }


def host_batch(n, stride, paired):
    """Allocate a numpy-backed host batch.  Returns (Batch, dict of arrays)."""
    arrs = {
        "seq1": np.zeros((n, stride), np.uint8), "qual1": np.zeros((n, stride), np.uint8), "len1": np.zeros(n, np.uint16),
    }
    if paired:
        arrs.update(seq2=np.zeros((n, stride), np.uint8), qual2=np.zeros((n, stride), np.uint8), len2=np.zeros(n, np.uint16))
    return batch_from_arrays(arrs), arrs


def batch_from_arrays(arrs):
    b = Batch()
    b.n = arrs["seq1"].shape[0]
    b.stride = arrs["seq1"].shape[1]
    for k in ("seq1", "qual1", "len1", "seq2", "qual2", "len2"):
        if k in arrs and arrs[k] is not None:
            a = arrs[k]
            assert a.flags["C_CONTIGUOUS"]
            setattr(b, k, a.ctypes.data)
    b._keepalive = arrs
    return b


def batch_from_strings(reads1, reads2=None, stride=None):
    """reads = list of (seq, qual) str/bytes pairs -> host batch."""
    mx = max([len(s) for s, _ in reads1] + ([len(s) for s, _ in reads2] if reads2 else []) + [1])
    stride = stride or ((mx + 15) // 16 * 16)
    b, arrs = host_batch(len(reads1), stride, reads2 is not None)
    for key, reads in (("1", reads1), ("2", reads2)):
        if reads is None:
            continue
        for i, (s, q) in enumerate(reads):
            s = s.encode() if isinstance(s, str) else s
            q = q.encode() if isinstance(q, str) else q
            assert len(s) == len(q)
            arrs["seq" + key][i, :len(s)] = np.frombuffer(s, np.uint8)
            arrs["qual" + key][i, :len(q)] = np.frombuffer(q, np.uint8)
            arrs["len" + key][i] = len(s)
    return b, arrs


def check(rc, lib=None):
    if rc != 0:
        msg = (lib or load()).fp_last_error()
        raise RuntimeError(f"fastp_b200 error {rc}: {msg.decode() if msg else ''}")
