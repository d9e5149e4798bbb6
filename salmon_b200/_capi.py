"""ctypes binding of libsalmon_b200.so (the C ABI in include/salmon_b200.h).

Plumbing only: numpy arrays in, numpy arrays out.  There is no CPU fallback --
if the shared library is missing or no CUDA device is usable, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsalmon_b200.so")

SB_OK = 0


class SalmonB200Error(RuntimeError):
    pass


class sb_eq_csr(C.Structure):
    _fields_ = [
        ("n_classes", C.c_uint64),
        ("n_txps", C.c_uint32),
        ("off", C.c_void_p),
        ("tids", C.c_void_p),
        ("weights", C.c_void_p),
        ("counts", C.c_void_p),
    ]


class sb_em_params(C.Structure):
    _fields_ = [
        ("use_vbem", C.c_int32),
        ("per_txp_prior", C.c_int32),
        ("init_uniform", C.c_int32),
        ("eq_class_mode", C.c_int32),
        ("no_rich_eq", C.c_int32),
        ("no_length_correction", C.c_int32),
        ("alt_init", C.c_int32),
        ("reserved", C.c_int32),
        ("vb_prior", C.c_double),
        ("tol", C.c_double),
        ("num_required_frags", C.c_double),
        ("min_iter", C.c_uint32),
        ("max_iter", C.c_uint32),
    ]


class sb_em_stats(C.Structure):
    _fields_ = [
        ("iters", C.c_uint32),
        ("converged", C.c_uint32),
        ("max_rel_diff", C.c_double),
        ("alpha_sum", C.c_double),
        ("n_degenerate", C.c_uint64),
        ("n_multi_classes", C.c_uint64),
        ("nnz_multi", C.c_uint64),
        ("n_active_txps", C.c_uint32),
        ("gpu_launches", C.c_uint32),
        ("prepare_ms", C.c_float),
        ("run_ms", C.c_float),
        ("loop_kernel_ms", C.c_float),
        ("loop_kernel_launches", C.c_uint32),
    ]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class sb_map_params(C.Structure):
    _fields_ = [
        ("k", C.c_uint32), ("stride", C.c_uint32), ("max_occs_per_hit", C.c_uint32), ("max_read_occ", C.c_uint32),
        ("max_frag_len", C.c_uint32), ("band", C.c_uint32), ("chain_gap", C.c_uint32), ("range_bins", C.c_uint32),
        ("ma", C.c_int32), ("mp", C.c_int32), ("go", C.c_int32), ("ge", C.c_int32),
        ("hard_filter", C.c_int32), ("first_decoy", C.c_int32),
        ("consensus_frac", C.c_double), ("min_score_fraction", C.c_double), ("score_exp", C.c_double),
        ("min_aln_prob", C.c_double), ("decoy_threshold", C.c_double), ("fld_mean", C.c_double), ("fld_sd", C.c_double),
        ("num_pre_burnin", C.c_uint64), ("num_burnin", C.c_uint64),
        ("seed", C.c_uint64), ("mini_batch", C.c_uint32), ("reserved2", C.c_uint32),
        ("pre_merge_thresh", C.c_double), ("post_merge_thresh", C.c_double), ("orphan_thresh", C.c_double),
        ("allow_dovetail", C.c_int32), ("allow_orphans", C.c_int32), ("lib_type", C.c_int32),
        ("recover_orphans", C.c_int32), ("softclip", C.c_int32),
        ("no_single_frag_prob", C.c_int32), ("no_frag_len_dist", C.c_int32), ("no_eff_len_correction", C.c_int32),
        ("incompat_prior", C.c_double),
    ]


class sb_map_batch_stats(C.Structure):
    _fields_ = [("n_pairs", C.c_uint32), ("gpu_launches", C.c_uint32)] + \
        [(k, C.c_uint64) for k in ("mapped", "lookups", "postings", "seeds", "candidates", "kept", "label_entries",
                                   "n_batch_classes")] + [("device_ms", C.c_float), ("reserved", C.c_uint32), ("full_dp", C.c_uint64),
                                                              ("seed_kernel_ms", C.c_float), ("seed_kernel_launches", C.c_uint32)] + \
        [(k, C.c_uint64) for k in ("orphans_rescued", "rescue_searches", "rescue_no_room")] + \
        [("rescue_kernel_ms", C.c_float), ("reserved2", C.c_uint32), ("compatible", C.c_uint64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class sb_map_result(C.Structure):
    _fields_ = [("n_classes", C.c_uint64), ("off", C.POINTER(C.c_uint64)), ("tids", C.POINTER(C.c_uint32)),
                ("weights", C.POINTER(C.c_double)), ("counts", C.POINTER(C.c_uint64)), ("bins", C.POINTER(C.c_uint32))] + \
        [(k, C.c_uint64) for k in ("n_mapped", "lookups", "postings", "seeds", "candidates", "kept", "label_entries")] + \
        [("n_txps", C.c_uint32), ("reserved", C.c_uint32), ("projected_counts", C.POINTER(C.c_double)),
         ("eff_len", C.POINTER(C.c_double)), ("unique_counts", C.POINTER(C.c_uint64)),
         ("total_counts", C.POINTER(C.c_uint64)), ("lib_format_counts", C.c_uint64 * 8)] + \
        [(k, C.c_uint64) for k in ("orphans_rescued", "rescue_searches", "rescue_no_room", "n_compatible")]


# every symbol include/salmon_b200.h declares: (name, restype, argtypes)
_P = C.c_void_p
class sb_map_partial(C.Structure):
    _fields_ = [("n_txps", C.c_uint32), ("n_fld", C.c_uint32), ("mass", C.POINTER(C.c_double)),
                ("fld_hist", C.POINTER(C.c_double)), ("fld_tot", C.c_double), ("fld_prior_hist", C.POINTER(C.c_double)),
                ("fld_prior_tot", C.c_double), ("fld_min", C.c_uint32), ("reserved", C.c_uint32),
                ("unique_counts", C.POINTER(C.c_uint64)), ("total_counts", C.POINTER(C.c_uint64)),
                ("cluster_hits", C.POINTER(C.c_uint64)), ("cluster_root", C.POINTER(C.c_uint32)), ("assigned", C.c_uint64),
                ("compatible", C.c_uint64)]


class sb_eq_file(C.Structure):
    _fields_ = [
        ("n_txps", C.c_uint32), ("has_weights", C.c_uint32), ("n_classes", C.c_uint64),
        ("names", C.POINTER(C.c_char_p)), ("off", C.c_void_p), ("tids", C.c_void_p), ("weights", C.c_void_p),
        ("counts", C.c_void_p), ("eff_len", C.c_void_p), ("n_missing_eff_len", C.c_uint32), ("reserved", C.c_uint32),
    ]


class sb_txome(C.Structure):
    _fields_ = [
        ("n_txps", C.c_uint32), ("first_decoy", C.c_uint32), ("names", C.POINTER(C.c_char_p)),
        ("seq_off", C.c_void_p), ("codes", C.c_void_p), ("complete_len", C.c_void_p),
        ("n_duplicates_removed", C.c_uint32), ("n_clipped", C.c_uint32), ("n_short", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


class sb_quant_opts(C.Structure):
    _fields_ = [("device", C.c_int32), ("batch", C.c_uint32), ("max_read_len", C.c_uint32), ("threads", C.c_uint32),
                ("dump_eq", C.c_int32), ("dump_eq_weights", C.c_int32), ("num_bootstraps", C.c_uint32),
                ("num_gibbs", C.c_uint32), ("thinning", C.c_uint32), ("no_gamma_draw", C.c_int32),
                ("shard_index", C.c_uint32), ("shard_count", C.c_uint32), ("seed", C.c_uint64), ("nccl_uid", C.c_void_p),
                ("write_mappings", C.c_char_p), ("write_qualities", C.c_int32), ("write_unmapped_names", C.c_int32),
                ("cmdline", C.c_char_p)]


class sb_read_meta(C.Structure):
    _fields_ = [("names", C.c_void_p), ("name_off", C.c_void_p), ("qual_left", C.c_void_p), ("qual_right", C.c_void_p)]


class sb_sam_stats(C.Structure):
    _fields_ = [("records", C.c_uint64), ("sam_bytes", C.c_uint64), ("unmapped_lines", C.c_uint64),
                ("batches", C.c_uint64), ("windows", C.c_uint64), ("format_ms", C.c_double), ("copy_ms", C.c_double),
                ("slot_wait_ms", C.c_double), ("write_ms", C.c_double)]


class sb_quant_summary(C.Structure):
    _fields_ = [("n_observed", C.c_uint64), ("n_mapped", C.c_uint64), ("n_too_short", C.c_uint64),
                ("n_trimmed_mates", C.c_uint64), ("n_classes", C.c_uint64), ("n_batches", C.c_uint64),
                ("n_read_lengths", C.c_uint32), ("em_iters", C.c_uint32), ("em_converged", C.c_uint32),
                ("reserved", C.c_uint32), ("map_seconds", C.c_double), ("em_seconds", C.c_double),
                ("total_seconds", C.c_double), ("map_device_ms", C.c_float), ("map_setup_ms", C.c_float)] + \
        [(k, C.c_uint64) for k in ("orphans_rescued", "rescue_searches", "rescue_no_room")]


SYMBOLS = {
    "sb_quant_default_opts": (None, [C.POINTER(sb_quant_opts)]),
    "sb_quant_files": (C.c_int, [_P, _P, _P, C.c_uint32, _P, _P, C.POINTER(sb_quant_opts), C.c_char_p, _P,
                                 C.POINTER(sb_quant_summary)]),
    "sb_reads_open": (_P, [_P, _P, C.c_uint32, C.c_uint32]),
    "sb_reads_next": (C.c_int64, [_P, C.c_uint32, C.c_uint32, _P, _P, _P, _P]),
    "sb_reads_close": (None, [_P]),
    "sb_reads_peek": (C.c_int64, [_P, C.c_uint32, _P]),
    "sb_reads_skip": (C.c_int64, [_P, C.c_uint32]),
    "sb_reads_paired": (C.c_int, [_P]),
    "sb_device_init": (C.c_int, [C.c_int]),
    "sb_map_lib_counts": (C.c_int, [_P, _P]),
    "sb_detect_lib_type": (C.c_int, [C.c_int, _P]),
    "sb_reads_bucketed": (C.c_int, [_P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, _P, _P, _P]),
    "sb_eq_file_read": (C.c_int, [C.c_char_p, C.POINTER(C.POINTER(sb_eq_file))]),
    "sb_eq_file_free": (None, [C.POINTER(sb_eq_file)]),
    "sb_bootstrap_writer_open": (_P, [C.c_char_p]),
    "sb_bootstrap_writer_write": (C.c_int, [_P, _P, C.c_uint32]),
    "sb_bootstrap_writer_close": (C.c_int64, [_P]),
    "sb_txome_read_fasta": (C.c_int, [C.c_char_p, C.c_uint32, C.c_int, C.c_char_p, C.c_int, C.c_int,
                                      C.POINTER(C.POINTER(sb_txome))]),
    "sb_txome_free": (None, [C.POINTER(sb_txome)]),
    "sb_version": (C.c_int, []),
    "sb_last_error": (C.c_char_p, []),
    "sb_device_count": (C.c_int, []),
    "sb_em_default_params": (None, [C.POINTER(sb_em_params)]),
    "sb_em_create": (_P, [C.c_int]),
    "sb_em_destroy": (None, [_P]),
    "sb_em_optimize": (C.c_int, [_P, C.POINTER(sb_eq_csr), C.POINTER(sb_em_params), _P, _P, _P, _P,
                                 C.POINTER(sb_em_stats)]),
    "sb_em_upload": (C.c_int, [_P, C.POINTER(sb_eq_csr), _P, _P, _P]),
    "sb_em_prepare": (C.c_int, [_P, C.POINTER(sb_em_params), C.POINTER(sb_em_stats)]),
    "sb_em_run": (C.c_int, [_P, C.POINTER(sb_em_stats)]),
    "sb_em_download": (C.c_int, [_P, _P, C.POINTER(sb_em_stats)]),
    "sb_em_get_combined": (C.c_int, [_P, _P, _P]),
    "sb_em_set_option": (C.c_int, [_P, C.c_char_p, C.c_int64]),
    "sb_em_get_info": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_int64)]),
    "sb_em_debug_timeline": (C.c_int, [_P, _P, C.c_uint32]),
    "sb_bootstrap": (C.c_int, [_P, C.POINTER(sb_em_params), C.c_double, C.c_uint32, C.c_uint64, _P, _P]),
    "sb_bootstrap_last_counts": (C.c_int, [_P, _P]),
    "sb_gibbs": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_double, C.c_uint32, C.c_uint32, C.c_int, C.c_double,
                           C.c_uint64, _P, _P]),
    "sb_gibbs_last_state": (C.c_int, [_P, _P, _P]),
    "sb_nccl_unique_id": (C.c_int, [_P]),
    "sb_em_comm_init": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "sb_em_comm_destroy": (C.c_int, [_P]),
    "sb_em_peer_handle": (C.c_int, [_P, C.c_uint32, _P]),
    "sb_em_peer_open": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "sb_flush_l2": (C.c_int, [_P]),
    "sb_index_build": (_P, [C.c_uint32, _P, _P, C.c_uint32]),
    "sb_index_free": (None, [_P]),
    "sb_index_set_meta": (C.c_int, [_P, _P, _P, C.c_uint32]),
    "sb_index_get_meta": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "sb_index_save": (C.c_int, [_P, C.c_char_p]),
    "sb_index_load": (_P, [C.c_char_p]),
    "sb_index_info": (C.c_int, [_P, _P]),
    "sb_index_host_arrays": (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    "sb_map_default_params": (None, [C.POINTER(sb_map_params)]),
    "sb_map_mimic_bt2": (C.c_int, [C.POINTER(sb_map_params), C.c_int]),
    "sb_map_create": (_P, [_P, C.POINTER(sb_map_params), C.c_int, C.c_uint32, C.c_uint32]),
    "sb_map_destroy": (None, [_P]),
    "sb_map_batch": (C.c_int, [_P, _P, _P, C.c_uint32, C.c_uint32, C.POINTER(sb_map_batch_stats)]),
    "sb_map_finish": (C.c_int, [_P, C.POINTER(sb_map_result)]),
    "sb_map_set_option": (C.c_int, [_P, C.c_char_p, C.c_int64]),
    "sb_comm_create": (_P, [C.c_int, C.c_int, _P, C.c_int]),
    "sb_comm_destroy": (None, [_P]),
    "sb_comm_rank": (C.c_int, [_P]),
    "sb_comm_size": (C.c_int, [_P]),
    "sb_comm_allreduce": (C.c_int, [_P, _P, C.c_size_t, C.c_int, C.c_int]),
    "sb_comm_allgather": (C.c_int, [_P, _P, _P, C.c_size_t]),
    "sb_em_peer_setup": (C.c_int, [_P, _P, C.c_uint32]),
    "sb_map_reduce_global": (C.c_int, [_P, _P, _P, _P]),
    "sb_quant_eqclasses": (C.c_int, [C.c_char_p, _P, _P, C.c_char_p, _P]),
    "sb_eq_create": (_P, [C.c_uint32, C.c_int]),
    "sb_eq_destroy": (None, [_P]),
    "sb_eq_add_batch": (C.c_int, [_P, C.c_uint32, _P, _P, _P, _P, _P]),
    "sb_eq_from_host": (C.c_int, [_P, C.POINTER(sb_eq_csr)]),
    "sb_eq_finish": (C.c_int, [_P, _P]),
    "sb_map_online_state": (C.c_int, [_P, _P, _P, _P, _P]),
    "sb_map_reset": (C.c_int, [_P]),
    "sb_tpm": (C.c_int, [C.c_uint32, _P, _P, C.c_double, _P]),
    "sb_write_quant_sf": (C.c_int, [C.c_char_p, C.c_uint32, _P, _P, _P, _P, C.c_double, C.c_int]),
    "sb_write_eq_classes": (C.c_int, [C.c_char_p, C.c_uint32, _P, C.c_uint64, _P, _P, _P, _P]),
    "sb_map_partial_get": (C.c_int, [_P, C.POINTER(sb_map_partial)]),
    "sb_map_project_global": (C.c_int, [_P, C.POINTER(sb_map_partial), C.c_uint32, _P, C.POINTER(sb_map_result)]),
    "sb_map_last_alignments": (C.c_int, [_P, C.c_uint32] + [_P] * 10),
    "sb_map_last_candidates": (C.c_int, [_P, C.c_uint32] + [_P] * 4),
    "sb_rescue_search_tap": (C.c_int, [C.c_int, C.c_uint32] + [_P] * 7),
    "sb_sam_open": (_P, [C.c_char_p, C.c_char_p, _P, C.c_char_p, C.c_uint32]),
    "sb_sam_close": (C.c_int, [_P]),
    "sb_sam_write_unmapped": (C.c_int, [_P, C.c_char_p, C.c_size_t]),
    "sb_sam_get_stats": (C.c_int, [_P, C.POINTER(sb_sam_stats)]),
    "sb_map_attach_sam": (C.c_int, [_P, _P]),
    "sb_map_batch_sam": (C.c_int, [_P, _P, _P, C.c_uint32, C.c_uint32, _P, _P, _P, _P, C.POINTER(sb_map_batch_stats)]),
    "sb_reads_next_meta": (C.c_int64, [_P, C.c_uint32, C.c_uint32, _P, _P, _P, _P, C.c_int, C.POINTER(sb_read_meta)]),
    "sb_reads_bucketed_meta": (C.c_int, [_P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                         C.c_int, _P, _P, _P, _P]),
    "sb_host_register": (C.c_int, [_P, C.c_size_t]),
    "sb_host_unregister": (C.c_int, [_P]),
}

_lib = None


def load():
    """Load the shared library (raises if it has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SalmonB200Error(
                f"{LIB_PATH} not found: build it with `make` (or __graft_entry__.build()); "
                "there is no CPU fallback")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def _check(rc, what):
    if rc < 0:
        raise SalmonB200Error(f"{what} failed ({rc}): {load().sb_last_error().decode()}")
    return rc


def default_params(**over) -> sb_em_params:
    p = sb_em_params()
    load().sb_em_default_params(C.byref(p))
    for k, v in over.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


class sb_eq_table(C.Structure):
    _fields_ = [("n_classes", C.c_uint64), ("n_txps", C.c_uint32), ("reserved", C.c_uint32), ("off", C.c_void_p),
                ("tids", C.c_void_p), ("weights", C.c_void_p), ("counts", C.c_void_p), ("n_txp_in_label", C.c_void_p),
                ("label_off", C.c_void_p), ("labels", C.c_void_p), ("n_groups", C.c_uint64)]


class EqBuilder:
    """B2 seam: EquivalenceClassBuilder::addGroup / finish through the C ABI (sb_eq_*)."""

    def __init__(self, n_txps: int, device: int = 0):
        self.lib = load()
        self.h = self.lib.sb_eq_create(int(n_txps), int(device))
        if not self.h:
            raise SalmonB200Error(f"sb_eq_create: {self.lib.sb_last_error().decode()}")
        self.n_txps = n_txps

    def add_batch(self, label_off, labels, weight_off, weights, counts=None):
        label_off = np.ascontiguousarray(label_off, dtype=np.uint64); labels = np.ascontiguousarray(labels, dtype=np.uint32)
        weight_off = np.ascontiguousarray(weight_off, dtype=np.uint64); weights = np.ascontiguousarray(weights, dtype=np.float64)
        cp = None
        if counts is not None:
            counts = np.ascontiguousarray(counts, dtype=np.uint64); cp = counts.ctypes.data
        _check(self.lib.sb_eq_add_batch(self.h, len(label_off) - 1, label_off.ctypes.data, labels.ctypes.data,
                                        weight_off.ctypes.data, weights.ctypes.data, cp), "sb_eq_add_batch")

    def from_host(self, eq):
        st = eq.as_struct()
        _check(self.lib.sb_eq_from_host(self.h, C.byref(st)), "sb_eq_from_host")

    def finish(self):
        t = sb_eq_table()
        _check(self.lib.sb_eq_finish(self.h, C.byref(t)), "sb_eq_finish")
        n = int(t.n_classes)

        def arr(ptr, dt, k):
            if k == 0:
                return np.zeros(0, dtype=dt)
            return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(dt))), shape=(k,)).copy()
        off = arr(t.off, np.uint64, n + 1) if n else np.zeros(1, dtype=np.uint64)
        loff = arr(t.label_off, np.uint64, n + 1) if n else np.zeros(1, dtype=np.uint64)
        nnz, nl = int(off[-1]), int(loff[-1])
        return dict(off=off, tids=arr(t.tids, np.uint32, nnz), weights=arr(t.weights, np.float64, nnz),
                    counts=arr(t.counts, np.uint64, n), ntx=arr(t.n_txp_in_label, np.uint32, n), label_off=loff,
                    labels=arr(t.labels, np.uint32, nl), n_groups=int(t.n_groups))

    def close(self):
        if self.h:
            self.lib.sb_eq_destroy(self.h)
            self.h = None


@dataclass
class EqClasses:
    """Host CSR view of EquivalenceClassBuilder::eqVec() (see sb_eq_csr)."""
    n_txps: int
    off: np.ndarray      # uint64 [C+1]
    tids: np.ndarray     # uint32 [nnz]
    weights: np.ndarray  # float64 [nnz]
    counts: np.ndarray   # uint64 [C]

    def __post_init__(self):
        self.off = np.ascontiguousarray(self.off, dtype=np.uint64)
        self.tids = np.ascontiguousarray(self.tids, dtype=np.uint32)
        self.weights = np.ascontiguousarray(self.weights, dtype=np.float64)
        self.counts = np.ascontiguousarray(self.counts, dtype=np.uint64)
        assert self.off.shape[0] == self.counts.shape[0] + 1
        assert self.tids.shape[0] == self.weights.shape[0] == int(self.off[-1])

    @property
    def n_classes(self):
        return int(self.counts.shape[0])

    @property
    def nnz(self):
        return int(self.tids.shape[0])

    def as_struct(self) -> sb_eq_csr:
        return sb_eq_csr(self.n_classes, self.n_txps, self.off.ctypes.data, self.tids.ctypes.data,
                         self.weights.ctypes.data, self.counts.ctypes.data)


class EMContext:
    """Thin RAII wrapper around sb_em_ctx."""

    def __init__(self, device: int = 0):
        self.lib = load()
        self.h = self.lib.sb_em_create(device)
        if not self.h:
            raise SalmonB200Error("sb_em_create failed: " + self.lib.sb_last_error().decode())
        self._keep = None
        self.M = 0

    def close(self):
        if self.h:
            self.lib.sb_em_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, key: str, value: int):
        _check(self.lib.sb_em_set_option(self.h, key.encode(), int(value)), "sb_em_set_option")

    def info(self, key: str) -> int:
        """sb_em_get_info: a figure of the prepared layout, e.g. "stream_bytes" or "fallback_rows_tm"."""
        v = C.c_int64(0)
        _check(self.lib.sb_em_get_info(self.h, key.encode(), C.byref(v)), "sb_em_get_info")
        return v.value

    @staticmethod
    def _txp_arrays(eq, projected, eff_len, unique):
        projected = np.ascontiguousarray(projected, dtype=np.float64)
        eff_len = np.ascontiguousarray(eff_len, dtype=np.float64)
        unique = np.ascontiguousarray(unique, dtype=np.uint64)
        assert projected.shape[0] == eff_len.shape[0] == unique.shape[0] == eq.n_txps
        return projected, eff_len, unique

    def optimize(self, eq: EqClasses, params: sb_em_params, projected, eff_len, unique):
        """sb_em_optimize: host buffers in, host alpha out.  Returns (alpha, stats, ok)."""
        projected, eff_len, unique = self._txp_arrays(eq, projected, eff_len, unique)
        alpha = np.empty(eq.n_txps, dtype=np.float64)
        st = sb_em_stats()
        s = eq.as_struct()
        rc = _check(self.lib.sb_em_optimize(self.h, C.byref(s), C.byref(params), projected.ctypes.data,
                                            eff_len.ctypes.data, unique.ctypes.data, alpha.ctypes.data,
                                            C.byref(st)), "sb_em_optimize")
        self.M = eq.n_txps
        self._nnz = eq.nnz
        self._C = eq.n_classes
        return alpha, st, rc == 0

    def upload(self, eq: EqClasses, projected, eff_len, unique):
        projected, eff_len, unique = self._txp_arrays(eq, projected, eff_len, unique)
        s = eq.as_struct()
        _check(self.lib.sb_em_upload(self.h, C.byref(s), projected.ctypes.data, eff_len.ctypes.data,
                                     unique.ctypes.data), "sb_em_upload")
        self.M = eq.n_txps
        self._nnz = eq.nnz
        self._C = eq.n_classes

    def prepare(self, params: sb_em_params) -> sb_em_stats:
        st = sb_em_stats()
        _check(self.lib.sb_em_prepare(self.h, C.byref(params), C.byref(st)), "sb_em_prepare")
        return st

    def run(self) -> sb_em_stats:
        st = sb_em_stats()
        _check(self.lib.sb_em_run(self.h, C.byref(st)), "sb_em_run")
        return st

    def download(self):
        alpha = np.empty(self.M, dtype=np.float64)
        st = sb_em_stats()
        rc = _check(self.lib.sb_em_download(self.h, alpha.ctypes.data, C.byref(st)), "sb_em_download")
        return alpha, st.alpha_sum, rc == 0

    def get_combined(self):
        cw = np.empty(self._nnz, dtype=np.float64)
        valid = np.empty(self._C, dtype=np.uint8)
        _check(self.lib.sb_em_get_combined(self.h, cw.ctypes.data, valid.ctypes.data), "sb_em_get_combined")
        return cw, valid

    def _collector(self):
        samples = []
        CB = C.CFUNCTYPE(C.c_int, C.POINTER(C.c_double), C.c_uint32, C.c_void_p)

        def cb(ptr, n, user):
            samples.append(np.ctypeslib.as_array(ptr, shape=(n,)).copy())
            return 0
        return samples, CB(cb)

    def bootstrap(self, params: sb_em_params, num_mapped_frags: float, n: int, seed: int):
        """sb_bootstrap -> (array [n, M], ok)."""
        samples, cb = self._collector()
        rc = _check(self.lib.sb_bootstrap(self.h, C.byref(params), float(num_mapped_frags), n, seed,
                                          C.cast(cb, C.c_void_p), None), "sb_bootstrap")
        return np.array(samples), rc == 0

    def bootstrap_last_counts(self):
        out = np.zeros(self._C, dtype=np.uint64)
        _check(self.lib.sb_bootstrap_last_counts(self.h, out.ctypes.data), "sb_bootstrap_last_counts")
        return out

    def gibbs(self, alphas_init, use_vbem, per_txp_prior, vb_prior, n_samples, thinning, no_gamma_draw,
              num_mapped_frags, seed):
        init = np.ascontiguousarray(alphas_init, dtype=np.float64)
        samples, cb = self._collector()
        _check(self.lib.sb_gibbs(self.h, init.ctypes.data, int(use_vbem), int(per_txp_prior), float(vb_prior),
                                 n_samples, thinning, int(no_gamma_draw), float(num_mapped_frags), seed,
                                 C.cast(cb, C.c_void_p), None), "sb_gibbs")
        return np.array(samples)

    def gibbs_last_state(self):
        """sb_gibbs_last_state -> (mu [M], cnt [M]) as the last Gibbs round left them."""
        mu = np.zeros(self.M, dtype=np.float64)
        cnt = np.zeros(self.M, dtype=np.float64)
        _check(self.lib.sb_gibbs_last_state(self.h, mu.ctypes.data, cnt.ctypes.data), "sb_gibbs_last_state")
        return mu, cnt

    def arm_timeline(self, iteration: int) -> int:
        return _check(self.lib.sb_em_debug_timeline(self.h, None, iteration), "sb_em_debug_timeline")

    def read_timeline(self, n_warps: int):
        out = np.zeros((n_warps, 16), dtype=np.uint64)   # DBG_SLOTS (em_kernels.cuh: SB_DBG)
        _check(self.lib.sb_em_debug_timeline(self.h, out.ctypes.data, 0), "sb_em_debug_timeline")
        return out

    def flush_l2(self):
        _check(self.lib.sb_flush_l2(self.h), "sb_flush_l2")

    def peer_setup(self, dist, max_txps: int):
        """fused multi-GPU all-reduce: exchange CUDA IPC handles of the per-rank blocks (torch.distributed) and map
        the peers (NVLink P2P).  Call before upload/prepare/optimize."""
        buf = C.create_string_buffer(64)
        _check(self.lib.sb_em_peer_handle(self.h, int(max_txps), buf), "sb_em_peer_handle")
        hs = [None] * dist.get_world_size()
        dist.all_gather_object(hs, buf.raw)
        allh = C.create_string_buffer(b"".join(hs), 64 * len(hs))
        _check(self.lib.sb_em_peer_open(self.h, dist.get_rank(), dist.get_world_size(), allh), "sb_em_peer_open")

    def peer_loopback(self, max_txps: int):
        """the fused multi-GPU kernel on ONE GPU: the rank is its own and only peer (exercises the push / owner /
        exchange-barrier logic without a second device)"""
        buf = C.create_string_buffer(64)
        _check(self.lib.sb_em_peer_handle(self.h, int(max_txps), buf), "sb_em_peer_handle")
        _check(self.lib.sb_em_peer_open(self.h, 0, 1, buf), "sb_em_peer_open")

    def comm_init(self, rank: int, nranks: int, uid: bytes):
        buf = C.create_string_buffer(uid, 128)
        _check(self.lib.sb_em_comm_init(self.h, rank, nranks, buf), "sb_em_comm_init")


def pin(arr: np.ndarray):
    """Page-lock a numpy array in place (returns the array)."""
    _check(load().sb_host_register(arr.ctypes.data, arr.nbytes), "sb_host_register")
    return arr


def unpin(arr: np.ndarray):
    _check(load().sb_host_unregister(arr.ctypes.data), "sb_host_unregister")


def nccl_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    _check(load().sb_nccl_unique_id(buf), "sb_nccl_unique_id")
    return buf.raw


# ------------------------------------------------------------------------------ Stage A
def map_default_params(**over) -> sb_map_params:
    p = sb_map_params()
    load().sb_map_default_params(C.byref(p))
    for k, v in over.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def map_mimic_bt2(p: sb_map_params, strict=False) -> sb_map_params:
    """sb_map_mimic_bt2: salmon's `--mimicBT2` (strict False) or `--mimicStrictBT2` (strict True) presets applied to p in
    place, overriding the values p holds for the same options (DESIGN.md section 14).  Returns p."""
    _check(load().sb_map_mimic_bt2(C.byref(p), 1 if strict else 0), "sb_map_mimic_bt2")
    return p


class Index:
    """sb_index: host-built k-mer hash index over a transcriptome (list of uint8 code arrays)."""

    def __init__(self, txps, k=31, names=None, complete_len=None, first_decoy=None, _handle=None):
        self.lib = load()
        if _handle is not None:
            self.h = _handle
            m = self.meta()
            self.n_txps, self.k = m["n_txps"], m["k"]
            return
        self._build(txps, k)
        if names is not None or complete_len is not None or first_decoy is not None:
            self.set_meta(names, complete_len, first_decoy)

    @classmethod
    def load(cls, path):
        """sb_index_load: the on-disk form written by save()."""
        lib = load()
        h = lib.sb_index_load(os.fsencode(path))
        if not h:
            raise SalmonB200Error("sb_index_load failed: " + lib.sb_last_error().decode())
        return cls(None, _handle=h)

    @classmethod
    def from_fasta(cls, path, k=31, **opts):
        """`salmon index -t path` (read_txome_fasta options: gencode, decoys, no_clip, keep_duplicates)."""
        t = read_txome_fasta(path, k=k, **opts)
        return cls(t["seqs"], k=k, names=t["names"], complete_len=t["complete_len"], first_decoy=t["first_decoy"])

    def save(self, path):
        _check(self.lib.sb_index_save(self.h, os.fsencode(path)), "sb_index_save")

    def set_meta(self, names=None, complete_len=None, first_decoy=None):
        na = (C.c_char_p * self.n_txps)(*[n.encode() for n in names]) if names is not None else None
        cl = np.ascontiguousarray(complete_len, dtype=np.uint32) if complete_len is not None else None
        _check(self.lib.sb_index_set_meta(self.h, na, cl.ctypes.data if cl is not None else None,
                                          self.n_txps if first_decoy is None else int(first_decoy)), "sb_index_set_meta")

    def meta(self):
        n, k, fd = C.c_uint32(), C.c_uint32(), C.c_uint32()
        names = C.POINTER(C.c_char_p)()
        cl = C.c_void_p()
        _check(self.lib.sb_index_get_meta(self.h, C.byref(n), C.byref(k), C.byref(fd), C.byref(names), C.byref(cl)),
               "sb_index_get_meta")
        return {"n_txps": n.value, "k": k.value, "first_decoy": fd.value,
                "names": [names[i].decode() for i in range(n.value)] if names else None,
                "complete_len": _view(cl.value, n.value, np.uint32) if cl.value else None}

    def tx_lengths(self):
        ha = self.host_arrays()
        off = _view(ha["tx_off"], self.n_txps + 1, np.uint64)
        return (off[1:] - off[:-1]).astype(np.uint32)

    def _build(self, txps, k):
        lens = np.array([t.shape[0] for t in txps], dtype=np.uint64)
        self.off = np.concatenate(([0], np.cumsum(lens))).astype(np.uint64)
        self.codes = np.ascontiguousarray(np.concatenate(txps).astype(np.uint8)) if len(txps) else np.zeros(0, np.uint8)
        self.n_txps = len(txps)
        self.k = k
        self.h = self.lib.sb_index_build(self.n_txps, self.off.ctypes.data, self.codes.ctypes.data, k)
        if not self.h:
            raise SalmonB200Error("sb_index_build failed: " + self.lib.sb_last_error().decode())

    def info(self):
        out = np.zeros(4, dtype=np.uint64)
        _check(self.lib.sb_index_info(self.h, out.ctypes.data), "sb_index_info")
        return dict(n_kmers=int(out[0]), n_postings=int(out[1]), table_capacity=int(out[2]), bytes=int(out[3]))

    def host_arrays(self):
        ptrs = [C.c_void_p() for _ in range(4)]
        cap, npost = C.c_uint64(), C.c_uint64()
        _check(self.lib.sb_index_host_arrays(self.h, C.byref(ptrs[0]), C.byref(ptrs[1]), C.byref(ptrs[2]), C.byref(cap),
                                             C.byref(ptrs[3]), C.byref(npost)), "sb_index_host_arrays")
        return dict(tx_off=ptrs[0].value, codes=ptrs[1].value, table=ptrs[2].value, table_capacity=cap.value,
                    postings=ptrs[3].value, n_postings=npost.value)

    def close(self):
        if self.h:
            self.lib.sb_index_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


CAND_DTYPE = np.dtype([("tid", np.uint32), ("diag_c", np.int32), ("ori_cov", np.uint32)])   # sbmap::Cand


def alloc_alignment_arrays(n, cap):
    return dict(n_aln=np.zeros(n, dtype=np.uint32), tid=np.zeros((n, cap), dtype=np.uint32),
                score=np.zeros((n, cap), dtype=np.int32), prob=np.zeros((n, cap)),
                pos=np.zeros((n, cap), dtype=np.int32), mate_pos=np.zeros((n, cap), dtype=np.int32),
                flags=np.zeros((n, cap), dtype=np.uint8), flen=np.zeros((n, cap), dtype=np.int32),
                label=np.zeros((n, 2 * cap), dtype=np.uint32), weight=np.zeros((n, cap)))


class MapContext:
    """sb_map_ctx: per-GPU mapping + equivalence-class builder."""

    def __init__(self, index: Index, params: sb_map_params, device=0, batch_cap=65536, max_read_len=150):
        self.lib = load()
        self.index = index
        self.p = params
        self.h = self.lib.sb_map_create(index.h, C.byref(params), device, batch_cap, max_read_len)
        if not self.h:
            raise SalmonB200Error("sb_map_create failed: " + self.lib.sb_last_error().decode())
        self.last_n = 0

    def map_batch(self, left, right=None) -> sb_map_batch_stats:
        """right=None: single-end reads (library types U / SF / SR)"""
        left = np.ascontiguousarray(left, dtype=np.uint8)
        n, L = left.shape
        rp = None
        if right is not None:
            right = np.ascontiguousarray(right, dtype=np.uint8)
            rp = right.ctypes.data
        st = sb_map_batch_stats()
        _check(self.lib.sb_map_batch(self.h, left.ctypes.data, rp, n, L, C.byref(st)), "sb_map_batch")
        self.last_n = n
        return st

    def map_batch_ptr(self, left_ptr: int, right_ptr: int, n: int, L: int) -> sb_map_batch_stats:
        """raw pointers (device pointers with set_option("input_on_device", 1))"""
        st = sb_map_batch_stats()
        _check(self.lib.sb_map_batch(self.h, C.c_void_p(left_ptr), C.c_void_p(right_ptr), n, L, C.byref(st)), "sb_map_batch")
        self.last_n = n
        return st

    def attach_sam(self, sam):
        """sb_map_attach_sam: a SamSink (None detaches)"""
        _check(self.lib.sb_map_attach_sam(self.h, sam.h if sam is not None else None), "sb_map_attach_sam")

    def map_batch_sam(self, left, right, names, quals=None) -> sb_map_batch_stats:
        """sb_map_batch_sam: the batch, plus its SAM records for the attached sink.  names: list of str / bytes (one
        per read); quals: (qual_left[n, L], qual_right[n, L] | None) as uint8 arrays when the sink writes qualities."""
        left = np.ascontiguousarray(left, dtype=np.uint8)
        n, L = left.shape
        rp = None
        if right is not None:
            right = np.ascontiguousarray(right, dtype=np.uint8)
            rp = right.ctypes.data
        blob, off = pack_names(names)
        q = [None, None]
        if quals is not None:
            q = [np.ascontiguousarray(x, dtype=np.uint8) if x is not None else None for x in quals]
        st = sb_map_batch_stats()
        _check(self.lib.sb_map_batch_sam(self.h, left.ctypes.data, rp, n, L, blob.ctypes.data, off.ctypes.data,
                                         q[0].ctypes.data if q[0] is not None else None,
                                         q[1].ctypes.data if q[1] is not None else None, C.byref(st)), "sb_map_batch_sam")
        self.last_n = n
        return st

    def reset(self):
        _check(self.lib.sb_map_reset(self.h), "sb_map_reset")

    def partial(self) -> dict:
        """this rank's statistics after finish() (multi-GPU: reduce them with salmon_b200.dist.reduce_partials)"""
        q = sb_map_partial()
        _check(self.lib.sb_map_partial_get(self.h, C.byref(q)), "sb_map_partial_get")
        M, nf = int(q.n_txps), int(q.n_fld)
        arr = lambda ptr, n, dt: (np.ctypeslib.as_array(ptr, shape=(n,)).copy() if n else np.zeros(0, dt))
        return dict(mass=arr(q.mass, M, np.float64), fld_hist=arr(q.fld_hist, nf, np.float64), fld_tot=float(q.fld_tot),
                    fld_prior_hist=arr(q.fld_prior_hist, nf, np.float64), fld_prior_tot=float(q.fld_prior_tot),
                    fld_min=int(q.fld_min), unique_counts=arr(q.unique_counts, M, np.uint64),
                    total_counts=arr(q.total_counts, M, np.uint64), cluster_hits=arr(q.cluster_hits, M, np.uint64),
                    cluster_root=arr(q.cluster_root, M, np.uint32), assigned=int(q.assigned),
                    compatible=int(q.compatible))

    def project_global(self, g: dict, roots_all: np.ndarray) -> dict:
        """normalizeAlphas with the statistics reduced over all ranks; returns the per-transcript EM inputs"""
        keep = {k: np.ascontiguousarray(g[k], dtype=dt) for k, dt in (
            ("mass", np.float64), ("fld_hist", np.float64), ("fld_prior_hist", np.float64), ("unique_counts", np.uint64),
            ("total_counts", np.uint64), ("cluster_hits", np.uint64))}
        roots_all = np.ascontiguousarray(roots_all, dtype=np.uint32)
        q = sb_map_partial()
        q.n_txps = keep["mass"].shape[0]; q.n_fld = keep["fld_hist"].shape[0]
        q.mass = keep["mass"].ctypes.data_as(C.POINTER(C.c_double))
        q.fld_hist = keep["fld_hist"].ctypes.data_as(C.POINTER(C.c_double)); q.fld_tot = float(g["fld_tot"])
        q.fld_prior_hist = keep["fld_prior_hist"].ctypes.data_as(C.POINTER(C.c_double)); q.fld_prior_tot = float(g["fld_prior_tot"])
        q.fld_min = int(g["fld_min"])
        q.unique_counts = keep["unique_counts"].ctypes.data_as(C.POINTER(C.c_uint64))
        q.total_counts = keep["total_counts"].ctypes.data_as(C.POINTER(C.c_uint64))
        q.cluster_hits = keep["cluster_hits"].ctypes.data_as(C.POINTER(C.c_uint64))
        q.cluster_root = None; q.assigned = int(g["assigned"]); q.compatible = int(g.get("compatible", 0))
        r = sb_map_result()
        _check(self.lib.sb_map_project_global(self.h, C.byref(q), roots_all.shape[0], roots_all.ctypes.data, C.byref(r)),
               "sb_map_project_global")
        M = int(r.n_txps)
        return {k: (np.ctypeslib.as_array(getattr(r, k), shape=(M,)).copy() if M else np.zeros(0))
                for k in ("projected_counts", "eff_len", "unique_counts", "total_counts")}

    def set_option(self, key: str, value: int):
        _check(self.lib.sb_map_set_option(self.h, key.encode(), int(value)), "sb_map_set_option")

    def last_alignments(self):
        n, cap = self.last_n, self.p.max_read_occ
        a = alloc_alignment_arrays(n, cap)
        _check(self.lib.sb_map_last_alignments(self.h, n, *[a[k].ctypes.data for k in (
            "n_aln", "tid", "score", "prob", "pos", "mate_pos", "flags", "flen", "label", "weight")]),
            "sb_map_last_alignments")
        return a

    def last_candidates(self):
        """the seed kernel's candidates of the last batch: n_l, n_r [n] (bit 31 of n_l: unmapped) and cand_l, cand_r
        [n, 64] records (tid, diag_c, ori_cov); refused after a batch of several chunks or with orphan rescue"""
        n = self.last_n
        out = dict(n_l=np.zeros(n, np.uint32), n_r=np.zeros(n, np.uint32), cand_l=np.zeros((n, 64), CAND_DTYPE),
                   cand_r=np.zeros((n, 64), CAND_DTYPE))
        _check(self.lib.sb_map_last_candidates(self.h, n, *[out[k].ctypes.data for k in ("n_l", "n_r", "cand_l", "cand_r")]),
               "sb_map_last_candidates")
        return out

    def finish(self):
        r = sb_map_result()
        _check(self.lib.sb_map_finish(self.h, C.byref(r)), "sb_map_finish")
        nc = int(r.n_classes)
        off = np.ctypeslib.as_array(r.off, shape=(nc + 1,)).copy() if nc else np.zeros(1, np.uint64)
        nn = int(off[-1])
        out = dict(off=off,
                   tids=np.ctypeslib.as_array(r.tids, shape=(nn,)).copy() if nn else np.zeros(0, np.uint32),
                   weights=np.ctypeslib.as_array(r.weights, shape=(nn,)).copy() if nn else np.zeros(0),
                   counts=np.ctypeslib.as_array(r.counts, shape=(nc,)).copy() if nc else np.zeros(0, np.uint64),
                   bins=(np.ctypeslib.as_array(r.bins, shape=(nn,)).copy() if (nn and r.bins) else None),
                   counters={k: int(getattr(r, k)) for k in ("n_mapped", "lookups", "postings", "seeds", "candidates",
                                                             "kept", "label_entries")})
        M = int(r.n_txps)
        for k, dt in (("projected_counts", np.float64), ("eff_len", np.float64), ("unique_counts", np.uint64),
                      ("total_counts", np.uint64)):
            out[k] = np.ctypeslib.as_array(getattr(r, k), shape=(M,)).copy() if M else np.zeros(0, dt)
        out["lib_format_counts"] = dict(zip(("ISF", "ISR", "SF", "SR"), [int(x) for x in r.lib_format_counts[:4]]))
        out["rescue"] = {k: int(getattr(r, k)) for k in ("orphans_rescued", "rescue_searches", "rescue_no_room")}
        out["counters"]["n_compatible"] = int(r.n_compatible)
        return out

    def online_state(self):
        M, nf = self.index.n_txps, self.p.max_frag_len + 1
        mass = np.zeros(M); hist = np.zeros(nf); le = np.zeros(M); sc = np.zeros(6, dtype=np.uint64)
        _check(self.lib.sb_map_online_state(self.h, mass.ctypes.data, hist.ctypes.data, le.ctypes.data, sc.ctypes.data),
               "sb_map_online_state")
        return dict(mass=mass, hist=hist, log_eff=le, assigned=int(sc[0]), frags_seen=int(sc[1]), timestep=int(sc[2]),
                    burned_in=int(sc[3]), min_val=int(sc[4]), tot=sc[5:6].view(np.float64)[0])

    def close(self):
        if self.h:
            self.lib.sb_map_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def rescue_search_tap(patterns, windows, K, device=0):
    """sb_rescue_search_tap: the orphan rescue's bit-vector infix search on the GPU.  patterns / windows: lists of uint8
    code arrays (0..3, 4 = N), K: edit limits.  Returns (dist, end) int32 arrays, -1 where nothing is within K."""
    n = len(patterns)
    def cat(xs):
        off = np.zeros(n + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(x) for x in xs], dtype=np.uint64)
        blob = np.ascontiguousarray(np.concatenate([np.asarray(x, dtype=np.uint8) for x in xs] + [np.zeros(1, np.uint8)]))
        return blob, off
    pb, po = cat(patterns)
    wb, wo = cat(windows)
    k = np.ascontiguousarray(K, dtype=np.int32)
    dist = np.zeros(n, dtype=np.int32); end = np.zeros(n, dtype=np.int32)
    _check(load().sb_rescue_search_tap(device, n, pb.ctypes.data, po.ctypes.data, wb.ctypes.data, wo.ctypes.data,
                                       k.ctypes.data, dist.ctypes.data, end.ctypes.data), "sb_rescue_search_tap")
    return dist, end


# ------------------------------------------------------------------------------ SAM output
def pack_names(names):
    """names -> (concatenated bytes as uint8[], offsets uint64[n+1]), the layout sb_map_batch_sam takes"""
    bs = [x.encode() if isinstance(x, str) else bytes(x) for x in names]
    off = np.zeros(len(bs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in bs], dtype=np.uint64)
    blob = np.frombuffer(b"".join(bs) + b"\0", dtype=np.uint8).copy()
    return blob, off


class SamSink:
    """sb_sam: SAM output (`--writeMappings`) and / or aux_info/unmapped_names.txt lines, written by a thread of its own."""

    def __init__(self, index: Index, sam_path=None, unmapped_path=None, cmdline="", qualities=False):
        self.lib = load()
        self.h = self.lib.sb_sam_open(os.fsencode(sam_path) if sam_path else None,
                                      os.fsencode(unmapped_path) if unmapped_path else None, index.h,
                                      cmdline.encode(), 1 if qualities else 0)
        if not self.h:
            raise SalmonB200Error("sb_sam_open failed: " + self.lib.sb_last_error().decode())

    def write_unmapped(self, text: bytes):
        _check(self.lib.sb_sam_write_unmapped(self.h, text, len(text)), "sb_sam_write_unmapped")

    def stats(self) -> dict:
        st = sb_sam_stats()
        _check(self.lib.sb_sam_get_stats(self.h, C.byref(st)), "sb_sam_get_stats")
        return {k: getattr(st, k) for k, _ in sb_sam_stats._fields_}

    def close(self):
        if self.h:
            h, self.h = self.h, None
            _check(self.lib.sb_sam_close(h), "sb_sam_close")

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _meta_arrays(m, n, shape, paired):
    """sb_read_meta of n reads -> (names: list of bytes, qual_left | None, qual_right | None)"""
    off = _view(m.name_off, n + 1, np.uint64)
    blob = C.string_at(m.names, int(off[-1])) if n and off[-1] else b""
    names = [blob[int(off[i]):int(off[i + 1])] for i in range(n)]
    ql = np.ctypeslib.as_array(C.cast(m.qual_left, C.POINTER(C.c_uint8)), shape=shape) if m.qual_left else None
    qr = np.ctypeslib.as_array(C.cast(m.qual_right, C.POINTER(C.c_uint8)), shape=shape) if (paired and m.qual_right) else None
    return names, ql, qr


# ------------------------------------------------------------------------------ output seam
def _names(names):
    arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
    return arr


def tpm(alpha, eff_len, num_mapped_frags=None):
    alpha = np.ascontiguousarray(alpha, dtype=np.float64); eff_len = np.ascontiguousarray(eff_len, dtype=np.float64)
    out = np.zeros_like(alpha)
    nm = float(alpha.sum()) if num_mapped_frags is None else float(num_mapped_frags)
    _check(load().sb_tpm(alpha.shape[0], alpha.ctypes.data, eff_len.ctypes.data, nm, out.ctypes.data), "sb_tpm")
    return out


def write_quant_sf(path, names, complete_len, eff_len, alpha, num_mapped_frags=None, sig_digits=3):
    alpha = np.ascontiguousarray(alpha, dtype=np.float64); eff_len = np.ascontiguousarray(eff_len, dtype=np.float64)
    cl = np.ascontiguousarray(complete_len, dtype=np.uint32)
    nm = float(alpha.sum()) if num_mapped_frags is None else float(num_mapped_frags)
    arr = _names(names)
    _check(load().sb_write_quant_sf(str(path).encode(), len(names), C.cast(arr, C.c_void_p), cl.ctypes.data,
                                    eff_len.ctypes.data, alpha.ctypes.data, nm, sig_digits), "sb_write_quant_sf")


def write_eq_classes(path, names, off, tids, counts, weights=None):
    off = np.ascontiguousarray(off, dtype=np.uint64); tids = np.ascontiguousarray(tids, dtype=np.uint32)
    counts = np.ascontiguousarray(counts, dtype=np.uint64)
    w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float64)
    arr = _names(names)
    _check(load().sb_write_eq_classes(str(path).encode(), len(names), C.cast(arr, C.c_void_p), counts.shape[0],
                                      off.ctypes.data, tids.ctypes.data, None if w is None else w.ctypes.data,
                                      counts.ctypes.data), "sb_write_eq_classes")


# ---- input seam (host code; no device needed) ------------------------------------------------------------------------
def _view(ptr, n, dtype):
    """Copy n items of dtype from a C pointer into a fresh numpy array."""
    if n == 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype, count=n).copy()


class ReadFiles:
    """FASTQ/FASTA reader (sb_reads_*): mirrors how salmon consumes fastx_parser<ReadPair> / <ReadSeq>
    (src/quant/SalmonQuantify.cpp:1118-1141): batches of reads, here as base codes."""

    def __init__(self, files1, files2=None, n_threads=4):
        lib = load()
        files1 = [files1] if isinstance(files1, (str, bytes, os.PathLike)) else list(files1)
        if files2 is not None:
            files2 = [files2] if isinstance(files2, (str, bytes, os.PathLike)) else list(files2)
            if len(files2) != len(files1):
                raise ValueError("the two mate file lists differ in length")
        self.paired = files2 is not None
        a1 = (C.c_char_p * len(files1))(*[os.fsencode(f) for f in files1])
        a2 = (C.c_char_p * len(files1))(*[os.fsencode(f) for f in files2]) if self.paired else None
        self.lib = lib
        self.h = lib.sb_reads_open(a1, a2, len(files1), n_threads)
        if not self.h:
            raise SalmonB200Error(lib.sb_last_error().decode())

    def next_batch(self, max_pairs, stride, out=None):
        """-> (n, left[n,stride], right[n,stride] | None, len_left[n], len_right[n] | None); n == 0 at the end."""
        if out is None:
            out = (np.empty((max_pairs, stride), np.uint8), np.empty((max_pairs, stride), np.uint8) if self.paired else None,
                   np.empty(max_pairs, np.uint32), np.empty(max_pairs, np.uint32) if self.paired else None)
        left, right, ll, lr = out
        n = self.lib.sb_reads_next(self.h, max_pairs, stride, left.ctypes.data,
                                   right.ctypes.data if self.paired else None, ll.ctypes.data,
                                   lr.ctypes.data if self.paired else None)
        _check(n, "sb_reads_next")
        return n, left[:n], (right[:n] if self.paired else None), ll[:n], (lr[:n] if self.paired else None)

    def next_batch_meta(self, max_pairs, stride, quals=False):
        """sb_reads_next_meta -> (n, left, right | None, len_left, len_right | None, names (bytes), qual_left | None,
        qual_right | None); the quality arrays are [n, stride] copies."""
        left = np.empty((max_pairs, stride), np.uint8)
        right = np.empty((max_pairs, stride), np.uint8) if self.paired else None
        ll = np.empty(max_pairs, np.uint32)
        lr = np.empty(max_pairs, np.uint32) if self.paired else None
        m = sb_read_meta()
        n = self.lib.sb_reads_next_meta(self.h, max_pairs, stride, left.ctypes.data,
                                        right.ctypes.data if self.paired else None, ll.ctypes.data,
                                        lr.ctypes.data if self.paired else None, int(quals), C.byref(m))
        _check(n, "sb_reads_next_meta")
        names, ql, qr = _meta_arrays(m, n, (n, stride), self.paired)
        return (n, left[:n], (right[:n] if self.paired else None), ll[:n], (lr[:n] if self.paired else None), names,
                None if ql is None else ql.copy(), None if qr is None else qr.copy())

    def bucketed_meta(self, fn, min_len=31, batch=65536, max_read_len=256, threads=4, shard_index=0, shard_count=1,
                      quals=False):
        """sb_reads_bucketed_meta: fn(left[n, L], right | None, L, names (list of bytes), qual_left | None, qual_right |
        None) per batch (views of the library's buffers).  -> (stats dict, names of the pairs dropped as too short)."""
        CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(sb_read_meta))
        NCB = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_size_t)
        raised, dropped = [], []

        def cb(user, lp, rp, n, L, mp):
            try:
                left = np.ctypeslib.as_array(C.cast(lp, C.POINTER(C.c_uint8)), shape=(n, L))
                right = np.ctypeslib.as_array(C.cast(rp, C.POINTER(C.c_uint8)), shape=(n, L)) if rp else None
                names, ql, qr = _meta_arrays(mp.contents, n, (n, L), rp is not None)
                r = fn(left, right, L, names, ql, qr)
                return int(r) if r else 0
            except Exception as e:  # noqa: BLE001  (an exception must not unwind through the C frames)
                raised.append(e)
                return -1

        def ncb(user, p, n):
            dropped.extend(C.string_at(p, n).splitlines())
        cbo, ncbo = CB(cb), NCB(ncb)
        st = (C.c_uint64 * 6)()
        rc = self.lib.sb_reads_bucketed_meta(self.h, min_len, batch, max_read_len, threads, shard_index, shard_count,
                                             int(quals), C.cast(cbo, C.c_void_p), C.cast(ncbo, C.c_void_p), None, st)
        if raised:
            raise raised[0]
        _check(rc, "sb_reads_bucketed_meta")
        return ({"n_observed": st[0], "n_delivered": st[1], "n_too_short": st[2], "n_trimmed_mates": st[3],
                 "n_batches": st[4], "n_read_lengths": st[5] & 0xffffffff}, dropped)

    def peek(self, max_pairs):
        """-> (n available up to max_pairs, their common read length or 0)"""
        L = C.c_uint32(0)
        n = _check(self.lib.sb_reads_peek(self.h, max_pairs, C.byref(L)), "sb_reads_peek")
        return n, L.value

    def skip(self, n):
        return _check(self.lib.sb_reads_skip(self.h, n), "sb_reads_skip")

    def bucketed(self, fn, min_len=31, batch=65536, max_read_len=256, threads=4, shard_index=0, shard_count=1):
        """sb_reads_bucketed: fn(left[n, L], right[n, L] | None, L) is called for every batch of one read length (the
        arrays are views of the library's buffers: copy what you keep).  -> stats dict."""
        CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32)

        raised = []

        def cb(user, lp, rp, n, L):
            try:
                left = np.ctypeslib.as_array(C.cast(lp, C.POINTER(C.c_uint8)), shape=(n, L))
                right = np.ctypeslib.as_array(C.cast(rp, C.POINTER(C.c_uint8)), shape=(n, L)) if rp else None
                r = fn(left, right, L)
                return int(r) if r else 0
            except Exception as e:  # noqa: BLE001  (an exception must not unwind through the C frames)
                raised.append(e)
                return -1
        cbo = CB(cb)
        st = (C.c_uint64 * 6)()
        rc = self.lib.sb_reads_bucketed(self.h, min_len, batch, max_read_len, threads, shard_index, shard_count,
                                        C.cast(cbo, C.c_void_p), None, st)
        if raised:
            raise raised[0]              # the callback's own exception, after the reader has wound down
        _check(rc, "sb_reads_bucketed")
        return {"n_observed": st[0], "n_delivered": st[1], "n_too_short": st[2], "n_trimmed_mates": st[3], "n_batches": st[4],
                "n_read_lengths": st[5] & 0xffffffff}

    def close(self):
        if self.h:
            self.lib.sb_reads_close(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def read_eq_classes(path):
    """--eqclasses reader (src/util/SalmonUtils.cpp:1024-1122) -> dict(names, eq=EqClasses, eff_len, has_weights, n_missing_eff_len)."""
    lib = load()
    pf = C.POINTER(sb_eq_file)()
    _check(lib.sb_eq_file_read(os.fsencode(path), C.byref(pf)), "sb_eq_file_read")
    f = pf.contents
    try:
        M, Cn = f.n_txps, f.n_classes
        off = _view(f.off, Cn + 1, np.uint64)
        nnz = int(off[-1]) if Cn else 0
        tids = _view(f.tids, nnz, np.uint32)
        w = _view(f.weights, nnz, np.float64) if f.has_weights else None
        counts = _view(f.counts, Cn, np.uint64)
        names = [f.names[i].decode() for i in range(M)]
        eff = _view(f.eff_len, M, np.float64)
        return {"names": names, "n_txps": M, "off": off, "tids": tids, "weights": w, "counts": counts,
                "eff_len": eff, "has_weights": bool(f.has_weights), "n_missing_eff_len": int(f.n_missing_eff_len)}
    finally:
        lib.sb_eq_file_free(pf)


class BootstrapWriter:
    """aux_info/bootstrap/bootstraps.gz (src/output/GZipWriter.cpp:765-789)."""

    def __init__(self, path):
        self.lib = load()
        self.h = self.lib.sb_bootstrap_writer_open(os.fsencode(path))
        if not self.h:
            raise SalmonB200Error(self.lib.sb_last_error().decode())

    def write(self, sample):
        sample = np.ascontiguousarray(sample, dtype=np.float64)
        _check(self.lib.sb_bootstrap_writer_write(self.h, sample.ctypes.data, sample.shape[0]), "sb_bootstrap_writer_write")

    def close(self):
        n = 0
        if self.h:
            n = self.lib.sb_bootstrap_writer_close(self.h)
            self.h = None
        return n


def read_txome_fasta(path, k=31, gencode=False, decoys=None, no_clip=False, keep_duplicates=False):
    """`salmon index -t` input handling -> dict(names, seqs (list of code arrays), complete_len, first_decoy, ...)."""
    lib = load()
    pt = C.POINTER(sb_txome)()
    _check(lib.sb_txome_read_fasta(os.fsencode(path), k, int(gencode), os.fsencode(decoys) if decoys else None,
                                   int(no_clip), int(keep_duplicates), C.byref(pt)), "sb_txome_read_fasta")
    t = pt.contents
    try:
        M = t.n_txps
        off = _view(t.seq_off, M + 1, np.uint64)
        codes = _view(t.codes, int(off[-1]) if M else 0, np.uint8)
        return {"names": [t.names[i].decode() for i in range(M)], "seq_off": off, "codes": codes,
                "seqs": [codes[int(off[i]):int(off[i + 1])] for i in range(M)],
                "complete_len": _view(t.complete_len, M, np.uint32), "first_decoy": int(t.first_decoy),
                "n_duplicates_removed": int(t.n_duplicates_removed), "n_clipped": int(t.n_clipped),
                "n_short": int(t.n_short)}
    finally:
        lib.sb_txome_free(pt)


def quant_files_native(index, mates1, mates2, out_dir=None, map_params=None, em_params=None, **opts):
    """sb_quant_files: the C++ host driver (reader thread + GPU thread, salmon_b200/csrc/pipeline.cu).
    opts: fields of sb_quant_opts.  -> (alpha[M], summary dict)."""
    lib = load()
    mates1 = [mates1] if isinstance(mates1, (str, bytes, os.PathLike)) else list(mates1)
    if mates2 is not None:
        mates2 = [mates2] if isinstance(mates2, (str, bytes, os.PathLike)) else list(mates2)
    o = sb_quant_opts()
    lib.sb_quant_default_opts(C.byref(o))
    for k, v in opts.items():
        if not hasattr(o, k):
            raise AttributeError(k)
        setattr(o, k, v)
    a1 = (C.c_char_p * len(mates1))(*[os.fsencode(f) for f in mates1])
    a2 = (C.c_char_p * len(mates2))(*[os.fsencode(f) for f in mates2]) if mates2 is not None else None   # None: single-end
    alpha = np.zeros(index.n_txps)
    sm = sb_quant_summary()
    _check(lib.sb_quant_files(index.h, a1, a2, len(mates1), C.byref(map_params) if map_params is not None else None,
                              C.byref(em_params) if em_params is not None else None, C.byref(o),
                              os.fsencode(out_dir) if out_dir else None, alpha.ctypes.data, C.byref(sm)), "sb_quant_files")
    return alpha, {k: getattr(sm, k) for k, _ in sb_quant_summary._fields_ if not k.startswith("reserved")}
