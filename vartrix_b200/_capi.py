"""ctypes binding of include/vartrix_b200.h (the C ABI a Rust/C++ host would bind the same way).

The shared library is built in-tree by ``make`` / ``__graft_entry__.build()`` into
``vartrix_b200/lib/libvartrix_b200.so``.  There is no fallback: if the library is missing or no
CUDA device is present, creating an engine raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# VTX_LIB lets kernel-tuning experiments load an alternative build of the same library
LIB_PATH = os.environ.get("VTX_LIB") or os.path.join(_HERE, "lib", "libvartrix_b200.so")

VTX_OK = 0
MODE_CONSENSUS, MODE_COVERAGE, MODE_ALT_FRAC = 0, 1, 2
MODES = {"consensus": MODE_CONSENSUS, "coverage": MODE_COVERAGE, "alt_frac": MODE_ALT_FRAC}
NO_CB = 0xFFFFFFFF
NO_UMI = 0xFFFFFFFFFFFFFFFF
F_KEEP_SCORES = 1
F_NO_SPLIT = 2
F_VALUES_ONLY = 4
F_NO_FOLD = 8
F_NAME_KEYS = 16        # vtx_submit_bam keys reads by QNAME instead of UB (--collapse-mates); needs use_umi

# every symbol include/vartrix_b200.h declares (tests check the library exports all of them)
SYMBOLS = [
    "vtx_abi_version", "vtx_create", "vtx_destroy", "vtx_last_error", "vtx_host_alloc", "vtx_host_free",
    "vtx_set_barcodes", "vtx_submit", "vtx_submit_device", "vtx_submit_device_ex", "vtx_finish",
    "vtx_finish_device", "vtx_fetch", "vtx_sync", "vtx_wait_copies", "vtx_score_pairs", "vtx_pack_umi", "vtx_last_timing", "vtx_last_tile_counts",
    "vtx_comm_unique_id", "vtx_comm_init", "vtx_gather", "vtx_gather_start", "vtx_gather_wait",
    "vtx_submit2", "vtx_submit2_device", "vtx_pack_cb", "vtx_bgzf_inflate", "vtx_submit_bam", "vtx_bam_metrics_get",
    "vtx_set_min_base_quality", "vtx_bam_low_base_quality", "vtx_set_locus_stats", "vtx_locus_stats_get",
    "vtx_set_donors", "vtx_donor_ll_get", "vtx_cluster_cells", "vtx_cluster_cells_pinned", "vtx_donors_ambient", "vtx_cluster_genotypes", "vtx_cluster_refine",
]
NO_CB_KEY = 0xFFFFFFFFFFFFFFFF
NO_LABEL = 0xFFFFFFFF     # VTX_NO_LABEL: a cell vtx_cluster_refine did not call singlet
CB_EXOTIC = 0x8000000000000000
GATHER_ALL = -1
BAND_FULL, BAND_MODEL = 0, 1
GT_MISSING = 0xFF
DONOR_LL_SCALE = 1 << 24


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("mode", C.c_int32), ("use_umi", C.c_int32), ("match", C.c_int32),
                ("mismatch", C.c_int32), ("gap_open", C.c_int32), ("gap_extend", C.c_int32),
                ("min_score", C.c_int32), ("stream", C.c_void_p), ("flags", C.c_uint32),
                ("band_k", C.c_int32), ("band_w", C.c_int32), ("band_mode", C.c_int32)]


class Batch(C.Structure):
    _fields_ = [
        ("n_loci", C.c_uint32), ("locus_row", C.c_void_p),
        ("hap_bytes", C.c_void_p), ("hap_bytes_len", C.c_uint64),
        ("ref_off", C.c_void_p), ("ref_len", C.c_void_p), ("alt_off", C.c_void_p), ("alt_len", C.c_void_p),
        ("cand_start", C.c_void_p),
        ("n_reads", C.c_uint32), ("read_nib", C.c_void_p), ("read_nib_len", C.c_uint64),
        ("read_off", C.c_void_p), ("read_len", C.c_void_p),
        ("cb_bytes", C.c_void_p), ("cb_bytes_len", C.c_uint64),
        ("read_cb_off", C.c_void_p), ("read_cb_len", C.c_void_p), ("read_umi_key", C.c_void_p),
        ("n_cand", C.c_uint64), ("cand_read", C.c_void_p),
    ]


class Batch2(C.Structure):          # vtx_batch2: the slim staging layout
    _fields_ = [
        ("n_loci", C.c_uint32), ("locus_row", C.c_void_p),
        ("hap_bytes", C.c_void_p), ("hap_bytes_len", C.c_uint64),
        ("ref_off", C.c_void_p), ("ref_len", C.c_void_p), ("alt_off", C.c_void_p), ("alt_len", C.c_void_p),
        ("cand_start", C.c_void_p),
        ("n_reads", C.c_uint32), ("read_nib", C.c_void_p), ("read_nib_len", C.c_uint64),
        ("read_off4", C.c_void_p), ("read_len", C.c_void_p), ("read_cb_key", C.c_void_p),
        ("n_exotic_cb", C.c_uint32), ("cb_bytes", C.c_void_p), ("cb_off", C.c_void_p),
        ("read_umi_key", C.c_void_p),
        ("n_cand", C.c_uint64), ("cand_read", C.c_void_p),
    ]


class BgzfBlock(C.Structure):      # vtx_bgzf_block
    _fields_ = [("in_off", C.c_uint64), ("in_len", C.c_uint32), ("out_len", C.c_uint32), ("out_off", C.c_uint64),
                ("crc32", C.c_uint32), ("reserved", C.c_uint32)]


class BamShard(C.Structure):       # vtx_bam_shard
    _fields_ = [
        ("n_loci", C.c_uint32), ("locus_row", C.c_void_p), ("locus_start", C.c_void_p), ("locus_end", C.c_void_p),
        ("hap_bytes", C.c_void_p), ("hap_bytes_len", C.c_uint64),
        ("ref_off", C.c_void_p), ("ref_len", C.c_void_p), ("alt_off", C.c_void_p), ("alt_len", C.c_void_p),
        ("tid", C.c_int32), ("n_members", C.c_uint32), ("members", C.c_void_p), ("comp", C.c_void_p), ("comp_len", C.c_uint64),
        ("n_entry", C.c_uint32), ("entry_off", C.c_void_p),
        ("mapq", C.c_uint32), ("primary_only", C.c_int32), ("no_duplicates", C.c_int32), ("bam_tag", C.c_char * 2),
    ]


class BamMetrics(C.Structure):     # vtx_bam_metrics
    _fields_ = [("num_reads", C.c_uint64), ("num_low_mapq", C.c_uint64), ("num_non_primary", C.c_uint64),
                ("num_duplicates", C.c_uint64), ("num_not_useful", C.c_uint64)]


LOCUS_STATS_FIELDS = ("row", "fetched", "low_mapq", "non_primary", "duplicate", "not_useful", "low_base_quality", "no_cell_barcode",
                      "no_umi", "scored", "reads_ref", "reads_alt", "reads_unknown", "reads_none", "calls_ref", "calls_alt",
                      "calls_unknown", "cells", "cells_ref_only", "cells_alt_only", "cells_both", "cells_multi_unknown")


class LocusStats(C.Structure):     # vtx_locus_stats
    _fields_ = [(f, C.c_uint32) for f in LOCUS_STATS_FIELDS]


class ClusterParams(C.Structure):  # vtx_cluster_params
    _fields_ = [("k", C.c_uint32), ("restarts", C.c_uint32), ("seed", C.c_uint64)]


class Clusters(C.Structure):       # vtx_clusters
    _fields_ = [("k", C.c_uint32), ("n_cols", C.c_uint32), ("n_hyp", C.c_uint32), ("best_restart", C.c_uint32),
                ("n_rows", C.c_uint64), ("rows_used", C.c_uint64), ("ll", C.POINTER(C.c_int64)), ("counts", C.POINTER(C.c_uint64)),
                ("row_used", C.POINTER(C.c_uint8)), ("alt_w", C.POINTER(C.c_int64)), ("depth_w", C.POINTER(C.c_int64)),
                ("restart_score", C.POINTER(C.c_int64)), ("restart_iters", C.POINTER(C.c_uint32))]


class ClusterPinnedParams(C.Structure):    # vtx_cluster_pinned_params
    _fields_ = [("k", C.c_uint32), ("restarts", C.c_uint32), ("seed", C.c_uint64), ("n_pinned", C.c_uint32),
                ("error_rate", C.c_double), ("rho_permille", C.c_int32)]


class AmbientParams(C.Structure):  # vtx_ambient_params
    _fields_ = [("n_donors", C.c_uint32), ("error_rate", C.c_double), ("rho_permille", C.c_int32), ("grid_batch", C.c_uint32)]


class Ambient(C.Structure):        # vtx_ambient
    _fields_ = [("n_donors", C.c_uint32), ("n_cols", C.c_uint32), ("n_hyp", C.c_uint32), ("rho_permille", C.c_uint32),
                ("n_evaluated", C.c_uint32), ("n_rows", C.c_uint64), ("rows_usable", C.c_uint64),
                ("ll", C.POINTER(C.c_int64)), ("counts", C.POINTER(C.c_uint64)), ("grid_permille", C.POINTER(C.c_uint16)),
                ("grid_objective", C.POINTER(C.c_int64)), ("grid_calls", C.POINTER(C.c_uint64)),
                ("row_alt", C.POINTER(C.c_uint64)), ("row_depth", C.POINTER(C.c_uint64))]


class ClusterGtParams(C.Structure):    # vtx_cluster_gt_params
    _fields_ = [("k", C.c_uint32), ("error_rate", C.c_double), ("rho_permille", C.c_int32), ("n_samples", C.c_uint32)]


class ClusterGt(C.Structure):          # vtx_cluster_gt
    _fields_ = [("k", C.c_uint32), ("n_samples", C.c_uint32), ("rho_permille", C.c_uint32), ("n_evaluated", C.c_uint32),
                ("n_rows", C.c_uint64), ("rows_fit", C.c_uint64), ("n_touched", C.c_uint64), ("rows_compared", C.c_uint64),
                ("grid_permille", C.POINTER(C.c_uint16)), ("grid_objective", C.POINTER(C.c_int64)), ("touched", C.POINTER(C.c_uint64)),
                ("gt", C.POINTER(C.c_uint8)), ("pl", C.POINTER(C.c_uint32)), ("match_ll", C.POINTER(C.c_int64)),
                ("match_discordant", C.POINTER(C.c_uint64)), ("match_rows", C.POINTER(C.c_uint64)), ("match_called", C.POINTER(C.c_uint64))]


class ClusterCallsParams(C.Structure):     # vtx_cluster_calls_params
    _fields_ = [("k", C.c_uint32), ("error_rate", C.c_double), ("max_rounds", C.c_uint32)]


class ClusterCallsRound(C.Structure):      # vtx_cluster_calls_round
    _fields_ = [("rho_permille", C.c_uint32), ("reserved", C.c_uint32), ("rows_fit", C.c_uint64), ("n_touched", C.c_uint64),
                ("rows_scored", C.c_uint64), ("calls", C.c_uint64 * 3), ("changed", C.c_uint64)]


class ClusterCalls(C.Structure):           # vtx_cluster_calls
    _fields_ = [("k", C.c_uint32), ("n_cols", C.c_uint32), ("n_hyp", C.c_uint32), ("n_rounds", C.c_uint32), ("converged", C.c_int32),
                ("reserved", C.c_uint32), ("n_rows", C.c_uint64), ("n_touched", C.c_uint64), ("ll", C.POINTER(C.c_int64)),
                ("counts", C.POINTER(C.c_uint64)), ("label", C.POINTER(C.c_uint32)), ("rounds", C.POINTER(ClusterCallsRound)),
                ("touched", C.POINTER(C.c_uint64)), ("gt", C.POINTER(C.c_uint8)), ("pl", C.POINTER(C.c_uint32))]


class Metrics(C.Structure):
    _fields_ = [("num_not_cell_bc", C.c_uint64), ("num_non_umi", C.c_uint64), ("num_scored", C.c_uint64)]


class Result(C.Structure):
    _fields_ = [("n", C.c_uint64), ("row", C.c_void_p), ("col", C.c_void_p), ("ref_cnt", C.c_void_p),
                ("alt_cnt", C.c_void_p), ("unk_cnt", C.c_void_p), ("val", C.c_void_p), ("val2", C.c_void_p),
                ("metrics", Metrics)]


class Timing(C.Structure):
    _fields_ = [("h2d_ms", C.c_float), ("prep_ms", C.c_float), ("sw_ms", C.c_float), ("post_ms", C.c_float),
                ("n_pairs", C.c_uint64), ("sw_launches", C.c_uint64), ("total_launches", C.c_uint64)]


_lib = None


def load():
    """dlopen the engine library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `make` (or __graft_entry__.build()) first; "
                           "vartrix_b200 has no CPU fallback")
    L = C.CDLL(LIB_PATH)
    L.vtx_abi_version.restype = C.c_int
    L.vtx_create.restype = C.c_int
    L.vtx_create.argtypes = [C.POINTER(Config), C.POINTER(C.c_void_p)]
    L.vtx_destroy.restype = None
    L.vtx_destroy.argtypes = [C.c_void_p]
    L.vtx_last_error.restype = C.c_char_p
    L.vtx_last_error.argtypes = [C.c_void_p]
    L.vtx_host_alloc.restype = C.c_int
    L.vtx_host_alloc.argtypes = [C.POINTER(C.c_void_p), C.c_uint64]
    L.vtx_host_free.restype = C.c_int
    L.vtx_host_free.argtypes = [C.c_void_p]
    L.vtx_set_barcodes.restype = C.c_int
    L.vtx_set_barcodes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    for name in ("vtx_submit", "vtx_submit_device"):
        f = getattr(L, name); f.restype = C.c_int; f.argtypes = [C.c_void_p, C.POINTER(Batch)]
    L.vtx_submit_device_ex.restype = C.c_int
    L.vtx_submit_device_ex.argtypes = [C.c_void_p, C.POINTER(Batch), C.c_uint32, C.c_uint32]
    for name in ("vtx_finish", "vtx_finish_device", "vtx_gather"):
        f = getattr(L, name); f.restype = C.c_int; f.argtypes = [C.c_void_p, C.POINTER(Result)]
    L.vtx_fetch.restype = C.c_int
    L.vtx_fetch.argtypes = [C.c_void_p, C.POINTER(Result), C.POINTER(Result)]
    L.vtx_sync.restype = C.c_int
    L.vtx_sync.argtypes = [C.c_void_p]
    L.vtx_wait_copies.restype = C.c_int
    L.vtx_wait_copies.argtypes = [C.c_void_p]
    L.vtx_score_pairs.restype = C.c_int
    L.vtx_score_pairs.argtypes = [C.c_void_p, C.POINTER(Batch), C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.vtx_pack_umi.restype = C.c_uint64
    L.vtx_pack_umi.argtypes = [C.c_char_p, C.c_uint32]
    L.vtx_last_timing.restype = C.c_int
    L.vtx_last_timing.argtypes = [C.c_void_p, C.POINTER(Timing)]
    L.vtx_last_tile_counts.restype = C.c_int
    L.vtx_last_tile_counts.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_uint32]
    L.vtx_submit2.restype = C.c_int
    L.vtx_submit2.argtypes = [C.c_void_p, C.POINTER(Batch2)]
    L.vtx_submit2_device.restype = C.c_int
    L.vtx_submit2_device.argtypes = [C.c_void_p, C.POINTER(Batch2), C.c_uint32, C.c_uint32]
    L.vtx_bgzf_inflate.restype = C.c_int
    L.vtx_bgzf_inflate.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32]
    L.vtx_submit_bam.restype = C.c_int
    L.vtx_submit_bam.argtypes = [C.c_void_p, C.POINTER(BamShard)]
    L.vtx_bam_metrics_get.restype = C.c_int
    L.vtx_bam_metrics_get.argtypes = [C.c_void_p, C.POINTER(BamMetrics)]
    L.vtx_set_min_base_quality.restype = C.c_int
    L.vtx_set_min_base_quality.argtypes = [C.c_void_p, C.c_uint32]
    L.vtx_bam_low_base_quality.restype = C.c_int
    L.vtx_bam_low_base_quality.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    L.vtx_set_locus_stats.restype = C.c_int
    L.vtx_set_locus_stats.argtypes = [C.c_void_p, C.c_int32]
    L.vtx_locus_stats_get.restype = C.c_int
    L.vtx_locus_stats_get.argtypes = [C.c_void_p, C.POINTER(C.POINTER(LocusStats)), C.POINTER(C.c_uint64)]
    L.vtx_set_donors.restype = C.c_int
    L.vtx_set_donors.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_double]
    L.vtx_donor_ll_get.restype = C.c_int
    L.vtx_donor_ll_get.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_int64)), C.POINTER(C.POINTER(C.c_uint64)),
                                   C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.vtx_cluster_cells.restype = C.c_int
    L.vtx_cluster_cells.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                                    C.POINTER(ClusterParams), C.POINTER(Clusters)]
    L.vtx_cluster_cells_pinned.restype = C.c_int
    L.vtx_cluster_cells_pinned.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                                           C.c_void_p, C.POINTER(ClusterPinnedParams), C.POINTER(Clusters)]
    L.vtx_donors_ambient.restype = C.c_int
    L.vtx_donors_ambient.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                                     C.c_void_p, C.POINTER(AmbientParams), C.POINTER(Ambient)]
    L.vtx_cluster_genotypes.restype = C.c_int
    L.vtx_cluster_genotypes.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.POINTER(ClusterGtParams), C.POINTER(ClusterGt)]
    L.vtx_cluster_refine.restype = C.c_int
    L.vtx_cluster_refine.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(ClusterCallsParams), C.POINTER(ClusterCalls)]
    L.vtx_pack_cb.restype = C.c_uint64
    L.vtx_pack_cb.argtypes = [C.c_char_p, C.c_uint32]
    L.vtx_gather_start.restype = C.c_int
    L.vtx_gather_start.argtypes = [C.c_void_p, C.c_int32]
    L.vtx_gather_wait.restype = C.c_int
    L.vtx_gather_wait.argtypes = [C.c_void_p, C.POINTER(Result)]
    L.vtx_comm_unique_id.restype = C.c_int
    L.vtx_comm_unique_id.argtypes = [C.c_void_p]
    L.vtx_comm_init.restype = C.c_int
    L.vtx_comm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
    _lib = L
    return L
