"""ctypes binding of libb200tip.so (the C ABI declared in include/b200tip.h).

There is no CPU fallback: if the shared library or a CUDA device is missing, every scoring
call raises.  `symbols()` lists what include/b200tip.h declares, so the CPU test-suite can
verify the export table without touching a GPU.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200tip.so")

TIP_F32, TIP_F64, TIP_BF16, TIP_I16, TIP_I32 = 0, 1, 2, 3, 4
COVER_NAC, COVER_SNAC, COVER_NBC = 0, 1, 2
CAM_MAX_BLOCKS = 1024
SC_CAM_MAX_SECTIONS = 4096      # TIP_SC_CAM_MAX_SECTIONS
ROLE_QUERY, ROLE_TRAIN = 0, 1
RANGE_SAME_CLASS, RANGE_OTHER_CLASSES = 0, 1
ROW_TILE, COL_TILE = 128, 256
STAT_GINI, STAT_MAX, STAT_PCS, STAT_ENTROPY = 0, 1, 2, 3
MC_LINEAR, MC_RELU, MC_SOFTMAX = 0, 1, 2
MC_OUTPUT, MC_PREACT = 0, 1


class RerankExtras(C.Structure):
    """tip_rerank_extras of include/b200tip.h"""
    _fields_ = [("q_idx", C.c_void_p), ("next_seed_ub", C.c_void_p), ("next_t_rmax", C.c_float),
                ("next_t_errmax", C.c_float), ("fin_dist_a", C.c_void_p), ("fin_gid", C.c_void_p),
                ("fin_idx", C.c_void_p), ("fin_n_total", C.c_int64), ("fin_out", C.c_void_p),
                ("count_overflow_only", C.c_int32), ("reserved", C.c_int32)]


class AdamTensor(C.Structure):
    """tip_adam_tensor of include/b200tip.h"""
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("m", C.c_void_p), ("v", C.c_void_p),
                ("numel", C.c_int64)]


class McLayer(C.Structure):
    """tip_mc_layer of include/b200tip.h"""
    _fields_ = [("kernel", C.c_void_p), ("bias", C.c_void_p), ("p", C.c_double), ("in_", C.c_int32),
                ("out", C.c_int32), ("activation", C.c_int32), ("reserved", C.c_int32)]


class CorruptTable(C.Structure):
    """tip_corrupt_table of include/b200tip.h"""
    _fields_ = [("arena", C.c_void_p), ("key_off", C.c_void_p), ("key_len", C.c_void_p), ("key_hash", C.c_void_p),
                ("val_begin", C.c_void_p), ("val_off", C.c_void_p), ("val_len", C.c_void_p), ("val_cdf", C.c_void_p),
                ("slots", C.c_void_p), ("n", C.c_int64), ("cap", C.c_int64)]


CORRUPT_CP_WORDS = 34816        # TIP_CORRUPT_CP_WORDS


class WorkItem(C.Structure):
    _fields_ = [("q_row0", C.c_int32), ("q_rows", C.c_int32), ("col0", C.c_int32), ("col1", C.c_int32),
                ("slot", C.c_int32), ("reserved", C.c_int32)]


_vp, _i32, _i64, _u64, _f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_float

# name -> (restype, argtypes); mirrors include/b200tip.h one to one
_SIGNATURES = {
    "tip_version": (C.c_int, []),
    "tip_last_error": (C.c_char_p, []),
    "tip_device_info": (C.c_int, [C.POINTER(C.c_int)] * 3),
    "tip_launch_count": (C.c_uint64, []),
    "tip_deepgini": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp, _vp]),
    "tip_softmax_stat": (C.c_int, [_vp, C.c_int, _i64, _i64, C.c_int, _vp, _vp, _vp]),
    "tip_vote_add": (C.c_int, [_vp, C.c_int, _i64, _i64, _i64, _i64, _i64, _vp, _vp]),
    "tip_vote_finish": (C.c_int, [_vp, _i64, _i64, _i64, _vp, _vp, _vp]),
    "tip_kmnc": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp, C.c_int, _i32, _vp, C.c_int, _vp, _vp]),
    "tip_kmnc_packed": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp, C.c_int, _i32, _vp, _vp, _vp]),
    "tip_cam_buckets": (C.c_int, [_vp, C.c_int, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _vp]),
    "tip_sc_cam": (C.c_int, [_vp, C.c_int, _i64, _vp, _i32, _vp, _vp, _vp, _vp]),
    "tip_cover_packed_words": (_i64, [_i64]),
    "tip_cover_threshold": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp, C.c_int, C.c_double, C.c_int, _vp, _vp, _vp, _vp]),
    "tip_tknc": (C.c_int, [_vp, C.c_int, _i64, _i64, _i32, _vp, _i64, _i64, _vp, _i64, _vp]),
    "tip_stats_update": (C.c_int, [_vp, C.c_int, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp]),
    "tip_pack_bool": (C.c_int, [_vp, _i64, _i64, _vp, _vp]),
    "tip_cam_bits": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp]),
    "tip_cam_bits_stack": (C.c_int, [_vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp]),
    "tip_pair_pitch": (_i64, [_i64, C.c_int]),
    "tip_pair_prep": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, C.c_int, C.c_int, _f32, _f32, _vp, _vp, _vp, _vp]),
    "tip_nn_filter": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _f32, _vp, _f32, _vp, _vp,
                                _vp, _i32, _i32, _vp, _vp]),
    "tip_nn_filter_live": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _f32, _vp, _f32, _vp,
                                     _vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    "tip_sizeof_rerank_extras": (_i32, []),
    "tip_nn_rerank_work_bytes": (_i64, [_i64, C.c_int]),
    "tip_nn_query_prep": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tip_nn_rerank": (C.c_int, [_vp, _vp, C.c_int, _i64, _i64, _i64, _vp, _vp, _i32, _vp, _vp, _i32, C.c_int,
                                _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tip_gather_rows": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _vp]),
    "tip_dsa_distinct_smem_bytes": (_i64, [_i64]),
    "tip_dsa_distinct_winners": (C.c_int, [_vp, _i64, _vp, _vp, _i32, _i64, _i32, _vp, C.c_int, _i64, _vp, _vp, _f32,
                                           _f32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tip_dsa_slot_out": (C.c_int, [_vp, C.c_int, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp]),
    "tip_dsa_pack_out": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _i64, _i64, _vp, _vp]),
    "tip_comm_bytes": (_i64, [_i32, _i64]),
    "tip_comm_alloc": (C.c_int, [_i32, _i64, C.POINTER(C.c_void_p), _vp]),
    "tip_comm_open": (C.c_int, [_i32, _i32, _vp, _vp, _i64, C.POINTER(C.c_void_p)]),
    "tip_comm_close": (C.c_int, [_vp]),
    "tip_comm_free_local": (C.c_int, [_vp]),
    "tip_comm_push_nn": (C.c_int, [_vp, _vp, C.c_int, _vp, _i64, _vp]),
    "tip_comm_push_lse": (C.c_int, [_vp, _vp, _vp, _i64, _vp]),
    "tip_comm_min": (C.c_int, [_vp, C.c_int, _i64, _vp, _vp]),
    "tip_comm_lse": (C.c_int, [_vp, _i64, _vp, _vp, _vp]),
    "tip_shard_winner_queries": (C.c_int, [_vp, _vp, _vp, C.c_int, _i64, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _vp,
                                           _vp, _vp, _vp, _vp, _vp]),
    "tip_whiten": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _i64, _vp, _vp, _vp, _vp]),
    "tip_row_sqnorm": (C.c_int, [_vp, _i64, _i64, _vp, _vp]),
    "tip_kde_lse": (C.c_int, [_vp, _i64, _vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _vp]),
    "tip_kde_lse_f16": (C.c_int, [_vp, _i64, _vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp, _vp]),
    "tip_pair_prep_f16": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, C.c_int, _f32, _f32, _vp, _vp, _vp, _vp]),
    "tip_kde_combine": (C.c_int, [_vp, _vp, _i64, _i32, _vp, _vp, _vp]),
    "tip_nn_filter_tile": (C.c_int, [_i64, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "tip_nn_filter_kind": (C.c_int, [_i64]),
    "tip_kde_tile_rows": (C.c_int, []),
    "tip_kde_slot_parts": (C.c_int, []),
    "tip_debug_timeline": (C.c_int, [_vp, _i32]),
    "tip_debug_cta_clock": (C.c_int, [_vp]),
    "tip_pair_probe": (C.c_int, [_vp, _i64, _vp, _i64, _i64, C.c_int, _i64, C.c_int, _vp, _vp]),
    "tip_kmeans_work_bytes": (_i64, [_i64, _i64, _i32, _i32, C.c_int]),
    "tip_kmeans_fit": (C.c_int, [_vp, C.c_int, _i64, _i64, _i32, _i32, _i32, C.c_double, C.c_uint64, _vp, _vp, _vp,
                                 _vp]),
    "tip_kmeans_predict": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _i32, _i32, _vp, _vp, _vp, _vp]),
    "tip_sil_prep": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tip_sil_dsum": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp, _i32, _vp, _vp]),
    "tip_sil_finish": (C.c_int, [_vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tip_gmm_scatter_chunks": (_i32, [_i64, _i64, _i32, _i32]),
    "tip_gmm_work_bytes": (_i64, [_i64, _i64, _i32, _i32]),
    "tip_gmm_quad": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp, _i32, _vp, _vp]),
    "tip_gmm_resp": (C.c_int, [_vp, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tip_gmm_moments": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "tip_gmm_scatter": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp, _i32, _vp, C.c_double, _i32, _vp, _vp, _vp]),
    "tip_cov_location": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp, _vp, _vp]),
    "tip_col_var": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp, _vp, _vp]),
    "tip_whiten_dmma": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _i64, _vp, _vp, _vp, _vp]),
    "tip_levenshtein": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _i64, _i32, C.c_int, _vp, _vp]),
    "tip_tok_count": (C.c_int, [_vp, _vp, _i64, _u64, _u64, C.c_int, _vp, _vp]),
    "tip_tok_emit": (C.c_int, [_vp, _vp, _i64, _u64, _u64, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp]),
    "tip_tok_vocab_table": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _i64, _vp]),
    "tip_tok_fit": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp,
                              _i64, _vp, _i64, _vp, _vp]),
    "tip_tok_lookup": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _i64, _vp, _i64,
                                 _vp, _vp, _vp, _vp, _i64, C.c_int, C.c_int, _i32, _vp]),
    "tip_corrupt_table_build": (C.c_int, [_vp, _vp]),
    "tip_corrupt_census": (C.c_int, [_vp, _i64, _vp, _vp]),
    "tip_corrupt_count": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _vp]),
    "tip_corrupt_texts": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _i64, C.c_double, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                    _vp, _vp]),
    "tip_corrupt_words": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tip_corrupt_layout": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "tip_corrupt_write": (C.c_int, [_vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tip_keras_adam": (C.c_int, [_vp, _i32, _i64, _vp, _f32, _f32, _f32, _f32, _vp]),
    "tip_softmax_xent": (C.c_int, [_vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp]),
    "tip_softmax_xent_seg": (C.c_int, [_vp, _vp, _i64, _i64, _i32, _vp, _vp, _vp, _vp]),
    "tip_stack_gather": (C.c_int, [_vp, _i32, _i64, _vp, _i64, _vp, _i64, _i64, _i64, _i64, _i64, _vp, _vp]),
    "tip_mc_head": (C.c_int, [_vp, _i64, _i64, _i64, _i64, _i64, _vp, _i32, _u64, _i32, _vp, _vp]),
    "tip_mc_head_stack": (C.c_int, [_vp, _i64, _i64, _i64, _i64, _i64, _i64, _i64, _vp, _i32, _vp, _i32, _vp, _vp]),
}

_lock = threading.Lock()
_lib = None


def symbols():
    return sorted(_SIGNATURES)


def load() -> C.CDLL:
    """Loads libb200tip.so; raises (never falls back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(
                    f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                    "(nvcc, sm_90a).  simple_tip_b200 has no CPU fallback.")
            lib = C.CDLL(LIB_PATH)
            for name, (res, args) in _SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype, fn.argtypes = res, args
            if lib.tip_sizeof_rerank_extras() != C.sizeof(RerankExtras):
                raise RuntimeError("libb200tip.so and simple_tip_b200/_lib.py disagree on tip_rerank_extras: rebuild the library")
            _lib = lib
    return _lib


class TipError(RuntimeError):
    pass


def check(rc: int, what: str):
    if rc != 0:
        msg = load().tip_last_error().decode(errors="replace")
        raise TipError(f"{what} failed with status {rc}: {msg}")


def launch_count() -> int:
    return int(load().tip_launch_count())
