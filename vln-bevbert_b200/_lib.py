"""ctypes binding of the C ABI in include/bevbert_b200.h (libbevbert_b200.so, built in-tree by
vln-bevbert_b200/csrc/Makefile or __graft_entry__.build()).

There is no fallback: if the shared library is missing or a symbol is absent, importing / calling fails
loudly.  This is the binding a maintainer of the reference would add (INTEGRATION.md).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbevbert_b200.so")

c_void_p, c_int, c_i32, c_i64, c_u32, c_u64, c_float = (C.c_void_p, C.c_int, C.c_int32, C.c_int64, C.c_uint32,
                                                         C.c_uint64, C.c_float)


class GemmArgs(C.Structure):
    """struct bb_gemm_args (include/bevbert_b200.h)."""
    _fields_ = [
        ("A", c_void_p), ("B", c_void_p), ("D", c_void_p),
        ("M", c_i32), ("N", c_i32), ("K", c_i32),
        ("nb1", c_i32), ("nb2", c_i32),
        ("a_mn", c_i32), ("b_mn", c_i32),
        ("lda", c_i64), ("a_s1", c_i64), ("a_s2", c_i64),
        ("ldb", c_i64), ("b_s1", c_i64), ("b_s2", c_i64),
        ("ldd", c_i64), ("d_s1", c_i64), ("d_s2", c_i64),
        ("out_f32", c_i32), ("accumulate", c_i32), ("split_k", c_i32),
        ("alpha", c_float),
        ("bias", c_void_p),
        ("act", c_i32),
        ("aux_out", c_void_p), ("aux_in", c_void_p),
        ("epi_mul", c_i32),
        ("drop_seed", c_u64), ("drop_thresh", c_u32), ("drop_scale", c_float),
        ("add_in", c_void_p),
        ("block_n", c_i32),
    ]


class AttnScoresArgs(C.Structure):
    """struct bb_attn_scores_args (include/bevbert_b200.h)."""
    _fields_ = [("A", c_void_p), ("lda", c_i64), ("a_s1", c_i64), ("a_s2", c_i64),
                ("Bm", c_void_p), ("ldb", c_i64), ("b_s1", c_i64), ("b_s2", c_i64)] + \
        [(n, c_i32) for n in ("B", "H", "nq", "nk", "ldp", "mode")] + [("alpha", c_float), ("out_scale", c_float)] + \
        [("kmask", c_void_p), ("bias", c_void_p), ("seed", c_u64), ("thresh", c_u32), ("scale", c_float)] + \
        [(n, c_void_p) for n in ("P", "Pd", "Pin", "dS", "dbias")]


class FlashArgs(C.Structure):
    """struct bb_flash_args (include/bevbert_b200.h)."""
    _fields_ = [(n, c_void_p) for n in ("q", "k", "v", "o")] + [(n, c_i64) for n in ("q_bs", "k_bs", "v_bs", "o_bs")] + \
        [(n, c_i32) for n in ("ldq", "ldk", "ldv", "ldo", "B", "H", "nq", "nk", "dh")] + [("alpha", c_float)] + \
        [("kmask", c_void_p), ("bias", c_void_p), ("lse", c_void_p), ("seed", c_u64), ("thresh", c_u32), ("scale", c_float)] + \
        [("dout", c_void_p), ("do_bs", c_i64), ("lddo", c_i32), ("pad0_", c_i32), ("dsum", c_void_p)] + \
        [(n, c_void_p) for n in ("dq", "dk", "dv")] + [(n, c_i64) for n in ("dq_bs", "dk_bs", "dv_bs")] + \
        [(n, c_i32) for n in ("lddq", "lddk", "lddv", "pad1_")] + [("dbias", c_void_p)]


class AttnDesc(C.Structure):
    """struct bb_attn_desc (include/bevbert_b200.h)."""
    _fields_ = [(n, c_i32) for n in ("B", "nq", "nk", "Hd", "heads", "cross", "want_dbias")] + [("eps", c_float)] + \
        [(n, c_void_p) for n in ("x", "c", "kmask", "bias", "w_qkv", "w_kv", "w_o", "b_qkv", "b_kv", "b_o", "gamma", "beta")] + \
        [("seed_attn", c_u64), ("th_attn", c_u32), ("sc_attn", c_float), ("seed_h", c_u64), ("th_h", c_u32), ("sc_h", c_float)] + \
        [(n, c_void_p) for n in ("ws", "y", "dy", "gws", "dx", "dc", "dw_qkv", "db_qkv", "dw_kv", "db_kv", "dw_o", "db_o",
                                  "dgamma", "dbeta", "dbias")]


class FfnDesc(C.Structure):
    """struct bb_ffn_desc (include/bevbert_b200.h)."""
    _fields_ = [("M", c_i64), ("Hd", c_i32), ("Fd", c_i32), ("eps", c_float)] + \
        [(n, c_void_p) for n in ("a", "w1", "w2", "b1", "b2", "gamma", "beta")] + \
        [("seed_h", c_u64), ("th_h", c_u32), ("sc_h", c_float)] + \
        [(n, c_void_p) for n in ("ws", "y", "dy", "gws", "da", "dw1", "db1", "dw2", "db2", "dgamma", "dbeta")]


class PanoDesc(C.Structure):
    """struct bb_pano_desc (include/bevbert_b200.h)."""
    _fields_ = [(n, c_i32) for n in ("N", "V", "Hd", "heads", "Fd", "pad_")] + \
        [(n, c_void_p) for n in ("x", "kmask", "w_in", "w_out", "w1", "w2", "b_in", "b_out", "b1", "b2", "g1", "be1", "g2",
                                  "be2")] + \
        [("seed_attn", c_u64), ("th_attn", c_u32), ("sc_attn", c_float), ("seed1", c_u64), ("seed2", c_u64),
         ("seed3", c_u64), ("th_h", c_u32), ("sc_h", c_float)] + \
        [(n, c_void_p) for n in ("ws", "y", "dy", "gws", "dx", "dw_in", "db_in", "dw_out", "db_out", "dw1", "db1", "dw2",
                                  "db2", "dg1", "dbe1", "dg2", "dbe2")]


class MtTensor(C.Structure):
    """struct bb_mt_tensor (include/bevbert_b200.h): one row of a multi-tensor launch table (64 bytes)."""
    _fields_ = [("p", c_void_p), ("g", c_void_p), ("m", c_void_p), ("v", c_void_p), ("p16", c_void_p), ("n", c_i64),
                ("step_size", c_float), ("decay", c_float), ("chunk0", c_i64)]


# name -> (restype, argtypes); mirrors include/bevbert_b200.h one to one
_SIGNATURES = {
    "bb_last_error": (C.c_char_p, []),
    "bb_abi_version": (c_int, []),
    "bb_launch_count": (c_i64, []),
    "bb_reset_launch_count": (None, []),
    "bb_gemm_bf16": (c_int, [C.POINTER(GemmArgs), c_void_p]),
    "bb_set_drop_salt_ptr": (c_int, [c_void_p]),
    "bb_set_deterministic": (c_int, [c_int]),
    "bb_set_det_workspace": (c_int, [c_void_p, c_void_p, c_i64]),
    "bb_set_act_f32": (c_int, [c_int]),
    "bb_get_act_f32": (c_int, []),
    "bb_gemm_trace": (c_int, [c_void_p]),
    "bb_gemm_profile_buffer": (c_int, [c_void_p, c_i64]),
    "bb_gemm_profile": (c_int, [c_int]),
    "bb_gemm_profile_count": (c_i64, []),
    "bb_gemm_profile_read": (c_int, [c_i64, C.POINTER(c_float), C.POINTER(c_i64)]),
    "bb_bev_lift_index": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_float] * 5 + [c_int, c_float, c_float, c_void_p,
                                                                                  c_void_p, c_void_p]),
    "bb_bev_lift_points": (c_int, [c_void_p, c_void_p] + [c_int] * 3 + [c_float] * 5 + [c_void_p] * 4),
    "bb_bev_cell_index": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_float, c_float, c_void_p, c_void_p]),
    "bb_bev_scatter_mean_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int] + [c_void_p] * 5),
    "bb_bev_scatter_mean_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int] + [c_void_p] * 5),
    "bb_bev_scatter_sem_f64": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "bb_bev_scatter_sem_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "bb_bev_splat_nodes": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                   c_float, c_float, c_void_p, c_void_p, c_void_p]),
    "bb_cast_f32_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_u64, c_u32, c_float, c_void_p]),
    "bb_cast_bf16_f32": (c_int, [c_void_p, c_void_p, c_i64, c_void_p]),
    "bb_layernorm_fwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_float, c_i64, c_int,
                                 c_u64, c_u32, c_float, c_u64, c_u32, c_float,
                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "bb_layernorm_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int,
                                 c_u64, c_u32, c_float, c_u64, c_u32, c_float,
                                 c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "bb_colsum_bf16": (c_int, [c_void_p, c_i64, c_int, c_i64, c_void_p, c_void_p]),
    "bb_softmax_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_u64, c_u32, c_float,
                               c_void_p, c_void_p, c_void_p]),
    "bb_softmax_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_u64, c_u32, c_float, c_float,
                               c_void_p, c_void_p, c_void_p]),
    "bb_embed_sum": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_int, c_void_p, c_void_p]),
    "bb_embed_scatter_grad": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_int, c_i64, c_void_p, c_void_p, c_void_p,
                                      c_void_p]),
    "bb_gather_rows_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_void_p, c_void_p]),
    "bb_scatter_add_rows": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_void_p, c_void_p]),
    "bb_scatter_rows_sorted": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p, c_void_p]),
    "bb_dropout_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_u64, c_u32, c_float, c_void_p]),
    "bb_act_bwd_bf16": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_i64, c_void_p]),
    "bb_add_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p, c_void_p]),
    "bb_add_rows3": (c_int, [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_i64,
                             c_int, c_void_p, c_i64, c_void_p]),
    "bb_image_patches": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_i64, c_i64, c_i64, c_i64, c_int,
                                 C.POINTER(c_float), C.POINTER(c_float), c_void_p, c_void_p]),
    "bb_vit_tokens": (c_int, [c_void_p] * 5 + [c_float, c_int, c_int, c_int, c_void_p, c_void_p]),
    "bb_waypoint_nms": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_float, c_int, c_void_p, c_void_p]),
    "bb_conv2d": (c_int, [c_void_p, c_void_p] + [c_int] * 8 + [c_void_p] * 3),
    "bb_depth_stem": (c_int, [c_void_p, c_int, c_int, c_int, c_i64, c_i64, c_i64, c_void_p, c_int, c_void_p, c_void_p,
                              c_void_p]),
    "bb_groupnorm_apply": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                   c_void_p, c_void_p] + [c_int] * 5 + [c_float, c_int, c_int, c_void_p, c_void_p]),
    "bb_ce_view_stack": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "bb_ce_waypoint_candidates": (c_int, [c_void_p, c_void_p, c_void_p, c_int] + [c_void_p] * 8 + [c_void_p]),
    "bb_ce_waypoint_candidates_aug": (c_int, [c_void_p] * 4 + [c_int] + [c_void_p] * 8 + [c_void_p]),
    "bb_ce_gmap_features": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "bb_ce_gmap_features_bwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "bb_scale_rows_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_i64, c_void_p]),
    "bb_segment_wsum": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p, c_void_p]),
    "bb_segment_wsum_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p, c_void_p]),
    "bb_add_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_void_p]),
    "bb_axpy_f32_from_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_void_p]),
    "bb_attn_scores": (c_int, [C.POINTER(AttnScoresArgs), c_void_p]),
    "bb_flash_fwd": (c_int, [C.POINTER(FlashArgs), c_void_p]),
    "bb_set_attn_tc": (c_int, [c_int]),
    "bb_attn_tc_trace": (c_int, [c_void_p]),
    "bb_flash_bwd": (c_int, [C.POINTER(FlashArgs), c_void_p]),
    "bb_set_side_stream": (c_int, [c_void_p]),
    "bb_side_join": (c_int, [c_void_p]),
    "bb_attn_ws_bytes": (c_int, [C.POINTER(AttnDesc), C.POINTER(c_i64), C.POINTER(c_i64)]),
    "bb_attn_fwd": (c_int, [C.POINTER(AttnDesc), c_void_p]),
    "bb_attn_bwd": (c_int, [C.POINTER(AttnDesc), c_void_p]),
    "bb_ffn_ws_bytes": (c_int, [C.POINTER(FfnDesc), C.POINTER(c_i64), C.POINTER(c_i64)]),
    "bb_ffn_fwd": (c_int, [C.POINTER(FfnDesc), c_void_p]),
    "bb_ffn_bwd": (c_int, [C.POINTER(FfnDesc), c_void_p]),
    "bb_pano_ws_bytes": (c_int, [C.POINTER(PanoDesc), C.POINTER(c_i64), C.POINTER(c_i64)]),
    "bb_pano_fwd": (c_int, [C.POINTER(PanoDesc), c_void_p]),
    "bb_pano_bwd": (c_int, [C.POINTER(PanoDesc), c_void_p]),
    "bb_mt_chunk_elems": (c_int, []),
    "bb_mt_sumsq": (c_int, [c_void_p, c_int, c_i64, c_void_p, c_void_p]),
    "bb_adamw_step": (c_int, [c_void_p, c_int, c_i64, c_float, c_float, c_float, c_void_p, c_float, c_float, c_void_p]),
    "bb_mt_cast_bf16": (c_int, [c_void_p, c_int, c_i64, c_void_p]),
    "bb_softmax_xent": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_i64, c_void_p, c_void_p, c_void_p, c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES.keys())

_lib = None


class BevbertLibraryError(RuntimeError):
    pass


def load():
    """Loads the shared library once and sets every prototype. Raises if it (or a symbol) is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise BevbertLibraryError(
            "%s not found: build it with `make -C vln-bevbert_b200/csrc` or `python -c 'import __graft_entry__ as g; "
            "g.build()'`. There is no CPU / PyTorch fallback for the hot path." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name, None)
        if fn is None:
            raise BevbertLibraryError("symbol %s missing from %s" % (name, LIB_PATH))
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().bb_last_error()
        raise BevbertLibraryError("%s failed (rc=%d): %s" % (what, rc, msg.decode() if msg else "?"))
