"""Tensor-level wrappers: one thin Python function per C-ABI entry point (include/bevbert_b200.h).

Each wrapper only extracts device pointers / sizes from torch tensors, passes torch's current CUDA stream and
raises on a non-zero status.  There is no arithmetic here and no fallback: without the CUDA library these
functions raise.  (tests/emu_kernels.py replaces this module's functions with torch restatements to
exercise the host-side block logic on CPU; that emulation is test infrastructure, never shipped.)
"""
import ctypes as C
import warnings

import torch

from . import _lib

ACT_NONE, ACT_GELU, ACT_RELU, ACT_QGELU = 0, 1, 2, 3     # ACT_QGELU: x * sigmoid(1.702 x), CLIP
EPI_NONE, EPI_DGELU, EPI_DRELU = 0, 1, 2
BF16 = torch.bfloat16


_FP32_ARM = False


def act_dtype():
    """dtype of activations between kernels: bf16 in the product, fp32 in the high-precision verification arm."""
    return torch.float32 if _FP32_ARM else BF16


def set_precision(fp32: bool) -> bool:
    """Switches the whole library between the bf16 product path and the fp32 VERIFICATION arm (bb_set_act_f32):
    activations, GEMM operands and every reduction in fp32 (a plain CUDA-core GEMM, the unfused attention sequence,
    the Python sub-layer composition).  It exists so that the parity tests can hold the model to 1e-3 against the fp32
    oracle and so separate kernel logic from bf16 rounding; it is far slower than the product path.  Returns the
    previous setting.  Build a fresh model (weight shadows are per precision) after switching."""
    global _FP32_ARM
    prev = _FP32_ARM
    _lib.load().bb_set_act_f32(1 if fp32 else 0)
    _FP32_ARM = bool(fp32)
    return prev


def use_flash():
    """fused attention core (bb_flash_*) or, in the fp32 arm, the unfused GEMM + softmax sequence"""
    return FLASH and not _FP32_ARM


def _p(t):
    return 0 if t is None else t.data_ptr()


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream():
    """raw cudaStream_t of torch's current stream on the current device (fast path avoids building a Stream object).
    Every launch asks for it, so this is also where the library's deterministic mode follows torch's flag."""
    if _det_mode() != _DET_MODE:
        _set_det_mode(_det_mode())
    if _raw_stream is not None:
        return _raw_stream(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------- deterministic mode
# torch.use_deterministic_algorithms(True) switches the library to fixed-order reductions (bb_set_deterministic):
# bit-identical results for bit-identical inputs on the same build and GPU model.  warn_only=True maps to mode 2, in
# which the one path without a deterministic kernel runs after a warning instead of raising.
DET_WS_BYTES = 32 << 20     # per stream; the largest user is a split-K weight gradient at about one wave of tiles
_DET_MODE = 0
_DET_WS = None


def _det_mode():
    if not torch._C._get_deterministic_algorithms():
        return 0
    return 2 if torch._C._get_deterministic_algorithms_warn_only() else 1


def _set_det_mode(mode):
    """Registers the zero-filled main / side workspaces before the first deterministic launch (they stay allocated at
    fixed addresses, so a CUDA graph captured later can use them), then sets the library's mode."""
    global _DET_MODE, _DET_WS
    lib = _lib.load()
    if mode and _DET_WS is None:
        if _capturing():
            raise RuntimeError("deterministic mode was switched on during a CUDA-graph capture; call "
                               "torch.use_deterministic_algorithms(True) and run one eager step before capturing")
        _DET_WS = [torch.zeros(DET_WS_BYTES, dtype=torch.uint8, device="cuda") for _ in range(2)]
        torch.cuda.synchronize()
        _lib.check(lib.bb_set_det_workspace(_DET_WS[0].data_ptr(), _DET_WS[1].data_ptr(), DET_WS_BYTES),
                   "bb_set_det_workspace")
    _lib.check(lib.bb_set_deterministic(mode), "bb_set_deterministic")
    _DET_MODE = mode


def _nondeterministic(what):
    """torch's contract for a path without a deterministic implementation: raise under the flag, or warn with
    warn_only=True."""
    mode = _det_mode()
    if mode == 1:
        raise RuntimeError("%s does not have a deterministic implementation, but torch.use_deterministic_algorithms"
                           "(True) is set" % what)
    if mode == 2:
        warnings.warn("%s does not have a deterministic implementation" % what)


def _scatter_sorted(src, dst, H, out_f32, src_row=None, w=None):
    """out_f32[dst[e]] += ((t_e1 + t_e2) + ...) in ascending source order e, t_e = (w[e] *) src[src_row[e] | e];
    dst < 0 is dropped (bb_scatter_rows_sorted after a stable sort of the destinations)."""
    keys, perm = torch.sort(dst, stable=True)
    rows = perm if src_row is None else src_row[perm]
    wp = w[perm].contiguous() if w is not None else None
    _lib.check(_lib.load().bb_scatter_rows_sorted(src.data_ptr(), int(src.dtype == torch.float32), rows.data_ptr(),
                                                  _p(wp), keys.data_ptr(), keys.numel(), H, out_f32.data_ptr(),
                                                  _stream()), "bb_scatter_rows_sorted")
    return out_f32


def _req(t, dtype, name):
    if t.dtype != dtype:
        raise TypeError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor (the hot path has no CPU implementation)" % name)


def drop_params(p: float):
    """(thresh, scale) of the counter-based dropout for probability p."""
    if p <= 0.0:
        return 0, 1.0
    return min(int(p * 4294967296.0), 4294967295), 1.0 / (1.0 - p)


def launch_count() -> int:
    return int(_lib.load().bb_launch_count())


def reset_launch_count():
    _lib.load().bb_reset_launch_count()


# ---------------------------------------------------------------------------------------------- GEMM
def gemm(a, b, out, M, N, K, lda, ldb, ldd, a_mn=False, b_mn=False, nb1=1, nb2=1, a_s=(0, 0), b_s=(0, 0),
         d_s=(0, 0), alpha=1.0, bias=None, act=ACT_NONE, aux_out=None, aux_in=None, epi_mul=EPI_NONE, add_in=None,
         accumulate=False, split_k=1, drop=(0, 0, 1.0), block_n=0):
    """out = epi(alpha * A @ B^T) on wgmma; a/b/out are base tensors (pointer = data_ptr()), strides in
    elements.  out dtype bf16 or f32 decides the output type.  drop = (seed, thresh, scale)."""
    lib = _lib.load()
    _req(a, act_dtype(), "a")
    _req(b, act_dtype(), "b")
    g = _lib.GemmArgs()
    g.A, g.B, g.D = a.data_ptr(), b.data_ptr(), out.data_ptr()
    g.M, g.N, g.K = M, N, K
    g.nb1, g.nb2 = nb1, nb2
    g.a_mn, g.b_mn = int(a_mn), int(b_mn)
    g.lda, g.a_s1, g.a_s2 = lda, a_s[0], a_s[1]
    g.ldb, g.b_s1, g.b_s2 = ldb, b_s[0], b_s[1]
    g.ldd, g.d_s1, g.d_s2 = ldd, d_s[0], d_s[1]
    if out.dtype == torch.float32:
        g.out_f32 = 1
    elif out.dtype == BF16 and not _FP32_ARM:
        g.out_f32 = 0
    else:
        raise TypeError("gemm output must be bf16 or f32 (f32 only in the fp32 verification arm)")
    g.accumulate, g.split_k = int(accumulate), split_k
    g.alpha = alpha
    g.bias = _p(bias)
    g.act = act
    g.aux_out, g.aux_in, g.epi_mul = _p(aux_out), _p(aux_in), epi_mul
    g.drop_seed, g.drop_thresh, g.drop_scale = drop
    g.add_in = _p(add_in)
    g.block_n = block_n
    _lib.check(lib.bb_gemm_bf16(C.byref(g), _stream()), "bb_gemm_bf16")
    return out


_PROF_BUF = None


def gemm_profile(enable: bool, capacity: int = 8192):
    """Start / stop the library's per-launch GEMM timing: every wgmma GEMM launch stamps %globaltimer (first CTA
    start, last CTA end) into its slot of a device buffer -- no events between launches."""
    global _PROF_BUF
    lib = _lib.load()
    if enable:
        if _PROF_BUF is None or _PROF_BUF.shape[0] < capacity:
            _PROF_BUF = torch.empty(capacity, 2, dtype=torch.int64, device="cuda")
        _PROF_BUF[:, 0] = -1          # all ones = "no start yet" for the unsigned atomicMin
        _PROF_BUF[:, 1] = 0
        torch.cuda.synchronize()
        _lib.check(lib.bb_gemm_profile_buffer(_PROF_BUF.data_ptr(), _PROF_BUF.shape[0]), "bb_gemm_profile_buffer")
    _lib.check(lib.bb_gemm_profile(int(enable)), "bb_gemm_profile")


def gemm_profile_records():
    """[(ms, (M, N, K, batches, a_mn, b_mn)), ...] for the launches recorded since gemm_profile(True)."""
    lib = _lib.load()
    out = []
    ms = C.c_float()
    dims = (C.c_int64 * 6)()
    for i in range(int(lib.bb_gemm_profile_count())):
        _lib.check(lib.bb_gemm_profile_read(i, C.byref(ms), dims), "bb_gemm_profile_read")
        out.append((float(ms.value), tuple(int(x) for x in dims)))
    return out


# ---------------------------------------------------------------------------------------------- native sub-layers
def native_sublayers():
    """True: blocks.py hands whole attention / FFN sub-layers to the C++ executors (csrc/layers.cu); the fp32
    verification arm runs the equivalent Python composition of the same kernels instead."""
    return not _FP32_ARM


_SIDE = None


def set_side_stream(stream):
    """torch.cuda.Stream (or None) for the weight-gradient GEMMs of the native backward executors (bb_set_side_stream)."""
    global _SIDE
    _SIDE = stream
    _lib.check(_lib.load().bb_set_side_stream(stream.cuda_stream if stream is not None else None), "bb_set_side_stream")


def side_stream():
    return _SIDE


def side_join():
    """the current stream waits for the side stream (no-op when nothing was forked since the last join)"""
    if _SIDE is not None:
        _lib.check(_lib.load().bb_side_join(_stream()), "bb_side_join")


def attn_desc():
    return _lib.AttnDesc()


def ffn_desc():
    return _lib.FfnDesc()


def pano_desc():
    return _lib.PanoDesc()


def sublayer_ws_bytes(d):
    lib = _lib.load()
    f, b = C.c_int64(), C.c_int64()
    fn = {_lib.AttnDesc: lib.bb_attn_ws_bytes, _lib.FfnDesc: lib.bb_ffn_ws_bytes, _lib.PanoDesc: lib.bb_pano_ws_bytes}[type(d)]
    _lib.check(fn(C.byref(d), C.byref(f), C.byref(b)), "bb_*_ws_bytes")
    return f.value, b.value


def sublayer_fwd(d):
    lib = _lib.load()
    fn = {_lib.AttnDesc: lib.bb_attn_fwd, _lib.FfnDesc: lib.bb_ffn_fwd, _lib.PanoDesc: lib.bb_pano_fwd}[type(d)]
    _lib.check(fn(C.byref(d), _stream()), "bb_sublayer_fwd")


def sublayer_bwd(d):
    lib = _lib.load()
    if isinstance(d, _lib.AttnDesc) and d.want_dbias and not FLASH and _fused_scores(d.nk, d.Hd // d.heads):
        _nondeterministic("the fused-scores (BB_FUSED_SCORES_MAX) graph-bias gradient")
    fn = {_lib.AttnDesc: lib.bb_attn_bwd, _lib.FfnDesc: lib.bb_ffn_bwd, _lib.PanoDesc: lib.bb_pano_bwd}[type(d)]
    _lib.check(fn(C.byref(d), _stream()), "bb_sublayer_bwd")


FUSED_SCORES_MAX_KEYS = min(512, int(__import__('os').environ.get('BB_FUSED_SCORES_MAX', '0')))


def _fused_scores(nk, dh):
    """the unfused attention path forms P / dS with bb_attn_scores (the BB_FUSED_SCORES_MAX experiment) instead of a
    GEMM and bb_softmax_fwd/bwd: bf16 operands only, so never in the fp32 verification arm"""
    return not _FP32_ARM and dh == 64 and nk <= FUSED_SCORES_MAX_KEYS


def attn_scores_fwd(q, ldq, k, ldk, B, H, nq, nk, dh, ldp, kmask, bias, drop):
    """fused P = softmax(Q K^T / sqrt(dh) + kmask + bias) (+ dropped copy): -> (P, Pd) bf16 (B,H,nq,ldp)."""
    lib = _lib.load()
    _req(q, BF16, "q")
    _req(k, BF16, "k")
    a = _lib.AttnScoresArgs()
    a.A, a.lda, a.a_s1, a.a_s2 = q.data_ptr(), ldq, dh, nq * ldq
    a.Bm, a.ldb, a.b_s1, a.b_s2 = k.data_ptr(), ldk, dh, nk * ldk
    a.B, a.H, a.nq, a.nk, a.ldp, a.mode = B, H, nq, nk, ldp, 0
    a.alpha = 1.0 / (dh ** 0.5)
    a.kmask, a.bias = _p(kmask), _p(bias)
    a.seed, a.thresh, a.scale = drop
    P = torch.empty(B, H, nq, ldp, dtype=BF16, device=q.device)
    Pd = torch.empty(B, H, nq, ldp, dtype=BF16, device=q.device) if drop[1] else None
    a.P, a.Pd = P.data_ptr(), _p(Pd)
    _lib.check(lib.bb_attn_scores(C.byref(a), _stream()), "bb_attn_scores")
    return P, (Pd if Pd is not None else P)


def attn_scores_bwd(dctx, ldd, v, ldv, P, B, H, nq, nk, dh, ldp, drop, dbias=None):
    """fused dS = P o (g - sum P g) / sqrt(dh), g = dropout-mask(dctx V^T): -> dS bf16 (B,H,nq,ldp)."""
    lib = _lib.load()
    for t, n in ((dctx, "dctx"), (v, "v"), (P, "P")):
        _req(t, BF16, n)
    if dbias is not None:
        _nondeterministic("the fused-scores (BB_FUSED_SCORES_MAX) graph-bias gradient")
    a = _lib.AttnScoresArgs()
    a.A, a.lda, a.a_s1, a.a_s2 = dctx.data_ptr(), ldd, dh, nq * ldd
    a.Bm, a.ldb, a.b_s1, a.b_s2 = v.data_ptr(), ldv, dh, nk * ldv
    a.B, a.H, a.nq, a.nk, a.ldp, a.mode = B, H, nq, nk, ldp, 1
    a.alpha, a.out_scale = 1.0, 1.0 / (dh ** 0.5)
    a.seed, a.thresh, a.scale = drop
    dS = torch.empty(B, H, nq, ldp, dtype=BF16, device=dctx.device)
    a.Pin, a.dS, a.dbias = P.data_ptr(), dS.data_ptr(), _p(dbias)
    _lib.check(lib.bb_attn_scores(C.byref(a), _stream()), "bb_attn_scores")
    return dS


NO_DROP = (0, 0, 1.0)
FLASH = __import__('os').environ.get('BB_FLASH', '1') != '0'     # fused attention core (csrc/attn_flash.cu), head dim 64


def _flash_args(q, k, v, o, lse, B, H, nq, nk, ldq, ldk, ldv, ldo, kmask, bias, drop):
    a = _lib.FlashArgs()
    a.q, a.k, a.v, a.o = q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr()
    a.q_bs, a.k_bs, a.v_bs, a.o_bs = nq * ldq, nk * ldk, nk * ldv, nq * ldo
    a.ldq, a.ldk, a.ldv, a.ldo = ldq, ldk, ldv, ldo
    a.B, a.H, a.nq, a.nk, a.dh = B, H, nq, nk, 64
    a.alpha = 0.125
    a.kmask, a.bias, a.lse = _p(kmask), _p(bias), lse.data_ptr()
    a.seed, a.thresh, a.scale = drop
    return a


def set_attn_tc(mode: int) -> int:
    """0: mma.sync attention kernels only; 1: wgmma kernels for nk >= 64 (default); 2: wgmma wherever supported."""
    return int(_lib.load().bb_set_attn_tc(int(mode)))


def flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask=None, bias=None, drop=NO_DROP):
    """fused attention core (bb_flash_fwd): q/k/v are bf16 tensors whose data_ptr is element (0,0,0,0) of the
    (B, rows, H, 64) view with row stride ld*; -> (o (B,nq,H*64) bf16, lse (B,H,nq) f32)."""
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _req(t, act_dtype(), n)
    o = torch.empty(B, nq, H * 64, dtype=act_dtype(), device=q.device)
    lse = torch.empty(B, H, nq, dtype=torch.float32, device=q.device)
    a = _flash_args(q, k, v, o, lse, B, H, nq, nk, ldq, ldk, ldv, H * 64, kmask, bias, drop)
    _lib.check(_lib.load().bb_flash_fwd(C.byref(a), _stream()), "bb_flash_fwd")
    return o, lse


def flash_bwd(q, k, v, o, lse, dout, B, H, nq, nk, ldq, ldk, ldv, kmask=None, bias=None, drop=NO_DROP, dbias=None,
              out=None):
    """backward of flash_fwd: -> (dq (B,nq,H*64), dk (B,nk,H*64), dv (B,nk,H*64)) bf16; dbias (B,nq,nk) f32 += .
    out = (dq, lddq, dk, lddk, dv, lddv) writes into existing views with the geometry of q / k / v instead."""
    Hd = H * 64
    a = _flash_args(q, k, v, o, lse, B, H, nq, nk, ldq, ldk, ldv, Hd, kmask, bias, drop)
    if out is None:
        dq = torch.empty(B, nq, Hd, dtype=act_dtype(), device=q.device)
        dk = torch.empty(B, nk, Hd, dtype=act_dtype(), device=q.device)
        dv = torch.empty(B, nk, Hd, dtype=act_dtype(), device=q.device)
        lddq = lddk = lddv = Hd
    else:
        dq, lddq, dk, lddk, dv, lddv = out
    dsum = torch.empty(B, H, nq, dtype=torch.float32, device=q.device)
    a.dout, a.do_bs, a.lddo, a.dsum = dout.data_ptr(), nq * Hd, Hd, dsum.data_ptr()
    a.dq, a.dk, a.dv = dq.data_ptr(), dk.data_ptr(), dv.data_ptr()
    a.dq_bs, a.dk_bs, a.dv_bs, a.lddq, a.lddk, a.lddv = nq * lddq, nk * lddk, nk * lddv, lddq, lddk, lddv
    a.dbias = _p(dbias)
    _lib.check(_lib.load().bb_flash_bwd(C.byref(a), _stream()), "bb_flash_bwd")
    return dq, dk, dv


# ---------------------------------------------------------------------------------------------- BEV
def bev_lift_index(depths, T_c2w, S_w2c, T_w2c, map_dim, map_res, depth_scale=10.0, fx=7.0, fy=7.0, cx=7.0, cy=7.0,
                   y_clip=0.5, want_pc=False):
    lib = _lib.load()
    for t, n in ((depths, "depths"), (T_c2w, "T_c2w"), (S_w2c, "S_w2c"), (T_w2c, "T_w2c")):
        _req(t, torch.float32, n)
    B, V = depths.shape[0], depths.shape[1]
    Hf, Wf = depths.shape[-2], depths.shape[-1]
    P = V * Hf * Wf
    idx = torch.empty(B, P, dtype=torch.int32, device=depths.device)
    pc = torch.empty(B, P, 3, dtype=torch.float32, device=depths.device) if want_pc else None
    _lib.check(lib.bb_bev_lift_index(depths.contiguous().data_ptr(), T_c2w.contiguous().data_ptr(),
                                     S_w2c.contiguous().data_ptr(), T_w2c.contiguous().data_ptr(), B, V, Hf, Wf,
                                     depth_scale, fx, fy, cx, cy, map_dim, map_res, y_clip, idx.data_ptr(), _p(pc),
                                     _stream()), "bb_bev_lift_index")
    return idx, pc


def bev_cell_index(pc, no_depth, map_dim, map_res, y_clip=0.5):
    """ego-frame cloud f32 (B,P,3) + no-depth mask bool (B,P) | None -> int32 cell index (B,P), -1 = dropped."""
    lib = _lib.load()
    _req(pc, torch.float32, "pc")
    pc = pc.contiguous()
    nd = no_depth.contiguous().to(torch.uint8) if no_depth is not None else None
    idx = torch.empty(pc.shape[:-1], dtype=torch.int32, device=pc.device)
    _lib.check(lib.bb_bev_cell_index(pc.data_ptr(), _p(nd), idx.numel(), map_dim, map_res, y_clip, idx.data_ptr(),
                                     _stream()), "bb_bev_cell_index")
    return idx


def bev_scatter_mean(feats, cell_idx, ncell, want_f32=True, want_bf16=True):
    """feats f32 or bf16 (B,P,C) -> (bev_f32 | None, bev_bf16 | None, ob_mask bool (B,ncell), counts int32)."""
    lib = _lib.load()
    if feats.dtype != BF16:
        _req(feats, torch.float32, "feats")
    elif not feats.is_cuda:
        raise RuntimeError("feats must be a CUDA tensor (the hot path has no CPU implementation)")
    fn = lib.bb_bev_scatter_mean_bf16 if feats.dtype == BF16 else lib.bb_bev_scatter_mean_f32
    B, P, Cc = feats.shape
    dev = feats.device
    if _FP32_ARM and want_bf16:          # the "activation copy" of the pooled map is the fp32 map itself
        o32, _, ob, cnt = bev_scatter_mean(feats, cell_idx, ncell, True, False)
        return (o32 if want_f32 else None), o32.clone(), ob, cnt
    o32 = torch.empty(B, ncell, Cc, dtype=torch.float32, device=dev) if want_f32 else None
    o16 = torch.empty(B, ncell, Cc, dtype=BF16, device=dev) if want_bf16 else None
    ob = torch.empty(B, ncell, dtype=torch.uint8, device=dev)
    cnt = torch.empty(B, ncell, dtype=torch.int32, device=dev)
    _lib.check(fn(feats.contiguous().data_ptr(), cell_idx.data_ptr(), B, P, Cc, ncell,
                  _p(o32), _p(o16), ob.data_ptr(), cnt.data_ptr(), _stream()), "bb_bev_scatter_mean")
    return o32, o16, ob.bool(), cnt


def bev_scatter_sem(sems, cell_idx, ncell, num_classes=40):
    """sems: float64 one-hots (B,P,S) as the reference collates them, or uint8 class ids (B,P) (wire format)."""
    lib = _lib.load()
    if sems.dtype == torch.uint8:
        if not sems.is_cuda:
            raise RuntimeError("sems must be a CUDA tensor (the hot path has no CPU implementation)")
        B, P = sems.shape
        out = torch.empty(B, ncell, num_classes, dtype=torch.float64, device=sems.device)
        m = torch.empty(B, ncell, dtype=torch.uint8, device=sems.device)
        _lib.check(lib.bb_bev_scatter_sem_u8(sems.contiguous().data_ptr(), cell_idx.data_ptr(), B, P, num_classes, ncell,
                                             out.data_ptr(), m.data_ptr(), _stream()), "bb_bev_scatter_sem_u8")
        return out, m.bool()
    _req(sems, torch.float64, "sems")
    B, P, S = sems.shape
    out = torch.empty(B, ncell, S, dtype=torch.float64, device=sems.device)
    m = torch.empty(B, ncell, dtype=torch.uint8, device=sems.device)
    _lib.check(lib.bb_bev_scatter_sem_f64(sems.contiguous().data_ptr(), cell_idx.data_ptr(), B, P, S, ncell,
                                          out.data_ptr(), m.data_ptr(), _stream()), "bb_bev_scatter_sem_f64")
    return out, m.bool()


# ---------------------------------------------------------------------------------------------- row kernels
def cast_to_act(src, drop=(0, 0, 1.0), out=None):
    """f32 -> activation dtype (bf16), optional inverted dropout. drop = (seed, thresh, scale)."""
    lib = _lib.load()
    _req(src, torch.float32, "src")
    src = src.contiguous()
    if out is None:
        out = torch.empty(src.shape, dtype=act_dtype(), device=src.device)
    _lib.check(lib.bb_cast_f32_bf16(src.data_ptr(), out.data_ptr(), src.numel(), drop[0], drop[1], drop[2],
                                    _stream()), "bb_cast_f32_bf16")
    return out


def cast_to_f32(src):
    lib = _lib.load()
    _req(src, act_dtype(), "src")
    src = src.contiguous()
    out = torch.empty(src.shape, dtype=torch.float32, device=src.device)
    _lib.check(lib.bb_cast_bf16_f32(src.data_ptr(), out.data_ptr(), src.numel(), _stream()), "bb_cast_bf16_f32")
    return out


def dropout_act(src, drop, out=None):
    lib = _lib.load()
    _req(src, act_dtype(), "src")
    if out is None:
        out = torch.empty_like(src)
    _lib.check(lib.bb_dropout_bf16(src.data_ptr(), out.data_ptr(), src.numel(), drop[0], drop[1], drop[2], _stream()),
               "bb_dropout_bf16")
    return out


def layernorm_fwd(x, residual, gamma, beta, eps, drop_in=(0, 0, 1.0), drop_out=(0, 0, 1.0), want_f32=False):
    """x (rows,H) bf16|f32, residual bf16|None -> (y bf16, y_f32|None, mean, rstd)."""
    lib = _lib.load()
    rows, H = x.shape
    dev = x.device
    y = torch.empty(rows, H, dtype=act_dtype(), device=dev)
    y32 = torch.empty(rows, H, dtype=torch.float32, device=dev) if want_f32 else None
    mean = torch.empty(rows, dtype=torch.float32, device=dev)
    rstd = torch.empty(rows, dtype=torch.float32, device=dev)
    _lib.check(lib.bb_layernorm_fwd(x.data_ptr(), int(x.dtype == torch.float32), _p(residual), gamma.data_ptr(),
                                    beta.data_ptr(), eps, rows, H, drop_in[0], drop_in[1], drop_in[2], drop_out[0],
                                    drop_out[1], drop_out[2], y.data_ptr(), _p(y32), mean.data_ptr(), rstd.data_ptr(),
                                    _stream()), "bb_layernorm_fwd")
    return y, y32, mean, rstd


def layernorm_bwd(dy, x, residual, gamma, mean, rstd, drop_in=(0, 0, 1.0), drop_out=(0, 0, 1.0), want_dx=True,
                  want_dres=False, dx_f32=False, dgamma=None, dbeta=None, dxsum=None):
    """-> (dx | None, dres | None); dgamma/dbeta/dxsum f32 [H] are accumulated into (dxsum = column sums of dx)."""
    lib = _lib.load()
    rows, H = x.shape
    dev = x.device
    dx_f32 = dx_f32 or _FP32_ARM
    dx = torch.empty(rows, H, dtype=torch.float32 if dx_f32 else act_dtype(), device=dev) if want_dx else None
    dres = torch.empty(rows, H, dtype=act_dtype(), device=dev) if want_dres else None
    _lib.check(lib.bb_layernorm_bwd(dy.data_ptr(), int(dy.dtype == torch.float32), x.data_ptr(),
                                    int(x.dtype == torch.float32), _p(residual), gamma.data_ptr(), mean.data_ptr(),
                                    rstd.data_ptr(), rows, H, drop_in[0], drop_in[1], drop_in[2], drop_out[0],
                                    drop_out[1], drop_out[2], _p(dx), int(dx_f32), _p(dres), _p(dgamma), _p(dbeta),
                                    _p(dxsum), _stream()), "bb_layernorm_bwd")
    return dx, dres


def colsum(x, N, out=None):
    """column sums of a bf16 (rows, N) row-major matrix -> f32 [N] (accumulated into `out` if given)."""
    lib = _lib.load()
    _req(x, act_dtype(), "x")
    rows = x.numel() // N
    if out is None:
        out = torch.zeros(N, dtype=torch.float32, device=x.device)
    _lib.check(lib.bb_colsum_bf16(x.data_ptr(), rows, N, N, out.data_ptr(), _stream()), "bb_colsum_bf16")
    return out


def softmax_fwd(scores, kmask, bias, nbatch, H, nq, nk, ld, drop=(0, 0, 1.0)):
    lib = _lib.load()
    dev = scores.device
    probs = torch.empty(nbatch, H, nq, ld, dtype=act_dtype(), device=dev)
    pd = torch.empty(nbatch, H, nq, ld, dtype=act_dtype(), device=dev) if drop[1] else None
    _lib.check(lib.bb_softmax_fwd(scores.data_ptr(), _p(kmask), _p(bias), nbatch, H, nq, nk, ld, drop[0], drop[1],
                                  drop[2], probs.data_ptr(), _p(pd), _stream()), "bb_softmax_fwd")
    return probs, (pd if pd is not None else probs)


def softmax_bwd(probs, dprobs, nbatch, H, nq, nk, ld, drop, out_scale, dbias=None):
    lib = _lib.load()
    ds = torch.empty(nbatch, H, nq, ld, dtype=act_dtype(), device=probs.device)
    _lib.check(lib.bb_softmax_bwd(probs.data_ptr(), dprobs.data_ptr(), nbatch, H, nq, nk, ld, drop[0], drop[1],
                                  drop[2], out_scale, ds.data_ptr(), _p(dbias), _stream()), "bb_softmax_bwd")
    return ds


def embed_sum(ids, word, pos, type0):
    lib = _lib.load()
    Bn, L = ids.shape
    H = word.shape[1]
    out = torch.empty(Bn * L, H, dtype=torch.float32, device=word.device)
    _lib.check(lib.bb_embed_sum(ids.contiguous().data_ptr(), word.data_ptr(), pos.data_ptr(), type0.data_ptr(),
                                Bn * L, L, H, out.data_ptr(), _stream()), "bb_embed_sum")
    return out


def embed_scatter_grad(ids, dz, L, padding_idx, dword, dpos, dtype0):
    lib = _lib.load()
    ntok, H = dz.shape
    if torch.are_deterministic_algorithms_enabled() and dword is not None:
        # the word table by destination here; the library sums the position and type tables in a fixed order
        ids1 = ids.reshape(-1)
        _scatter_sorted(dz, torch.where(ids1 == padding_idx, -1, ids1), H, dword)
        dword = None
    _lib.check(lib.bb_embed_scatter_grad(ids.contiguous().data_ptr(), dz.data_ptr(), ntok, L, H, padding_idx,
                                         _p(dword), _p(dpos), _p(dtype0), _stream()), "bb_embed_scatter_grad")


def gather_rows(src, idx, H):
    """out[r] = src[idx[r]] (bf16 rows of width H); idx int64, negative -> zero row."""
    lib = _lib.load()
    out = torch.empty(idx.numel(), H, dtype=act_dtype(), device=src.device)
    _lib.check(lib.bb_gather_rows_bf16(src.data_ptr(), idx.data_ptr(), idx.numel(), H, out.data_ptr(), _stream()),
               "bb_gather_rows_bf16")
    return out


def scatter_add_rows(src, idx, H, out_f32):
    """out_f32[idx[r]] += src[r]."""
    if torch.are_deterministic_algorithms_enabled():
        return _scatter_sorted(src, idx.reshape(-1), H, out_f32)
    lib = _lib.load()
    _lib.check(lib.bb_scatter_add_rows(src.data_ptr(), idx.data_ptr(), idx.numel(), H, out_f32.data_ptr(), _stream()),
               "bb_scatter_add_rows")
    return out_f32


def _act_bwd(dy, aux, mode):
    lib = _lib.load()
    out = torch.empty_like(dy)
    _lib.check(lib.bb_act_bwd_bf16(dy.data_ptr(), aux.data_ptr(), mode, out.data_ptr(), dy.numel(), _stream()),
               "bb_act_bwd_bf16")
    return out


def gelu_bwd(dy, pre):
    """dy * gelu'(pre) (exact erf form, vilmodel.py:31-37)."""
    return _act_bwd(dy, pre, 1)


def relu_bwd(dy, post):
    """dy * (post > 0)."""
    return _act_bwd(dy, post, 2)


def add_rows(a, b=None, table=None, idx=None, vec=None, c=None, out=None):
    """a (+ b) (+ table[idx]) (+ vec) over activation rows (rows,H) (bb_add_rows).  With a third row operand `c` (and
    `b`): ((a + b) + c) (+ table[idx]) (+ vec) in one bb_add_rows3 launch, where a / b / c / `out` may be row-strided
    views with unit column stride; `out` (only with `c`) is the (rows,H) destination, else a new contiguous tensor."""
    lib = _lib.load()
    rows, H = a.shape
    if c is None:
        if out is not None:
            raise ValueError("add_rows: `out` is taken only with the third row operand `c` (bb_add_rows3)")
        out = torch.empty(rows, H, dtype=act_dtype(), device=a.device)
        _lib.check(lib.bb_add_rows(a.data_ptr(), _p(b), _p(table), _p(idx), _p(vec), rows, H, out.data_ptr(),
                                   _stream()), "bb_add_rows")
        return out
    if out is None:
        out = torch.empty(rows, H, dtype=act_dtype(), device=a.device)
    for t in (a, b, c, out):
        if t is None or t.dim() != 2 or t.shape[0] != rows or t.shape[1] != H or t.stride(1) != 1:
            raise ValueError("add_rows with c: a, b, c and out must be (rows, H) matrices with unit column stride")
    _lib.check(lib.bb_add_rows3(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), c.data_ptr(), c.stride(0),
                                _p(table), _p(idx), _p(vec), rows, H, out.data_ptr(), out.stride(0), _stream()),
               "bb_add_rows3")
    return out


def scale_rows_(x, g, rows, ld):
    lib = _lib.load()
    _lib.check(lib.bb_scale_rows_bf16(x.data_ptr(), g.data_ptr(), rows, ld, _stream()), "bb_scale_rows_bf16")
    return x


def segment_wsum(src, seg_off, idx, w, nseg, H):
    lib = _lib.load()
    out = torch.empty(nseg, H, dtype=act_dtype(), device=src.device)
    _lib.check(lib.bb_segment_wsum(src.data_ptr(), seg_off.data_ptr(), idx.data_ptr(), w.data_ptr(), nseg, H,
                                   out.data_ptr(), _stream()), "bb_segment_wsum")
    return out


def segment_wsum_bwd(dout, seg_off, idx, w, nseg, H, dsrc_f32):
    if torch.are_deterministic_algorithms_enabled():
        # by destination: entry e of segment s adds w[e] * dout[s] to dsrc[idx[e]]
        e = torch.arange(idx.numel(), dtype=seg_off.dtype, device=idx.device)
        seg = torch.searchsorted(seg_off, e, right=True) - 1
        dst = torch.where((seg >= 0) & (seg < nseg), idx.long(), -1)
        return _scatter_sorted(dout, dst, H, dsrc_f32, src_row=seg.clamp(0, max(nseg - 1, 0)), w=w)
    lib = _lib.load()
    _lib.check(lib.bb_segment_wsum_bwd(dout.data_ptr(), seg_off.data_ptr(), idx.data_ptr(), w.data_ptr(), nseg, H,
                                       dsrc_f32.data_ptr(), _stream()), "bb_segment_wsum_bwd")
    return dsrc_f32


def add_act(a, b):
    lib = _lib.load()
    out = torch.empty_like(a)
    _lib.check(lib.bb_add_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), _stream()), "bb_add_bf16")
    return out


def axpy_f32_from_act(x, y):
    """y (f32) += x (bf16)."""
    lib = _lib.load()
    _lib.check(lib.bb_axpy_f32_from_bf16(x.data_ptr(), y.data_ptr(), x.numel(), _stream()), "bb_axpy_f32_from_bf16")
    return y


def softmax_xent(logits, labels, V, ld, want_grad=True):
    """logits f32 (rows, ld) -> (loss f32 (rows,), dlogits bf16 (rows, ld) | None) with dlogits = softmax - onehot."""
    lib = _lib.load()
    rows = logits.shape[0]
    loss = torch.empty(rows, dtype=torch.float32, device=logits.device)
    dl = torch.empty(rows, ld, dtype=act_dtype(), device=logits.device) if want_grad else None
    _lib.check(lib.bb_softmax_xent(logits.data_ptr(), labels.data_ptr(), rows, V, ld, loss.data_ptr(), 0, _p(dl),
                                   _stream()), "bb_softmax_xent")
    return loss, dl


# ---------------------------------------------------------------------------------------------- multi-tensor
class MtTable:
    """Device copy of a `bb_mt_tensor` table (include/bevbert_b200.h): rows = (p, g, m, v, p16, n, step_size, decay);
    chunk offsets are filled in here.  The host rows live in a pinned numpy-backed tensor so that per-step updates
    of the gradient pointers / step sizes are one asynchronous copy."""

    def __init__(self, rows, device):
        import numpy as np
        self.dt = np.dtype([("p", "<u8"), ("g", "<u8"), ("m", "<u8"), ("v", "<u8"), ("p16", "<u8"), ("n", "<i8"),
                            ("step_size", "<f4"), ("decay", "<f4"), ("chunk0", "<i8")])
        assert self.dt.itemsize == C.sizeof(_lib.MtTensor)
        self.nt = len(rows)
        self.host = torch.empty(max(self.nt, 1) * self.dt.itemsize, dtype=torch.uint8)
        if torch.cuda.is_available():
            self.host = self.host.pin_memory()
        self.np = self.host.numpy().view(self.dt)
        chunk = int(_lib.load().bb_mt_chunk_elems())
        c0 = 0
        for i, r in enumerate(rows):
            self.np[i] = tuple(r) + (c0,)
            c0 += (int(r[5]) + chunk - 1) // chunk
        self.chunks = c0
        self.dev = torch.empty(self.host.numel(), dtype=torch.uint8, device=device)
        self.busy = None        # event behind the last enqueued copy that reads the pinned rows
        self.upload()

    def upload(self):
        self.dev.copy_(self.host, non_blocking=True)

    # The pinned rows are read by an ASYNCHRONOUS copy (a plain one in eager steps, a memcpy node of the step graph in
    # replay), while the host rewrites them for the next step that uses this table.  `mark_busy` is called after the
    # work that reads the rows has been enqueued, `wait_idle` before the host touches them again: the host then never
    # runs more than one step of THIS table ahead of the device (with two tasks alternating it waits on a step that
    # finished long ago).  Neither is a graph node; both are skipped while the stream is capturing.
    def mark_busy(self):
        if self.dev.is_cuda and not _capturing():
            self.busy = torch.cuda.Event()
            self.busy.record()

    def wait_idle(self):
        if self.busy is not None and not _capturing():
            self.busy.synchronize()
            self.busy = None


def _capturing():
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


def mt_cast_bf16(table: MtTable):
    _lib.check(_lib.load().bb_mt_cast_bf16(table.dev.data_ptr(), table.nt, table.chunks, _stream()), "bb_mt_cast_bf16")


def mt_sumsq(table: MtTable, out):
    _lib.check(_lib.load().bb_mt_sumsq(table.dev.data_ptr(), table.nt, table.chunks, out.data_ptr(), _stream()),
               "bb_mt_sumsq")
    return out


def adamw_step(table: MtTable, beta1, beta2, eps, sumsq=None, max_norm=0.0, grad_scale=1.0):
    _lib.check(_lib.load().bb_adamw_step(table.dev.data_ptr(), table.nt, table.chunks, beta1, beta2, eps, _p(sumsq),
                                         max_norm, grad_scale, _stream()), "bb_adamw_step")
