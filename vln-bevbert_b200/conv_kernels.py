"""Tensor-level wrappers of the depth-encoder kernels (csrc/conv.cu: bb_conv2d, bb_depth_stem, bb_groupnorm_apply), in
the style of kernels.py: pointers, sizes and torch's current stream in, a raised error on a non-zero status, no
arithmetic and no fallback.  Only the depth tower (model/depth_resnet.py) calls them.

Activations are NHWC tensors (N, H, W, C) in `conv_dtype()`: fp16 in the product path, fp32 in the verification arm
(kernels.set_precision(True)).  A conv or the stem returns its output together with a `Partials`: the GroupNorm partial
statistics of the stored values (include/bevbert_b200.h describes their layout) and the stat tile height."""
from collections import namedtuple

import torch

from . import _lib
from . import kernels as K

CONV_TM = 128       # stat tile of bb_conv2d: one CTA's 128 output pixels
Partials = namedtuple("Partials", "stats tm groups")


def conv_dtype():
    """activation dtype of the depth tower: fp16, or fp32 in the verification arm"""
    return torch.float32 if K._FP32_ARM else torch.float16


def stats_len(n, h, w, c, groups, tm):
    """float4 count of the partials of an (n, h, w, c) map with stat tiles of tm rows"""
    hw = h * w
    seg = (tm + hw - 2) // hw + 1
    cb = min(c // groups, 32)
    return -(-n * hw // tm) * seg * (c // cb)


def _new_stats(n, h, w, c, groups, tm, dev):
    return torch.empty(stats_len(n, h, w, c, groups, tm), 4, dtype=torch.float32, device=dev)


def conv2d(x, w, stride, groups):
    """bb_conv2d: x (N, H, W, Cin), w (Cout, R, R, Cin), both contiguous in conv_dtype() -> (y (N, Ho, Wo, Cout),
    Partials of y for GroupNorm(groups))."""
    dt = conv_dtype()
    for t, name in ((x, "x"), (w, "w")):
        if t.dtype != dt or not t.is_cuda or not t.is_contiguous():
            raise ValueError("%s must be a contiguous CUDA %s tensor, got %s" % (name, dt, t.dtype))
    N, H, W, Cin = x.shape
    Cout, R, S, Cw = w.shape
    if R != S or Cw != Cin:
        raise ValueError("w must be (Cout, R, R, Cin) with Cin = %d, got %s" % (Cin, tuple(w.shape)))
    pad = (R - 1) // 2
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    y = torch.empty(N, Ho, Wo, Cout, dtype=dt, device=x.device)
    st = _new_stats(N, Ho, Wo, Cout, groups, CONV_TM, x.device)
    _lib.check(_lib.load().bb_conv2d(x.data_ptr(), w.data_ptr(), N, H, W, Cin, Cout, R, stride, groups, y.data_ptr(),
                                     st.data_ptr(), K._stream()), "bb_conv2d")
    return y, Partials(st, CONV_TM, groups)


def depth_stem(depth, w, groups):
    """bb_depth_stem: depth f32 (N, Hd, Wd) or (N, Hd, Wd, 1), any strides; w f32 (32, 1, 7, 7) contiguous ->
    (y (N, Ho, Wo, 32) in conv_dtype(), Partials) of conv7x7/2(avg_pool2d(depth, 2))."""
    if depth.dtype != torch.float32 or not depth.is_cuda:
        raise ValueError("depth must be a CUDA float32 tensor, got %s" % depth.dtype)
    if depth.dim() == 4:
        if depth.shape[3] != 1:
            raise ValueError("depth must have one channel, got %s" % (tuple(depth.shape),))
        depth = depth[..., 0]
    if w.dtype != torch.float32 or tuple(w.shape) != (32, 1, 7, 7) or not w.is_contiguous():
        raise ValueError("the stem weight must be a contiguous float32 (32, 1, 7, 7) tensor")
    N, Hd, Wd = depth.shape
    Hp, Wp = Hd // 2, Wd // 2
    Ho, Wo = (Hp - 1) // 2 + 1, (Wp - 1) // 2 + 1
    y = torch.empty(N, Ho, Wo, 32, dtype=conv_dtype(), device=depth.device)
    st = _new_stats(N, Ho, Wo, 32, groups, Wo, depth.device)
    _lib.check(_lib.load().bb_depth_stem(depth.data_ptr(), N, Hd, Wd, *depth.stride(), w.data_ptr(), groups,
                                         y.data_ptr(), st.data_ptr(), K._stream()), "bb_depth_stem")
    return y, Partials(st, Wo, groups)


GN_RELU, GN_ADD_RELU, GN_ADD_NORM_RELU, GN_RELU_MAXPOOL = 0, 1, 2, 3


def groupnorm_apply(x, p, gamma, beta, eps, mode=GN_RELU, identity=None, x2=None, p2=None, gamma2=None, beta2=None,
                    out_f32=False):
    """bb_groupnorm_apply on x (N, H, W, C) with its Partials p and f32 gamma / beta: relu(GN(x)) (mode 0),
    relu(GN(x) + identity) (1), relu(GN(x) + GN2(x2)) (2), maxpool3x3/2(relu(GN(x))) (3).  -> a new NHWC tensor in
    conv_dtype(), or with out_f32 (mode 0) a new f32 NCHW tensor (N, C, H, W)."""
    N, H, W, C = x.shape
    if mode == GN_RELU_MAXPOOL:
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    else:
        Ho, Wo = H, W
    for t, name in ((x, "x"), (identity, "identity"), (x2, "x2")):
        if t is not None and (t.dtype != conv_dtype() or not t.is_contiguous() or tuple(t.shape) != tuple(x.shape)):
            raise ValueError("%s must be a contiguous %s tensor of x's shape" % (name, conv_dtype()))
    for t in (gamma, beta, gamma2, beta2):
        if t is not None and (t.dtype != torch.float32 or t.numel() != C):
            raise ValueError("gamma / beta must be float32 vectors of %d channels" % C)
    if out_f32:
        out = torch.empty(N, C, Ho, Wo, dtype=torch.float32, device=x.device)
    else:
        out = torch.empty(N, Ho, Wo, C, dtype=conv_dtype(), device=x.device)
    p2s, tm2 = (p2.stats.data_ptr(), p2.tm) if p2 is not None else (0, 0)
    _lib.check(_lib.load().bb_groupnorm_apply(
        x.data_ptr(), p.stats.data_ptr(), p.tm, gamma.data_ptr(), beta.data_ptr(), K._p(x2), p2s, tm2, K._p(gamma2),
        K._p(beta2), K._p(identity), N, H, W, C, p.groups, float(eps), mode, int(out_f32), out.data_ptr(),
        K._stream()), "bb_groupnorm_apply")
    return out
