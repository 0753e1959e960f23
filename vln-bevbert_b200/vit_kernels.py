"""Tensor-level wrappers of the ViT image-tower input kernels (csrc/vit.cu: bb_image_patches, bb_vit_tokens), in
the style of kernels.py: pointers, sizes and torch's current stream in, a raised error on a non-zero status, no
arithmetic and no fallback.  They live in their own module because only the CLIP tower (model/clip_visual.py) calls
them, and kernels.py is the surface tests/emu_kernels.py restates for the CPU host-logic tests."""
import ctypes as C

import torch

from . import _lib
from . import kernels as K


def image_patches(img, patch, mean, std, out=None):
    """Patch rows of a ViT's stride-`patch` conv1 (bb_image_patches) with ConvertImageDtype(float) + Normalize(mean,
    std) fused: img (N, H, W, 3) uint8 or f32, any strides (an NCHW tensor passes as img.permute(0, 2, 3, 1)) ->
    (N * (H/P) * (W/P), 3 * P * P) in the activation dtype, columns in conv1.weight's flatten order."""
    if img.dtype not in (torch.uint8, torch.float32):
        raise TypeError("img must be uint8 or float32, got %s" % img.dtype)
    if not img.is_cuda:
        raise RuntimeError("img must be a CUDA tensor (the hot path has no CPU implementation)")
    if img.dim() != 4 or img.shape[3] != 3:
        raise ValueError("img must be (N, H, W, 3), got %s" % (tuple(img.shape),))
    N, H, W, _ = img.shape
    if N == 0:
        raise ValueError("img holds no image")
    rows = N * (H // patch) * (W // patch)
    if out is None:
        out = torch.empty(rows, 3 * patch * patch, dtype=K.act_dtype(), device=img.device)
    m, s = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
    _lib.check(_lib.load().bb_image_patches(img.data_ptr(), int(img.dtype == torch.uint8), N, H, W, *img.stride(), patch,
                                            m, s, out.data_ptr(), K._stream()), "bb_image_patches")
    return out


def vit_tokens(patch_out, cls, pos, gamma, beta, eps, N):
    """First-block input of a ViT (bb_vit_tokens): patch_out f32 (N*(T-1), H), cls f32 (H), pos f32 (T, H) ->
    LN([cls; patch rows] + pos) as (N*T, H) in the activation dtype."""
    for t, n in ((patch_out, "patch_out"), (cls, "cls"), (pos, "pos"), (gamma, "gamma"), (beta, "beta")):
        K._req(t, torch.float32, n)
    T, H = pos.shape
    if patch_out.numel() != N * (T - 1) * H or not patch_out.is_contiguous():
        raise ValueError("patch_out must be a contiguous (N*(T-1), H) = (%d, %d) tensor" % (N * (T - 1), H))
    out = torch.empty(N * T, H, dtype=K.act_dtype(), device=pos.device)
    _lib.check(_lib.load().bb_vit_tokens(patch_out.data_ptr(), cls.data_ptr(), pos.data_ptr(), gamma.data_ptr(),
                                         beta.data_ptr(), eps, N, T, H, out.data_ptr(), K._stream()), "bb_vit_tokens")
    return out
