"""OpenAI CLIP's ViT image tower on the H100 kernels, forward only: the VLN-CE policy's RGB encoder (`CLIPEncoderB16`,
bevbert_ce/vlnce_baselines/models/encoders/resnet_encoders.py:280-314, over clip/model.py:206-237).

`VisionTransformer` has the reference class's constructor, parameter names and shapes; `ClipTower` runs the same
forward over the parameters of any module with that layout, such as the reference's own `rgb_encoder.model.visual`
(graphs.install_ce_rgb_encoder).  Per call:
    patch rows of the images (bb_image_patches: ConvertImageDtype(float) + Normalize fused) -> GEMM with conv1 (fp32)
    -> class token + positional embedding + ln_pre (bb_vit_tokens) -> `layers` pre-norm blocks (blocks.PanoLayerImpl
    with QuickGELU: LN, packed QKV GEMM, wgmma attention over all tokens, out-projection GEMM + residual, LN, FFN-up
    GEMM with the QuickGELU epilogue, FFN-down GEMM + residual) -> fp32 copy of the token rows; ln_post of the class
    rows, then @ proj as a GEMM with an MN-major B operand.
Weights may be fp16 (what clip.load leaves for conv1, the Linear / in_proj weights and biases and proj) or fp32: the
bf16 GEMM operands and fp32 bias copies are WeightCache shadows, re-made when a parameter's version or storage changes
(load_state_dict between calls).  The tower is frozen in the reference; a call with grad enabled while a tower
parameter requires grad raises, because nothing here runs backward.  Autocast is disabled inside the call, so the
trainer's autocast() changes no bit of the outputs.
"""
from collections import OrderedDict

import torch
from torch import nn

from .. import blocks
from .. import kernels as K
from .. import vit_kernels as VK

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)     # resnet_encoders.py:300-303
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
_IDENTITY = ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0))
LN_EPS = 1e-5


def check_geometry(input_resolution, patch_size, width, heads, output_dim):
    """What the kernels need of the tower's shape; raises ValueError otherwise."""
    if heads <= 0 or width != 64 * heads:
        raise ValueError("the attention kernels need a head dim of 64: width %d, heads %d" % (width, heads))
    if width % 8 or width > 1024:
        raise ValueError("width must be a multiple of 8 and at most 1024, got %d" % width)
    if input_resolution % patch_size:
        raise ValueError("input_resolution %d is not divisible by patch_size %d" % (input_resolution, patch_size))
    if (3 * patch_size * patch_size) % 8 or output_dim % 8:
        raise ValueError("3 * patch_size^2 and output_dim must be multiples of 8 (patch %d, output_dim %d)" % (
            patch_size, output_dim))


class ClipTower:
    """The kernels' forward over `visual`, a module laid out as clip/model.py's VisionTransformer (conv1,
    class_embedding, positional_embedding, ln_pre, transformer.resblocks[i].{attn, ln_1, mlp.c_fc, mlp.c_proj, ln_2},
    ln_post, proj).  `owner` (default `visual`) is the module whose train / eval mode the caller goes by."""

    def __init__(self, visual, mean=CLIP_MEAN, std=CLIP_STD, owner=None):
        self.v, self.owner = visual, owner if owner is not None else visual
        self.mean, self.std = tuple(float(m) for m in mean), tuple(float(s) for s in std)
        w = visual.conv1.weight
        self.width, self.patch = w.shape[0], w.shape[-1]
        self.res = int(visual.input_resolution)
        self.heads = visual.transformer.resblocks[0].attn.num_heads
        self.out_dim = visual.proj.shape[1]
        check_geometry(self.res, self.patch, self.width, self.heads, self.out_dim)
        self.tokens = (self.res // self.patch) ** 2 + 1
        self.rt = blocks.Runtime()
        self.layer = blocks.PanoLayerImpl(self.rt, self.heads, act=K.ACT_QGELU)
        self._cls_idx = {}
        self._sig = None

    @property
    def training(self):
        return self.owner.training

    def parameters(self):
        return self.v.parameters()

    def changed(self):
        """True when a parameter's storage or version moved since the previous call of this method."""
        sig = tuple((p.data_ptr(), p._version) for p in self.v.parameters())
        moved, self._sig = sig != self._sig, sig
        return moved

    def check_grad(self):
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.v.parameters()):
            raise RuntimeError("the CLIP image tower runs forward only: call it under torch.no_grad() or freeze its "
                               "parameters (requires_grad_(False)), as CLIPEncoderB16 does")

    def encode_rgb(self, rgb):
        """CLIPEncoderB16.forward on observations["rgb"] (N, H, W, 3), uint8 or float32 -> (rgb_vector (N, output_dim),
        rgb_grid (N, grid^2, width)), both fresh fp32 tensors."""
        return self.encode(rgb, self.mean, self.std)

    def encode(self, img, mean, std):
        """img (N, H, W, 3) (any strides) -> (x_proj, x_patch) in fp32"""
        self.check_grad()
        if img.dim() != 4 or img.shape[1] != self.res or img.shape[2] != self.res or img.shape[3] != 3:
            raise ValueError("expected images of shape (N, %d, %d, 3), got %s" % (self.res, self.res, tuple(img.shape)))
        with torch.autocast("cuda", enabled=False), torch.no_grad():
            return self._encode(img, mean, std)

    def _encode(self, img, mean, std):
        v, wc, D, P, T = self.v, self.rt.wc, self.width, self.patch, self.tokens
        f32 = wc.f32
        N = img.shape[0]
        kp = 3 * P * P
        patches = VK.image_patches(img, P, mean, std)
        pe = torch.empty(N * (T - 1), D, dtype=torch.float32, device=img.device)
        K.gemm(patches, wc.get(v.conv1.weight.view(D, kp)), pe, N * (T - 1), D, kp, lda=kp, ldb=kp, ldd=D)
        x = VK.vit_tokens(pe, f32(v.class_embedding), f32(v.positional_embedding), f32(v.ln_pre.weight),
                         f32(v.ln_pre.bias), LN_EPS, N).view(N, T, D)
        for b in v.transformer.resblocks:
            p = (b.attn.in_proj_weight, f32(b.attn.in_proj_bias), b.attn.out_proj.weight, f32(b.attn.out_proj.bias),
                 b.mlp.c_fc.weight, f32(b.mlp.c_fc.bias), b.mlp.c_proj.weight, f32(b.mlp.c_proj.bias),
                 f32(b.ln_1.weight), f32(b.ln_1.bias), f32(b.ln_2.weight), f32(b.ln_2.bias))
            x = self.layer.fwd({}, (x, None), p)
        y = x.reshape(N * T, D)
        grid = K.cast_to_f32(y).view(N, T, D)[:, 1:]
        key = (N, img.device)
        if key not in self._cls_idx:
            self._cls_idx[key] = torch.arange(N, dtype=torch.int64, device=img.device) * T
        h, _, _, _ = K.layernorm_fwd(K.gather_rows(y, self._cls_idx[key], D), None, f32(v.ln_post.weight),
                                     f32(v.ln_post.bias), LN_EPS)
        out = torch.empty(N, self.out_dim, dtype=torch.float32, device=img.device)
        K.gemm(h, wc.get(v.proj), out, N, self.out_dim, D, lda=D, ldb=self.out_dim, ldd=self.out_dim, b_mn=True)
        return out, grid


class _Mlp(nn.Module):
    def __init__(self, width):
        super().__init__()
        self.c_fc = nn.Linear(width, 4 * width)
        self.c_proj = nn.Linear(4 * width, width)


class _Block(nn.Module):
    """parameters of clip/model.py's ResidualAttentionBlock, under its names"""

    def __init__(self, width, heads):
        super().__init__()
        self.attn = nn.MultiheadAttention(width, heads)
        self.ln_1 = nn.LayerNorm(width)
        self.mlp = _Mlp(width)
        self.ln_2 = nn.LayerNorm(width)


class _Transformer(nn.Module):
    def __init__(self, width, layers, heads):
        super().__init__()
        self.width, self.layers = width, layers
        self.resblocks = nn.Sequential(OrderedDict((str(i), _Block(width, heads)) for i in range(layers)))


class VisionTransformer(nn.Module):
    """clip/model.py's VisionTransformer on the kernels: same constructor, state_dict keys and shapes.  `forward(x)`
    takes normalized images (N, 3, R, R) in fp32 and returns (x_proj (N, output_dim), x_patch (N, grid^2, width)) in
    fp32; `encode_rgb(rgb)` is CLIPEncoderB16.forward on observations["rgb"] (N, R, R, 3), preprocessing included."""

    def __init__(self, input_resolution, patch_size, width, layers, heads, output_dim):
        super().__init__()
        check_geometry(input_resolution, patch_size, width, heads, output_dim)
        self.input_resolution = input_resolution
        self.output_dim = output_dim
        self.conv1 = nn.Conv2d(3, width, kernel_size=patch_size, stride=patch_size, bias=False)
        scale = width ** -0.5
        self.class_embedding = nn.Parameter(scale * torch.randn(width))
        self.positional_embedding = nn.Parameter(scale * torch.randn((input_resolution // patch_size) ** 2 + 1, width))
        self.ln_pre = nn.LayerNorm(width)
        self.transformer = _Transformer(width, layers, heads)
        self.ln_post = nn.LayerNorm(width)
        self.proj = nn.Parameter(scale * torch.randn(width, output_dim))
        object.__setattr__(self, "_tower", None)

    @property
    def tower(self):
        if self._tower is None:
            object.__setattr__(self, "_tower", ClipTower(self))
        return self._tower

    def forward(self, x):
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("expected normalized fp32 images (N, 3, R, R), got %s %s" % (x.dtype, tuple(x.shape)))
        return self.tower.encode(x.permute(0, 2, 3, 1), *_IDENTITY)

    def encode_rgb(self, rgb):
        return self.tower.encode_rgb(rgb)
