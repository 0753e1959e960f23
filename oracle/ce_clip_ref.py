"""TEST INFRASTRUCTURE ONLY -- oracle for the VLN-CE policy's CLIP ViT image tower (model/clip_visual.py).

A functional restatement of CLIPEncoderB16.forward (bevbert_ce/vlnce_baselines/models/encoders/resnet_encoders.py:
305-314) and VisionTransformer.forward (encoders/clip/model.py:220-237) over a flat state_dict with the tower's keys
(`conv1.weight`, `transformer.resblocks.<i>.attn.in_proj_weight`, ...; a `visual.` prefix is stripped), in two arms:

  * `forward(sd, rgb, dtype)`: every operation in `dtype` (fp32 or fp64) on the device of the tensors;
  * `forward_fp16(sd, rgb)`: the reference's dtype flow on the GPU -- weights as clip's convert_weights leaves them
    (conv1, Linear / in_proj weights and biases, proj in fp16; embeddings and LayerNorms fp32), the image cast to fp16
    before conv1, LayerNorm in fp32 and cast back, seq-first nn.MultiheadAttention and QuickGELU x * sigmoid(1.702 x)
    on fp16 activations.  scripts/bench_ce_clip.py times it as the reference path.

`preprocess(rgb)` is ConvertImageDtype(float) + Normalize as torchvision computes them (`image.to(float32) / 255.0`
for uint8, then `.sub_(mean).div_(std)` with (3, 1, 1) tensors), on the device of `rgb`.  Pinned against the
unmodified reference and torchvision by tests/golden/small_ce_clip.pt (tests/golden/make_ce_clip_golden.py).  The
product never imports it.
"""
import torch
import torch.nn.functional as F
from torch import nn

MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)
EPS = 1e-5


def strip(sd):
    return {(k[len("visual."):] if k.startswith("visual.") else k): v for k, v in sd.items()}


def layers(sd):
    return len([k for k in sd if k.endswith(".attn.in_proj_weight")])


def preprocess(rgb, mean=MEAN, std=STD):
    """observations["rgb"] (N, H, W, 3) -> normalized fp32 (N, 3, H, W), torchvision's operations"""
    x = rgb.permute(0, 3, 1, 2)
    if not x.is_floating_point():
        x = x.to(torch.float32) / 255.0
    elif x.dtype != torch.float32:
        x = x.to(torch.float32)
    m = torch.as_tensor(mean, dtype=torch.float32, device=x.device).view(-1, 1, 1)
    s = torch.as_tensor(std, dtype=torch.float32, device=x.device).view(-1, 1, 1)
    return x.clone().sub_(m).div_(s)


def _ln(x, sd, k):
    return F.layer_norm(x, x.shape[-1:], sd[k + ".weight"].to(x.dtype), sd[k + ".bias"].to(x.dtype), EPS)


def tower(sd, x, dtype=torch.float32):
    """VisionTransformer.forward on normalized images x (N, 3, R, R) -> (x_proj, x_patch), all in `dtype`"""
    sd = {k: v.to(dtype) for k, v in strip(sd).items()}
    x = x.to(dtype)
    w = sd["conv1.weight"]
    P, D = w.shape[-1], w.shape[0]
    x = F.conv2d(x, w, stride=P).flatten(2).transpose(1, 2)                       # (N, G, D)
    N = x.shape[0]
    x = torch.cat([sd["class_embedding"].expand(N, 1, D), x], 1) + sd["positional_embedding"]
    x = _ln(x, sd, "ln_pre")
    T = x.shape[1]
    H = D // 64
    for i in range(layers(sd)):
        b = "transformer.resblocks.%d." % i
        h = _ln(x, sd, b + "ln_1")
        qkv = h @ sd[b + "attn.in_proj_weight"].t() + sd[b + "attn.in_proj_bias"]
        q, k, v = (t.view(N, T, H, 64).transpose(1, 2) for t in qkv.split(D, -1))
        a = torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1) @ v
        a = a.transpose(1, 2).reshape(N, T, D)
        x = x + a @ sd[b + "attn.out_proj.weight"].t() + sd[b + "attn.out_proj.bias"]
        h = _ln(x, sd, b + "ln_2")
        f = h @ sd[b + "mlp.c_fc.weight"].t() + sd[b + "mlp.c_fc.bias"]
        f = f * torch.sigmoid(1.702 * f)
        x = x + f @ sd[b + "mlp.c_proj.weight"].t() + sd[b + "mlp.c_proj.bias"]
    return _ln(x[:, 0], sd, "ln_post") @ sd["proj"], x[:, 1:]


def forward(sd, rgb, dtype=torch.float32, mean=MEAN, std=STD):
    """CLIPEncoderB16.forward: observations["rgb"] -> (rgb_vector, rgb_grid) in `dtype`"""
    return tower(sd, preprocess(rgb, mean, std), dtype)


# ------------------------------------------------------------------------------------------------ fp16 arm
FP16_KEYS = ("conv1.weight", "proj", ".attn.in_proj_weight", ".attn.in_proj_bias", ".attn.out_proj.weight",
             ".attn.out_proj.bias", ".mlp.c_fc.weight", ".mlp.c_fc.bias", ".mlp.c_proj.weight", ".mlp.c_proj.bias")


def converted(sd):
    """the state_dict in the dtypes clip.load leaves it on the GPU (clip/model.py:372-393)"""
    return {k: v.to(torch.float16 if k.endswith(FP16_KEYS) else torch.float32) for k, v in strip(sd).items()}


class _LN(nn.LayerNorm):
    def forward(self, x):
        return super().forward(x.float()).to(x.dtype)


class _QuickGELU(nn.Module):
    def forward(self, x):
        return x * torch.sigmoid(1.702 * x)


class _Block(nn.Module):
    def __init__(self, d, h):
        super().__init__()
        self.attn = nn.MultiheadAttention(d, h)
        self.ln_1 = _LN(d)
        self.mlp = nn.Sequential()
        self.mlp.add_module("c_fc", nn.Linear(d, 4 * d))
        self.mlp.add_module("gelu", _QuickGELU())
        self.mlp.add_module("c_proj", nn.Linear(4 * d, d))
        self.ln_2 = _LN(d)

    def forward(self, x):                       # x (L, N, D), seq-first
        h = self.ln_1(x)
        x = x + self.attn(h, h, h, need_weights=False)[0]
        return x + self.mlp(self.ln_2(x))


class Fp16Tower(nn.Module):
    """The reference's GPU dtype flow, built from the torch modules it uses, loaded from a state_dict."""

    def __init__(self, sd):
        super().__init__()
        sd = converted(sd)
        D, P = sd["conv1.weight"].shape[0], sd["conv1.weight"].shape[-1]
        self.conv1 = nn.Conv2d(3, D, P, P, bias=False)
        self.class_embedding = nn.Parameter(torch.empty(D))
        self.positional_embedding = nn.Parameter(torch.empty_like(sd["positional_embedding"]))
        self.ln_pre = _LN(D)
        self.transformer = nn.Module()
        self.transformer.resblocks = nn.Sequential(*[_Block(D, D // 64) for _ in range(layers(sd))])
        self.ln_post = _LN(D)
        self.proj = nn.Parameter(torch.empty_like(sd["proj"]))
        for k, v in sd.items():                 # dtypes first, then values
            mod, _, name = k.rpartition(".")
            owner = self.get_submodule(mod) if mod else self
            getattr(owner, name).data = v.clone()
        self.requires_grad_(False).eval()

    def forward(self, x):
        x = self.conv1(x.to(self.conv1.weight.dtype)).flatten(2).transpose(1, 2)
        N, _, D = x.shape
        x = torch.cat([self.class_embedding.to(x.dtype).expand(N, 1, D), x], 1) + self.positional_embedding.to(x.dtype)
        x = self.ln_pre(x).permute(1, 0, 2)
        x = self.transformer.resblocks(x).permute(1, 0, 2)
        return self.ln_post(x[:, 0]) @ self.proj, x[:, 1:]


def forward_fp16(model, rgb, mean=MEAN, std=STD):
    """CLIPEncoderB16.forward through an Fp16Tower on the GPU -> (rgb_vector, rgb_grid) as fp32"""
    with torch.no_grad():
        v, g = model(preprocess(rgb, mean, std))
    return v.float(), g.float()
