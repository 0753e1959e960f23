"""Functional restatement of the VLN-CE policy's depth encoder (resnet_encoders.py VlnResnetDepthEncoder.visual_encoder:
habitat-lab v0.1.7's ResNetEncoder over a GroupNorm ResNet-50 with 32 base planes and GroupNorm(16); compression to
128 channels with GroupNorm(1)) over a flat state_dict, with F.conv2d, F.group_norm, F.max_pool2d and F.avg_pool2d.

Two arms:
  * `forward(sd, depth, dtype)`: everything in `dtype` (fp64 or fp32), the yardstick;
  * `forward_fp16(sd, depth)`: CUDA autocast's dtype flow (torch.autocast("cuda", torch.float16), as the trainer runs
    the policy): each convolution takes fp16 operands and returns fp16 (an fp32 conv of fp16-rounded operands,
    rounded to fp16: cuDNN accumulates in fp32); group_norm is on autocast's fp32 list, so it returns fp32, and the
    ReLUs, the residual adds and the max-pool stay in fp32; avg_pool2d of the fp32 depth is fp32.
The depth arrives as observations["depth"], (N, H, W, 1) fp32.  The output is (N, 128, h, w) fp32 (fp64 in the fp64
arm)."""
import torch
import torch.nn.functional as F

LAYERS = (3, 4, 6, 3)
NGROUPS, EPS = 16, 1e-5


def _conv_exact(x, w, stride, pad):
    return F.conv2d(x, w.to(x.dtype), stride=stride, padding=pad)


def _conv_fp16(x, w, stride, pad):
    return F.conv2d(x.half().float(), w.half().float(), stride=stride, padding=pad).half()


def _gn(x, sd, k, groups, dtype):
    return F.group_norm(x.to(dtype), groups, sd[k + ".weight"].to(dtype), sd[k + ".bias"].to(dtype), EPS)


def _forward(sd, depth, conv, dtype):
    x = F.avg_pool2d(depth.to(dtype).permute(0, 3, 1, 2), 2)
    x = conv(x, sd["backbone.conv1.0.weight"], 2, 3)
    x = F.relu(_gn(x, sd, "backbone.conv1.1", NGROUPS, dtype))
    x = F.max_pool2d(x, 3, 2, 1)
    for li, n in enumerate(LAYERS):
        for bi in range(n):
            b = "backbone.layer%d.%d." % (li + 1, bi)
            stride = 2 if (bi == 0 and li > 0) else 1
            h = F.relu(_gn(conv(x, sd[b + "convs.0.weight"], 1, 0), sd, b + "convs.1", NGROUPS, dtype))
            h = F.relu(_gn(conv(h, sd[b + "convs.3.weight"], stride, 1), sd, b + "convs.4", NGROUPS, dtype))
            h = _gn(conv(h, sd[b + "convs.6.weight"], 1, 0), sd, b + "convs.7", NGROUPS, dtype)
            if bi == 0:
                idn = _gn(conv(x, sd[b + "downsample.0.weight"], stride, 0), sd, b + "downsample.1", NGROUPS, dtype)
            else:
                idn = x
            x = F.relu(h + idn)
    x = conv(x, sd["compression.0.weight"], 1, 1)
    return F.relu(_gn(x, sd, "compression.1", 1, dtype))


def forward(sd, depth, dtype=torch.float64):
    """the encoder in `dtype` throughout"""
    return _forward(sd, depth, _conv_exact, dtype)


def forward_fp16(sd, depth):
    """the encoder under CUDA fp16 autocast's dtype flow -> fp32"""
    return _forward(sd, depth, _conv_fp16, torch.float32)


def visual_keys(sd):
    """key -> shape, in order"""
    return [(k, tuple(v.shape)) for k, v in sd.items()]
