"""The VLN-CE policy's depth encoder on the H100 kernels, forward only: `VlnResnetDepthEncoder.visual_encoder`
(bevbert_ce/vlnce_baselines/models/encoders/resnet_encoders.py:13-107), habitat-lab v0.1.7's DD-PPO `ResNetEncoder` over
a GroupNorm ResNet-50 (`habitat_baselines/rl/ddppo/policy/resnet.py::resnet50`, `resnet_policy.py::ResNetEncoder`).

`ResNetEncoder` and `resnet50` restate habitat-lab's classes from their documented structure (constructor signature,
module names, state_dict keys, shapes and order); habitat-lab's source is not part of this project.  `DepthTower` runs
the kernels' forward over any module with that layout, such as the user's own habitat `ResNetEncoder`
(graphs.install_ce_depth_encoder).  Per call, with N depth images (N, H, W, 1) in fp32:
    bb_depth_stem (avg_pool2d 2 + conv 7x7/2, Cin 1) -> bb_groupnorm_apply (GN, ReLU, max-pool 3x3/2)
    -> 16 bottlenecks: bb_conv2d 1x1 -> GN + ReLU -> bb_conv2d 3x3 (stride on the first block of layers 2-4) -> GN +
       ReLU -> bb_conv2d 1x1 -> GN + identity + ReLU, or, on the first block of a layer, GN + GN(downsample conv 1x1)
       + ReLU in one bb_groupnorm_apply
    -> compression bb_conv2d 3x3 (1024 -> 128) -> GN(1, 128) + ReLU written as fp32 NCHW (N, 128, h, w).
Every conv writes the GroupNorm partial statistics of its stored output, so a GroupNorm costs one pass over its input.
Activations are fp16 between kernels (fp32 in the verification arm, kernels.set_precision(True)); conv weights are fp16
(K-major (Cout, R, S, Cin)) WeightCache shadows, re-made when a parameter's version or storage changes.  Autocast is
disabled inside the call, and the output is a fresh fp32 tensor.
"""
from collections import OrderedDict

import torch
from torch import nn
import torch.nn.functional as F

from .. import blocks
from .. import conv_kernels as CK
from .. import kernels as K

GN_EPS = 1e-5
BASE_PLANES, NGROUPS = 32, 16
LAYERS = (3, 4, 6, 3)
COMPRESSION_FLAT = 2048


# ------------------------------------------------------------------------------------ habitat-lab v0.1.7 layout
def conv3x3(in_planes, out_planes, stride=1, groups=1):
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False, groups=groups)


def conv1x1(in_planes, out_planes, stride=1):
    return nn.Conv2d(in_planes, out_planes, kernel_size=1, stride=stride, bias=False)


class Bottleneck(nn.Module):
    expansion = 4
    resneXt = False

    def __init__(self, inplanes, planes, ngroups, stride=1, downsample=None, cardinality=1):
        super().__init__()
        self.convs = nn.Sequential(
            conv1x1(inplanes, planes), nn.GroupNorm(ngroups, planes), nn.ReLU(True),
            conv3x3(planes, planes, stride, groups=cardinality), nn.GroupNorm(ngroups, planes), nn.ReLU(True),
            conv1x1(planes, planes * self.expansion), nn.GroupNorm(ngroups, planes * self.expansion))
        self.downsample = downsample
        self.relu = nn.ReLU(True)

    def forward(self, x):
        identity = x
        out = self.convs(x)
        if self.downsample is not None:
            identity = self.downsample(x)
        return self.relu(out + identity)


class ResNet(nn.Module):
    def __init__(self, in_channels, base_planes, ngroups, block, layers, cardinality=1):
        super().__init__()
        self.conv1 = nn.Sequential(
            nn.Conv2d(in_channels, base_planes, kernel_size=7, stride=2, padding=3, bias=False),
            nn.GroupNorm(ngroups, base_planes), nn.ReLU(True))
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.cardinality = cardinality
        self.inplanes = base_planes
        if block.resneXt:
            base_planes *= 2
        self.layer1 = self._make_layer(block, ngroups, base_planes, layers[0])
        self.layer2 = self._make_layer(block, ngroups, base_planes * 2, layers[1], stride=2)
        self.layer3 = self._make_layer(block, ngroups, base_planes * 2 * 2, layers[2], stride=2)
        self.layer4 = self._make_layer(block, ngroups, base_planes * 2 * 2 * 2, layers[3], stride=2)
        self.final_channels = self.inplanes
        self.final_spatial_compress = 1.0 / (2 ** 5)

    def _make_layer(self, block, ngroups, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(conv1x1(self.inplanes, planes * block.expansion, stride),
                                       nn.GroupNorm(ngroups, planes * block.expansion))
        layers = [block(self.inplanes, planes, ngroups, stride, downsample, cardinality=self.cardinality)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes, ngroups))
        return nn.Sequential(*layers)

    def forward(self, x):
        x = self.maxpool(self.conv1(x))
        return self.layer4(self.layer3(self.layer2(self.layer1(x))))


def resnet50(in_channels, base_planes, ngroups):
    return ResNet(in_channels, base_planes, ngroups, Bottleneck, list(LAYERS))


class RunningMeanAndVar(nn.Module):
    """the `normalize_visual_inputs=True` input normaliser's buffers (layout only: DepthTower rejects it)"""

    def __init__(self, n_channels):
        super().__init__()
        self.register_buffer("_mean", torch.zeros(1, n_channels, 1, 1))
        self.register_buffer("_var", torch.zeros(1, n_channels, 1, 1))
        self.register_buffer("_count", torch.zeros(()))


class ResNetEncoder(nn.Module):
    """habitat-lab's ResNetEncoder: `observation_space.spaces` maps "rgb" / "depth" to spaces with a (H, W, C) shape."""

    def __init__(self, observation_space, baseplanes=32, ngroups=32, spatial_size=128, make_backbone=None,
                 normalize_visual_inputs=False):
        super().__init__()
        spaces = observation_space.spaces
        self._n_input_rgb = spaces["rgb"].shape[2] if "rgb" in spaces else 0
        if "rgb" in spaces:
            spatial_size = spaces["rgb"].shape[0] // 2
        self._n_input_depth = spaces["depth"].shape[2] if "depth" in spaces else 0
        if "depth" in spaces:
            spatial_size = spaces["depth"].shape[0] // 2
        if normalize_visual_inputs:
            self.running_mean_and_var = RunningMeanAndVar(self._n_input_depth + self._n_input_rgb)
        else:
            self.running_mean_and_var = nn.Sequential()
        if not self.is_blind:
            input_channels = self._n_input_depth + self._n_input_rgb
            self.backbone = make_backbone(input_channels, baseplanes, ngroups)
            final_spatial = int(spatial_size * self.backbone.final_spatial_compress)
            num_compression_channels = int(round(COMPRESSION_FLAT / (final_spatial ** 2)))
            self.compression = nn.Sequential(
                nn.Conv2d(self.backbone.final_channels, num_compression_channels, kernel_size=3, padding=1,
                          bias=False),
                nn.GroupNorm(1, num_compression_channels), nn.ReLU(True))
            self.output_shape = (num_compression_channels, final_spatial, final_spatial)

    @property
    def is_blind(self):
        return self._n_input_rgb + self._n_input_depth == 0

    def forward(self, observations):
        """the reference PyTorch forward (the tests' and the benchmark's yardstick; DepthTower is the kernels')"""
        if self.is_blind:
            return None
        cnn_input = []
        if self._n_input_rgb > 0:
            cnn_input.append(observations["rgb"].permute(0, 3, 1, 2) / 255.0)
        if self._n_input_depth > 0:
            cnn_input.append(observations["depth"].permute(0, 3, 1, 2))
        x = F.avg_pool2d(torch.cat(cnn_input, dim=1), 2)
        x = self.running_mean_and_var(x)
        return self.compression(self.backbone(x))


class Box:
    """a space with a shape, enough for ResNetEncoder (gym.spaces.Box stands in when gym is installed)"""

    def __init__(self, shape):
        self.shape = tuple(shape)


class Spaces:
    def __init__(self, spaces):
        self.spaces = dict(spaces)


def depth_encoder(height=256, width=256, baseplanes=BASE_PLANES, ngroups=NGROUPS):
    """The VLN-CE policy's `visual_encoder` as VlnResnetDepthEncoder builds it (baseplanes 32, ngroups 16, resnet50)."""
    return ResNetEncoder(Spaces({"depth": Box((height, width, 1))}), baseplanes=baseplanes, ngroups=ngroups,
                         make_backbone=resnet50, normalize_visual_inputs=False)


# ------------------------------------------------------------------------------------------ the kernels' forward
def _check_conv(conv, name, cin, cout, k, stride, pad):
    if not isinstance(conv, nn.Conv2d):
        raise ValueError("%s must be a Conv2d" % name)
    got = (conv.in_channels, conv.out_channels, conv.kernel_size, conv.stride, conv.padding, conv.dilation,
           conv.groups, conv.bias is None, conv.padding_mode)
    want = (cin, cout, (k, k), (stride, stride), (pad, pad), (1, 1), 1, True, "zeros")
    if got != want:
        raise ValueError("%s: conv geometry %s, the kernels need %s (in, out, kernel, stride, padding, dilation, "
                         "groups, no bias, zero padding)" % (name, got, want))


def _check_gn(gn, name, groups, channels):
    if not isinstance(gn, nn.GroupNorm):
        raise ValueError("%s must be a GroupNorm" % name)
    if (gn.num_groups, gn.num_channels, gn.eps, gn.affine) != (groups, channels, GN_EPS, True):
        raise ValueError("%s: GroupNorm(%d, %d, eps=%g, affine=%s), the spec is GroupNorm(%d, %d, eps=%g) with an "
                         "affine" % (name, gn.num_groups, gn.num_channels, gn.eps, gn.affine, groups, channels,
                                     GN_EPS))


def check_layout(enc):
    """Validates a ResNetEncoder-layout module against the depth encoder the kernels run (depth only, no input
    normaliser, resnet50 with 32 base planes and GroupNorm(16), compression to 128 channels with GroupNorm(1));
    raises ValueError otherwise.  -> the list of (planes, stride, block) of the 16 bottlenecks."""
    if getattr(enc, "_n_input_rgb", 0):
        raise ValueError("the depth kernels take depth only: the encoder has %d RGB input channels" % enc._n_input_rgb)
    if getattr(enc, "_n_input_depth", 1) != 1:
        raise ValueError("the depth kernels take one depth channel, got %s" % enc._n_input_depth)
    rmv = getattr(enc, "running_mean_and_var", None)
    if not isinstance(rmv, nn.Sequential) or len(rmv) or len(list(rmv.buffers())):
        raise ValueError("normalize_visual_inputs=True (a RunningMeanAndVar input normaliser) is not supported")
    bb = getattr(enc, "backbone", None)
    if bb is None:
        raise ValueError("the encoder has no backbone (blind)")
    _check_conv(bb.conv1[0], "backbone.conv1.0", 1, BASE_PLANES, 7, 2, 3)
    _check_gn(bb.conv1[1], "backbone.conv1.1", NGROUPS, BASE_PLANES)
    mp = bb.maxpool
    if not isinstance(mp, nn.MaxPool2d) or (mp.kernel_size, mp.stride, mp.padding, mp.dilation, mp.ceil_mode) not in (
            (3, 2, 1, 1, False), ((3, 3), (2, 2), (1, 1), (1, 1), False)):
        raise ValueError("backbone.maxpool must be MaxPool2d(3, stride 2, padding 1)")
    plan, inplanes = [], BASE_PLANES
    for li, (n, planes) in enumerate(zip(LAYERS, (32, 64, 128, 256))):
        layer = getattr(bb, "layer%d" % (li + 1))
        if len(layer) != n:
            raise ValueError("backbone.layer%d has %d blocks, resnet50 has %d" % (li + 1, len(layer), n))
        for bi, blk in enumerate(layer):
            name = "backbone.layer%d.%d" % (li + 1, bi)
            stride = 2 if (bi == 0 and li > 0) else 1
            c = blk.convs
            _check_conv(c[0], name + ".convs.0", inplanes, planes, 1, 1, 0)
            _check_gn(c[1], name + ".convs.1", NGROUPS, planes)
            _check_conv(c[3], name + ".convs.3", planes, planes, 3, stride, 1)
            _check_gn(c[4], name + ".convs.4", NGROUPS, planes)
            _check_conv(c[6], name + ".convs.6", planes, 4 * planes, 1, 1, 0)
            _check_gn(c[7], name + ".convs.7", NGROUPS, 4 * planes)
            if bi == 0:
                if blk.downsample is None:
                    raise ValueError("%s needs its downsample branch" % name)
                _check_conv(blk.downsample[0], name + ".downsample.0", inplanes, 4 * planes, 1, stride, 0)
                _check_gn(blk.downsample[1], name + ".downsample.1", NGROUPS, 4 * planes)
            elif blk.downsample is not None:
                raise ValueError("%s must not have a downsample branch" % name)
            plan.append((planes, stride, blk))
            inplanes = 4 * planes
    comp = enc.compression
    cc = comp[0].out_channels if isinstance(comp[0], nn.Conv2d) else -1
    _check_conv(comp[0], "compression.0", inplanes, 128, 3, 1, 1)
    _check_gn(comp[1], "compression.1", 1, cc)
    return plan


class DepthTower:
    """The kernels' forward over `enc`, a module laid out as habitat-lab's ResNetEncoder for one depth channel
    (check_layout).  `owner` (default `enc`) is the module whose train / eval mode the caller goes by."""

    def __init__(self, enc, owner=None):
        self.enc, self.owner = enc, owner if owner is not None else enc
        self.plan = check_layout(enc)
        self.rt = blocks.Runtime()
        self._sig = None

    @property
    def training(self):
        return self.owner.training

    def parameters(self):
        return self.enc.parameters()

    def changed(self):
        """True when a parameter's storage or version moved since the previous call of this method."""
        sig = tuple((p.data_ptr(), p._version) for p in self.enc.parameters())
        moved, self._sig = sig != self._sig, sig
        return moved

    def check_grad(self):
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.enc.parameters()):
            raise RuntimeError("the depth encoder runs forward only: call it under torch.no_grad() or freeze its "
                               "parameters (trainable=False), as VlnResnetDepthEncoder does by default")

    def encode(self, depth):
        """visual_encoder(observations) on observations["depth"] (N, H, W, 1) float32 (any strides) -> (N, 128, h, w)
        fp32, h = ceil(ceil(H/2 / 2) / 16) after the stem, max-pool and three stride-2 layers (4 x 4 at 256 x 256)."""
        self.check_grad()
        if depth.dim() != 4 or depth.shape[3] != 1 or depth.dtype != torch.float32:
            raise ValueError("expected depth of shape (N, H, W, 1) in float32, got %s %s" % (
                depth.dtype, tuple(depth.shape)))
        with torch.autocast("cuda", enabled=False), torch.no_grad():
            return self._encode(depth)

    def _encode(self, depth):
        wc, dt, eps = self.rt.wc, CK.conv_dtype(), GN_EPS
        f32, w16 = wc.f32, (lambda conv: wc.conv_nhwc(conv.weight, dt))
        bb = self.enc.backbone
        stem_w = wc.conv_nhwc(bb.conv1[0].weight, torch.float32).view(BASE_PLANES, 1, 7, 7)
        y, p = CK.depth_stem(depth, stem_w, NGROUPS)
        gn = bb.conv1[1]
        x = CK.groupnorm_apply(y, p, f32(gn.weight), f32(gn.bias), eps, CK.GN_RELU_MAXPOOL)
        for planes, stride, blk in self.plan:
            c = blk.convs
            h, ph = CK.conv2d(x, w16(c[0]), 1, NGROUPS)
            h = CK.groupnorm_apply(h, ph, f32(c[1].weight), f32(c[1].bias), eps)
            h, ph = CK.conv2d(h, w16(c[3]), stride, NGROUPS)
            h = CK.groupnorm_apply(h, ph, f32(c[4].weight), f32(c[4].bias), eps)
            h, ph = CK.conv2d(h, w16(c[6]), 1, NGROUPS)
            if blk.downsample is not None:
                d, pd = CK.conv2d(x, w16(blk.downsample[0]), stride, NGROUPS)
                ds = blk.downsample[1]
                x = CK.groupnorm_apply(h, ph, f32(c[7].weight), f32(c[7].bias), eps, CK.GN_ADD_NORM_RELU, x2=d,
                                       p2=pd, gamma2=f32(ds.weight), beta2=f32(ds.bias))
            else:
                x = CK.groupnorm_apply(h, ph, f32(c[7].weight), f32(c[7].bias), eps, CK.GN_ADD_RELU, identity=x)
        comp = self.enc.compression
        h, ph = CK.conv2d(x, w16(comp[0]), 1, 1)
        return CK.groupnorm_apply(h, ph, f32(comp[1].weight), f32(comp[1].bias), eps, out_f32=True)


def ddppo_visual_keys(enc):
    """state_dict key -> shape of a ResNetEncoder, in order (the strict-load contract with DD-PPO checkpoints)"""
    return OrderedDict((k, tuple(v.shape)) for k, v in enc.state_dict().items())
