"""CPU checks of the VLN-CE depth encoder: oracle/ce_depth_ref.py against tests/golden/small_ce_depth.pt (made by the
reference's unmodified VlnResnetDepthEncoder over the restated habitat-lab layout), the key layout, DepthTower's layout
validation, the oracle's fp16 dtype flow, and the install host logic."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevbert_b200 import graphs, synth  # noqa: E402
from bevbert_b200.model import depth_resnet as D  # noqa: E402
from oracle import ce_depth_ref as R  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "small_ce_depth.pt")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


def test_oracle_against_golden(golden):
    sd = synth.depth_encoder_state(golden["seed"])
    depth = synth.depth_images(golden["n"], golden["depth_seed"])
    out32 = R.forward(sd, depth, torch.float32)
    out64 = R.forward(sd, depth, torch.float64)
    assert ((out32 - golden["out_fp32"]).norm() / golden["out_fp32"].norm()) <= 1e-5
    assert ((out64 - golden["out_fp64"]).norm() / golden["out_fp64"].norm()) <= 1e-12
    assert golden["passthrough"] and golden["spatial_shape"] == (2, 192, 4, 4)
    assert not golden["params_requires_grad"]


def test_key_map_and_order(golden):
    enc = D.depth_encoder()
    keys = D.ddppo_visual_keys(enc)
    assert list(keys.items()) == [tuple(kv) for kv in golden["keys"]]
    assert len(keys) == 162 and list(keys)[:4] == ["backbone.conv1.0.weight", "backbone.conv1.1.weight",
                                                   "backbone.conv1.1.bias", "backbone.layer1.0.convs.0.weight"]
    assert sum(p.numel() for p in enc.parameters()) == 7069408
    assert [(k, tuple(v.shape)) for k, v in synth.depth_encoder_state(0).items()] == list(keys.items())
    ck = synth.ddppo_checkpoint(0)["state_dict"]
    remap = {".".join(k.split(".")[3:]): v for k, v in ck.items() if k.split(".")[2] == "visual_encoder"}
    enc.load_state_dict(remap, strict=True)


def test_oracle_matches_restated_module():
    sd = synth.depth_encoder_state(3)
    enc = D.depth_encoder(256, 341)
    enc.load_state_dict(sd)
    depth = synth.depth_images(1, 4, 256, 341)
    with torch.no_grad():
        ref = enc.eval()({"depth": depth})
    out = R.forward(sd, depth, torch.float32)
    assert out.shape == ref.shape == (1, 128, 4, 6)
    assert (out - ref).norm() / ref.norm() <= 1e-5


def test_fp16_arm_dtype_flow():
    """CUDA autocast: conv2d on fp16 operands returns fp16, group_norm returns fp32, the rest follows in fp32"""
    seen = []
    orig = R.F.group_norm

    def spy(x, *a, **k):
        seen.append(x.dtype)
        return orig(x, *a, **k)
    sd = synth.depth_encoder_state(5)
    depth = synth.depth_images(1, 6, 64, 64)
    x, w = torch.randn(1, 32, 8, 8), torch.randn(32, 32, 3, 3)
    y = R._conv_fp16(x, w, 1, 1)
    assert y.dtype == torch.float16
    assert torch.equal(y, torch.nn.functional.conv2d(x.half().float(), w.half().float(), padding=1).half())
    R.F.group_norm = spy
    try:
        out = R.forward_fp16(sd, depth)
    finally:
        R.F.group_norm = orig
    assert out.dtype == torch.float32 and set(seen) == {torch.float32} and len(seen) == 54
    ref = R.forward(sd, depth, torch.float64)
    assert 0 < float((out.double() - ref).norm() / ref.norm()) < 2e-2


def test_fp16_arm_against_cpu_autocast():
    """where the CPU's autocast runs convolutions in fp16, the restated module under it follows the same flow"""
    sd = synth.depth_encoder_state(7)
    enc = D.depth_encoder().eval()
    enc.load_state_dict(sd)
    depth = synth.depth_images(1, 8, 64, 64)
    try:
        with torch.no_grad(), torch.autocast("cpu", dtype=torch.float16):
            got = enc({"depth": depth})
    except RuntimeError as e:
        pytest.skip("CPU autocast has no fp16 convolution here: %s" % str(e)[:80])
    ref = R.forward_fp16(sd, depth)
    assert (got.float() - ref).norm() / ref.norm() <= 1e-2


def _rejects(mutate, match):
    enc = D.depth_encoder()
    mutate(enc)
    with pytest.raises(ValueError, match=match):
        D.DepthTower(enc)


def test_layout_validation():
    plan = D.check_layout(D.depth_encoder())
    assert len(plan) == 16 and [s for _, s, _ in plan].count(2) == 3
    rgbd = D.ResNetEncoder(D.Spaces({"rgb": D.Box((256, 256, 3)), "depth": D.Box((256, 256, 1))}), 32, 16,
                           make_backbone=D.resnet50)
    with pytest.raises(ValueError, match="RGB"):
        D.DepthTower(rgbd)
    norm = D.ResNetEncoder(D.Spaces({"depth": D.Box((256, 256, 1))}), 32, 16, make_backbone=D.resnet50,
                           normalize_visual_inputs=True)
    with pytest.raises(ValueError, match="normalize_visual_inputs"):
        D.DepthTower(norm)
    with pytest.raises(ValueError, match="GroupNorm"):
        D.DepthTower(D.depth_encoder(ngroups=32))
    _rejects(lambda e: setattr(e.backbone.layer2[1].convs[1], "eps", 1e-6), "GroupNorm")
    _rejects(lambda e: setattr(e.compression[1], "num_groups", 2), "GroupNorm")
    _rejects(lambda e: setattr(e.backbone.layer3[0].convs[3], "stride", (1, 1)), "conv geometry")
    _rejects(lambda e: setattr(e.backbone.layer1[0].convs[3], "padding", (2, 2)), "conv geometry")
    _rejects(lambda e: setattr(e.backbone.layer1[0].convs[3], "dilation", (2, 2)), "conv geometry")
    _rejects(lambda e: setattr(e.backbone.conv1[0], "kernel_size", (5, 5)), "conv geometry")
    with pytest.raises(ValueError, match="conv geometry"):
        D.DepthTower(D.depth_encoder(baseplanes=64))


class _Wrapper(torch.nn.Module):
    """VlnResnetDepthEncoder's attribute layout: .visual_encoder, frozen"""

    def __init__(self):
        super().__init__()
        self.visual_encoder = D.depth_encoder()
        for p in self.visual_encoder.parameters():
            p.requires_grad_(False)


def test_install_host_logic():
    policy = torch.nn.Module()
    policy.net = torch.nn.Module()
    policy.net.depth_encoder = enc = _Wrapper()
    before = {k: v.clone() for k, v in policy.state_dict().items()}
    replay = graphs.install_ce_depth_encoder(enc)
    after = policy.state_dict()
    assert list(after) == list(before) and all(torch.equal(after[k], v) for k, v in before.items())
    tower = replay.model
    assert replay.s is graphs.CE_DEPTH and replay.s.grad_ok and tower.enc is enc.visual_encoder
    assert "forward" in enc.visual_encoder.__dict__ and "forward" not in enc.__dict__
    enc.train()
    assert tower.training
    enc.eval()
    assert not tower.training
    # a parameter that requires grad, with grad enabled, is refused before anything runs
    enc.visual_encoder.compression[1].weight.requires_grad_(True)
    with pytest.raises(RuntimeError, match="forward only"):
        enc.visual_encoder({"depth": torch.zeros(1, 256, 256, 1)})
    assert tower.changed() and not tower.changed()
    with torch.no_grad():
        enc.visual_encoder.compression[1].bias.add_(1.0)
    assert tower.changed() and not tower.changed()


def test_replay_key_is_the_exact_image_count():
    def key(n, dt=torch.float32):
        return graphs._bucket(graphs.CE_DEPTH_DIMS, "depth", {"depth": torch.zeros(n, 256, 256, 1, dtype=dt)})
    assert key(96) != key(84) != key(12)
    assert key(12) == key(12) and key(12) != key(12, torch.float64)
    assert key(12)[2] == ((12, 256, 256, 1), torch.float32)
