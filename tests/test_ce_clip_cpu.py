"""CPU checks of the VLN-CE policy's CLIP image tower (model/clip_visual.py): the oracle (oracle/ce_clip_ref.py) against
the unmodified reference (tests/golden/small_ce_clip.pt), the state_dict surface, the preprocessing restatement against
torchvision, the patch-row layout of conv1 as a GEMM, and the host logic of the encoder install and its replay key."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevbert_b200 import graphs, synth  # noqa: E402
from bevbert_b200.model import clip_visual as CV  # noqa: E402
from oracle import ce_clip_ref as R  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "small_ce_clip.pt")
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_ce_clip_golden as MG  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def state(golden):
    return synth.clip_visual_state(golden["seed"])


def test_oracle_matches_reference_golden(golden, state):
    rgb = synth.clip_images(3, golden["img_seed"])
    vec, grid = R.forward(state, rgb, torch.float64)
    got = MG.summarize(vec, grid)
    for k, ref in got.items():
        g = golden[k].double()
        err = float((ref - g).norm() / g.norm())
        assert err < 2e-5, (k, err)       # reference: fp32 on the CPU; oracle: fp64


def test_state_dict_surface(golden):
    m = CV.VisionTransformer(**synth.CLIP_B16)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [tuple(x) for x in golden["keys"]]
    assert list(synth.clip_visual_state(0, layers=1).keys()) == list(
        CV.VisionTransformer(**dict(synth.CLIP_B16, layers=1)).state_dict().keys())


def test_preprocessing_restatement_is_torchvisions(golden):
    rgb = synth.clip_images(3, golden["img_seed"])
    x = R.preprocess(rgb)
    assert torch.equal(x[:, :, :4, :4], golden["pre_corner"])
    assert torch.equal(x.double().sum(dim=(1, 2, 3)), golden["pre_sum"])
    transforms = pytest.importorskip("torchvision.transforms")
    tf = torch.nn.Sequential(transforms.ConvertImageDtype(torch.float), transforms.Normalize(R.MEAN, R.STD))
    for img in (rgb, rgb.float()):
        ref = tf(img.permute(0, 3, 1, 2))
        assert torch.equal(R.preprocess(img).view(torch.int32), ref.view(torch.int32))


def patch_rows(x, P):
    """the kernel's patch-row layout (bb_image_patches) of normalized NCHW images: row (n, py, px), column (c, ky, kx)"""
    N, _, H, W = x.shape
    return x.reshape(N, 3, H // P, P, W // P, P).permute(0, 2, 4, 1, 3, 5).reshape(N * (H // P) * (W // P), 3 * P * P)


@pytest.mark.parametrize("P,R_", [(16, 224), (16, 64), (8, 40)])
def test_patch_gemm_is_conv1(P, R_):
    g = torch.Generator().manual_seed(P + R_)
    x = torch.randn(3, 3, R_, R_, generator=g, dtype=torch.float64)
    w = torch.randn(24, 3, P, P, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, w, stride=P).flatten(2).transpose(1, 2).reshape(-1, 24)
    got = patch_rows(x, P) @ w.reshape(24, -1).t()
    assert torch.allclose(got, ref, rtol=0, atol=1e-12)
    assert torch.equal(patch_rows(x, P), F.unfold(x, P, stride=P).transpose(1, 2).reshape(-1, 3 * P * P))


def test_geometry_is_validated():
    CV.check_geometry(224, 16, 768, 12, 512)
    for args in ((224, 16, 768, 8, 512), (224, 16, 1088, 17, 512), (225, 16, 768, 12, 512), (224, 14, 768, 12, 512),
                 (224, 16, 768, 12, 500)):
        with pytest.raises(ValueError):
            CV.check_geometry(*args)
    with pytest.raises(ValueError):
        CV.VisionTransformer(224, 16, 768, 1, 8, 512)


class _Normalize(torch.nn.Module):
    def __init__(self, mean, std):
        super().__init__()
        self.mean, self.std = list(mean), list(std)


class _Encoder(torch.nn.Module):
    """CLIPEncoderB16's attribute layout: .model.visual and .rgb_transform"""

    def __init__(self, layers=1):
        super().__init__()
        self.model = torch.nn.Module()
        self.model.visual = CV.VisionTransformer(**dict(synth.CLIP_B16, layers=layers))
        self.rgb_transform = torch.nn.Sequential(torch.nn.Identity(), _Normalize(R.MEAN, R.STD))
        for p in self.model.parameters():
            p.requires_grad_(False)
        self.model.eval()


def test_install_host_logic():
    policy = torch.nn.Module()
    policy.net = torch.nn.Module()
    policy.net.rgb_encoder = enc = _Encoder()
    before = {k: v.clone() for k, v in policy.state_dict().items()}
    replay = graphs.install_ce_rgb_encoder(enc)
    after = policy.state_dict()
    assert list(after) == list(before) and all(torch.equal(after[k], v) for k, v in before.items())
    tower = replay.model
    assert tower.mean == tuple(float(m) for m in R.MEAN) and tower.std == tuple(float(s) for s in R.STD)
    assert (tower.width, tower.patch, tower.heads, tower.tokens, tower.out_dim) == (768, 16, 12, 197, 512)
    assert replay.s is graphs.CE_RGB and replay.s.grad_ok
    # replay follows the encoder's own train / eval switch
    enc.train()
    assert tower.training
    enc.eval()
    assert not tower.training
    # a tower parameter that requires grad, with grad enabled, is refused before anything runs
    enc.model.visual.proj.requires_grad_(True)
    with pytest.raises(RuntimeError, match="forward only"):
        enc({"rgb": torch.zeros(1, 224, 224, 3, dtype=torch.uint8)})
    # weight changes are seen through storage and version
    assert tower.changed() and not tower.changed()
    with torch.no_grad():
        enc.model.visual.ln_post.weight.add_(1.0)
    assert tower.changed() and not tower.changed()


def test_replay_key_is_the_exact_image_count():
    def key(n, dt=torch.uint8):
        return graphs._bucket(graphs.CE_RGB_DIMS, "rgb", {"rgb": torch.zeros(n, 224, 224, 3, dtype=dt)})
    assert key(96) != key(84) != key(12)
    assert key(12) == key(12) and key(12) != key(12, torch.float32)
    assert key(12)[2] == ((12, 224, 224, 3), torch.uint8)
