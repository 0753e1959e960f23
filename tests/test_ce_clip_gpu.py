"""GPU checks of the VLN-CE policy's CLIP image tower: bb_image_patches (bit-exact against torch's own preprocessing
operations on the device), the QuickGELU GEMM epilogue (integer-operand harness of tests/gemm_cases.py), bb_vit_tokens
against fp64, the whole tower against oracle/ce_clip_ref.py in both arms, autocast and deterministic mode, and the
encoder install with graph replay on a stand-in with CLIPEncoderB16's attribute layout."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import gemm_cases as G  # noqa: E402
from helpers import rel_l2  # noqa: E402
from bevbert_b200 import _lib, graphs, synth  # noqa: E402
from bevbert_b200 import kernels as K  # noqa: E402
from bevbert_b200 import vit_kernels as VK  # noqa: E402
from bevbert_b200.model import clip_visual as CV  # noqa: E402
from oracle import ce_clip_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 11


def patch_rows(x, P):
    N, _, H, W = x.shape
    return x.reshape(N, 3, H // P, P, W // P, P).permute(0, 2, 4, 1, 3, 5).reshape(N * (H // P) * (W // P), 3 * P * P)


def images(n, dt, seed=3):
    rgb = synth.clip_images(n, seed).to(DEV)
    return rgb if dt == torch.uint8 else rgb.float() + 0.25     # float pixels are not scaled


# --------------------------------------------------------------------------------------------- bb_image_patches
@pytest.mark.parametrize("n", [1, 12, 96])
@pytest.mark.parametrize("dt", [torch.uint8, torch.float32])
def test_image_patches_bit_exact(n, dt):
    rgb = images(n, dt)
    ref = patch_rows(R.preprocess(rgb), 16)          # torch's operations, on the device
    prev = K.set_precision(True)
    try:
        got32 = VK.image_patches(rgb, 16, R.MEAN, R.STD)
    finally:
        K.set_precision(prev)
    assert torch.equal(got32.view(torch.int32), ref.view(torch.int32))
    got = VK.image_patches(rgb, 16, R.MEAN, R.STD)
    assert got.dtype == torch.bfloat16
    assert torch.equal(got.view(torch.int16), ref.to(torch.bfloat16).view(torch.int16))


def test_image_patches_strides_unread_memory_and_guards():
    rgb = images(5, torch.float32)
    # a padded NHWC layout whose gaps hold NaN, and an NCHW tensor passed as its permuted view
    big = torch.full((5, 224, 230, 4), float("nan"), device=DEV)
    big[:, :, :224, :3] = rgb
    nchw = rgb.permute(0, 3, 1, 2).contiguous()
    ref = patch_rows(R.preprocess(rgb), 16).to(torch.bfloat16)
    rows = 5 * 196 * 768
    for src in (big[:, :, :224, :3], nchw.permute(0, 2, 3, 1)):
        buf = torch.full((rows + 2 * 64,), float("nan"), dtype=torch.bfloat16, device=DEV)
        init = buf.clone()
        VK.image_patches(src, 16, R.MEAN, R.STD, out=buf[64:64 + rows].view(-1, 768))
        assert torch.equal(buf[64:64 + rows].view(torch.int16), ref.reshape(-1).view(torch.int16))
        assert torch.equal(buf[:64].view(torch.int16), init[:64].view(torch.int16))
        assert torch.equal(buf[64 + rows:].view(torch.int16), init[64 + rows:].view(torch.int16))
    # forward(x) passes normalized images with an identity Normalize: the values themselves
    x = R.preprocess(rgb)
    got = VK.image_patches(x.permute(0, 2, 3, 1), 16, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0))
    assert torch.equal(got.view(torch.int16), patch_rows(x, 16).to(torch.bfloat16).view(torch.int16))


def test_image_patches_rejections():
    rgb = images(2, torch.uint8)
    with pytest.raises(_lib.BevbertLibraryError, match="multiples of the patch size"):
        VK.image_patches(rgb[:, :220], 16, R.MEAN, R.STD)
    with pytest.raises(_lib.BevbertLibraryError, match="3 \\* P \\* P"):
        VK.image_patches(rgb, 14, R.MEAN, R.STD)
    buf = torch.empty(2 * 196 * 768 + 8, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(_lib.BevbertLibraryError, match="aligned"):
        VK.image_patches(rgb, 16, R.MEAN, R.STD, out=buf[1:1 + 2 * 196 * 768].view(-1, 768))
    with pytest.raises(TypeError):
        VK.image_patches(rgb.to(torch.int32), 16, R.MEAN, R.STD)
    with pytest.raises(ValueError):
        VK.image_patches(rgb[..., :2], 16, R.MEAN, R.STD)
    with pytest.raises(RuntimeError):
        VK.image_patches(rgb.cpu(), 16, R.MEAN, R.STD)


# --------------------------------------------------------------------------------------------- QuickGELU epilogue
def qgelu64(x):
    return x * torch.sigmoid(1.702 * x)


# base variants of the harness whose reference keeps the pre-activation exact: "auxout" stores it, "add" adds add_in
QG_CASES = [G.Case("auxout", 128 + r, bn + 1 + (3 * r) % 7, k, maj=maj, block_n=bn, bias=b, alpha=a)
            for r, bn, k, maj, b, a in [(1, 64, 40, "NT", True, 1.0), (17, 128, 72, "NN", True, 0.125),
                                        (63, 64, 136, "NT", False, 1.0), (100, 128, 1000, "NN", True, 1.0)]] + \
    [G.Case("add", 333, 3072 + 5, 768, bias=True, block_n=0), G.Case("add", 77, 136, 64, maj="NN", block_n=64)]


@pytest.mark.parametrize("arm", ["bf16", "fp32"])
@pytest.mark.parametrize("case", QG_CASES, ids=lambda c: c.id)
def test_qgelu_epilogue(case, arm):
    """act = 3 on integer operands: the accumulator (aux_out) is bit-exact, and x*sigmoid(1.702x) of the exact
    pre-activation x is within 4 fp32 ulps of |x| of fp64 (expf and a correctly rounded division), plus one output
    rounding."""
    arm32 = arm == "fp32"
    prev = K.set_precision(arm32)
    try:
        L = G.Launch(case, DEV, arm32=arm32)
        pre = L.ref["aux_out"] if "aux_out" in L.ref else L.ref["D"] - L.logical("add_in").double()
        ref_D = qgelu64(pre) + (L.logical("add_in").double() if case.feats["add_in"] else 0.0)
        L.ref = {k: v for k, v in L.ref.items() if k == "aux_out"}
        L.run(K.gemm, act=K.ACT_QGELU)
        L.check()                                      # aux_out bit-exact, guards / inputs unchanged
        got = L.logical("D").double()
        tol = G.ulp(ref_D, L.odt) + 4 * 2.0 ** -24 * pre.abs()
        err = (got - ref_D).abs()
        assert bool((err <= tol).all()), float((err - tol).max())
        pos = (L.start["D"] + L.loff).reshape(-1)
        outside = torch.ones(L.buflen, dtype=torch.bool, device=DEV)
        outside[pos] = False
        assert torch.equal(G.bits(L.bufs["D"])[outside], G.bits(L.init["D"])[outside])
    finally:
        K.set_precision(prev)


@pytest.mark.parametrize("arm", ["bf16", "fp32"])
def test_gemm_rejects_unknown_act(arm):
    prev = K.set_precision(arm == "fp32")
    try:
        L = G.Launch(G.Case("plain", 64, 64, 64), DEV, arm32=arm == "fp32")
        for act in (4, -1):
            with pytest.raises(_lib.BevbertLibraryError, match="act must be"):
                L.run(K.gemm, act=act)
        L.untouched()
    finally:
        K.set_precision(prev)


# --------------------------------------------------------------------------------------------- bb_vit_tokens
@pytest.mark.parametrize("arm", ["bf16", "fp32"])
@pytest.mark.parametrize("N,T,H", [(3, 197, 768), (2, 5, 40), (1, 2, 1024)])
def test_vit_tokens_fp64(N, T, H, arm):
    g = torch.Generator().manual_seed(N * T + H)
    patch = (torch.randn(N * (T - 1), H, generator=g) * 2 + 0.5).to(DEV)
    cls, gamma, beta = (torch.randn(H, generator=g).to(DEV) for _ in range(3))
    pos = torch.randn(T, H, generator=g).to(DEV)
    x = torch.cat([cls.expand(N, 1, H), patch.view(N, T - 1, H)], 1).double() + pos.double()
    ref = torch.nn.functional.layer_norm(x, (H,), gamma.double(), beta.double(), 1e-5).reshape(N * T, H)
    prev = K.set_precision(arm == "fp32")
    try:
        got = VK.vit_tokens(patch, cls, pos, gamma, beta, 1e-5, N).double()
    finally:
        K.set_precision(prev)
    scale = ref.abs() + gamma.double().abs() + beta.double().abs()
    bound = 2.0 ** -8 * ref.abs() + 1e-5 * scale if arm == "bf16" else 1e-5 * scale
    assert bool(((got - ref).abs() <= bound).all()), float((got - ref).abs().max())


def test_vit_tokens_rejections():
    z = torch.zeros(2 * 196, 768, device=DEV)
    v = torch.zeros(768, device=DEV)
    pos = torch.zeros(197, 768, device=DEV)
    with pytest.raises(ValueError):
        VK.vit_tokens(z[:-1], v, pos, v, v, 1e-5, 2)
    with pytest.raises(_lib.BevbertLibraryError, match="aligned"):
        VK.vit_tokens(z, torch.zeros(776, device=DEV)[1:769], pos, v, v, 1e-5, 2)
    with pytest.raises(_lib.BevbertLibraryError, match="1024"):
        VK.vit_tokens(torch.zeros(2, 1032, device=DEV), torch.zeros(1032, device=DEV), torch.zeros(2, 1032, device=DEV),
                     torch.zeros(1032, device=DEV), torch.zeros(1032, device=DEV), 1e-5, 2)


# --------------------------------------------------------------------------------------------- whole tower
@pytest.fixture(scope="module")
def state():
    return synth.clip_visual_state(SEED)


def fp16_params_(vit):
    """the dtypes clip.load leaves on the GPU (convert_weights)"""
    for name, p in vit.named_parameters():
        if name.endswith(R.FP16_KEYS):
            p.data = p.data.half()
    return vit


@pytest.fixture(scope="module")
def vit(state):
    m = CV.VisionTransformer(**synth.CLIP_B16)
    m.load_state_dict(state)
    return fp16_params_(m.to(DEV)).requires_grad_(False).eval()


@pytest.fixture(scope="module")
def fp16_ref(state):
    return R.Fp16Tower(state).to(DEV)


@pytest.mark.parametrize("n", [12, 48, 96])
@pytest.mark.parametrize("dt", [torch.uint8, torch.float32])
def test_tower_against_oracle(state, vit, fp16_ref, n, dt):
    rgb = images(n, dt, seed=20 + n)
    sd64 = {k: v.to(DEV) for k, v in state.items()}
    ref = R.forward(sd64, rgb, torch.float64)
    e16 = [rel_l2(o, r) for o, r in zip(R.forward_fp16(fp16_ref, rgb), ref)]
    out = vit.encode_rgb(rgb)
    assert all(o.dtype == torch.float32 for o in out)
    assert out[0].shape == (n, 512) and out[1].shape == (n, 196, 768)
    e = [rel_l2(o, r) for o, r in zip(out, ref)]
    prev = K.set_precision(True)
    try:
        m32 = CV.VisionTransformer(**synth.CLIP_B16)
        m32.load_state_dict(state)
        m32 = fp16_params_(m32.to(DEV)).requires_grad_(False)
        out32 = m32.encode_rgb(rgb)
    finally:
        K.set_precision(prev)
    e32 = [rel_l2(o, r) for o, r in zip(out32, ref)]
    print("n=%d %s: fp32 arm %s | bf16 %s | fp16 reference %s" % (n, dt, e32, e, e16))
    assert max(e32) <= 1e-3, e32
    for got, ref16 in zip(e, e16):
        assert got <= max(1e-2, 2.5 * ref16), (e, e16)


def test_forward_takes_normalized_images(vit):
    rgb = images(4, torch.uint8, seed=5)
    a = vit.encode_rgb(rgb)
    b = vit(R.preprocess(rgb))
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_autocast_changes_no_bit(vit):
    rgb = images(12, torch.uint8, seed=6)
    a = vit.encode_rgb(rgb)
    with torch.autocast("cuda", dtype=torch.float16):
        b = vit.encode_rgb(rgb)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_deterministic_repeats(vit):
    rgb = images(48, torch.uint8, seed=7)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a = vit.encode_rgb(rgb)
        b = vit.encode_rgb(rgb)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_grad_with_trainable_tower_raises(state):
    m = CV.VisionTransformer(**dict(synth.CLIP_B16, layers=1)).to(DEV)
    with pytest.raises(RuntimeError, match="forward only"):
        m.encode_rgb(images(1, torch.uint8))
    with torch.no_grad():
        m.encode_rgb(images(1, torch.uint8))


# --------------------------------------------------------------------------------------------- install + replay
class _Normalize(torch.nn.Module):
    def __init__(self, mean, std):
        super().__init__()
        self.mean, self.std = list(mean), list(std)


class _Encoder(torch.nn.Module):
    """CLIPEncoderB16's attribute layout, weights in clip.load's dtypes, frozen and in eval mode"""

    def __init__(self, state):
        super().__init__()
        self.model = torch.nn.Module()
        self.model.visual = CV.VisionTransformer(**synth.CLIP_B16)
        self.model.visual.load_state_dict(state)
        fp16_params_(self.model.visual)
        self.rgb_transform = torch.nn.Sequential(torch.nn.Identity(), _Normalize(R.MEAN, R.STD))
        for p in self.model.parameters():
            p.requires_grad_(False)
        self.model.eval()


def test_install_replay(state):
    policy = torch.nn.Module()
    policy.net = torch.nn.Module()
    policy.net.rgb_encoder = enc = _Encoder(state)
    policy.to(DEV).eval()
    before = {k: v.clone() for k, v in policy.state_dict().items()}
    replay = graphs.install_ce_rgb_encoder(enc)
    after = policy.state_dict()
    assert list(after) == list(before) and all(torch.equal(after[k], v) for k, v in before.items())

    def eager(rgb):
        enc.train()                     # training mode: the same kernels, launched eagerly
        try:
            return enc({"rgb": rgb})
        finally:
            enc.eval()

    obs = {n: images(n, torch.uint8, seed=40 + n) for n in (96, 84, 12)}
    for i, n in enumerate([96, 84, 12, 96, 12]):
        rgb = obs[n]
        if i % 2:
            got = enc({"rgb": rgb})     # grad enabled: a frozen tower replays too
        else:
            with torch.no_grad():
                got = enc({"rgb": rgb})
        assert replay.launches("rgb", {"rgb": rgb}) is not None
        exp = eager(rgb)
        assert all(torch.equal(a, b) for a, b in zip(got, exp)), n
        assert got[0].data_ptr() != replay.entries[graphs._bucket(graphs.CE_RGB_DIMS, "rgb", {"rgb": rgb})]["out"][0] \
            .data_ptr()
    # load_state_dict on the policy between calls is seen, replayed and eager
    sd = policy.state_dict()
    sd2 = {k: (v * 1.25 if k.endswith(("ln_post.weight", "mlp.c_fc.weight", "attn.in_proj_bias")) else v)
           for k, v in sd.items()}
    old = enc({"rgb": obs[12]})
    policy.load_state_dict(sd2)
    new = enc({"rgb": obs[12]})
    assert not torch.equal(old[0], new[0]) and not torch.equal(old[1], new[1])
    exp = eager(obs[12])
    assert all(torch.equal(a, b) for a, b in zip(new, exp))
    fresh = CV.ClipTower(enc.model.visual)
    ref = fresh.encode_rgb(obs[12])
    assert all(torch.equal(a, b) for a, b in zip(new, ref))
    assert len(replay.entries) == 3
