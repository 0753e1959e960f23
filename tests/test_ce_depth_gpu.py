"""GPU checks of the VLN-CE depth encoder on the kernels (csrc/conv.cu, model/depth_resnet.py): bb_conv2d bit for bit on
integer operands over every conv shape of the network, with NaN in unread memory and untouched guards; the GroupNorm
partials and every bb_groupnorm_apply variant against fp64 GroupNorm of the same stored tensor; the stem against fp64;
the whole encoder at 12, 48 and 96 images in both arms against oracle/ce_depth_ref.py; autocast and deterministic mode;
the install with graph replay; and the composition depth encoder -> waypoint predictor -> bb_waypoint_nms."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from helpers import rel_l2  # noqa: E402
from bevbert_b200 import _lib, graphs, synth  # noqa: E402
from bevbert_b200 import conv_kernels as CK  # noqa: E402
from bevbert_b200 import kernels as K  # noqa: E402
from bevbert_b200.model import depth_resnet as D  # noqa: E402
from oracle import ce_depth_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 31
GUARD = 64          # elements of NaN / sentinel around every operand (keeps 16-byte alignment)

# (Cin, Cout, R, stride, H = W of the input): every conv of the network, plus 64-pixel maps, Cin % 32 == 16 and a
# Cout that needs three 32-wide tiles
NET_CONVS = [(32, 32, 1, 1, 32), (32, 32, 3, 1, 32), (32, 128, 1, 1, 32), (128, 32, 1, 1, 32),
             (128, 64, 1, 1, 32), (64, 64, 3, 2, 32), (64, 256, 1, 1, 16), (128, 256, 1, 2, 32), (256, 64, 1, 1, 16),
             (64, 64, 3, 1, 16), (256, 128, 1, 1, 16), (128, 128, 3, 2, 16), (128, 512, 1, 1, 8), (256, 512, 1, 2, 16),
             (512, 128, 1, 1, 8), (128, 128, 3, 1, 8), (512, 256, 1, 1, 8), (256, 256, 3, 2, 8), (256, 1024, 1, 1, 4),
             (512, 1024, 1, 2, 8), (1024, 256, 1, 1, 4), (256, 256, 3, 1, 4), (1024, 128, 3, 1, 4)]
EXTRA_CONVS = [(32, 32, 3, 1, 64), (32, 128, 1, 1, 64), (64, 64, 3, 2, 64), (16, 32, 3, 1, 8), (48, 96, 3, 2, 16),
               (16, 64, 1, 1, 4), (96, 96, 1, 2, 4)]


def bits16(x):
    return x.detach().contiguous().view(torch.int16)


def guarded(n, dtype, fill=float("nan")):
    buf = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device=DEV)
    return buf, buf[GUARD:GUARD + n]


def int_tensor(shape, seed, lo=-1, hi=1):
    return synth.det_randint(shape, seed, 3, lo, hi).to(DEV)


def raw_conv(x, w, stride, groups, sentinel=-7.0):
    """bb_conv2d on NaN-guarded copies of x (N, H, W, Cin) and w (Cout, R, R, Cin), into a sentinel-guarded y ->
    (y, stats, y buffer, stats buffer)"""
    dt = x.dtype
    N, H, W, Cin = x.shape
    Cout, Rk = w.shape[0], w.shape[1]
    pad = (Rk - 1) // 2
    Ho, Wo = (H + 2 * pad - Rk) // stride + 1, (W + 2 * pad - Rk) // stride + 1
    xb, xv = guarded(x.numel(), dt)
    xv.copy_(x.reshape(-1))
    wb, wv = guarded(w.numel(), dt)
    wv.copy_(w.reshape(-1))
    yb, yv = guarded(N * Ho * Wo * Cout, dt, sentinel)
    ns = CK.stats_len(N, Ho, Wo, Cout, groups, CK.CONV_TM) * 4
    sb, sv = guarded(ns, torch.float32, sentinel)
    _lib.check(_lib.load().bb_conv2d(xv.data_ptr(), wv.data_ptr(), N, H, W, Cin, Cout, Rk, stride, groups,
                                     yv.data_ptr(), sv.data_ptr(), K._stream()), "bb_conv2d")
    return yv.view(N, Ho, Wo, Cout), CK.Partials(sv.view(-1, 4), CK.CONV_TM, groups), yb, sb


def conv_ref64(x, w, stride):
    return F.conv2d(x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2), stride=stride,
                    padding=(w.shape[1] - 1) // 2).permute(0, 2, 3, 1)


def check_guards(buf, sentinel=-7.0):
    assert bool((buf[:GUARD] == sentinel).all()) and bool((buf[-GUARD:] == sentinel).all())


# ----------------------------------------------------------------------------------------------------- bb_conv2d
@pytest.mark.parametrize("case", NET_CONVS + EXTRA_CONVS, ids=lambda c: "x".join(map(str, c)))
@pytest.mark.parametrize("n", [1, 3])
def test_conv_bit_exact_on_integers(case, n):
    """integer operands in {-1, 0, 1}: every fp32 partial sum is an exact integer below 2^11, so the fp16 output must
    equal the fp64 convolution bit for bit; n = 3 makes tiles span images and leaves a partial last tile"""
    Cin, Cout, Rk, stride, H = case
    x = int_tensor((n, H, H, Cin), 1000 + Cin + H).half()
    w = int_tensor((Cout, Rk, Rk, Cin), 2000 + Cout).half()
    groups = 1 if (Cin, Rk) == (1024, 3) or Cout == 96 else 16
    y, p, yb, sb = raw_conv(x, w, stride, groups)
    ref = conv_ref64(x, w, stride)
    assert ref.abs().max() < 2048
    assert torch.equal(y.double(), ref), (y.double() - ref).abs().max()
    check_guards(yb)
    check_guards(sb)
    assert bool(torch.isfinite(p.stats).all())


def test_conv_rejections():
    x = torch.zeros(1, 8, 8, 64, dtype=torch.float16, device=DEV)
    w = torch.zeros(64, 3, 3, 64, dtype=torch.float16, device=DEV)
    y = torch.zeros(1, 8, 8, 64, dtype=torch.float16, device=DEV)
    st = torch.zeros(4096, dtype=torch.float32, device=DEV)
    lib = _lib.load()
    s = K._stream()
    for args, msg in (((x.data_ptr(), w.data_ptr(), 1, 8, 8, 24, 64, 3, 1, 16), "Cin"),
                      ((x.data_ptr(), w.data_ptr(), 1, 8, 8, 64, 48, 3, 1, 16), "Cout"),
                      ((x.data_ptr(), w.data_ptr(), 1, 8, 8, 64, 64, 5, 1, 16), "1x1 or 3x3"),
                      ((x.data_ptr(), w.data_ptr(), 1, 8, 8, 64, 64, 3, 3, 16), "stride"),
                      ((x.data_ptr() + 2, w.data_ptr(), 1, 8, 8, 64, 64, 3, 1, 16), "aligned"),
                      ((x.data_ptr(), w.data_ptr() + 8, 1, 8, 8, 64, 64, 3, 1, 16), "aligned"),
                      ((x.data_ptr(), w.data_ptr(), 1, 8, 8, 64, 64, 3, 1, 3), "groups")):
        with pytest.raises(_lib.BevbertLibraryError, match=msg):
            _lib.check(lib.bb_conv2d(*args, y.data_ptr(), st.data_ptr(), s), "bb_conv2d")
    with pytest.raises(_lib.BevbertLibraryError, match="aligned"):
        _lib.check(lib.bb_conv2d(x.data_ptr(), w.data_ptr(), 1, 8, 8, 64, 64, 3, 1, 16, y.data_ptr() + 4,
                                 st.data_ptr(), s), "bb_conv2d")


# ------------------------------------------------------------------------------------------ GroupNorm partials, apply
def gn64(y, groups, gamma, beta):
    """fp64 GroupNorm of the stored NHWC tensor y"""
    return F.group_norm(y.double().permute(0, 3, 1, 2), groups, gamma.double(), beta.double(), 1e-5).permute(0, 2, 3, 1)


def gn_bound(ref):
    """fp16 output rounding (2^-11 relative) plus the fp32 statistics and affine (well below 1e-4 at these scales)"""
    return ref.abs() * 2.0 ** -10 + 1e-4


def affine(C, seed):
    return (synth.det_uniform((C,), seed, 1, 0.8, 1.2).to(DEV), synth.det_uniform((C,), seed, 2, -0.1, 0.1).to(DEV))


# (Cin, Cout, R, stride, H, groups): the group shapes of the network (2 .. 64 channels per group, one group of 128)
GN_CASES = [(32, 32, 3, 1, 32, 16), (32, 128, 1, 1, 32, 16), (64, 256, 1, 1, 16, 16), (128, 512, 1, 1, 8, 16),
            (256, 1024, 1, 1, 4, 16), (1024, 128, 3, 1, 4, 1), (64, 64, 3, 2, 32, 16)]


@pytest.mark.parametrize("case", GN_CASES, ids=lambda c: "x".join(map(str, c)))
@pytest.mark.parametrize("n", [1, 5])
def test_groupnorm_apply_variants(case, n):
    Cin, Cout, Rk, stride, H, groups = case
    x = synth.det_uniform((n, H, H, Cin), 7, Cin, -1.0, 1.0).to(DEV).half()
    w = (synth.det_uniform((Cout, Rk, Rk, Cin), 8, Cout, -1.0, 1.0) * (Rk * Rk * Cin) ** -0.5).to(DEV).half()
    y, p = CK.conv2d(x, w, stride, groups)
    g1, b1 = affine(Cout, 1)
    ref = gn64(y, groups, g1, b1)
    out = CK.groupnorm_apply(y, p, g1, b1, 1e-5)
    r = ref.clamp_min(0)
    assert bool(((out.double() - r).abs() <= gn_bound(r)).all()), (out.double() - r).abs().max()
    # + identity
    idn = synth.det_uniform(tuple(y.shape), 9, 1, -1.0, 1.0).to(DEV).half()
    out = CK.groupnorm_apply(y, p, g1, b1, 1e-5, CK.GN_ADD_RELU, identity=idn)
    r = (ref + idn.double()).clamp_min(0)
    assert bool(((out.double() - r).abs() <= gn_bound(r)).all())
    # + a second normalized tensor with its own partials and affine
    x2 = synth.det_uniform(tuple(x.shape), 10, 1, -1.0, 1.0).to(DEV).half()
    y2, p2 = CK.conv2d(x2, w, stride, groups)
    g2, b2 = affine(Cout, 2)
    out = CK.groupnorm_apply(y, p, g1, b1, 1e-5, CK.GN_ADD_NORM_RELU, x2=y2, p2=p2, gamma2=g2, beta2=b2)
    r = (ref + gn64(y2, groups, g2, b2)).clamp_min(0)
    assert bool(((out.double() - r).abs() <= gn_bound(r)).all())
    # fp32 NCHW output (the compression's)
    out = CK.groupnorm_apply(y, p, g1, b1, 1e-5, out_f32=True)
    r = ref.clamp_min(0).permute(0, 3, 1, 2)
    assert out.dtype == torch.float32 and out.shape == r.shape
    assert bool(((out.double() - r).abs() <= r.abs() * 1e-5 + 1e-5).all()), (out.double() - r).abs().max()
    # max-pool variant
    out = CK.groupnorm_apply(y, p, g1, b1, 1e-5, CK.GN_RELU_MAXPOOL)
    r = F.max_pool2d(ref.clamp_min(0).permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert out.shape == r.shape
    assert bool(((out.double() - r).abs() <= gn_bound(r)).all())
    # deterministic: a repeat of the conv and the normalisation gives the same bits
    y_, p_ = CK.conv2d(x, w, stride, groups)
    assert torch.equal(bits16(y_), bits16(y))
    a1 = CK.groupnorm_apply(y, p, g1, b1, 1e-5, out_f32=True)
    a2 = CK.groupnorm_apply(y_, p_, g1, b1, 1e-5, out_f32=True)
    assert torch.equal(a1.view(torch.int32), a2.view(torch.int32))


# ------------------------------------------------------------------------------------------------------ stem
@pytest.mark.parametrize("shape", [(3, 256, 256), (2, 256, 341), (1, 30, 18)])
def test_stem_against_fp64(shape):
    n, h, w = shape
    depth = synth.depth_images(n, 4, h, w).to(DEV)
    wt = (synth.det_uniform((32, 1, 7, 7), 5, 0, -1.0, 1.0) * 0.2).to(DEV)
    ref = F.conv2d(F.avg_pool2d(depth.double().permute(0, 3, 1, 2), 2), wt.double(), stride=2, padding=3)
    ref = ref.permute(0, 2, 3, 1)
    y, p = CK.depth_stem(depth, wt, 16)
    assert y.shape == ref.shape and y.dtype == torch.float16
    assert bool(((y.double() - ref).abs() <= ref.abs() * 2.0 ** -11 + 1e-5).all()), (y.double() - ref).abs().max()
    # a strided (NCHW-permuted) depth gives the same bits
    y2, _ = CK.depth_stem(depth.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1), wt, 16)
    assert torch.equal(bits16(y2), bits16(y))
    g, b = affine(32, 3)
    out = CK.groupnorm_apply(y, p, g, b, 1e-5, CK.GN_RELU_MAXPOOL)
    r = F.max_pool2d(gn64(y, 16, g, b).clamp_min(0).permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert bool(((out.double() - r).abs() <= gn_bound(r)).all())
    prev = K.set_precision(True)
    try:
        y32, _ = CK.depth_stem(depth, wt, 16)
    finally:
        K.set_precision(prev)
    assert y32.dtype == torch.float32
    assert bool(((y32.double() - ref).abs() <= ref.abs() * 1e-6 + 1e-6).all()), (y32.double() - ref).abs().max()


# ---------------------------------------------------------------------------------------------- whole encoder
@pytest.fixture(scope="module")
def state():
    return synth.depth_encoder_state(SEED)


def encoder(state, h=256, w=256):
    m = D.depth_encoder(h, w)
    m.load_state_dict(state)
    return m.to(DEV).requires_grad_(False).eval()


@pytest.mark.parametrize("n", [12, 48, 96])
def test_encoder_against_oracle(state, n):
    depth = synth.depth_images(n, 40 + n).to(DEV)
    sd = {k: v.to(DEV) for k, v in state.items()}
    ref = R.forward(sd, depth, torch.float64)
    e16 = rel_l2(R.forward_fp16(sd, depth), ref)
    enc = encoder(state)
    out = D.DepthTower(enc).encode(depth)
    assert out.dtype == torch.float32 and out.shape == (n, 128, 4, 4) and out.is_contiguous()
    with torch.autocast("cuda", dtype=torch.float16):
        mod = enc({"depth": depth})
    assert mod.dtype == out.dtype and mod.shape == out.shape
    e = rel_l2(out, ref)
    prev = K.set_precision(True)
    try:
        out32 = D.DepthTower(encoder(state)).encode(depth)
    finally:
        K.set_precision(prev)
    e32 = rel_l2(out32, ref)
    print("n=%d: fp32 arm %.3e | fp16 %.3e | fp16 autocast reference %.3e | restated module under autocast %.3e" % (
        n, e32, e, e16, rel_l2(mod, ref)))
    assert e32 <= 1e-3, e32
    assert e <= max(1e-2, 2.5 * e16), (e, e16)


def test_non_square_depth(state):
    depth = synth.depth_images(3, 9, 256, 341).to(DEV)
    enc = encoder(state, 256, 341)
    ref = R.forward({k: v.to(DEV) for k, v in state.items()}, depth, torch.float64)
    out = D.DepthTower(enc).encode(depth)
    assert out.shape == ref.shape == (3, 128, 4, 6)
    assert rel_l2(out, ref) <= 1e-2


def test_autocast_and_deterministic_change_no_bit(state):
    depth = synth.depth_images(24, 5).to(DEV)
    tower = D.DepthTower(encoder(state))
    base = tower.encode(depth)
    with torch.autocast("cuda", dtype=torch.float16):
        a = tower.encode(depth)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        d = tower.encode(depth)
    finally:
        torch.use_deterministic_algorithms(prev)
    for t in (a, d, tower.encode(depth)):
        assert torch.equal(t.view(torch.int32), base.view(torch.int32))


def test_grad_with_trainable_parameter_raises(state):
    enc = encoder(state)
    enc.compression[1].weight.requires_grad_(True)
    with pytest.raises(RuntimeError, match="forward only"):
        D.DepthTower(enc).encode(synth.depth_images(1, 1).to(DEV))


class _Wrapper(torch.nn.Module):
    """VlnResnetDepthEncoder's attribute layout: .visual_encoder"""

    def __init__(self, enc):
        super().__init__()
        self.visual_encoder = enc

    def forward(self, observations):
        return self.visual_encoder(observations)


def test_install_replay(state):
    enc = encoder(state)
    wrap = _Wrapper(enc).eval()
    eager = D.DepthTower(encoder(state))
    replay = graphs.install_ce_depth_encoder(wrap)
    seq = [96, 84, 12, 96]
    for i, n in enumerate(seq):
        depth = synth.depth_images(n, 60 + i).to(DEV)
        got = wrap({"depth": depth})
        assert replay.launches("depth", {"depth": depth}) is not None
        assert torch.equal(got.view(torch.int32), eager.encode(depth).view(torch.int32)), n
    # a load_state_dict between calls is seen, replayed and eager
    new = synth.depth_encoder_state(SEED + 1)
    enc.load_state_dict(new)
    eager2 = D.DepthTower(encoder(new))
    depth = synth.depth_images(12, 70).to(DEV)
    got = wrap({"depth": depth})
    assert torch.equal(got.view(torch.int32), eager2.encode(depth).view(torch.int32))
    with torch.enable_grad():
        got = wrap({"depth": depth})        # frozen encoder: grad-enabled eval calls replay too
    assert torch.equal(got.view(torch.int32), eager2.encode(depth).view(torch.int32))
    wrap.train()
    got = wrap({"depth": depth})
    assert torch.equal(got.view(torch.int32), eager2.encode(depth).view(torch.int32))


def test_depth_encoder_into_waypoint_predictor(state):
    """depth encoder -> J7 predictor -> bb_waypoint_nms: the picks equal the fp64 chain's wherever the fp64 margin
    exceeds 4x the logit error"""
    import test_ce_waypoint_gpu as TW
    from oracle import ce_waypoint_ref as RW
    wstate = synth.waypoint_state(TW.SEED)
    wp = TW.predictor(wstate)
    n = 48
    depth = synth.depth_images(n, 80).to(DEV)
    ref_feats = R.forward({k: v.to(DEV) for k, v in state.items()}, depth, torch.float64)
    ref = RW.forward({k: v.to(DEV) for k, v in wstate.items()}, ref_feats, torch.float64)
    feats = D.DepthTower(encoder(state)).encode(depth)
    logits = wp(torch.zeros(n, 512, device=DEV), feats)
    checked, unsure = TW.check_picks(logits, ref)
    print("depth -> waypoint chain: logits rel err %.3e, NMS rounds checked %d, unchecked %d" % (
        rel_l2(logits, ref), checked, unsure))
    assert checked > 0
