"""GPU checks of the VLN-CE waypoint predictor and its heatmap NMS: bb_waypoint_nms bit-identical to the reference
(tests/golden/small_ce_waypoint.pt) and to oracle/ce_waypoint_ref.py on seeded sweeps, with NaN in unread memory and
untouched guards; the predictor's logits against the oracle in both arms; the NMS picks of the kernel logits against
those of fp64 logits; autocast and deterministic mode; and the install with graph replay."""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from helpers import rel_l2  # noqa: E402
from bevbert_b200 import _lib, graphs, synth  # noqa: E402
from bevbert_b200 import kernels as K  # noqa: E402
from bevbert_b200.model import waypoint as WP  # noqa: E402
from oracle import ce_waypoint_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 21
GOLDEN = os.path.join(ROOT, "tests", "golden", "small_ce_waypoint.pt")


def bits(x):
    return x.detach().cpu().contiguous().view(torch.int32)


# --------------------------------------------------------------------------------------------- bb_waypoint_nms
def test_nms_golden_cases_bit_identical():
    g = torch.load(GOLDEN)
    for name, c in g["nms"].items():
        got = WP.nms(c["pred"].to(DEV), max_predictions=c["k"], sigma=c["sigma"])
        assert got.shape == c["pred"].shape and got.dtype == torch.float32
        assert torch.equal(bits(got), bits(c["out"])), name


def sweep_map(B, H, W, seed, kind):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, 1, H, W, generator=g)
    if kind == "ties":                                  # few distinct values: ties everywhere
        x = torch.floor(x * 4) / 4
    elif kind == "signed":                              # both signs and both zeros
        x = torch.floor((x - 0.5) * 8) / 8
        x[torch.rand(B, 1, H, W, generator=g) < 0.2] = -0.0
    elif kind == "nan":
        x = x - 0.3
        x[torch.rand(B, 1, H, W, generator=g) < 0.002] = float("nan")
        x[torch.rand(B, 1, H, W, generator=g) < 0.002] = float("inf")
    elif kind == "softmax":                             # the policy's heatmap of random logits
        x = torch.softmax((torch.randn(B, H * W, generator=g) * 2), dim=1).view(B, 1, H, W)
    return x


SWEEP = [(122, 12, (7.0, 5.0), 5), (122, 12, (3.0, 2.0), 12), (24, 48, (1.0, 1.0), 10), (7, 5, (1.5, 0.5), 4),
         (64, 128, (10.0, 4.0), 6), (1, 1, (0.0, 0.0), 3), (13, 7, (0.3, 2.7), 40), (90, 90, (5.0, 7.0), 8)]


@pytest.mark.parametrize("B", [1, 8, 96])
@pytest.mark.parametrize("kind", ["uniform", "ties", "signed", "nan", "softmax"])
def test_nms_sweep_bit_identical(B, kind):
    for i, (H, W, sigma, k) in enumerate(SWEEP):
        pred = sweep_map(B, H, W, 1000 * B + 10 * i + len(kind), kind)
        got = WP.nms(pred.to(DEV), k, sigma)
        ref = R.nms(pred, k, sigma)
        assert torch.equal(bits(got), bits(ref)), (H, W, sigma, k)


def test_nms_reads_and_writes_only_its_rows():
    """NaN in device memory just past the input must not be read; the guards around the output stay untouched"""
    B, H, W = 8, 122, 12
    n = B * H * W
    pred = sweep_map(B, H, W, 7, "uniform")
    src = torch.full((n + 4096,), float("nan"), device=DEV)
    src[:n] = pred.reshape(-1).to(DEV)
    out = torch.full((n + 2 * 64,), float("nan"), device=DEV)
    init = out.clone()
    lib = _lib.load()
    _lib.check(lib.bb_waypoint_nms(src.data_ptr(), B, H, W, 7.0, 5.0, 5, out[64:].data_ptr(), K._stream()), "nms")
    assert torch.equal(bits(out[64:64 + n]), bits(R.nms(pred, 5, (7.0, 5.0)).reshape(-1)))
    assert torch.equal(bits(out[:64]), bits(init[:64])) and torch.equal(bits(out[64 + n:]), bits(init[64 + n:]))
    # a strided input is made contiguous first and gives the same map
    wide = torch.full((B, 1, H, W + 4), float("nan"), device=DEV)
    wide[..., :W] = pred.to(DEV)
    assert torch.equal(bits(WP.nms(wide[..., :W], 5, (7.0, 5.0))), bits(R.nms(pred, 5, (7.0, 5.0))))
    # B = 0 and max_predictions <= 0, as range() treats them
    assert WP.nms(torch.zeros(0, 1, H, W, device=DEV), 5, (7.0, 5.0)).shape == (0, 1, H, W)
    assert torch.equal(bits(WP.nms(pred.to(DEV), -2, (7.0, 5.0))), bits(torch.zeros(B, 1, H, W)))


def test_nms_rejections():
    x = torch.rand(2, 1, 122, 12, device=DEV)
    lib = _lib.load()
    with pytest.raises(NotImplementedError):
        WP.nms(x, 5, (7.0, 5.0), gaussian=True)
    with pytest.raises(TypeError):
        WP.nms(x.double(), 5, (7.0, 5.0))
    with pytest.raises(RuntimeError, match="CUDA"):
        WP.nms(x.cpu(), 5, (7.0, 5.0))
    with pytest.raises(ValueError):
        WP.nms(torch.rand(1, 1, 91, 91, device=DEV), 5, (7.0, 5.0))
    with pytest.raises(ValueError):
        WP.nms(x[:, 0], 5, (7.0, 5.0))
    with pytest.raises(_lib.BevbertLibraryError, match="positive"):
        WP.nms(torch.rand(1, 1, 0, 12, device=DEV), 5, (7.0, 5.0))
    st = K._stream()
    for args, msg in (((x.data_ptr(), 2, 91, 91, 7.0, 5.0, 5, x.data_ptr() + 4 * 2 * 91 * 91), "8192"),
                      ((x.data_ptr(), 2, 122, 12, 7.0, 5.0, 5, x.data_ptr() + 4 * 100), "overlap"),
                      ((x.data_ptr() + 2, 1, 122, 12, 7.0, 5.0, 5, x.data_ptr() + 4 * 2000), "aligned"),
                      ((x.data_ptr(), 1, 122, 12, 7.0, 5.0, -1, x.data_ptr() + 4 * 2000), "non-negative")):
        with pytest.raises(_lib.BevbertLibraryError, match=msg):
            _lib.check(lib.bb_waypoint_nms(*args, st), "bb_waypoint_nms")


# --------------------------------------------------------------------------------------------- predictor
@pytest.fixture(scope="module")
def state():
    return synth.waypoint_state(SEED)


def predictor(state):
    m = WP.BinaryDistPredictor_TRM()
    m.load_state_dict(state)
    return m.to(DEV).requires_grad_(False).eval()


@pytest.fixture(scope="module")
def wp(state):
    return predictor(state)


def feats(n, seed):
    return synth.det_uniform((n, 128, 4, 4), seed, 5, 0.0, 1.0).to(DEV)


def policy_heatmap(logits):
    B = logits.shape[0]
    x = torch.softmax(logits.reshape(B, -1), dim=1).reshape(B, 120, 12)
    return torch.cat((x[:, -1:], x, x[:, :1]), dim=1).unsqueeze(1)


def rounds_fp64(logits64, k=5, sigma=(7.0, 5.0)):
    """the policy's NMS on fp64 logits, per environment and round: the cells picked in rounds 1..r and the logit
    margin of round r, between its pick and the best other unsuppressed cell of a different source cell (a heatmap
    cell's order is its logit's: softmax is monotonic and suppressed cells are 0)"""
    src = torch.cat((torch.arange(1428, 1440), torch.arange(1440), torch.arange(12)))   # wrapped cell -> logit cell
    res = []
    for b in range(logits64.shape[0]):
        lg = logits64[b].reshape(-1).cpu()[src]
        alive = torch.ones(122 * 12, dtype=torch.bool)
        picks, rounds = [], []
        for _ in range(k):
            v = torch.where(alive, lg, torch.full_like(lg, -math.inf))
            ix = int(v.argmax())
            other = torch.where(src == src[ix], torch.full_like(v, -math.inf), v)
            picks.append(ix)
            rounds.append((sorted(set(picks)), float(v[ix] - other.max())))
            alive &= ~R.neighbourhood(torch.tensor([ix]), 122, 12, sigma).reshape(-1)
        res.append(rounds)
    return res


def check_picks(logits, ref):
    """NMS on `logits` picks the cells NMS picks on fp64 `ref` in rounds 1..r, for every r up to the first round whose
    fp64 margin is within 4x the environment's measured logit error -> (rounds checked, rounds left unchecked)"""
    heat = policy_heatmap(logits)
    checked = unsure = 0
    for b, rounds in enumerate(rounds_fp64(ref)):
        err = float((logits[b].double() - ref[b]).abs().max())
        for r, (picks, margin) in enumerate(rounds, 1):
            if margin <= 4 * err:
                unsure += len(rounds) - r + 1
                break
            got = WP.nms(heat[b:b + 1], r, (7.0, 5.0))
            assert sorted(torch.nonzero(got.reshape(-1).cpu()).view(-1).tolist()) == picks, (b, r)
            checked += 1
    return checked, unsure


@pytest.mark.parametrize("n", [12, 48, 96])
def test_predictor_against_oracle(state, wp, n):
    dep = feats(n, 30 + n)
    rgb = torch.zeros(n, 512, device=DEV)
    sd64 = {k: v.to(DEV) for k, v in state.items()}
    ref = R.forward(sd64, dep, torch.float64)
    e16 = rel_l2(R.forward_fp16(sd64, dep), ref)
    out = wp(rgb, dep)
    assert out.dtype == torch.float32 and out.shape == (n // 12, 120, 12)
    e = rel_l2(out, ref)
    prev = K.set_precision(True)
    try:
        out32 = predictor(state)(rgb, dep)
    finally:
        K.set_precision(prev)
    e32 = rel_l2(out32, ref)
    print("n=%d: fp32 arm %.3e | bf16 %.3e | fp16 autocast reference %.3e" % (n, e32, e, e16))
    assert e32 <= 1e-3, e32
    assert e <= max(1e-2, 2.5 * e16), (e, e16)
    # NMS on kernel logits picks the fp64 logits' cells wherever the fp64 margin exceeds 4x the logit error
    for arm, logits in (("bf16", out), ("fp32 arm", out32)):
        checked, unsure = check_picks(logits, ref)
        print("n=%d %s: NMS rounds checked %d, left unchecked (margin within 4x the logit error) %d" % (
            n, arm, checked, unsure))


def test_fp16_depth_features_are_converted(wp):
    dep = feats(24, 3).half()
    rgb = torch.zeros(24, 512, device=DEV)
    assert torch.equal(bits(wp(rgb, dep)), bits(wp(rgb, dep.float())))


def test_autocast_and_deterministic_change_no_bit(wp):
    dep = feats(48, 6)
    rgb = torch.zeros(48, 512, device=DEV)
    a = wp(rgb, dep)
    with torch.autocast("cuda", dtype=torch.float16):
        b = wp(rgb, dep)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        c = wp(rgb, dep)
        d = wp(rgb, dep)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.equal(bits(a), bits(x)) for x in (b, c, d))
    h = policy_heatmap(a)
    with torch.autocast("cuda", dtype=torch.float16):
        assert torch.equal(bits(WP.nms(h, 5, (7.0, 5.0))), bits(R.nms(h, 5, (7.0, 5.0))))


def test_training_mode_and_grad_raise(state):
    m = predictor(state)
    dep, rgb = feats(12, 1), torch.zeros(12, 512, device=DEV)
    m.train()
    with pytest.raises(RuntimeError, match="eval mode"):
        m(rgb, dep)
    m.eval()
    m.vis_classifier[0].weight.requires_grad_(True)
    with pytest.raises(RuntimeError, match="forward only"):
        m(rgb, dep)
    with torch.no_grad():
        m(rgb, dep)


# --------------------------------------------------------------------------------------------- install + replay
@pytest.mark.parametrize("wrap", [False, True])
def test_install_replay(state, wrap):
    ref_mod = predictor(state)                          # stands in for the reference instance: same layout
    outer = torch.nn.DataParallel(ref_mod, device_ids=[0], output_device=0) if wrap else ref_mod
    before = {k: v.clone() for k, v in outer.state_dict().items()}
    replay = graphs.install_ce_waypoint_predictor(outer)
    after = outer.state_dict()
    assert list(after) == list(before) and all(torch.equal(after[k], v) for k, v in before.items())
    # expected outputs from a second module: runners re-home the packed q / k / v biases of the module they run
    fresh = WP.WaypointRunner(predictor(state))
    obs = {n: feats(n, 40 + n) for n in (96, 84, 12)}
    for i, n in enumerate([96, 84, 12, 96, 12]):
        dep, rgb = obs[n], torch.zeros(n, 512, device=DEV)
        if i % 2:
            got = outer(rgb, dep)                       # grad enabled: a frozen predictor replays too
        else:
            with torch.no_grad():
                got = outer(rgb, dep)
        assert replay.launches("waypoint", {"depth_feats": dep}) is not None
        assert torch.equal(bits(got), bits(fresh(rgb, dep))), n
        ent = replay.entries[graphs._bucket(graphs.CE_WAYPOINT_DIMS, "waypoint", {"depth_feats": dep})]
        assert got.data_ptr() != ent["out"].data_ptr()
    assert len(replay.entries) == 3
    # load_state_dict between calls is seen under replay
    rgb = torch.zeros(12, 512, device=DEV)
    old = outer(rgb, obs[12])
    outer.load_state_dict({k: (v * 1.25 if k.endswith(("vis_classifier.2.weight", "intermediate.dense.weight",
                                                          "query.bias")) else v) for k, v in before.items()})
    new = outer(rgb, obs[12])
    assert not torch.equal(old, new)
    changed = WP.BinaryDistPredictor_TRM()
    changed.load_state_dict(ref_mod.state_dict())
    changed = changed.to(DEV).requires_grad_(False).eval()
    assert torch.equal(bits(new), bits(changed(rgb, obs[12])))
    assert len(replay.entries) == 3
    outer.train()
    with pytest.raises(RuntimeError, match="eval mode"):
        outer(rgb, obs[12])
