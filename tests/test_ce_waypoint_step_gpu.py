"""GPU checks of the VLN-CE policy's waypoint step: bb_ce_view_stack bit-exact (grid against the CUDA
AdaptiveAvgPool2d((14, 14))), bb_ce_waypoint_candidates against torch softmax + wrap + bb_waypoint_nms + nonzero, the
installed step against the reference branch (oracle/ce_waypoint_step_ref.py) around the same eager towers, replay
across batch sizes and weight changes, fallbacks, and the single host synchronisation per step."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import ce_waypoint_step_cases as C  # noqa: E402
from bevbert_b200 import _lib, graphs, synth  # noqa: E402
from bevbert_b200.model import ce_waypoint_step as CS  # noqa: E402
from bevbert_b200.model import waypoint as WP  # noqa: E402
from oracle import ce_waypoint_step_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 31


def bits(x):
    return x.detach().contiguous().view(torch.int32)


def ulps(a, b):
    """elementwise distance in fp32 ulps (same-sign finite values)"""
    return (bits(a).long() - bits(b).long()).abs()


def ref_stack(obs):
    depth = torch.zeros_like(obs["depth"]).repeat(12, 1, 1, 1)
    rgb = torch.zeros_like(obs["rgb"]).repeat(12, 1, 1, 1)
    for a, (r, d) in enumerate(CS.view_pairs(obs)):
        for b in range(obs[d].shape[0]):
            depth[(12 - a) % 12 + 12 * b] = obs[d][b]
            rgb[(12 - a) % 12 + 12 * b] = obs[r][b]
    grid = torch.flatten(F.adaptive_avg_pool2d(depth.permute(0, 3, 1, 2), (14, 14)), 1)
    return rgb, depth, grid


# --------------------------------------------------------------------------------------------- bb_ce_view_stack
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("crop", [False, True])
@pytest.mark.parametrize("depth_hw", [(256, 256), (240, 320)])
def test_view_stack_bit_exact(B, crop, depth_hw):
    obs = C.observations(B, 100 + B, DEV, crop=crop, depth_hw=depth_hw)
    if B == 3:          # order-sensitive grid sums: magnitudes over 2^-20 .. 2^20
        g = torch.Generator().manual_seed(5)
        for _, d in CS.view_pairs(obs):
            e = torch.randint(-20, 21, obs[d].shape, generator=g).float().to(DEV)
            obs[d].mul_(torch.exp2(e))
    pairs, geom = CS.covered(obs, 224, torch.device(DEV, torch.cuda.current_device()))
    assert geom == (B, 224, 224) + depth_hw
    table = CS.view_table(obs, pairs).to(DEV)
    rgb, depth, grid = CS.view_stack(table, B, (224, 224), depth_hw, DEV)
    r_rgb, r_depth, r_grid = ref_stack(obs)
    assert torch.equal(rgb, r_rgb)
    assert torch.equal(bits(depth), bits(r_depth))
    assert torch.equal(bits(grid), bits(r_grid))


def test_view_stack_guards_and_rejections():
    B, (Hd, Wd) = 2, (64, 48)
    obs = C.observations(B, 7, DEV, depth_hw=(Hd, Wd))
    pairs, _ = CS.covered(obs, 224, torch.device(DEV, torch.cuda.current_device()))
    table = CS.view_table(obs, pairs).to(DEV)
    n, pad = 12 * B, 64
    dep = torch.full((n * Hd * Wd + 2 * pad,), -7.0, device=DEV)
    grid = torch.full((n * 196 + 2 * pad,), -7.0, device=DEV)
    rgb = torch.full((n * 224 * 224 * 3 + 2 * pad,), 77, dtype=torch.uint8, device=DEV)
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.bb_ce_view_stack(table.data_ptr(), B, 224, 224, Hd, Wd, rgb[pad:].data_ptr(), dep[pad:].data_ptr(),
                                    grid[pad:].data_ptr(), stream), "bb_ce_view_stack")
    for buf, fill in ((dep, -7.0), (grid, -7.0), (rgb, 77)):
        assert bool((buf[:pad] == fill).all()) and bool((buf[-pad:] == fill).all())
    r_rgb, r_depth, r_grid = ref_stack(obs)
    assert torch.equal(bits(grid[pad:-pad]), bits(r_grid.reshape(-1)))
    args = [table.data_ptr(), B, 224, 224, Hd, Wd, rgb.data_ptr(), dep[pad:].data_ptr(), grid[pad:].data_ptr(), stream]
    for i, bad in ((1, 0), (4, 13), (5, 0), (0, None), (6, None), (7, dep.data_ptr() + 2), (8, dep[pad:].data_ptr())):
        a = list(args)
        a[i] = bad
        assert lib.bb_ce_view_stack(*a) != 0, i
    with pytest.raises(ValueError):
        CS.view_stack(table[:12], B, (224, 224), (Hd, Wd), DEV)


# ------------------------------------------------------------------------------------ bb_ce_waypoint_candidates
def ref_candidates(logits, rgb_vec, dep):
    B = logits.shape[0]
    x = torch.softmax(logits.reshape(B, -1), dim=1).reshape(B, 120, 12)
    heat = torch.cat((x[:, -1:], x, x[:, :1]), dim=1).unsqueeze(1)
    out = WP.nms(heat, 5, (7.0, 5.0)).squeeze(1)[:, 1:-1]
    rgb_r = rgb_vec.reshape(B, 12, 512)
    rgb_feats = torch.cat([rgb_r[:, 0:1], torch.flip(rgb_r[:, 1:], [1])], dim=1)
    dep_r = dep.reshape(B, 12, 128, 4, 4)
    dep_feats = torch.flatten(F.adaptive_avg_pool2d(torch.cat([dep_r[:, 0:1], torch.flip(dep_r[:, 1:], [1])], 1),
                                                    (1, 1)), 2)
    return x, out, rgb_feats, dep_feats


@pytest.mark.parametrize("B", [1, 5, 8, 64])
@pytest.mark.parametrize("kind", ["seeded", "constructed"])
def test_candidates_against_torch(B, kind):
    g = torch.Generator().manual_seed(B)
    logits = (torch.randn(B, 120, 12, generator=g) * 3 if kind == "seeded" else C.constructed_logits(B, B)).to(DEV)
    rgb_vec = torch.randn(12 * B, 512, generator=g).to(DEV)
    dep = torch.rand(12 * B, 128, 4, 4, generator=g).mul(torch.exp2(torch.randint(-8, 9, (12 * B, 128, 4, 4),
                                                                                  generator=g).float())).to(DEV)
    got = CS.waypoint_candidates(logits, rgb_vec, dep, prob=True)
    prob, out, rgb_feats, dep_feats = ref_candidates(logits, rgb_vec, dep)
    du = int(ulps(got["prob"], prob).max())
    print("softmax vs torch: max %d ulp" % du)
    assert du <= 16
    picks = got["picks"].cpu()
    assert torch.equal(bits(got["pano_rgb"]), bits(rgb_feats))
    assert torch.equal(bits(got["pano_depth"]), bits(dep_feats))
    for b in range(B):
        nz = out[b].nonzero().cpu()
        k = int(picks[b, 10])
        assert k == nz.shape[0], b
        assert picks[b, 0:2 * k].view(k, 2).long().tolist() == nz.tolist(), b
        img = 12 - (nz[:, 0].numpy() + 5) // 10
        img[img == 12] = 0
        cand = np.zeros(12, dtype=bool)
        cand[img] = True
        assert int(picks[b, 11]) == k + 12 - int(cand.sum())
        rows_r = torch.cat([got["pano_rgb"][b, img], got["pano_rgb"][b, torch.from_numpy(~cand).to(DEV)]])
        rows_d = torch.cat([got["pano_depth"][b, img], got["pano_depth"][b, torch.from_numpy(~cand).to(DEV)]])
        L = rows_r.shape[0]
        assert torch.equal(bits(got["cand_rgb"][b, :k]), bits(rgb_feats[b, img]))
        assert torch.equal(bits(got["cand_depth"][b, :k]), bits(got["pano_depth"][b, img]))
        assert not bool(got["cand_rgb"][b, k:].any()) and not bool(got["cand_depth"][b, k:].any())
        assert torch.equal(bits(got["rgb_fts"][b, :L]), bits(rows_r))
        assert torch.equal(bits(got["dep_fts"][b, :L]), bits(rows_d))
        assert not bool(got["rgb_fts"][b, L:].any()) and not bool(got["dep_fts"][b, L:].any())
    if kind == "constructed" and B >= 5:
        counts = picks[:, 10].tolist()
        assert min(counts) < 5 and 1 in counts


def test_candidates_rejections():
    x = torch.zeros(2, 120, 12, device=DEV)
    with pytest.raises(ValueError):
        CS.waypoint_candidates(x, torch.zeros(23, 512, device=DEV), torch.zeros(24, 128, 4, 4, device=DEV))
    with pytest.raises(TypeError):
        CS.waypoint_candidates(x.double(), torch.zeros(24, 512, device=DEV), torch.zeros(24, 128, 4, 4, device=DEV))
    lib = _lib.load()
    args = [x.data_ptr(), x.data_ptr(), x.data_ptr(), 0] + [x.data_ptr()] * 8 + [None]
    assert lib.bb_ce_waypoint_candidates(*args) != 0
    args[3] = 2
    args[4] = None
    assert lib.bb_ce_waypoint_candidates(*args) != 0


# ------------------------------------------------------------------------------------------------ whole step
@pytest.fixture(scope="module")
def setup():
    net = C.Net(SEED, DEV)
    wp = C.predictor(SEED, DEV)
    step = graphs.install_ce_waypoint_step(net)
    trainer = type("Trainer", (), {})()
    trainer._vp_feature_variable = lambda obs: R.vp_feature_variable(obs, DEV)
    graphs.install_ce_vp_features(trainer)
    # the reference runs on its own modules: two weight caches over one module would move its packed biases back
    # and forth, and every move drops the step's graphs
    REF["net"], REF["wp"] = C.Net(SEED, DEV), C.predictor(SEED, DEV)
    return net, wp, step, trainer


REF = {}


def reference(net, wp, obs):
    """the reference branch on the twin modules of `net` / `wp` (same weights)"""
    if "wp_twin" not in REF:
        REF["wp_twin"] = C.predictor(SEED, DEV)
    REF["wp_twin"].load_state_dict(wp.state_dict())
    net_ref = REF["net"]
    net_ref.load_state_dict(net.state_dict())
    return type(net_ref).forward(net_ref, mode="waypoint", waypoint_predictor=REF["wp_twin"], observations=obs,
                                 in_train=False)


def check_same(got, ref, depth_ulps=0):
    assert isinstance(got, CS.StepOutputs) and list(got.keys()) == list(ref.keys())
    for k, r in ref.items():
        g = got[k]
        assert type(g) is type(r), k
        if isinstance(r, list):
            assert len(g) == len(r), k
            for a, b in zip(g, r):
                assert type(a) is type(b), k
                if isinstance(b, torch.Tensor):
                    assert a.dtype == b.dtype and a.device == b.device and a.shape == b.shape, k
                    if k == "cand_depth":
                        assert (int(ulps(a, b).max()) if a.numel() else 0) <= depth_ulps, k
                    else:
                        assert torch.equal(bits(a), bits(b)), k
                elif isinstance(b, np.ndarray):
                    assert a.dtype == b.dtype and np.array_equal(a, b), k
                else:
                    assert a == b, k
        elif isinstance(r, torch.Tensor):
            assert g.dtype == r.dtype and g.device == r.device and g.shape == r.shape, k
            if k == "pano_depth":
                assert int(ulps(g, r).max()) <= depth_ulps, k
            elif r.dtype == torch.float32:
                assert torch.equal(bits(g), bits(r)), k
            else:
                assert torch.equal(g, r), k
        else:
            assert np.array_equal(g, r) and g.dtype == r.dtype, k


def check_vp(trainer, got, ref):
    v, r = trainer._vp_feature_variable(got), R.vp_feature_variable(ref, DEV)
    assert list(v.keys()) == list(r.keys())
    for k in r:
        assert v[k].dtype == r[k].dtype and v[k].shape == r[k].shape and v[k].device == r[k].device, k
        if v[k].dtype == torch.float32:
            assert torch.equal(bits(v[k]), bits(r[k])), k
        else:
            assert torch.equal(v[k], r[k]), k


def test_step_replay_against_reference_branch(setup):
    net, wp, step, trainer = setup
    with torch.no_grad():
        for i, B in enumerate([8, 5, 1, 8]):
            obs = C.observations(B, 200 + i, DEV, crop=bool(i % 2))
            calls = net.calls
            got = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)
            assert net.calls == calls, "the step must not run the original forward"
            ref = reference(net, wp, obs)
            check_same(got, ref)
            check_vp(trainer, got, ref)
        assert len(step.replay.entries) == 3 and all(e["graph"] is not None for e in step.replay.entries.values())


def test_step_sees_weight_changes(setup):
    net, wp, step, trainer = setup
    obs = C.observations(4, 300, DEV)
    with torch.no_grad():
        for load in (lambda: net.rgb_encoder.model.visual.load_state_dict(synth.clip_visual_state(SEED + 1)),
                     lambda: net.depth_encoder.visual_encoder.load_state_dict(synth.depth_encoder_state(SEED + 1)),
                     lambda: wp.load_state_dict(synth.waypoint_state(SEED + 1))):
            load()
            got = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)
            check_same(got, reference(net, wp, obs))
        # a different predictor module rebuilds the step
        wp2 = C.predictor(SEED + 2, DEV)
        got = net(mode="waypoint", waypoint_predictor=torch.nn.DataParallel(wp2), observations=obs, in_train=False)
        check_same(got, reference(net, wp2, obs))


def test_step_bucket_without_graph_returns_reference_dict(setup):
    """a bucket whose capture failed runs the step eagerly and still returns the reference's output dict"""
    net, wp, step, trainer = setup
    obs = C.observations(2, 450, DEV)
    with torch.no_grad():
        net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)
        ents = [e for k, e in step.replay.entries.items() if k[-1][0] == 2]
        assert len(ents) == 1
        ents[0]["failed"] = True
        try:
            got = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)
        finally:
            ents[0]["failed"] = False
        ref = reference(net, wp, obs)
    check_same(got, ref)
    check_vp(trainer, got, ref)


def test_step_fallbacks(setup):
    net, wp, step, trainer = setup
    obs = C.observations(2, 400, DEV)
    calls = net.calls
    assert net(mode="language") == "language"
    out = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=True)
    assert not isinstance(out, CS.StepOutputs)
    bad = dict(obs)
    bad["depth_30"] = bad["depth_30"].double().float().cpu()
    assert not isinstance(net(mode="waypoint", waypoint_predictor=wp, observations=bad, in_train=False), CS.StepOutputs)
    assert net.calls == calls + 3
    wp.train()
    try:
        with pytest.raises(RuntimeError, match="eval mode"):
            net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)
    finally:
        wp.eval()
    # plain dicts reach the trainer's own method
    ref = reference(net, wp, obs)
    v = trainer._vp_feature_variable(ref)
    assert torch.equal(v["view_lens"], R.vp_feature_variable(ref, DEV)["view_lens"])


def test_step_autocast_and_deterministic_change_no_bit(setup):
    net, wp, step, trainer = setup
    obs = C.observations(3, 500, DEV)
    with torch.no_grad():
        base = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)
        with torch.autocast("cuda", dtype=torch.float16):
            amp = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True, warn_only=True)
        try:
            det = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)
        finally:
            torch.use_deterministic_algorithms(prev)
    check_same(amp, base, depth_ulps=0)
    check_same(det, base, depth_ulps=0)


def test_step_one_synchronisation(setup):
    net, wp, step, trainer = setup
    obs = C.observations(4, 600, DEV)
    with torch.no_grad():
        out = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)   # captured
        trainer._vp_feature_variable(out)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                out = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)
                trainer._vp_feature_variable(out)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [str(x.message) for x in w if "synchroniz" in str(x.message).lower()]
    assert len(syncs) == 1, syncs


def rel(x, ref):
    return float((x.double() - ref.double()).norm() / ref.double().norm())


def ccw(v, B):
    """(12 B, ...) clockwise per-image rows -> (B, 12, -1) counter-clockwise views"""
    v = v.reshape(B, 12, -1)
    return torch.cat([v[:, :1], torch.flip(v[:, 1:], [1])], 1)


def test_step_against_full_reference(setup):
    """The step's own candidates and features against the full reference towers (ce_clip_ref, ce_depth_ref,
    ce_waypoint_ref) at B = 1, 4 and 8.  Candidates: for every environment, the cells the fp64 chain picks in the rounds
    whose fp64 margin exceeds 4x the step's logit error (the convention of test_ce_waypoint_gpu.py) are among the
    step's candidates when they survive the strip.  Features: pano_rgb and pano_depth within max(1e-2, 2.5 x the error
    of the reference's fp16-autocast towers) of fp64, the towers' existing bar."""
    import test_ce_waypoint_gpu as TW
    from oracle import ce_clip_ref as RC, ce_depth_ref as RD, ce_waypoint_ref as RW
    net, wp, step, trainer = setup
    vis_sd = dict(net.rgb_encoder.model.visual.state_dict())
    dep_sd = dict(net.depth_encoder.visual_encoder.state_dict())
    wp_sd = dict(wp.state_dict())
    fp16_clip = RC.Fp16Tower({k: v.cpu() for k, v in vis_sd.items()}).to(DEV)
    checked = 0
    for B in (1, 4, 8):
        obs = C.observations(B, 700 + B, DEV)
        rgb_b, depth_b, _ = ref_stack(obs)
        with torch.no_grad():
            got = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=False)
            logits = step.runner.logits(step.depth.encode(depth_b))     # the graph's logits (bit-equal, eager)
            rgb64 = RC.forward(vis_sd, rgb_b, torch.float64)[0]
            dep64 = RD.forward(dep_sd, depth_b, torch.float64)
            logits64 = RW.forward(wp_sd, dep64, torch.float64)
            rgb16 = RC.forward_fp16(fp16_clip, rgb_b)[0]
            dep16 = RD.forward_fp16(dep_sd, depth_b)
        for b, rounds in enumerate(TW.rounds_fp64(logits64)):
            k = int(got.picks[b, 10])
            mine = {(int(got.picks[b, 2 * q]), int(got.picks[b, 2 * q + 1])) for q in range(k)}
            err = float((logits[b].double() - logits64[b]).abs().max())
            for picks, margin in rounds:
                if margin <= 4 * err:
                    break
                sure = {(ix // 12 - 1, ix % 12) for ix in picks if 1 <= ix // 12 <= 120}
                assert sure <= mine, (B, b, sure, mine)
                checked += 1
        ref_rgb, ref_dep = ccw(rgb64, B), ccw(dep64, B).reshape(B, 12, 128, 16).mean(-1)
        e16_rgb, e16_dep = rel(ccw(rgb16, B), ref_rgb), rel(ccw(dep16, B).reshape(B, 12, 128, 16).mean(-1), ref_dep)
        e_rgb, e_dep = rel(got["pano_rgb"], ref_rgb), rel(got["pano_depth"], ref_dep)
        print("B=%d: pano_rgb rel err %.3e (fp16 reference %.3e), pano_depth %.3e (fp16 reference %.3e)" % (
            B, e_rgb, e16_rgb, e_dep, e16_dep))
        assert e_rgb <= max(1e-2, 2.5 * e16_rgb) and e_dep <= max(1e-2, 2.5 * e16_dep)
    print("NMS rounds checked against fp64: %d" % checked)
    assert checked > 0
