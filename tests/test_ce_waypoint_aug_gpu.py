"""GPU checks of the VLN-CE waypoint step with waypoint augmentation (in_train=True): bb_ce_waypoint_candidates_aug
against a torch restatement on the device given the same noise (NMS picks, samples, every feature), forced samples of
every image, ties and NaN, guards and rejections; the installed step (waypoint_aug=True) against the reference branch
(oracle/ce_waypoint_aug_ref.py) fed the step's own noise; the sampled distribution against the fp64 regional softmax;
seeding, replay, autocast and deterministic invariance; and both graphs of a geometry living side by side."""
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
from bevbert_b200 import _lib, graphs  # noqa: E402
from bevbert_b200.model import ce_waypoint_step as CS  # noqa: E402
from bevbert_b200.model import waypoint as WP  # noqa: E402
from oracle import ce_waypoint_aug_ref as RA  # noqa: E402
from oracle import ce_waypoint_step_ref as R  # noqa: E402
from test_ce_waypoint_aug_cpu import expected_cell  # noqa: E402
from test_ce_waypoint_step_gpu import bits, check_same, check_vp, ref_candidates  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 37


def features(B, g):
    rgb_vec = torch.randn(12 * B, 512, generator=g).to(DEV)
    dep = torch.rand(12 * B, 128, 4, 4, generator=g).mul(torch.exp2(torch.randint(-8, 9, (12 * B, 128, 4, 4),
                                                                                  generator=g).float())).to(DEV)
    return rgb_vec, dep


def ref_samples(logits, noise, nms_picks):
    """the reference's lines 229-264 on the device for the kernel's NMS picks: per environment the sampled indices"""
    B = logits.shape[0]
    regional = torch.cat((logits[:, -5:], logits[:, :-5]), dim=1).reshape(B, 12, 10, 12)
    out = []
    for b in range(B):
        k = int(nms_picks[b, 10])
        img = (nms_picks[b, 0:2 * k:2].numpy() + 5) // 10
        img[img == 12] = 0
        p = F.softmax(regional[b][img].view(k, -1), 1)
        s = RA.sample_candidates(p, noise[b, :k]).cpu().tolist()
        out.append([(x // 12 + ((i - 1) * 10 + 5 if i != 0 else 0), x % 12) for x, i in zip(s, img.tolist())])
    return out


def check_kernel(logits, noise, rgb_vec, dep):
    B = logits.shape[0]
    got = CS.waypoint_candidates_aug(logits, noise, rgb_vec, dep, nms_picks=True)
    base = CS.waypoint_candidates(logits, rgb_vec, dep)
    nms_picks, picks = got["nms_picks"].cpu(), got["picks"].cpu()
    assert torch.equal(nms_picks, base["picks"].cpu())
    _, _, rgb_feats, dep_feats = ref_candidates(logits, rgb_vec, dep)
    assert torch.equal(bits(got["pano_rgb"]), bits(rgb_feats)) and torch.equal(bits(got["pano_depth"]), bits(dep_feats))
    for b, cells in enumerate(ref_samples(logits, noise, nms_picks)):
        k = len(cells)
        assert int(picks[b, 10]) == k and picks[b, 0:2 * k].view(k, 2).tolist() == [list(c) for c in cells], b
        img = 12 - (np.array([a for a, _ in cells], dtype=np.int64) + 5) // 10
        img[img == 12] = 0
        cand = np.zeros(12, dtype=bool)
        cand[img] = True
        assert int(picks[b, 11]) == k + 12 - int(cand.sum())
        rest = torch.from_numpy(~cand).to(DEV)
        rows_r = torch.cat([got["pano_rgb"][b, img], got["pano_rgb"][b, rest]])
        rows_d = torch.cat([got["pano_depth"][b, img], got["pano_depth"][b, rest]])
        L = rows_r.shape[0]
        assert torch.equal(bits(got["cand_rgb"][b, :k]), bits(rgb_feats[b, img]))
        assert torch.equal(bits(got["cand_depth"][b, :k]), bits(dep_feats[b, img]))
        assert not bool(got["cand_rgb"][b, k:].any()) and not bool(got["cand_depth"][b, k:].any())
        assert torch.equal(bits(got["rgb_fts"][b, :L]), bits(rows_r))
        assert torch.equal(bits(got["dep_fts"][b, :L]), bits(rows_d))
        assert not bool(got["rgb_fts"][b, L:].any()) and not bool(got["dep_fts"][b, L:].any())
    return got


@pytest.mark.parametrize("B", [1, 5, 8, 64])
@pytest.mark.parametrize("kind", ["seeded", "constructed"])
def test_aug_candidates_against_torch(B, kind):
    g = torch.Generator().manual_seed(100 + B)
    logits = (torch.randn(B, 120, 12, generator=g) * 3 if kind == "seeded" else C.constructed_logits(B, B)).to(DEV)
    rgb_vec, dep = features(B, g)
    torch.manual_seed(B)
    for _ in range(3):
        check_kernel(logits, CS.draw_noise(B, DEV), rgb_vec, dep)


def test_aug_forced_samples_every_image():
    """noise 1e-30 at sample s and 1 elsewhere forces s for every pick: the sampled cells of every clockwise image, and
    image 0 from both of its sides, follow the reference's pointer arithmetic"""
    angles = [10 * i for i in range(12)] + [117]
    B = len(angles)
    logits = torch.zeros(B, 120, 12)
    for j, a in enumerate(angles):
        logits[j, a, 4] = 6.0
    logits = logits.to(DEV)
    rgb_vec, dep = features(B, torch.Generator().manual_seed(1))
    images = set()
    for s in range(120):
        noise = torch.ones(B, 5, 120, device=DEV)
        noise[:, :, s] = 1e-30
        got = check_kernel(logits, noise, rgb_vec, dep)
        nms_picks, picks = got["nms_picks"].cpu(), got["picks"].cpu()
        for b in range(B):
            for q in range(int(nms_picks[b, 10])):
                img = ((int(nms_picks[b, 2 * q]) + 5) // 10) % 12
                images.add(img)
                angle, d, _ = expected_cell(img, s)
                assert (int(picks[b, 2 * q]), int(picks[b, 2 * q + 1])) == (angle, d), (b, q, s)
    assert images == set(range(12))


def test_aug_ties_and_nan():
    """equal logits and equal noise tie every cell: the lowest index wins; a NaN ratio is the maximum (the lowest NaN
    index wins)"""
    B = 3
    rgb_vec, dep = features(B, torch.Generator().manual_seed(2))
    logits = torch.zeros(B, 120, 12, device=DEV)
    noise = torch.ones(B, 5, 120, device=DEV)
    got = check_kernel(logits, noise, rgb_vec, dep)
    nms_picks, picks = got["nms_picks"].cpu(), got["picks"].cpu()
    for b in range(B):
        for q in range(int(nms_picks[b, 10])):
            img = ((int(nms_picks[b, 2 * q]) + 5) // 10) % 12
            assert (int(picks[b, 2 * q]), int(picks[b, 2 * q + 1])) == expected_cell(img, 0)[:2]
    noise[:, :, 50] = float("nan")
    noise[:, :, 7] = float("nan")
    got = check_kernel(logits, noise, rgb_vec, dep)
    assert int(got["picks"][0, 1]) == 7


def test_aug_guards_and_rejections():
    B, pad = 2, 64
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(B, 120, 12, generator=g).to(DEV)
    rgb_vec, dep = features(B, g)
    noise = CS.draw_noise(B, DEV)
    ref = CS.waypoint_candidates_aug(logits, noise, rgb_vec, dep, nms_picks=True)
    sizes = {"picks": 12, "nms_picks": 12, "pano_rgb": 12 * 512, "pano_depth": 12 * 128, "cand_rgb": 5 * 512,
             "cand_depth": 5 * 128, "rgb_fts": 17 * 512, "dep_fts": 17 * 128}
    bufs = {k: torch.full((B * n + 2 * pad,), -7, dtype=torch.int32 if "picks" in k else torch.float32, device=DEV)
            for k, n in sizes.items()}
    o = {k: v[pad:].data_ptr() for k, v in bufs.items()}
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    args = [logits.data_ptr(), noise.data_ptr(), rgb_vec.data_ptr(), dep.data_ptr(), B, o["picks"], o["nms_picks"],
            o["pano_rgb"], o["pano_depth"], o["cand_rgb"], o["cand_depth"], o["rgb_fts"], o["dep_fts"], stream]
    _lib.check(lib.bb_ce_waypoint_candidates_aug(*args), "bb_ce_waypoint_candidates_aug")
    for k, buf in bufs.items():
        assert bool((buf[:pad] == -7).all()) and bool((buf[-pad:] == -7).all()), k
        assert torch.equal(bits(buf[pad:-pad]), bits(ref[k].reshape(-1))), k
    a = list(args)
    a[6] = None                                             # nms_picks may be NULL
    _lib.check(lib.bb_ce_waypoint_candidates_aug(*a), "bb_ce_waypoint_candidates_aug")
    for i, bad in ((4, 0), (4, 65536), (0, None), (1, None), (5, None), (1, noise.data_ptr() + 2),
                   (5, noise.data_ptr()), (6, o["picks"]), (7, o["pano_depth"])):
        a = list(args)
        a[i] = bad
        assert lib.bb_ce_waypoint_candidates_aug(*a) != 0, i
    with pytest.raises(ValueError):
        CS.waypoint_candidates_aug(logits, noise[:, :4].contiguous(), rgb_vec, dep)
    with pytest.raises(TypeError):
        CS.waypoint_candidates_aug(logits, noise.double(), rgb_vec, dep)
    with pytest.raises(TypeError):
        CS.waypoint_candidates_aug(logits, noise.cpu(), rgb_vec, dep)


def test_aug_distribution():
    """B = 2048 copies of one environment, noise drawn as the step draws it: the sampled cells of each pick follow the
    fp64 regional softmax (chi-square at a fixed seed)"""
    from scipy.stats import chisquare
    B = 2048
    g = torch.Generator().manual_seed(6)
    one = torch.randn(1, 120, 12, generator=g) * 1.5
    logits = one.expand(B, 120, 12).contiguous().to(DEV)
    rgb_vec, dep = features(1, g)
    rgb_vec, dep = rgb_vec.repeat(B, 1), dep.repeat(B, 1, 1, 1)
    torch.manual_seed(7)
    got = CS.waypoint_candidates_aug(logits, CS.draw_noise(B, DEV), rgb_vec, dep, nms_picks=True)
    nms_picks, picks = got["nms_picks"].cpu(), got["picks"].cpu()
    assert bool((nms_picks == nms_picks[0]).all())
    regional = torch.cat((one[:, -5:], one[:, :-5]), dim=1).reshape(12, 120).double()
    k = int(nms_picks[0, 10])
    assert k >= 2
    for q in range(k):
        img = ((int(nms_picks[0, 2 * q]) + 5) // 10) % 12
        ptr = (img - 1) * 10 + 5 if img != 0 else 0
        s = (picks[:, 2 * q].long() - ptr) * 12 + picks[:, 2 * q + 1].long()
        assert bool(((s >= 0) & (s < 120)).all())
        counts = torch.bincount(s, minlength=120).double()
        expect = torch.softmax(regional[img], 0) * B
        big = expect >= 5
        obs = torch.cat([counts[big], counts[~big].sum().view(1)]).numpy()
        exp = torch.cat([expect[big], expect[~big].sum().view(1)]).numpy()
        if exp[-1] == 0:
            obs, exp = obs[:-1], exp[:-1]
        p = chisquare(obs, exp * obs.sum() / exp.sum()).pvalue
        print("pick %d (image %d): chi-square p = %.3g over %d bins" % (q, img, p, len(obs)))
        assert p > 1e-4, (q, p)


# ------------------------------------------------------------------------------------------------ whole step
class AugNet(C.Net):
    """C.Net whose forward honours in_train (the reference branch with the reference's own sampling)"""

    def forward(self, mode=None, txt_ids=None, txt_masks=None, txt_embeds=None, waypoint_predictor=None,
                observations=None, in_train=True):
        self.calls += 1
        if mode != "waypoint":
            return mode
        return RA.waypoint_branch(observations, lambda o: self.depth.encode(o["depth"]),
                                  lambda o: self.clip.encode_rgb(o["rgb"]), waypoint_predictor, WP.nms,
                                  self.pano_angle_fts, self.pano_img_idxes, in_train=in_train)


REF = {}


@pytest.fixture(scope="module")
def setup():
    net = AugNet(SEED, DEV)
    wp = C.predictor(SEED, DEV)
    step = graphs.install_ce_waypoint_step(net, waypoint_aug=True)
    trainer = type("Trainer", (), {})()
    trainer._vp_feature_variable = lambda obs: R.vp_feature_variable(obs, DEV)
    graphs.install_ce_vp_features(trainer)
    REF["net"], REF["wp"] = AugNet(SEED, DEV), C.predictor(SEED, DEV)
    return net, wp, step, trainer


def reference(obs, noise):
    n = REF["net"]
    return RA.waypoint_branch(obs, lambda o: n.depth.encode(o["depth"]), lambda o: n.clip.encode_rgb(o["rgb"]),
                              REF["wp"], WP.nms, n.pano_angle_fts, n.pano_img_idxes, in_train=True, noise=noise)


def call(net, wp, obs, in_train=True):
    return net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=in_train)


def test_aug_step_against_reference_branch(setup):
    net, wp, step, trainer = setup
    with torch.no_grad():
        for i, B in enumerate([8, 5, 1, 8]):
            obs = C.observations(B, 800 + i, DEV, crop=bool(i % 2))
            calls = net.calls
            got = call(net, wp, obs)
            assert net.calls == calls, "the step must not run the original forward"
            assert got.noise.shape == (B, 5, 120) and got.noise.dtype == torch.float32
            ref = reference(obs, got.noise)
            check_same(got, ref)
            check_vp(trainer, got, ref)
            for lst in got["cand_angles"] + got["cand_distances"]:
                assert all(type(x) is float for x in lst)
    keys = [k for k in step.replay.entries if k[-1][-1]]
    assert len(keys) == 3 and all(step.replay.entries[k]["graph"] is not None for k in keys)


def test_aug_bucket_without_graph(setup):
    net, wp, step, trainer = setup
    obs = C.observations(2, 850, DEV)
    with torch.no_grad():
        call(net, wp, obs)
        ents = [e for k, e in step.replay.entries.items() if k[-1][0] == 2 and k[-1][-1]]
        assert len(ents) == 1
        ents[0]["failed"] = True
        try:
            got = call(net, wp, obs)
        finally:
            ents[0]["failed"] = False
        ref = reference(obs, got.noise)
    check_same(got, ref)
    check_vp(trainer, got, ref)


def test_aug_seeding_and_replay(setup):
    net, wp, step, trainer = setup
    obs = C.observations(4, 900, DEV)
    with torch.no_grad():
        call(net, wp, obs)                                  # captured: its eager warm-up drew noise too
        outs = []
        for _ in range(2):
            torch.manual_seed(1234)
            outs.append(call(net, wp, obs))
        nxt = call(net, wp, obs)
    check_same(outs[1], outs[0])
    assert torch.equal(outs[0].noise, outs[1].noise) and torch.equal(outs[0].picks, outs[1].picks)
    assert not torch.equal(nxt.noise, outs[1].noise)


def test_aug_autocast_and_deterministic_change_no_bit(setup):
    net, wp, step, trainer = setup
    obs = C.observations(3, 950, DEV)
    prev = torch.are_deterministic_algorithms_enabled()
    with torch.no_grad():
        call(net, wp, obs)
        torch.use_deterministic_algorithms(True, warn_only=True)
        try:
            call(net, wp, obs)                              # the deterministic-mode bucket's capture
            torch.manual_seed(77)
            det = call(net, wp, obs)
        finally:
            torch.use_deterministic_algorithms(prev)
        torch.manual_seed(77)
        base = call(net, wp, obs)
        torch.manual_seed(77)
        with torch.autocast("cuda", dtype=torch.float16):
            amp = call(net, wp, obs)
    check_same(amp, base)
    check_same(det, base)
    assert torch.equal(det.noise, base.noise) and torch.equal(amp.noise, base.noise)


def test_aug_and_eval_graphs_live_side_by_side(setup):
    """alternating in_train=True and in_train=False calls of one geometry keep both graphs (no recapture), and every
    call makes exactly one synchronising copy"""
    net, wp, step, trainer = setup
    obs = C.observations(6, 1000, DEV)
    with torch.no_grad():
        for in_train in (True, False):
            trainer._vp_feature_variable(call(net, wp, obs, in_train))
        ents = {k: e for k, e in step.replay.entries.items() if k[-1][0] == 6}
        assert sorted(k[-1][-1] for k in ents) == [False, True]
        graphs_before = {k: e["graph"] for k, e in ents.items()}
        torch.cuda.synchronize()
        for i in range(4):
            in_train = i % 2 == 0
            torch.cuda.set_sync_debug_mode("warn")
            try:
                with warnings.catch_warnings(record=True) as w:
                    warnings.simplefilter("always")
                    out = call(net, wp, obs, in_train)
                    trainer._vp_feature_variable(out)
            finally:
                torch.cuda.set_sync_debug_mode("default")
            syncs = [str(x.message) for x in w if "synchroniz" in str(x.message).lower()]
            assert len(syncs) == 1, (in_train, syncs)
            assert (out.noise is not None) == in_train
    after = {k: e["graph"] for k, e in step.replay.entries.items() if k[-1][0] == 6}
    assert after.keys() == graphs_before.keys() and all(after[k] is graphs_before[k] for k in after)
