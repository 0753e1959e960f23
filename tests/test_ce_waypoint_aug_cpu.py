"""CPU checks of the VLN-CE waypoint step with waypoint augmentation (in_train=True): the oracle
(oracle/ce_waypoint_aug_ref.py) against the golden of the unmodified reference branch
(tests/golden/small_ce_waypoint_aug.pt), with the reference's own sampling and with the recorded noise; the recorded
noise against a re-seeded draw; the host dict builder and the restated _vp_feature_variable on the sampled indices; the
sampled-cell arithmetic for every image; and the install's routing of in_train=True calls."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import ce_waypoint_step_cases as C  # noqa: E402
import make_ce_waypoint_aug_golden as MA  # noqa: E402
import make_ce_waypoint_step_golden as MG  # noqa: E402
from bevbert_b200 import graphs  # noqa: E402
from bevbert_b200.model import ce_waypoint_step as CS  # noqa: E402
from oracle import ce_waypoint_aug_ref as RA  # noqa: E402
from oracle import ce_waypoint_ref as RW  # noqa: E402
from oracle import ce_waypoint_step_ref as R  # noqa: E402
from test_ce_waypoint_step_cpu import same_value  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "small_ce_waypoint_aug.pt")


def golden():
    return torch.load(GOLDEN, weights_only=False)


def run_oracle(case, noise=None):
    stored, logits = MA.case_inputs(case)
    obs = MG.observations(stored)
    enc = MG.Encoders(case["enc_seed"], logits)
    idx, fts = R.pano_features()
    with torch.no_grad():
        return RA.waypoint_branch(obs, enc.depth, enc.rgb, enc.predictor, RW.nms, fts, idx, in_train=True, noise=noise)


def check_against(out, case):
    grid = out.pop("pano_rgb_grid")
    ref = case["outputs"]
    assert list(out) == list(ref)
    for k in ref:
        same_value(out[k], ref[k], k)
    gg = case["pano_rgb_grid"]
    assert tuple(grid.shape) == gg["shape"] and grid.dtype == gg["dtype"]
    assert torch.equal(grid.double().sum((2, 3)), gg["sums"])


@pytest.mark.parametrize("B", MA.BATCHES)
def test_oracle_against_golden(B):
    """the oracle reproduces the unmodified reference branch bit for bit, Python and numpy types included: under the
    golden's seed with the reference's own Categorical(...).sample(), and with the recorded noise"""
    g = golden()
    case = g["B%d" % B]
    torch.manual_seed(g["seed"] + B)
    check_against(run_oracle(case), case)
    check_against(run_oracle(case, noise=case["noise"]), case)


def test_golden_covers_the_cases():
    """picks in image 0 with samples in both halves (one in counter-clockwise view 11), two picks in one sector, a
    wrap-row pick and fewer than five picks, at B = 1 and 8"""
    g = golden()
    halves, shared, wrap, fewer = set(), False, False, False
    for B in MA.BATCHES:
        case = g["B%d" % B]
        for j, ang in enumerate(nms_angles(case)):
            imgs = [((a + 5) // 10) % 12 for a in ang]
            samp = sampled_indices(case["outputs"], j)[0]
            halves |= {a >= 5 for a, i in zip(samp, imgs) if i == 0}
            shared |= len(set(imgs)) < len(imgs)
            wrap |= any(a in (0, 119) for a in ang)
            fewer |= len(ang) < 5
    assert halves == {False, True} and shared and wrap and fewer
    assert any(11 in o.tolist() for o in g["B8"]["outputs"]["cand_img_idxes"])


def nms_angles(case):
    """per environment, the angles of the branch's NMS picks (before sampling) on the logits it saw (the stand-in
    predictor adds its depth term)"""
    stored, logits = MA.case_inputs(case)
    obs = MG.observations(stored)
    enc = MG.Encoders(case["enc_seed"], logits)
    B = case["B"]
    logits = enc.predictor(torch.zeros(12 * B, 512), enc.depth({"depth": MG._stacked_depth(obs)}))
    x = torch.softmax(logits.reshape(B, 1440), dim=1).reshape(B, 120, 12)
    x = torch.cat((x[:, -1:], x, x[:, :1]), dim=1)
    out = RW.nms(x.unsqueeze(1), max_predictions=5, sigma=(7.0, 5.0)).squeeze(1)[:, 1:-1]
    return [out[j].nonzero()[:, 0].tolist() for j in range(B)]


def test_noise_redraw():
    """re-seeding and drawing exponential_ of shape (K_j, 120) in environment order reproduces the recorded noise"""
    g = golden()
    for B in MA.BATCHES:
        case = g["B%d" % B]
        counts = [len(a) for a in case["outputs"]["cand_angles"]]
        again = MA.redraw_noise(g["seed"] + B, counts)
        assert all(torch.equal(a, b) for a, b in zip(again, case["noise"]))


def sampled_indices(out, j):
    """environment j's sampled (angle, distance) indices, read back from the golden's outputs"""
    ang = [int(round((2 * math.pi - a) * 120 / (2 * math.pi))) for a in out["cand_angles"][j]]
    dist = [int(round(d / 0.25)) - 1 for d in out["cand_distances"][j]]
    return ang, dist


def golden_picks(out):
    """(B, 12) int32 picks of the golden's sampled indices"""
    B = len(out["cand_angles"])
    picks = torch.zeros(B, CS.PICK_COLS, dtype=torch.int32)
    for j in range(B):
        ang, dist = sampled_indices(out, j)
        k = len(ang)
        picks[j, 0:2 * k:2], picks[j, 1:2 * k:2] = torch.tensor(ang), torch.tensor(dist)
        img = 12 - (np.array(ang) + 5) // 10
        img[img == 12] = 0
        picks[j, 10], picks[j, 11] = k, k + 12 - len(set(img.tolist()))
    return picks


def test_host_outputs_and_vp_on_golden_samples():
    """host_outputs(..., "cpu") on the sampled indices gives the reference's candidate outputs (its index tensors are
    CPU tensors), and the restated _vp_feature_variable agrees with vp_host_inputs and the picks' view lengths"""
    g = golden()
    for B in MA.BATCHES:
        out = g["B%d" % B]["outputs"]
        picks = golden_picks(out)
        got = CS.host_outputs(picks, device_type="cpu")
        for k in ("cand_angle_fts", "cand_img_idxes", "cand_angles", "cand_distances"):
            same_value(got[k], out[k], k)
        ref = R.vp_feature_variable(out, "cpu")
        loc, nav, lens = CS.vp_host_inputs(out)
        assert torch.equal(loc, ref["loc_fts"]) and torch.equal(nav, ref["nav_types"])
        assert torch.equal(lens, ref["view_lens"]) and lens.tolist() == picks[:, 11].tolist()


def expected_cell(img, s):
    """the reference's sampled (angle, distance, counter-clockwise view) for sample s of clockwise image img: the
    angle of the logit row the sample came from, except in image 0, whose pointer is 0 rather than -5"""
    r, d = divmod(s, 12)
    angle = r if img == 0 else 10 * img - 5 + r
    view = 12 - (angle + 5) // 10
    return angle, d, 0 if view == 12 else view


def test_sampled_cell_arithmetic(monkeypatch):
    """every sample s of every clockwise image, through the oracle's candidate loop: one environment per image with a
    single pick (the other cells underflow), image 0 from both of its sides (angles 0 and 117)"""
    angles = [10 * i for i in range(12)] + [117]
    B = len(angles)
    logits = torch.full((B, 120, 12), -300.0)
    for j, a in enumerate(angles):
        logits[j, a, 4] = 0.0
    stored = MG.inputs(B, 3)
    obs = MG.observations(stored)
    enc = MG.Encoders(4, logits)
    idx, fts = R.pano_features()
    forced = {}
    monkeypatch.setattr(RA, "sample_candidates", lambda probs, noise_rows=None: forced["s"].expand(probs.shape[0]))
    for s in range(120):
        forced["s"] = torch.tensor([s])
        with torch.no_grad():
            out = RA.waypoint_branch(obs, enc.depth, enc.rgb, enc.predictor, RW.nms, fts, idx, in_train=True)
        for j, a in enumerate(angles):
            img = ((a + 5) // 10) % 12
            angle, d, view = expected_cell(img, s)
            assert out["cand_distances"][j] == [(d + 1) * 0.25]
            assert out["cand_img_idxes"][j].tolist() == [view], (a, s)
            assert out["cand_angles"][j] == (2 * math.pi - torch.tensor([angle]).float() / 120 * 2 * math.pi).tolist()
    # the image-0 quirk: the second half of its samples lands in view 11, as the sampled angle 5..9 says
    assert [expected_cell(0, s)[2] for s in (0, 59, 60, 119)] == [0, 0, 11, 11]


class _Covered(Exception):
    pass


class _Net(C.Net):
    def forward(self, mode=None, txt_ids=None, txt_masks=None, txt_embeds=None, waypoint_predictor=None,
                observations=None, in_train=True):
        self.calls += 1
        return "original"


@pytest.mark.parametrize("waypoint_aug", [False, True])
def test_install_routing(waypoint_aug):
    """default: in_train=True falls through to the original forward; waypoint_aug=True: covered in_train=True calls
    reach the step, uncovered ones still fall through"""
    net = _Net(1, "cpu")
    step = graphs.install_ce_waypoint_step(net, waypoint_aug=waypoint_aug)

    def reached(_):
        raise _Covered()
    step.set_predictor = reached
    obs = C.observations(1, 5, "cpu", depth_hw=(16, 16))
    for in_train in (False, True):
        covered = not in_train or waypoint_aug
        if covered:
            with pytest.raises(_Covered):
                net(mode="waypoint", waypoint_predictor=None, observations=obs, in_train=in_train)
        else:
            assert net(mode="waypoint", waypoint_predictor=None, observations=obs, in_train=in_train) == "original"
        bad = dict(obs, depth_30=obs["depth_30"].double())
        assert net(mode="waypoint", waypoint_predictor=None, observations=bad, in_train=in_train) == "original"
    assert net(mode="language") == "original"
