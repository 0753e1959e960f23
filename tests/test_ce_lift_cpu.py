"""CPU checks of the VLN-CE trainer's lift (agent_bev.ce_lift, graphs.install_ce_lift): the oracle
(tests/ce_lift_oracle.py) against the unmodified reference's golden (tests/golden/small_ce_lift.pt), the host fan
builder bit for bit, the install's routing, the projector checks and the wrapper's argument checks."""
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [p for p in (ROOT, os.path.join(ROOT, "tests")) if p not in sys.path]

import ce_lift_cases as C  # noqa: E402
import ce_lift_oracle as O  # noqa: E402
from bevbert_b200 import agent_bev, bev_nodes, graphs  # noqa: E402

GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "small_ce_lift.pt"), weights_only=False)


def bits(x):
    return x.contiguous().view(torch.int32)


def dot_error(pc, ref, xyz1, T):
    """|pc - ref| in units of the fp32 spacing at sum_k |T[j,k] xyz1[k]|, per coordinate"""
    S = (T[:, None, :3, :] * xyz1[:, :, None, :]).abs().sum(-1).reshape(pc.shape)
    return (pc - ref).abs() / torch.from_numpy(np.spacing(S.numpy()))


@pytest.fixture(params=range(len(C.CASES)), ids=["B%d" % c["B"] for c in C.CASES])
def gold(request):
    g = GOLD["cases"][request.param]
    cur_pos, cur_ori, depth, shift, digests = C.case_inputs(g["case"])
    assert digests == g["input_digests"]            # the seeds regenerate the inputs the golden was made from
    return g, cur_pos, cur_ori, depth, shift


def test_cases_cover_what_lift_sees():
    B = [c["B"] for c in C.CASES]
    assert B == [1, 3, 8]
    d = torch.cat([C.case_inputs(c)[2].reshape(-1) for c in C.CASES])
    assert (d == 0).any() and ((d > 0) & (d < 1.1754944e-38)).sum() >= 5 and d.max() <= 1.0
    heads = [h for g in GOLD["cases"] for h in g["headings"]]
    assert len({round(h, 6) for h in heads}) >= 8


def test_headings_restated_from_habitat(gold):
    g, _, cur_ori, _, _ = gold
    assert [C.heading_from_quaternion(o) for o in cur_ori] == g["headings"]


def test_oracle_against_reference_golden(gold):
    g, cur_pos, _, depth, shift = gold
    o = O.lift(cur_pos, g["headings"], depth, shift)
    assert torch.equal(bits(o["T"]), bits(g["T"]))
    assert C.sha(o["xyz1"].numpy()) == g["xyz1_digest"] and tuple(o["xyz1"].shape) == g["xyz1_shape"]
    assert torch.equal(o["pc_mask"], g["pc_mask"])
    # the reference leaves the 4-term dot to bmm, whose order differs: where the terms cancel, a rounding of the
    # largest partial sum is many ulps of the result, so the pin is in ulps of the sum of the terms' magnitudes
    assert o["pc"].shape == g["pc"].shape
    assert float(dot_error(o["pc"], g["pc"], o["xyz1"], o["T"]).max()) <= 2.0


def test_host_fan_builder_equals_golden_T(gold):
    g, cur_pos, _, _, _ = gold
    T = agent_bev.lift_frames(cur_pos, g["headings"])
    assert T.dtype == np.float32 and torch.equal(bits(torch.from_numpy(T)), bits(g["T"]))


def test_heading_frames_is_transfrom3D():
    from ce_nav_bev_oracle import transfrom3D
    h = np.array([0.0, 0.3, -1.2, math.pi, 2.5, 4.0])
    xyzhe = np.zeros((len(h), 5))
    xyzhe[:, 3] = h
    _, T = agent_bev.heading_frames(np.zeros((len(h), 3)), h)
    assert np.array_equal(T.view(np.int32), transfrom3D(xyzhe).view(np.int32))


def test_intrinsics_are_compute_intrinsic_matrix():
    fx, fy, cx, cy = agent_bev.lift_intrinsics(C.Projector("cpu"))
    assert (fx, fy, cx, cy) == tuple(float(v) for v in O.intrinsics())
    fx2, fy2, _, _ = agent_bev.lift_intrinsics(C.Projector("cpu", vfov=math.radians(79)))
    assert (fx2, fy2) == tuple(float(v) for v in O.intrinsics(math.radians(79))[:2])


@pytest.mark.parametrize("kw", [{"fmh": 16}, {"fmw": 7}, {"vfov": 0.0}, {"vfov": float("nan")}, {"vfov": "90"}])
def test_projector_rejected(kw):
    with pytest.raises(ValueError):
        agent_bev.lift_intrinsics(C.Projector("cpu", **kw))


@pytest.mark.parametrize("shift", [[0.0, 0.0], torch.zeros(3, dtype=torch.float64), torch.zeros(1), torch.zeros(3, 1),
                                   (0.0, 0.0, 0.0)])
def test_world_shift_rejected(shift):
    p = C.Projector("cpu")
    p.world_shift_origin = torch.tensor(shift) if isinstance(shift, list) else shift
    with pytest.raises(ValueError):
        agent_bev.lift_intrinsics(p)
    trainer = types.SimpleNamespace(projector=p)
    with pytest.raises(ValueError):
        graphs.install_ce_lift(trainer)
    assert not hasattr(trainer, "lift")


def test_world_shift_shapes_accepted():
    for s in (torch.zeros(3), torch.zeros(1, 3), torch.zeros(1, 1, 3)):
        p = C.Projector("cpu")
        p.world_shift_origin = s
        agent_bev.lift_intrinsics(p)


def test_depth_grid_rejected():
    tr = C.LiftTrainer(2, "cpu")
    pos, ori = [np.zeros(3)] * 2, [C.quaternion_at(0.0)] * 2
    rgb = torch.zeros(2, 12, 196, 768)
    for d in (torch.zeros(2, 12, 196, 1),                    # not on the GPU
              torch.zeros(2, 12, 196, 1, dtype=torch.float64), np.zeros((2, 12, 196, 1), np.float32)):
        with pytest.raises(ValueError):
            agent_bev.ce_lift(tr, pos, ori, rgb, d)


def test_install_routes_to_ce_lift(monkeypatch):
    tr = C.LiftTrainer(2, "cpu")
    calls = []
    monkeypatch.setattr(agent_bev, "ce_lift", lambda *a: calls.append(a) or "lifted")
    lift = graphs.install_ce_lift(tr)
    assert tr.lift is lift
    assert tr.lift("pos", "ori", "rgb", "depth") == "lifted"
    assert calls == [(tr, "pos", "ori", "rgb", "depth")]


def test_wrapper_argument_checks():
    d, T, s = torch.zeros(2, 14, 14), torch.zeros(2, 4, 4), torch.zeros(3)
    with pytest.raises(RuntimeError):                           # CPU tensors: the lift has no CPU implementation
        bev_nodes.bev_lift_points(d, T, s, 10.0, 7.0, 7.0, 7.0, 7.0)
    with pytest.raises(TypeError):
        bev_nodes.bev_lift_points(d.double(), T, s, 10.0, 7.0, 7.0, 7.0, 7.0)
