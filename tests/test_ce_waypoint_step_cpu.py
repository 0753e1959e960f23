"""CPU checks of the VLN-CE waypoint step's host logic: the view permutation from the observation dict's order, the
fallback conditions, the oracle (oracle/ce_waypoint_step_ref.py) against the golden of the unmodified reference branch (tests/golden/small_ce_waypoint_step.pt), the host
dict builder on the reference's own indices, and the restated _vp_feature_variable on the reference's outputs."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import ce_waypoint_step_cases as C  # noqa: E402
from bevbert_b200.model import ce_waypoint_step as CS  # noqa: E402
from oracle import ce_waypoint_ref as RW  # noqa: E402
from oracle import ce_waypoint_step_ref as R  # noqa: E402

CPU = torch.device("cpu")


def small_obs(B, seed, hw=(16, 18)):
    """observations with tiny images (224 x 224 rgb is not needed for the host logic)"""
    g = torch.Generator().manual_seed(seed)
    obs = {"instruction": torch.zeros(B, 3)}
    for h in C.HEADINGS:
        obs["rgb" + h] = torch.randint(0, 256, (B, 4, 4, 3), generator=g, dtype=torch.uint8)
        obs["depth" + h] = torch.rand(B, hw[0], hw[1], 1, generator=g)
    return obs


def test_view_permutation_follows_dict_order():
    obs = small_obs(2, 1)
    pairs = CS.view_pairs(obs)
    assert pairs == [("rgb" + h, "depth" + h) for h in C.HEADINGS]
    assert [CS.image_slot(k) for k in range(12)] == [0] + list(range(11, 0, -1))
    # the reference's stacking puts view k of environment b at image slot(k) + 12 b
    dep = torch.zeros_like(obs["depth"]).repeat(12, 1, 1, 1)
    for k, (_, d) in enumerate(pairs):
        for b in range(2):
            dep[CS.image_slot(k) + 12 * b] = obs[d][b]
    a_count = 0
    ref = torch.zeros_like(dep)
    for key, v in obs.items():
        if "depth" in key:
            for bi in range(v.size(0)):
                ref[(12 - a_count) % 12 + bi * 12] = v[bi]
            a_count += 1
    assert torch.equal(dep, ref)
    # another key order permutes the views accordingly
    keys = list(obs)
    reordered = {k: obs[k] for k in keys[::-1]}
    assert [d for _, d in CS.view_pairs(reordered)] == ["depth" + h for h in C.HEADINGS[::-1]]


def test_fallback_conditions():
    obs = small_obs(2, 2)
    assert CS.covered(obs, 4, CPU) is not None
    assert CS.covered(obs, 4, CPU)[1] == (2, 4, 4, 16, 18)
    assert CS.covered(obs, 4, torch.device("cuda", 0)) is None            # CPU tensors
    assert CS.covered(obs, 8, CPU) is None                                # not the tower's resolution
    missing = {k: v for k, v in obs.items() if k != "depth_90"}
    assert CS.covered(missing, 4, CPU) is None                            # 11 depth keys
    extra = dict(obs, depth_extra=obs["depth"], rgb_extra=obs["rgb"])
    assert CS.covered(extra, 4, CPU) is None                              # 13 depth keys
    nopartner = {k: v for k, v in obs.items() if k != "rgb_60"}
    assert CS.covered(nopartner, 4, CPU) is None
    for key, bad in (("depth_30", obs["depth_30"].double()), ("rgb_30", obs["rgb_30"].float()),
                     ("depth_30", obs["depth_30"][:1]), ("depth", torch.rand(2, 10, 18, 1))):
        assert CS.covered(dict(obs, **{key: bad}), 4, CPU) is None, key


GOLDEN = os.path.join(ROOT, "tests", "golden", "small_ce_waypoint_step.pt")


def golden():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_ce_waypoint_step_golden as MG
    return MG, torch.load(GOLDEN, weights_only=False)


def same_value(a, b, key):
    assert type(a) is type(b), key
    if isinstance(b, list):
        assert len(a) == len(b), key
        for x, y in zip(a, b):
            same_value(x, y, key)
    elif isinstance(b, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape and a.device == b.device, key
        assert torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8)), key
    elif isinstance(b, np.ndarray):
        assert a.dtype == b.dtype and np.array_equal(a, b), key
    else:
        assert a == b, key


def test_oracle_against_golden():
    """oracle/ce_waypoint_step_ref.py on the golden's inputs and stand-in encoders reproduces the unmodified reference
    branch bit for bit, with the same keys, key order, Python and numpy types"""
    MG, g = golden()
    for B in MG.BATCHES:
        case = g["B%d" % B]
        obs = MG.observations(case["inputs"])
        assert list(obs) == g["key_order"]
        enc = MG.Encoders(case["enc_seed"], case["logits"])
        idx, fts = R.pano_features()
        with torch.no_grad():
            out = R.waypoint_branch(obs, enc.depth, enc.rgb, enc.predictor, RW.nms, fts, idx)
        grid = out.pop("pano_rgb_grid")
        ref = case["outputs"]
        assert list(out) == list(ref)
        for k in ref:
            same_value(out[k], ref[k], k)
        gg = case["pano_rgb_grid"]
        assert tuple(grid.shape) == gg["shape"] and grid.dtype == gg["dtype"]
        assert torch.equal(grid.double().sum((2, 3)), gg["sums"])


def test_host_outputs_on_golden_indices():
    """host_outputs on the reference's own nonzero indices gives the reference's candidate outputs (its CPU arithmetic)"""
    MG, g = golden()
    for B in MG.BATCHES:
        case = g["B%d" % B]
        got = CS.host_outputs(case["picks"], device_type="cpu")
        for k in ("cand_angle_fts", "cand_img_idxes", "cand_angles", "cand_distances"):
            same_value(got[k], case["outputs"][k], k)
        for b, lst in enumerate(got["cand_angles"]):
            assert all(type(x) is float for x in lst) and all(type(x) is float for x in got["cand_distances"][b])
    counts = [int(c) for B in MG.BATCHES for c in g["B%d" % B]["picks"][:, 10]]
    assert min(counts) < 5 and 1 in counts


def test_vp_restatement_on_golden_outputs():
    """the restated _vp_feature_variable on the reference's outputs: the host part equals vp_host_inputs, the view
    lengths equal the picks' column 11, and the feature rows are the candidates, then the other views, then zeros"""
    MG, g = golden()
    for B in MG.BATCHES:
        case = g["B%d" % B]
        out = case["outputs"]
        ref = R.vp_feature_variable(out, "cpu")
        loc, nav, lens = CS.vp_host_inputs(out)
        assert loc.dtype == ref["loc_fts"].dtype and torch.equal(loc, ref["loc_fts"])
        assert torch.equal(nav, ref["nav_types"]) and torch.equal(lens, ref["view_lens"])
        assert lens.tolist() == case["picks"][:, 11].tolist()
        L = int(lens.max())
        for b in range(B):
            img = out["cand_img_idxes"][b]
            rest = [j for j in range(12) if j not in set(img.tolist())]
            rows = torch.cat([out["pano_rgb"][b, img], out["pano_rgb"][b, rest]])
            n = rows.shape[0]
            assert torch.equal(ref["rgb_fts"][b, :n], rows) and not bool(ref["rgb_fts"][b, n:L].any())
            drows = torch.cat([out["pano_depth"][b, img], out["pano_depth"][b, rest]])
            assert torch.equal(ref["dep_fts"][b, :n], drows)


def test_device_angle_rule():
    """a CUDA index tensor divided by 120 is multiplied by the fp32 reciprocal; the CPU divides"""
    picks = torch.zeros(1, CS.PICK_COLS, dtype=torch.int32)
    picks[0, 0], picks[0, 10] = 23, 1
    a = np.float32(23) * (np.float32(1) / np.float32(120)) * np.float32(2) * np.float32(np.pi)
    assert CS.host_outputs(picks, "cuda")["cand_angles"][0] == [float(np.float32(2 * np.pi) - a)]
    assert CS.host_outputs(picks, "cpu")["cand_angles"][0] == (2 * np.pi - torch.tensor([23.0]) / 120 * 2 * np.pi).tolist()
