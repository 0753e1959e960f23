"""Generates tests/golden/small_ce_waypoint_aug.pt by running the UNMODIFIED `waypoint` branch of the VLN-CE policy
with waypoint augmentation (bevbert_ce/vlnce_baselines/models/Policy_ViewSelection_BEV.py BEV.forward, mode='waypoint',
in_train=True) on the CPU under a fixed torch.manual_seed, from the reference checkout located by oracle/ref_shim.py
(env BEVBERT_REFERENCE):

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_ce_waypoint_aug_golden.py

The stub modules, stand-in encoders, cropped inputs and constructed logits are make_ce_waypoint_step_golden.py's (its
own output is not touched).  Cases, B = 1 and 8: picks in image 0 (angles 115-119 and 0-4) whose samples land in
counter-clockwise view 11, the wrap rows, two picks in one sector, and a single pick (the other cells underflow).

Stored (data only): the seed; per B the inputs as the seeds of make_ce_waypoint_step_golden.py's `inputs` and
`constructed_logits` with the SHA-256 of every buffer they generate (`case_inputs` regenerates them and checks the
digests, so the file stays small), the reference's output dict as returned (pano_rgb_grid as its shape and
per-(environment, view) fp64 sums), and the Exp(1) noise the sampling drew, re-drawn by re-seeding and drawing exponential_ of shape (K_j, 120) per environment in environment order (the
only draws of the branch: Categorical.sample() is torch.multinomial's argmax(p / q), q = empty_like(p).exponential_(1)).
The script checks that the re-drawn noise reproduces every sample before it writes."""
import hashlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(os.path.dirname(HERE))]

import make_ce_waypoint_step_golden as MG  # noqa: E402
from oracle import ce_waypoint_aug_ref as RA  # noqa: E402

OUT = os.path.join(HERE, "small_ce_waypoint_aug.pt")
BATCHES = (1, 8)
SEED = 2024


def digest(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def case_inputs(case):
    """-> (stored inputs, logits) of one stored case, regenerated from its seeds and checked against its digests"""
    B = case["B"]
    stored = MG.inputs(B, case["input_seed"])
    logits = MG.constructed_logits(B, case["logits_seed"])
    assert {k: (digest(buf), box) for k, (buf, box) in stored.items()} == case["input_digests"]
    assert digest(logits) == case["logits_digest"]
    return stored, logits


def redraw_noise(seed, counts):
    """the noise the branch drew after torch.manual_seed(seed): one (K_j, 120) exponential_ draw per environment"""
    torch.manual_seed(seed)
    return [torch.empty(k, 120).exponential_(1) for k in counts]


def main():
    policy, utils, mutils = MG.load_reference()
    out = {"key_order": MG.key_order(), "seed": SEED}
    view11 = 0
    for B in BATCHES:
        stored = MG.inputs(B, 40 + B)
        logits = MG.constructed_logits(B, 50 + B)
        enc = MG.Encoders(60 + B, logits)
        self = MG.stand_in_self(enc, mutils.angle_feature_torch)
        obs = MG.observations(stored)
        torch.manual_seed(SEED + B)
        with torch.no_grad():
            res = policy.BEV.forward(self, mode="waypoint", waypoint_predictor=enc.predictor, observations=obs,
                                     in_train=True)
        counts = [len(a) for a in res["cand_angles"]]
        noise = redraw_noise(SEED + B, counts)
        # the recorded noise reproduces the reference's samples
        idx, fts = self.pano_img_idxes, self.pano_angle_fts
        with torch.no_grad():
            again = RA.waypoint_branch(obs, enc.depth, enc.rgb, enc.predictor, utils.nms, fts, idx, in_train=True,
                                       noise=noise)
        for j in range(B):
            assert again["cand_angles"][j] == res["cand_angles"][j], j
            assert again["cand_distances"][j] == res["cand_distances"][j], j
            view11 += int((res["cand_img_idxes"][j] == 11).sum())
        grid = res.pop("pano_rgb_grid")
        out["B%d" % B] = {"B": B, "input_seed": 40 + B, "logits_seed": 50 + B, "enc_seed": 60 + B,
                          "input_digests": {k: (digest(buf), box) for k, (buf, box) in stored.items()},
                          "logits_digest": digest(logits), "outputs": res, "noise": noise,
                          "pano_rgb_grid": {"shape": tuple(grid.shape), "dtype": grid.dtype,
                                            "sums": grid.double().sum((2, 3))}}
    assert view11 > 0, "no image-0 sample landed in view 11"
    torch.save(out, OUT)
    print("wrote %s" % OUT)


if __name__ == "__main__":
    main()
