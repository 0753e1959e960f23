"""Generates tests/golden/small_ce_waypoint_step.pt by running the UNMODIFIED `waypoint` branch of the VLN-CE policy
(bevbert_ce/vlnce_baselines/models/Policy_ViewSelection_BEV.py BEV.forward, mode='waypoint', in_train=False) on the
CPU, with the reference's own waypoint_pred/utils.py `nms` and models/utils.py `angle_feature_torch`, from the reference
checkout located by oracle/ref_shim.py (env BEVBERT_REFERENCE):

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_ce_waypoint_step_golden.py

Policy_ViewSelection_BEV.py imports gym, habitat, habitat_baselines and the policy's other modules at its top, and
models/utils.py imports `turtle`; those are stub modules here (none of them is used by the branch).  BEV.forward runs
as a plain function on a stand-in `self` whose encoders and predictor are small seeded functions of their inputs:
    depth_encoder(obs)  -> the 4 x 4 average pool of obs['depth'] times a seeded per-channel scale, (12 B, 128, 4, 4)
    rgb_encoder(obs)    -> (pixel means of obs['rgb'] @ a seeded (3, 512) matrix, a (12 B, 196, 768) grid of
                           them @ a seeded (3, 768) matrix)
    predictor(rgb, dep) -> constructed logits (`logits`) + 1e-3 x each view's mean depth feature, broadcast per angle
and the pools and pano features BEV.__init__ builds.  Inputs: B = 1 and 3, the trainer's key order with 'instruction'
and 'progress' among the 12 rgb<h> / depth<h> pairs, every view a crop of a NaN-bordered buffer (non-contiguous), and
logits whose picks cover the wrap rows, two candidates in one view, angles 115-119 and 0-4 (image 0), fewer than five
candidates and softmax values that underflow to 0.

Stored (data only): per B the inputs (buffers, crop box, key order, encoder seeds), the reference's output dict with
every value as returned (Python floats, numpy int64 arrays, CPU tensors) except `pano_rgb_grid`, kept as its shape and
per-(environment, view) fp64 sums; and the (B, 12) int32 picks (angle, distance pairs, count, view length) of the
reference `nms` on the same heatmap, taken with `nonzero` as the branch does."""
import importlib
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT]

from oracle import ref_shim  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "small_ce_waypoint_step.pt")
BATCHES = (1, 3)
HEADINGS = [""] + ["_%d" % (30 * a) for a in range(1, 12)]
RGB_HW, DEPTH_HW, PAD = (20, 18), (30, 28), (3, 2)


def key_order():
    keys = ["instruction"]
    for i, h in enumerate(HEADINGS):
        keys += ["rgb" + h, "depth" + h]
        if i == 5:
            keys.append("progress")
    return keys


def inputs(B, seed):
    """-> {key: (buffer, crop box or None)}: views are [:, r0:r0 + H, c0:c0 + W] of NaN / 255-bordered buffers"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    (Hr, Wr), (Hd, Wd), (r0, c0) = RGB_HW, DEPTH_HW, PAD
    for k in key_order():
        if k.startswith("rgb"):
            buf = torch.full((B, Hr + 2 * r0, Wr + 2 * c0, 3), 255, dtype=torch.uint8)
            buf[:, r0:r0 + Hr, c0:c0 + Wr] = torch.randint(0, 256, (B, Hr, Wr, 3), generator=g, dtype=torch.uint8)
            out[k] = (buf, (r0, c0, Hr, Wr))
        elif k.startswith("depth"):
            buf = torch.full((B, Hd + 2 * r0, Wd + 2 * c0, 1), float("nan"))
            buf[:, r0:r0 + Hd, c0:c0 + Wd] = torch.rand(B, Hd, Wd, 1, generator=g) * torch.exp2(
                torch.randint(-6, 7, (B, Hd, Wd, 1), generator=g).float())
            out[k] = (buf, (r0, c0, Hd, Wd))
        else:
            out[k] = (torch.randint(0, 100, (B, 7), generator=g), None)
    return out


def observations(stored):
    """the observation dict of stored inputs, views as crops (non-contiguous)"""
    obs = {}
    for k, (buf, box) in stored.items():
        obs[k] = buf if box is None else buf[:, box[0]:box[0] + box[2], box[1]:box[1] + box[3]]
    return obs


def constructed_logits(B, seed):
    """(B, 120, 12): per environment one of: peaks at angles 119 / 0 (wrap rows) and 116 / 2; two candidates in one view
    (angles 21 and 23); one dominant cell, the rest underflowing to 0"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 120, 12, generator=g)
    for b in range(B):
        kind = b % 3
        if kind == 0:
            x[b, 119, 3] = x[b, 0, 9] = 9.0
            x[b, 116, 0] = x[b, 2, 11] = 8.0
            x[b, 115, 6] = x[b, 4, 1] = 7.5
        elif kind == 1:
            x[b, 21, 0] = 9.0
            x[b, 23, 11] = 8.5
        else:
            x[b] = -200.0
            x[b, 60, 6] = 200.0
    return x


class Encoders:
    """the seeded stand-in encoders and predictor (pure torch, CPU or CUDA)"""

    def __init__(self, seed, logits):
        g = torch.Generator().manual_seed(seed)
        self.dscale = torch.rand(128, generator=g) + 0.5
        self.wrgb = torch.randn(3, 512, generator=g)
        self.wgrid = torch.randn(3, 768, generator=g)
        self.logits = logits

    def depth(self, obs):
        d = obs["depth"].permute(0, 3, 1, 2)
        return F.adaptive_avg_pool2d(d, (4, 4)) * self.dscale.to(d.device).view(1, 128, 1, 1)

    def rgb(self, obs):
        x = obs["rgb"].float()
        vec = x.mean((1, 2)) @ self.wrgb.to(x.device)
        grid = F.adaptive_avg_pool2d(x.permute(0, 3, 1, 2), (14, 14)).flatten(2).transpose(1, 2)
        return vec, grid @ self.wgrid.to(x.device)

    def predictor(self, rgb, dep):
        B = rgb.shape[0] // 12
        view = dep.reshape(B, 12, -1).mean(-1)                      # (B, 12)
        return self.logits.to(dep.device) + 1e-3 * view.repeat_interleave(10, 1).unsqueeze(-1)


def stand_in_self(enc, angle_feature_torch):
    """the attributes BEV.forward's waypoint branch reads, built as BEV.__init__ builds them"""
    s = types.SimpleNamespace()
    s.depth_encoder, s.rgb_encoder = enc.depth, enc.rgb
    s.space_pool_depth = nn.Sequential(nn.AdaptiveAvgPool2d((1, 1)), nn.Flatten(start_dim=2))
    s.grid_pool_depth = nn.Sequential(nn.AdaptiveAvgPool2d((14, 14)), nn.Flatten(start_dim=1))
    s.space_pool_rgb = nn.Sequential(nn.AdaptiveAvgPool2d((1, 1)), nn.Flatten(start_dim=2))
    s.pano_img_idxes = np.arange(0, 12, dtype=np.int64)
    s.pano_angle_fts = angle_feature_torch(torch.from_numpy((1 - s.pano_img_idxes / 12) * 2 * math.pi))
    return s


def _pkg(name, path=None, **attrs):
    m = types.ModuleType(name)
    if path is not None:
        m.__path__ = [path]
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def load_reference():
    """-> (Policy_ViewSelection_BEV module, waypoint_pred utils module, models utils module) of the unmodified reference"""
    base = os.path.join(ref_shim.REF_ROOT, "bevbert_ce", "vlnce_baselines")
    if not os.path.isdir(base):
        raise RuntimeError("CE reference tree not found under %s" % ref_shim.REF_ROOT)
    sys.dont_write_bytecode = True
    stub_class = lambda name: type(name, (nn.Module,), {})   # noqa: E731
    _pkg("gym", Space=stub_class("Space"))
    _pkg("habitat", Config=stub_class("Config"))
    _pkg("turtle", heading=None)
    _pkg("habitat_baselines", "")
    _pkg("habitat_baselines.common", "")
    _pkg("habitat_baselines.common.baseline_registry",
         baseline_registry=types.SimpleNamespace(register_policy=lambda cls: cls))
    _pkg("habitat_baselines.rl", "")
    _pkg("habitat_baselines.rl.models", "")
    _pkg("habitat_baselines.rl.models.rnn_state_encoder", build_rnn_state_encoder=None)
    _pkg("habitat_baselines.rl.ppo", "")
    _pkg("habitat_baselines.rl.ppo.policy", Net=stub_class("Net"))
    _pkg("vlnce_baselines", base)
    _pkg("vlnce_baselines.models", os.path.join(base, "models"))
    _pkg("vlnce_baselines.models.bev", "")
    _pkg("vlnce_baselines.models.bev.vlnbert_init", get_vlnbert_models=None)
    _pkg("vlnce_baselines.common", "")
    _pkg("vlnce_baselines.common.aux_losses", AuxLosses=None)
    _pkg("vlnce_baselines.models.encoders", "")
    _pkg("vlnce_baselines.models.encoders.instruction_encoder", InstructionEncoder=None)
    _pkg("vlnce_baselines.models.encoders.resnet_encoders", TorchVisionResNet50=None, VlnResnetDepthEncoder=None,
         CLIPEncoder=None, CLIPEncoderB16=None)
    _pkg("vlnce_baselines.models.policy", ILPolicy=stub_class("ILPolicy"))
    _pkg("vlnce_baselines.waypoint_pred", os.path.join(base, "waypoint_pred"))
    _pkg("vlnce_baselines.waypoint_pred.TRM_net", BinaryDistPredictor_TRM=None)
    utils = importlib.import_module("vlnce_baselines.waypoint_pred.utils")
    mutils = importlib.import_module("vlnce_baselines.models.utils")
    policy = importlib.import_module("vlnce_baselines.models.Policy_ViewSelection_BEV")
    for m in (utils, mutils, policy):
        assert m.__file__.startswith(base), m.__file__
    return policy, utils, mutils


def reference_picks(utils, logits):
    """the branch's nonzero indices of the stripped NMS map, as (B, 12) int32 picks"""
    B = logits.shape[0]
    x = torch.softmax(logits.reshape(B, 1440), dim=1).reshape(B, 120, 12)
    x = torch.cat((x[:, -1:, :], x, x[:, :1, :]), dim=1)
    out = utils.nms(x.unsqueeze(1), max_predictions=5, sigma=(7.0, 5.0)).squeeze(1)[:, 1:-1, :]
    picks = torch.zeros(B, 12, dtype=torch.int32)
    for b in range(B):
        nz = out[b].nonzero()
        K = nz.shape[0]
        picks[b, :2 * K] = nz.reshape(-1).to(torch.int32)
        img = 12 - (nz[:, 0].numpy() + 5) // 10
        img[img == 12] = 0
        picks[b, 10], picks[b, 11] = K, K + 12 - len(set(img.tolist()))
    return picks


def main():
    policy, utils, mutils = load_reference()
    out = {"key_order": key_order()}
    for B in BATCHES:
        stored = inputs(B, 10 + B)
        logits = constructed_logits(B, 20 + B)
        # the predictor adds 1e-3 x the mean depth feature to these logits; the picks below are taken on the logits the
        # branch actually sees
        enc = Encoders(30 + B, logits)
        self = stand_in_self(enc, mutils.angle_feature_torch)
        obs = observations(stored)
        with torch.no_grad():
            res = policy.BEV.forward(self, mode="waypoint", waypoint_predictor=enc.predictor, observations=obs,
                                     in_train=False)
            seen = enc.predictor(torch.zeros(12 * B, 512), enc.depth({"depth": _stacked_depth(obs)}))
        grid = res.pop("pano_rgb_grid")
        out["B%d" % B] = {"inputs": stored, "logits": logits, "enc_seed": 30 + B, "outputs": res,
                          "pano_rgb_grid": {"shape": tuple(grid.shape), "dtype": grid.dtype,
                                            "sums": grid.double().sum((2, 3))},
                          "picks": reference_picks(utils, seen)}
    torch.save(out, OUT)
    print("wrote %s" % OUT)


def _stacked_depth(obs):
    """the branch's clockwise depth batch (restated only to evaluate the stand-in predictor's logits for the picks)"""
    depth_keys = [k for k in obs if "depth" in k]
    B = obs["depth"].shape[0]
    d = torch.zeros(12 * B, *obs["depth"].shape[1:])
    for a, k in enumerate(depth_keys):
        for b in range(B):
            d[(12 - a) % 12 + 12 * b] = obs[k][b]
    return d


if __name__ == "__main__":
    main()
