"""Shared inputs of the CE waypoint-step tests and benchmark: a stand-in policy network over the project's encoder
modules (the reference's attribute layout), per-heading observation dicts in the trainer's key order, and constructed
heatmap logits."""
import types

import torch

from bevbert_b200 import synth
from bevbert_b200.model import clip_visual as CV
from bevbert_b200.model import depth_resnet as D
from bevbert_b200.model import waypoint as WP
from oracle import ce_waypoint_step_ref as R

HEADINGS = [""] + ["_%d" % (30 * a) for a in range(1, 12)]


def observations(B, seed, device, crop=False, depth_hw=(256, 256)):
    """The trainer's batch: 'instruction' and 'progress' mixed among rgb<h> / depth<h> keys of 12 headings.  crop=True
    hands over center-cropped views of larger NaN-bordered buffers, as habitat's crop transform does."""
    g = torch.Generator().manual_seed(seed)
    obs = {"instruction": torch.randint(0, 100, (B, 20), generator=g).to(device)}
    Hd, Wd = depth_hw
    for i, h in enumerate(HEADINGS):
        rgb = torch.randint(0, 256, (B, 224, 224, 3), generator=g, dtype=torch.uint8)
        dep = torch.rand(B, Hd, Wd, 1, generator=g)
        if crop:
            big = torch.randint(0, 256, (B, 240, 232, 3), generator=g, dtype=torch.uint8)
            big[:, 8:232, 4:228] = rgb
            rgb = big.to(device)[:, 8:232, 4:228]
            bigd = torch.full((B, Hd + 6, Wd + 10, 1), float("nan"))
            bigd[:, 3:3 + Hd, 5:5 + Wd] = dep
            dep = bigd.to(device)[:, 3:3 + Hd, 5:5 + Wd]
        obs["rgb" + h] = rgb.to(device)
        obs["depth" + h] = dep.to(device)
        if i == 5:
            obs["progress"] = torch.zeros(B, device=device)
    return obs


class Net(torch.nn.Module):
    """BEV's attributes the waypoint call reads (rgb_encoder.model.visual, rgb_encoder.rgb_transform,
    depth_encoder.visual_encoder, pano_angle_fts, pano_img_idxes); forward is the reference branch
    (oracle/ce_waypoint_step_ref.py) around the eager towers and bb_waypoint_nms.  `calls` counts its runs."""

    def __init__(self, seed, device):
        super().__init__()
        vis = CV.VisionTransformer(**synth.CLIP_B16)
        vis.load_state_dict(synth.clip_visual_state(seed))
        self.rgb_encoder = torch.nn.Module()
        self.rgb_encoder.model = torch.nn.Module()
        self.rgb_encoder.model.visual = vis
        self.rgb_encoder.rgb_transform = [types.SimpleNamespace(mean=CV.CLIP_MEAN, std=CV.CLIP_STD)]
        enc = D.depth_encoder(256, 256)
        enc.load_state_dict(synth.depth_encoder_state(seed))
        self.depth_encoder = torch.nn.Module()
        self.depth_encoder.visual_encoder = enc
        self.depth_encoder.spatial_output = False
        self.pano_img_idxes, self.pano_angle_fts = R.pano_features()
        self.to(device).requires_grad_(False)
        self.clip = CV.ClipTower(vis, owner=self.rgb_encoder)
        self.depth = D.DepthTower(enc, owner=self.depth_encoder)
        self.calls = 0

    def forward(self, mode=None, txt_ids=None, txt_masks=None, txt_embeds=None, waypoint_predictor=None,
                observations=None, in_train=True):
        self.calls += 1
        if mode != "waypoint":
            return mode
        return R.waypoint_branch(observations, lambda o: self.depth.encode(o["depth"]),
                                 lambda o: self.clip.encode_rgb(o["rgb"]), waypoint_predictor, WP.nms,
                                 self.pano_angle_fts, self.pano_img_idxes)


def predictor(seed, device):
    m = WP.BinaryDistPredictor_TRM()
    m.load_state_dict(synth.waypoint_state(seed))
    return m.to(device).requires_grad_(False).eval()


def constructed_logits(B, seed):
    """(B, 120, 12) logits whose picks cover the wrap rows, candidates sharing a view, angles 115-119 and 0-4 (image 0),
    fewer than 5 candidates, and softmax values that underflow to 0"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 120, 12, generator=g)
    for b in range(B):
        kind = b % 5
        if kind == 0:       # peaks at angles 119 and 0 (wrap rows of the padded map) and 116, 2
            x[b, 119, 3] = x[b, 0, 9] = 9.0
            x[b, 116, 0] = x[b, 2, 11] = 8.0
        elif kind == 1:     # two candidates in one view (angles 21 and 23 -> image 10), far apart in distance
            x[b, 21, 0] = 9.0
            x[b, 23, 11] = 8.5
        elif kind == 2:     # one dominant cell: every other probability underflows to 0 -> a single candidate
            x[b] = -200.0
            x[b, 60, 6] = 200.0
        elif kind == 3:     # two cells, the rest underflows: picks in later rounds are zeros (fewer than 5)
            x[b] = -300.0
            x[b, 30, 2] = x[b, 90, 7] = 0.0
        else:               # angles 115-119 and 0-4 all map to image 0
            x[b, 115, 1] = x[b, 4, 10] = 9.0
    return x
