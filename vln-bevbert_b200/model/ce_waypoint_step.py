"""The VLN-CE policy's whole `waypoint` call on the H100 kernels, forward only: BEV.forward(mode='waypoint',
in_train=False) (bevbert_ce/vlnce_baselines/models/Policy_ViewSelection_BEV.py:166-321) and the trainer's
_vp_feature_variable (ss_trainer_BEV.py:347-384), which turns the call's outputs into the `panorama` call's inputs.

`WaypointStep` composes the three existing towers over the policy's own modules, in the reference's order:
    bb_ce_view_stack (the 12 + 12 per-heading observations -> clockwise image batches, and the 14 x 14 depth grid)
    -> DepthTower (policy.net.depth_encoder.visual_encoder) -> ClipTower (policy.net.rgb_encoder.model.visual)
    -> WaypointRunner (the trainer's predictor) -> bb_ce_waypoint_candidates (softmax, wrap, NMS, strip, nonzero
    picks, the counter-clockwise pano features, the candidate gathers and the padded panorama inputs).
Every step reads device memory only, so graphs.install_ce_waypoint_step replays it as one CUDA graph per (B, image
sizes); the observation tensors reach the graph through a 24-entry table of pointers and strides, copied to the device
before each replay.  After the replay one device-to-host copy of the picks (B, 12) int32 feeds the host-side
outputs, which use the reference's own expressions on the copied indices (`host_outputs`).

With in_train=True (waypoint augmentation, lines 229-264; graphs.install_ce_waypoint_step(net, waypoint_aug=True)) the
call draws Exp(1) noise inside the graph and bb_ce_waypoint_candidates_aug replaces each NMS pick by a sample of its
image's regional softmax, the draw torch.multinomial makes for the reference's Categorical(...).sample().

Autocast is disabled inside the call (as in the towers), so the trainer's autocast() changes no bit.  The step runs
forward only: a call with grad enabled while an encoder or predictor parameter requires grad raises, and so does a call
while the predictor is in training mode (the reference applies dropout there).
"""
import copy
import math
import types

import numpy as np
import torch

from .. import _lib
from .. import kernels as K
from .clip_visual import ClipTower
from .depth_resnet import DepthTower
from .waypoint import WaypointRunner

NUM_IMGS, NUM_ANGLES, NUM_CLASSES = 12, 120, 12
MAX_PRED, PICK_COLS, VIEW_ROWS = 5, 12, 17       # PICK_COLS: BB_CE_PICK_COLS of include/bevbert_b200.h
GRID, RGB_DIM, DEP_DIM = 14, 512, 128
_INV_120 = float(np.float32(1) / np.float32(120))


# ------------------------------------------------------------------------------------------------------ kernels
def view_stack(table, B, rgb_hw, depth_hw, device):
    """bb_ce_view_stack: `table` (24, 5) int64 on `device`, rows (ptr, sb, sh, sw, sc) of the k-th rgb view (row k) and
    depth view (row 12 + k) in element strides -> (rgb (12 B, Hr, Wr, 3) uint8, depth (12 B, Hd, Wd, 1) fp32,
    grid (12 B, 196) fp32), image (12 - k) % 12 + 12 b holding view k of environment b."""
    if table.dtype != torch.int64 or tuple(table.shape) != (2 * NUM_IMGS, 5) or not table.is_contiguous():
        raise ValueError("table must be a contiguous (24, 5) int64 tensor")
    device = torch.device(device)
    if not table.is_cuda or device.type != "cuda" or (device.index is not None and table.device != device):
        raise ValueError("table must be on the CUDA device %s, got %s" % (device, table.device))
    device = table.device
    (Hr, Wr), (Hd, Wd) = rgb_hw, depth_hw
    n = B * NUM_IMGS
    rgb = torch.empty(n, Hr, Wr, 3, dtype=torch.uint8, device=device)
    depth = torch.empty(n, Hd, Wd, 1, dtype=torch.float32, device=device)
    grid = torch.empty(n, GRID * GRID, dtype=torch.float32, device=device)
    _lib.check(_lib.load().bb_ce_view_stack(table.data_ptr(), B, Hr, Wr, Hd, Wd, rgb.data_ptr(), depth.data_ptr(),
                                            grid.data_ptr(), K._stream()), "bb_ce_view_stack")
    return rgb, depth, grid


def _candidate_outputs(logits, rgb_vec, depth_feats, noise=None):
    """checks the candidate kernels' inputs -> (B, dict of their fresh outputs)"""
    B = logits.shape[0] if logits.dim() == 3 else 0
    want = {"logits": (logits, (B, NUM_ANGLES, NUM_CLASSES)), "rgb_vec": (rgb_vec, (B * NUM_IMGS, RGB_DIM)),
            "depth_feats": (depth_feats, (B * NUM_IMGS, DEP_DIM, 4, 4))}
    if noise is not None:
        want["noise"] = (noise, (B, MAX_PRED, NUM_ANGLES))
    for name, (t, shape) in want.items():
        if t.dtype != torch.float32 or not t.is_cuda:
            raise TypeError("%s must be a float32 CUDA tensor, got %s on %s" % (name, t.dtype, t.device))
        if B == 0 or tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError("%s must be contiguous %s, got %s" % (name, shape, tuple(t.shape)))
    f = dict(dtype=torch.float32, device=logits.device)
    return B, {"picks": torch.empty(B, PICK_COLS, dtype=torch.int32, device=logits.device),
               "pano_rgb": torch.empty(B, NUM_IMGS, RGB_DIM, **f), "pano_depth": torch.empty(B, NUM_IMGS, DEP_DIM, **f),
               "cand_rgb": torch.empty(B, MAX_PRED, RGB_DIM, **f), "cand_depth": torch.empty(B, MAX_PRED, DEP_DIM, **f),
               "rgb_fts": torch.empty(B, VIEW_ROWS, RGB_DIM, **f), "dep_fts": torch.empty(B, VIEW_ROWS, DEP_DIM, **f)}


def waypoint_candidates(logits, rgb_vec, depth_feats, prob=False):
    """bb_ce_waypoint_candidates: logits (B, 120, 12), rgb_vec (12 B, 512) and depth_feats (12 B, 128, 4, 4), fp32 CUDA,
    images in clockwise order -> dict of fresh tensors: picks (B, 12) int32 (pairs, count, view length), pano_rgb,
    pano_depth, cand_rgb, cand_depth, rgb_fts, dep_fts, and with prob=True the softmax (B, 120, 12)."""
    B, out = _candidate_outputs(logits, rgb_vec, depth_feats)
    f = dict(dtype=torch.float32, device=logits.device)
    if prob:
        out["prob"] = torch.empty(B, NUM_ANGLES, NUM_CLASSES, **f)
    o = out
    _lib.check(_lib.load().bb_ce_waypoint_candidates(
        logits.data_ptr(), rgb_vec.data_ptr(), depth_feats.data_ptr(), B, o["picks"].data_ptr(),
        o["prob"].data_ptr() if prob else None, o["pano_rgb"].data_ptr(), o["pano_depth"].data_ptr(),
        o["cand_rgb"].data_ptr(), o["cand_depth"].data_ptr(), o["rgb_fts"].data_ptr(), o["dep_fts"].data_ptr(),
        K._stream()), "bb_ce_waypoint_candidates")
    return out


def waypoint_candidates_aug(logits, noise, rgb_vec, depth_feats, nms_picks=False):
    """bb_ce_waypoint_candidates_aug (in_train=True): as waypoint_candidates, with each NMS pick k of environment b
    replaced by the cell sampled from its image's regional softmax under the Exp(1) noise row noise[b, k] (noise
    (B, 5, 120) fp32 CUDA).  picks and the features follow the sampled cells; with nms_picks=True the dict also holds
    the pre-sampling picks (B, 12) int32 as "nms_picks"."""
    B, out = _candidate_outputs(logits, rgb_vec, depth_feats, noise)
    if nms_picks:
        out["nms_picks"] = torch.empty(B, PICK_COLS, dtype=torch.int32, device=logits.device)
    o = out
    _lib.check(_lib.load().bb_ce_waypoint_candidates_aug(
        logits.data_ptr(), noise.data_ptr(), rgb_vec.data_ptr(), depth_feats.data_ptr(), B, o["picks"].data_ptr(),
        o["nms_picks"].data_ptr() if nms_picks else None, o["pano_rgb"].data_ptr(), o["pano_depth"].data_ptr(),
        o["cand_rgb"].data_ptr(), o["cand_depth"].data_ptr(), o["rgb_fts"].data_ptr(), o["dep_fts"].data_ptr(),
        K._stream()), "bb_ce_waypoint_candidates_aug")
    return out


def draw_noise(B, device):
    """the Exp(1) noise of one in_train=True call, (B, 5, 120) fp32, from torch's default generator of `device` on the
    current stream: torch.multinomial's single draw is argmax(p / q) with q = empty_like(p).exponential_(1)"""
    return torch.empty(B, MAX_PRED, NUM_ANGLES, dtype=torch.float32, device=device).exponential_(1)


# ------------------------------------------------------------------------------------------------- host logic
def view_pairs(observations):
    """The (rgb key, depth key) of each view in the order BEV.forward stacks them: every key containing 'depth', in the
    dict's order, with its partner k.replace('depth', 'rgb').  None unless there are exactly 12 such keys, each with
    its partner, and the dict also has 'rgb' and 'depth' (the reference's batch templates)."""
    depth_keys = [k for k in observations.keys() if "depth" in k]
    if len(depth_keys) != NUM_IMGS or "rgb" not in observations or "depth" not in observations:
        return None
    pairs = [(k.replace("depth", "rgb"), k) for k in depth_keys]
    if any(r not in observations for r, _ in pairs):
        return None
    return pairs


def image_slot(k):
    """the clockwise image (within one environment) of the k-th view in dict order"""
    return (NUM_IMGS - k) % NUM_IMGS


def covered(observations, rgb_res, device):
    """-> (pairs, (B, Hr, Wr, Hd, Wd)) when the step computes this call, else None: 12 depth keys with rgb partners,
    uint8 rgb views (B, rgb_res, rgb_res, 3) and float32 depth views (B, Hd, Wd, 1), Hd, Wd >= 14, all on `device`
    and shaped like observations['rgb'] / ['depth']."""
    pairs = view_pairs(observations)
    if pairs is None:
        return None
    rgb0, dep0 = observations["rgb"], observations["depth"]
    if not isinstance(rgb0, torch.Tensor) or not isinstance(dep0, torch.Tensor) or rgb0.dim() != 4 or dep0.dim() != 4:
        return None
    B, Hd, Wd = dep0.shape[0], dep0.shape[1], dep0.shape[2]
    if tuple(rgb0.shape) != (B, rgb_res, rgb_res, 3) or dep0.shape[3] != 1 or B == 0 or Hd < GRID or Wd < GRID:
        return None
    for r, d in pairs:
        for t, like, dtype in ((observations[r], rgb0, torch.uint8), (observations[d], dep0, torch.float32)):
            if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.shape != like.shape or t.device != device:
                return None
    return pairs, (B, rgb_res, rgb_res, Hd, Wd)


def view_table(observations, pairs):
    """(24, 5) int64 rows (data_ptr, strides...) of the rgb views (rows 0..11) and depth views (rows 12..23)"""
    rows = [[observations[r].data_ptr()] + list(observations[r].stride()) for r, _ in pairs]
    rows += [[observations[d].data_ptr()] + list(observations[d].stride()) for _, d in pairs]
    return torch.tensor(rows, dtype=torch.int64)


def angle_features(headings):
    """models/utils.py angle_feature_torch: (sin, cos, sin 0, cos 0) per heading, as fp32 (K, 4)"""
    return torch.stack([torch.sin(headings), torch.cos(headings), torch.sin(torch.zeros_like(headings)),
                        torch.cos(torch.zeros_like(headings))]).float().T


def host_outputs(picks, device_type="cuda"):
    """The candidate outputs the reference builds per environment from nonzero's indices, from the copied picks
    (B, 12) int32 (CPU): cand_angle_fts (CPU fp32 tensors), cand_angles and cand_distances (lists of floats),
    cand_img_idxes (numpy int64).  `device_type` is where the reference's index tensors live: its counter-clockwise
    angle divides them by 120 there, and torch divides a CUDA tensor by a Python number as a multiply by the fp32
    reciprocal, which differs from the CPU's division in the last bit for 55 of the 120 angles."""
    out = {"cand_angle_fts": [], "cand_img_idxes": [], "cand_angles": [], "cand_distances": []}
    for row in picks.tolist():
        k = row[2 * MAX_PRED]
        angle_idxes = torch.tensor(row[0:2 * k:2], dtype=torch.int64)
        distance_idxes = torch.tensor(row[1:2 * k:2], dtype=torch.int64)
        angle_rad_c = angle_idxes.float() / 120 * 2 * math.pi
        a = angle_idxes.float()
        a = a * _INV_120 if device_type == "cuda" else a / 120
        angle_rad_cc = 2 * math.pi - a * 2 * math.pi
        out["cand_angle_fts"].append(angle_features(angle_rad_c))
        out["cand_angles"].append(angle_rad_cc.tolist())
        out["cand_distances"].append(((distance_idxes + 1) * 0.25).tolist())
        img_idxes = 12 - (angle_idxes.numpy() + 5) // 10
        img_idxes[img_idxes == 12] = 0
        out["cand_img_idxes"].append(img_idxes)
    return out


def vp_host_inputs(obs):
    """_vp_feature_variable's host-built inputs from the outputs dict: loc_fts (B, L, 4) fp32, nav_types (B, L) int64 and
    view_lens (B,) int64 on the CPU, L the longest view list, with the reference's per-environment expressions."""
    locs, navs = [], []
    for i in range(len(obs["cand_angles"])):
        cand = np.zeros(NUM_IMGS, dtype=bool)
        cand[obs["cand_img_idxes"][i]] = True
        locs.append(torch.cat([obs["cand_angle_fts"][i], obs["pano_angle_fts"][~cand]], dim=0))
        navs.append(torch.LongTensor([1] * len(obs["cand_angles"][i]) + [0] * (NUM_IMGS - int(np.sum(cand)))))
    L = max(x.shape[0] for x in locs)
    loc = torch.zeros(len(locs), L, 4, dtype=locs[0].dtype)
    nav = torch.zeros(len(locs), L, dtype=torch.int64)
    for i, (x, n) in enumerate(zip(locs, navs)):
        loc[i, :x.shape[0]] = x
        nav[i, :n.shape[0]] = n
    return loc, nav, torch.LongTensor([x.shape[0] for x in locs])


class StepOutputs(dict):
    """The reference's `waypoint` output dict (same keys, value types, devices and dtypes), computed by the step.  It
    also carries the step's picks (B, 12) int32 on the host (`picks`), the padded panorama inputs of the same replay
    (`padded`), which graphs.install_ce_vp_features hands to the
    `panorama` call in place of _vp_feature_variable's per-environment concatenations, and for an in_train=True call
    the (B, 5, 120) Exp(1) noise its candidates were sampled with (`noise`, else None)."""

    def vp_inputs(self):
        """_vp_feature_variable(self): rgb_fts, dep_fts (device, sliced to the longest view list), loc_fts, nav_types
        and view_lens, the last three built on the host and uploaded in one copy"""
        rgb_fts, dep_fts = self.padded
        loc, nav, lens = vp_host_inputs(self)
        parts = [loc.reshape(-1).view(torch.uint8), nav.reshape(-1).view(torch.uint8), lens.view(torch.uint8)]
        dev = torch.cat(parts).pin_memory().to(rgb_fts.device, non_blocking=True)
        n0, n1 = parts[0].numel(), parts[0].numel() + parts[1].numel()
        return {"rgb_fts": rgb_fts, "dep_fts": dep_fts,
                "loc_fts": dev[:n0].view(loc.dtype).view(loc.shape),
                "nav_types": dev[n0:n1].view(torch.int64).view(nav.shape),
                "view_lens": dev[n1:].view(torch.int64)}


class _Shadows:
    """the weight caches of the three towers, re-cast together (GraphedNavigation.refresh)"""

    def __init__(self, runtimes):
        self.runtimes = runtimes

    def refresh_all(self, padded=False):
        for rt in self.runtimes:
            rt.wc.refresh_all(padded=padded)


class WaypointStep:
    """The `waypoint` call over `net` (the policy's network: .rgb_encoder a CLIPEncoderB16, .depth_encoder a
    VlnResnetDepthEncoder without spatial output, .pano_angle_fts / .pano_img_idxes) and the predictor of the current
    call (set_predictor)."""

    def __init__(self, net):
        if getattr(net.depth_encoder, "spatial_output", False):
            raise ValueError("the waypoint step covers VlnResnetDepthEncoder with spatial_output=False (R2R-CE)")
        norm = net.rgb_encoder.rgb_transform[-1]
        self.net = net
        self.clip = ClipTower(net.rgb_encoder.model.visual, mean=norm.mean, std=norm.std, owner=net.rgb_encoder)
        self.depth = DepthTower(net.depth_encoder.visual_encoder, owner=net.depth_encoder)
        self.predictor = self.runner = None
        self.device = next(net.rgb_encoder.model.visual.parameters()).device

    training = False        # nothing in the branch depends on the network's train / eval switch

    @property
    def rt(self):
        return types.SimpleNamespace(wc=_Shadows([self.clip.rt, self.depth.rt, self.runner.rt]))

    def parameters(self):
        return [*self.clip.parameters(), *self.depth.parameters(), *self.runner.parameters()]

    def changed(self):
        """True when a parameter of any of the three modules moved since the previous call of this method."""
        moved = [self.clip.changed(), self.depth.changed(), self.runner.changed()]
        return any(moved)

    def set_predictor(self, waypoint_predictor):
        """Use `waypoint_predictor` (DataParallel-wrapped or not); -> True when the runner was (re)built."""
        module = waypoint_predictor
        if isinstance(module, (torch.nn.DataParallel, torch.nn.parallel.DistributedDataParallel)):
            module = module.module
        if module is self.predictor:
            return False
        self.predictor, self.runner = module, WaypointRunner(module)
        return True

    def check_call(self):
        self.clip.check_grad()
        self.depth.check_grad()
        self.runner.check_call()

    def run(self, table, geom, in_train=False):
        """the call on a staged view table (24, 5) and its geometry (B, Hr, Wr, Hd, Wd) -> dict of device tensors.
        in_train=True draws the call's noise (draw_noise; inside a graph every replay draws afresh) and samples the
        candidates from it; the noise is returned as "noise"."""
        B, Hr, Wr, Hd, Wd = geom
        with torch.autocast("cuda", enabled=False), torch.no_grad():
            rgb, depth, grid = view_stack(table, B, (Hr, Wr), (Hd, Wd), self.device)
            depth_feats = self.depth._encode(depth)
            rgb_vec, rgb_grid = self.clip._encode(rgb, self.clip.mean, self.clip.std)
            logits = self.runner._forward(depth_feats, B)
            if in_train:
                noise = draw_noise(B, self.device)
                out = waypoint_candidates_aug(logits, noise, rgb_vec, depth_feats.contiguous())
                out["noise"] = noise
            else:
                out = waypoint_candidates(logits, rgb_vec, depth_feats.contiguous())
        out.update(rgb_grid=rgb_grid, depth_grid=grid)
        return out

    def outputs(self, out, B):
        """the reference's output dict from the step's device outputs `out`; the copy of the picks is the call's one
        host synchronisation.  For an in_train=True call (`out` holds "noise") the reference's sampled index tensors
        are CPU tensors (torch.tensor over a list of 0-d tensors), so the angles divide on the CPU, and the result
        carries a copy of the noise as `noise`."""
        c = torch.Tensor.clone
        cand_rgb, cand_depth = c(out["cand_rgb"]), c(out["cand_depth"])
        res = {"pano_rgb": c(out["pano_rgb"]), "pano_depth": c(out["pano_depth"]),
               "pano_rgb_grid": c(out["rgb_grid"].reshape(B, NUM_IMGS, GRID * GRID, -1)),
               "pano_depth_grid": c(out["depth_grid"].view(B, NUM_IMGS, GRID * GRID, 1))}
        picks = out["picks"].cpu()
        L = int(picks[:, 2 * MAX_PRED + 1].max())
        padded = (c(out["rgb_fts"][:, :L]), c(out["dep_fts"][:, :L]))
        host = host_outputs(picks, "cpu" if "noise" in out else self.device.type)
        counts = picks[:, 2 * MAX_PRED].tolist()
        o = StepOutputs(cand_rgb=[cand_rgb[j, :k] for j, k in enumerate(counts)],
                        cand_depth=[cand_depth[j, :k] for j, k in enumerate(counts)],
                        cand_angle_fts=host["cand_angle_fts"], cand_img_idxes=host["cand_img_idxes"],
                        cand_angles=host["cand_angles"], cand_distances=host["cand_distances"],
                        pano_rgb=res["pano_rgb"], pano_depth=res["pano_depth"], pano_rgb_grid=res["pano_rgb_grid"],
                        pano_depth_grid=res["pano_depth_grid"],
                        pano_angle_fts=copy.deepcopy(self.net.pano_angle_fts),
                        pano_img_idxes=copy.deepcopy(self.net.pano_img_idxes))
        o.padded, o.picks = padded, picks
        o.noise = c(out["noise"]) if "noise" in out else None
        return o
