"""Seeded VLN-CE rollouts for the global-map image glue (oracle/ce_gmap_ref.py, bevbert_b200/ce_gmap.py).

`Trainer` stands in for ss_trainer_BEV's trainer: `policy.net` answers the `panorama` call with pano_embeds =
rgb_fts * scale (+ bias) and the `navigation` call with fused_logits = gmap_img_fts . w over the map (both
differentiable in their parameters, fp32 under autocast), and `_nav_gmap_variable` is the reference's loop restricted to
gmap_vp_ids, gmap_img_fts, gmap_masks and no_vp_left, on the CPU except the embeddings.  `rollout` restates the
rollout's per-step order (ss_trainer_BEV.py:1013-1180): panorama, masked mean, one update_graph per environment with
its candidate rows, _nav_gmap_variable, navigation, consume the chosen ghost, drop finished environments.  Candidates
sit at random places in each row, land on nodes, merge into ghosts or open new ones, and some environments have none."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ce_gmap_ref as R  # noqa: E402

H = 768
SCHEDULE = [8] * 5 + [5] * 5 + [1] * 5      # environments per step: episodes finish at different steps


class Net(torch.nn.Module):
    def __init__(self, seed, device):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.scale = torch.nn.Parameter((1 + torch.rand(H, generator=g)).to(device))
        self.bias = torch.nn.Parameter(torch.randn(H, generator=g).to(device))
        self.w = torch.nn.Parameter(torch.randn(H, generator=g).to(device))

    def forward(self, mode, **kw):
        if mode == "panorama":
            masks = torch.arange(kw["rgb_fts"].shape[1], device=self.w.device)[None] < kw["view_lens"][:, None]
            return kw["rgb_fts"] * self.scale + self.bias, masks
        logits = (kw["gmap_img_fts"] * self.w).sum(-1)
        return {"fused_logits": logits.masked_fill(~kw["gmap_masks"], -float("inf"))}


class Trainer:
    def __init__(self, seed, device, merge_ghost=True):
        self.policy = type("Policy", (), {})()
        self.policy.net = Net(seed, device)
        self.merge_ghost, self.device = merge_ghost, device

    def _nav_gmap_variable(self, cur_vp, cur_pos, cur_ori):
        ids, fts, lens, no_vp_left = [], [], [], []
        for gmap in self.gmaps:
            nodes, ghosts = list(gmap.node_pos.keys()), list(gmap.ghost_pos.keys())
            no_vp_left.append(len(ghosts) == 0)
            ids.append([None] + nodes + ghosts)
            rows = [gmap.get_node_embeds(vp) for vp in nodes] + [gmap.get_node_embeds(vp) for vp in ghosts]
            fts.append(torch.stack([torch.zeros_like(rows[0])] + rows, 0))
            lens.append(len(ids[-1]))
        masks = torch.arange(max(lens))[None] < torch.tensor(lens)[:, None]
        return {"gmap_vp_ids": ids, "gmap_img_fts": R.pad_tensors_wgrad(fts), "gmap_masks": masks,
                "no_vp_left": no_vp_left}


def step_inputs(rng, B, device, empty_env=None):
    """panorama inputs of one step: rgb_fts (B, V, H), nav_types (B, V) int64 with the candidates at random places
    within each row's view_lens, view_lens (B,); the environments `empty_env` (an index or a list) have no candidate"""
    ncand = rng.integers(0, 6, B)
    if empty_env is not None:
        ncand[empty_env] = 0
    lens = 12 + ncand
    V = int(lens.max())
    nav = np.zeros((B, V), np.int64)
    for i in range(B):
        nav[i, rng.choice(lens[i], ncand[i], replace=False)] = 1
    # magnitudes over 2^-12 .. 2^12 make the order of every sum show in the rounding
    x = rng.standard_normal((B, V, H)).astype(np.float32) * np.exp2(rng.integers(-12, 13, (B, V, 1))).astype(np.float32)
    return {"rgb_fts": torch.from_numpy(x).to(device), "nav_types": torch.from_numpy(nav).to(device),
            "view_lens": torch.from_numpy(lens).to(device)}, ncand


def positions(rng, gmap, cur_pos, n):
    """n candidate positions: on a node, on a ghost (a merge), or new"""
    out = []
    for _ in range(n):
        u = rng.random()
        if u < 0.2 and gmap.node_pos:
            p = list(gmap.node_pos.values())[rng.integers(len(gmap.node_pos))] + 0.1
        elif u < 0.6 and gmap.ghost_mean_pos:
            p = list(gmap.ghost_mean_pos.values())[rng.integers(len(gmap.ghost_mean_pos))] + 0.1
        else:
            p = cur_pos + rng.uniform(-20, 20, 3)
        out.append(np.asarray(p, np.float64))
    return out


def rollout(trainer, seed, schedule=SCHEDULE, train=True, reference_glue=True):
    """-> (fused_logits per step, actions per step, loss).  reference_glue=False passes None for update_graph's
    embeddings, as a rollout that no longer computes them would."""
    rng = np.random.default_rng(seed)
    net, dev = trainer.policy.net, trainer.device
    trainer.gmaps = [R.GraphMap(False, 0.5, trainer.merge_ghost, 0) for _ in range(schedule[0])]
    cur_pos = [rng.uniform(-50, 50, 3) for _ in range(schedule[0])]
    logits_all, actions_all, loss = [], [], 0.0
    for stepk, B in enumerate(schedule):
        while len(trainer.gmaps) > B:           # a middle environment's episode ends, as ss_trainer_BEV.py:1238-1246 pops
            j = len(trainer.gmaps) // 2
            trainer.gmaps.pop(j)
            cur_pos.pop(j)
        vp_inputs, ncand = step_inputs(rng, B, dev, empty_env=0 if stepk == 3 else None)
        pano_embeds, pano_masks = net(mode="panorama", **vp_inputs)
        cur_vp = [str(len(g.node_pos)) for g in trainer.gmaps]
        cand_vp = [["%s_%d" % (cur_vp[i], k) for k in range(ncand[i])] for i in range(B)]
        cand_pos = [positions(rng, g, cur_pos[i], ncand[i]) for i, g in enumerate(trainer.gmaps)]
        if reference_glue:
            R.update_graphs(trainer.gmaps, stepk + 1, pano_embeds, pano_masks, vp_inputs["nav_types"], cur_vp,
                            cur_pos, cand_vp, cand_pos)
        else:
            for i, g in enumerate(trainer.gmaps):
                g.update_graph(None, stepk + 1, cur_vp[i], cur_pos[i], None, cand_vp[i], cand_pos[i], None, None)
        nav_inputs = trainer._nav_gmap_variable(cur_vp, cur_pos, None)
        nav_inputs["gmap_masks"] = nav_inputs["gmap_masks"].to(dev)
        no_vp_left = nav_inputs.pop("no_vp_left")
        logits = net(mode="navigation", **nav_inputs)["fused_logits"]
        if train:
            teacher = torch.tensor([len(ids) - 1 for ids in nav_inputs["gmap_vp_ids"]], device=dev)
            loss = loss + torch.nn.functional.cross_entropy(logits, teacher, reduction="sum")
        a = logits.argmax(-1).cpu().numpy()
        logits_all.append(logits.detach())
        actions_all.append(a)
        for i, g in enumerate(trainer.gmaps):
            vp = nav_inputs["gmap_vp_ids"][i][a[i]]
            if not no_vp_left[i] and vp is not None and vp.startswith("g"):
                cur_pos[i] = g.ghost_mean_pos[vp]
                g.delete_ghost(vp)
            else:
                cur_pos[i] = cur_pos[i] + rng.uniform(-3, 3, 3)
    return logits_all, actions_all, loss


# Episodes of the golden file (tests/golden/make_ce_gmap_golden.py): the reference GraphMap's own constructor arguments,
# environments per step (a middle one finishes), and a step where no environment has a candidate.
GOLDEN_CASES = [
    {"seed": 41, "has_real_pos": True, "merge_ghost": True, "ghost_aug": 0.3, "schedule": [5, 5, 5, 4, 4, 3, 3, 2],
     "empty_step": 2},
    {"seed": 42, "has_real_pos": False, "merge_ghost": False, "ghost_aug": 0.0, "schedule": [4, 4, 3, 3, 3, 1],
     "empty_step": 4},
]


def label(h):
    """a ce_gmap handle as data: ("n", s, i) for a node, the (s, i, k) terms in merge order for a ghost"""
    return ("n", h.s, h.i) if hasattr(h, "s") else tuple(tuple(t) for t in h.terms)


def golden_episode(case, graph_map, trainer, nav_gmap_variable, handles=False):
    """One seeded episode of the rollout's graph steps on the CPU: per step the panorama inputs (pano_embeds = rgb_fts),
    update_graph for every environment, nav_gmap_variable(cur_vp, cur_pos, cur_ori) (cur_ori a heading), then a seeded
    action that consumes the chosen ghost.  handles=False passes the rollout's embeddings (lines 1032-1033, 1060-1066);
    handles=True is the install's host half: GraphMaps attached to a ce_gmap.Memory, None embeddings, and the method
    run by ce_gmap.trainer_method.  -> per step (the method's dict, its rows as labels or None, input digests)"""
    import hashlib
    from bevbert_b200 import ce_gmap
    np.random.seed(case["seed"])            # GraphMap's ghost_aug noise draws from numpy's global generator
    rng = np.random.default_rng(case["seed"])
    sched = case["schedule"]
    trainer.gmaps = [graph_map(case["has_real_pos"], 0.5, case["merge_ghost"], case["ghost_aug"]) for _ in range(sched[0])]
    mem = ce_gmap.Memory() if handles else None
    if handles:
        for g in trainer.gmaps:
            ce_gmap.attach(trainer, g, mem)
    pos = [rng.uniform(-50, 50, 3) for _ in range(sched[0])]
    ori = [float(rng.uniform(0, 2 * np.pi)) for _ in range(sched[0])]
    prev = [None] * sched[0]
    steps = []
    for stepk, B in enumerate(sched):
        while len(trainer.gmaps) > B:
            j = len(trainer.gmaps) // 2
            for lst in (trainer.gmaps, pos, ori, prev):
                lst.pop(j)
        inputs, ncand = step_inputs(rng, B, "cpu", empty_env=list(range(B)) if stepk == case["empty_step"] else None)
        digests = {k: hashlib.sha256(v.numpy().tobytes()).hexdigest() for k, v in inputs.items()}
        pano, nav = inputs["rgb_fts"], inputs["nav_types"]
        masks = torch.arange(pano.shape[1])[None] < inputs["view_lens"][:, None]
        cur_vp = [str(len(g.node_pos)) for g in trainer.gmaps]
        cand_pos = [positions(rng, g, pos[i], ncand[i]) for i, g in enumerate(trainer.gmaps)]
        if handles:
            mem.steps.append(None)
        else:
            avg = torch.sum(pano * masks.unsqueeze(2), 1) / torch.sum(masks, 1, keepdim=True)
        for i, g in enumerate(trainer.gmaps):
            cand_vp = ["%s_%d" % (cur_vp[i], k) for k in range(ncand[i])]
            real = [p + 0.05 for p in cand_pos[i]] if case["has_real_pos"] else None
            cur_e, cand_e = (None, None) if handles else (avg[i], pano[i][nav[i] == 1])
            g.update_graph(prev[i], stepk + 1, cur_vp[i], pos[i], cur_e, cand_vp, cand_pos[i], cand_e, real)
        if handles:
            out, rows = ce_gmap.trainer_method(nav_gmap_variable, trainer.gmaps, cur_vp, pos, ori)
            rows = [[label(h) for h in r] for r in rows]
        else:
            out, rows = nav_gmap_variable(cur_vp, pos, ori), None
        steps.append((out, rows, digests))
        for i, g in enumerate(trainer.gmaps):
            ids = out["gmap_vp_ids"][i]
            vp = ids[int(rng.integers(len(ids)))]
            prev[i] = cur_vp[i]
            if vp is not None and vp.startswith("g"):
                pos[i] = np.asarray(g.ghost_mean_pos[vp], np.float64)
                g.delete_ghost(vp)
            else:
                pos[i] = pos[i] + rng.uniform(-3, 3, 3)
            ori[i] = float(rng.uniform(0, 2 * np.pi))
    return steps
