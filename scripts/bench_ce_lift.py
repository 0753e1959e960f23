"""The VLN-CE trainer's `lift` (ss_trainer_BEV.py:386-410) on one H100, and a whole stand-in rollout step with every
install composed.  Prints the card's name and power limit from the same run, a table per part, and one JSON line.

1. `lift` alone: the reference's torch chain on the device (heading fan uploaded by a blocking copy,
   PointCloud.forward's elementwise ops and cuBLAS bmm; restated in tests/test_ce_lift_gpu.py) against
   graphs.install_ce_lift (one pinned upload, one bb_bev_lift_points launch), at B = 1, 4 and 8 on the waypoint step's
   grid sizes.  Outputs are compared at every timed size: identical masks, and the largest ulp difference of the points.
   The arms alternate over windows; min-max over windows of ms per call, each window ending in a device synchronise.

2. A rollout step (ss_trainer_BEV.py:1013-1180) over 15-step episodes at a fixed B, in eval (no_grad, argmax) and in
   training (IL.waypoint_aug waypoint calls, the teacher-forced loss, its backward once per episode), with every
   install: install_ce_waypoint_step (waypoint_aug in training) + install_ce_vp_features, the CE navigation network
   (model/ce_nav.py, full-size configuration, seeded weights) behind the panorama / navigation calls with
   install_ce_replay, install_ce_gmap_features, install_ce_lift, and agent_bev.ce_nav_bev_variable.  It is a stand-in:
   the observations are seeded tensors (the same each step), node positions follow the predicted candidates, every
   step makes a new node linked to the previous one, and the rollout passes None for update_graph's embeddings (as
   INTEGRATION describes for an installed rollout).  The gmap keys the installs do not build (step ids, positions,
   pair distances, visited masks) come from host loops, as in the reference.  Two ways of running the same episodes:
     * `step`: ms per step, nothing added;
     * the split: the same, with a device synchronise after each part, ms per step of each part: the waypoint call,
       the panorama call (with _vp_feature_variable), the lift, gmap + BEV (_nav_gmap_variable and
       _nav_bev_variable), the navigation call, and the host glue (identify_node's stand-in and update_graph,
       update_node_pc, the stop-score .item() per environment, softmax, the action choice and its copy to the host, the
       loss).  In training the episode's backward is a part of its own, per step.  The parts of the split add up to
       more than `step`, because each synchronise stops the host from running ahead."""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import ce_lift_cases as C  # noqa: E402
import ce_nav_cases as NC  # noqa: E402
import ce_waypoint_step_cases as WC  # noqa: E402
from bevbert_b200 import agent_bev, graphs, synth  # noqa: E402
from bevbert_b200.config import make_ce_nav_config  # noqa: E402
from bevbert_b200.model.ce_nav import GlocalTextPathNavCMT  # noqa: E402
from ce_nav_bev_cases import StubGraphMap  # noqa: E402
from oracle import ce_gmap_ref as GR  # noqa: E402
from oracle import ce_waypoint_step_ref as WR  # noqa: E402
from test_ce_lift_gpu import reference_lift, ulps  # noqa: E402

DEV = "cuda"
STEPS = 15
PARTS = ("waypoint", "panorama", "lift", "gmap_bev", "navigation", "host_glue", "backward")


def bench_lift(windows, calls):
    rows = []
    for B in (1, 4, 8):
        rng = np.random.default_rng(B)
        pos = [rng.uniform(-50, 50, 3) for _ in range(B)]
        ori = [C.quaternion_at(float(rng.uniform(0, 2 * np.pi))) for _ in range(B)]
        depth = C.depth_grid(rng, B).cuda()
        rgb = C.rgb_grid(B, DEV)
        ref, ins = C.LiftTrainer(B, DEV), C.LiftTrainer(B, DEV)
        graphs.install_ce_lift(ins)
        arms = {"reference": lambda: reference_lift(ref, pos, ori, rgb, depth),
                "installed": lambda: ins.lift(pos, ori, rgb, depth)}
        got, want = arms["installed"](), arms["reference"]()
        assert torch.equal(got[1], want[1]) and got[2].data_ptr() == want[2].data_ptr()
        worst = int(ulps(got[0], want[0]).max())
        for f in arms.values():
            for _ in range(20):
                f()
        times = {k: [] for k in arms}
        for w in range(windows):
            for name in (("reference", "installed") if w % 2 == 0 else ("installed", "reference")):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(calls):
                    arms[name]()
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t0) * 1e3 / calls)
        row = {"B": B, "max_ulp_vs_bmm": worst}
        for k, v in times.items():
            row[k] = [round(min(v), 4), round(max(v), 4)]
        rows.append(row)
        print("lift B=%d  reference %.4f-%.4f ms/call  installed %.4f-%.4f ms/call  points vs bmm: %d ulp" % (
            B, *row["reference"], *row["installed"], worst))
    return rows


# --------------------------------------------------------------------------------------------- the composed step
class Policy(WC.Net):
    """The policy network's calls as BEV.forward dispatches them: `waypoint` is tests/ce_waypoint_step_cases.Net's
    branch over the project's encoders (replaced by install_ce_waypoint_step), `language` / `panorama` / `navigation`
    go to the CE navigation network `vln_bert`."""

    def __init__(self, seed, device):
        super().__init__(seed, device)
        self.vln_bert = synth.det_init_(GlocalTextPathNavCMT(make_ce_nav_config()), seed=seed).to(device)

    def forward(self, mode=None, txt_ids=None, txt_masks=None, txt_embeds=None, waypoint_predictor=None,
                observations=None, in_train=True, **kw):
        if mode == "waypoint":
            return super().forward(mode=mode, waypoint_predictor=waypoint_predictor, observations=observations,
                                   in_train=in_train)
        if mode == "language":
            return self.vln_bert.forward_txt(txt_ids, txt_masks)
        if mode == "panorama":
            return self.vln_bert.forward_panorama(*[kw[k] for k in NC.PANO_ARGS])
        kw.update(txt_embeds=txt_embeds, txt_masks=txt_masks)
        return self.vln_bert.forward_navigation(*[kw[k] for k in NC.NAV_ARGS])


class Trainer:
    """what the rollout step reads of the CE trainer: policy.net, gmaps, _vp_feature_variable and _nav_gmap_variable
    (the reference's loop, on the host but for the embeddings); `bev` is the LiftTrainer whose graph maps keep the node
    clouds (lift, update_node_pc, _nav_bev_variable)"""

    def __init__(self, net, device):
        self.policy = types.SimpleNamespace(net=net)
        self.device = device
        self._vp_feature_variable = lambda obs: WR.vp_feature_variable(obs, device)

    def _nav_gmap_variable(self, cur_vp, cur_pos, cur_ori):
        ids, fts, steps, visited = [], [], [], []
        for gmap in self.gmaps:
            nodes, ghosts = list(gmap.node_pos.keys()), list(gmap.ghost_pos.keys())
            ids.append([None] + nodes + ghosts)
            rows = [gmap.get_node_embeds(vp) for vp in nodes] + [gmap.get_node_embeds(vp) for vp in ghosts]
            fts.append(torch.stack([torch.zeros_like(rows[0])] + rows, 0))
            steps.append([0] + [gmap.node_stepId[vp] for vp in nodes] + [0] * len(ghosts))
            visited.append([False] + [True] * len(nodes) + [False] * len(ghosts))
        B, G = len(ids), max(len(i) for i in ids)
        pad = lambda rows, v: torch.tensor([r + [v] * (G - len(r)) for r in rows])       # noqa: E731
        lens = torch.tensor([len(i) for i in ids])
        dev = self.device
        return {"gmap_vp_ids": ids, "gmap_img_fts": GR.pad_tensors_wgrad(fts),
                "gmap_masks": (torch.arange(G)[None] < lens[:, None]).to(dev), "gmap_step_ids": pad(steps, 0).to(dev),
                "gmap_pos_fts": torch.zeros(B, G, 7, device=dev), "gmap_visited_masks": pad(visited, False).to(dev),
                "gmap_pair_dists": torch.zeros(B, G, G, device=dev),
                "no_vp_left": [len(i) == 1 + len(g.node_pos) for i, g in zip(ids, self.gmaps)]}


class Split:
    """times the parts of a step: each part ends in a device synchronise (off: no synchronise, nothing recorded)"""

    def __init__(self, on):
        self.on, self.ms = on, dict.fromkeys(PARTS, 0.0)

    @contextlib.contextmanager
    def __call__(self, part):
        if not self.on:
            yield
            return
        t0 = time.perf_counter()
        yield
        torch.cuda.synchronize()
        self.ms[part] += (time.perf_counter() - t0) * 1e3


def episode(tr, bev, wp, obs, lang, B, train, split):
    net = tr.policy.net
    tr.gmaps = [GR.GraphMap(False, 0.5, True, 0) for _ in range(B)]
    bev.gmaps = [StubGraphMap() for _ in range(B)]
    rng = np.random.default_rng(B)
    pos = [tuple(rng.uniform(-20, 20, 3)) for _ in range(B)]
    head = [float(rng.uniform(0, 2 * np.pi)) for _ in range(B)]
    prev = [None] * B
    stop_scores = [{} for _ in range(B)]
    loss = 0.0
    with torch.no_grad() if not train else contextlib.nullcontext():
        txt = net(mode="language", txt_ids=lang["txt_ids"], txt_masks=lang["txt_masks"])
        for k in range(STEPS):
            ori = [C.quaternion_at(h) for h in head]
            with split("waypoint"):
                wp_out = net(mode="waypoint", waypoint_predictor=wp, observations=obs, in_train=train)
            with split("panorama"):
                vp_inputs = tr._vp_feature_variable(wp_out)
                net(mode="panorama", **vp_inputs)
            with split("host_glue"):                    # identify_node's stand-in, update_graph
                cur_vp = ["s%d" % k] * B
                for i, g in enumerate(tr.gmaps):
                    ang, dis = wp_out["cand_angles"][i], wp_out["cand_distances"][i]
                    cand_pos = [np.add(pos[i], [d * np.sin(head[i] + a), 0.0, -d * np.cos(head[i] + a)])
                                for a, d in zip(ang, dis)]
                    g.update_graph(prev[i] and prev[i][0], k + 1, cur_vp[i], np.asarray(pos[i]), None,
                                   ["s%d_%d" % (k, j) for j in range(len(ang))], cand_pos, None, None)
            with split("lift"):
                pc, pc_mask, pc_feat = bev.lift(pos, ori, wp_out["pano_rgb_grid"], wp_out["pano_depth_grid"])
            with split("host_glue"):                    # update_node_pc
                for i, g in enumerate(bev.gmaps):
                    g.visit(cur_vp[i], pos[i], [prev[i]] if prev[i] else [], (pc[i], pc_mask[i], pc_feat[i]))
            with split("gmap_bev"):
                nav_inputs = tr._nav_gmap_variable(cur_vp, pos, ori)
                nav_inputs.update(bev._nav_bev_variable(cur_vp, pos, ori))
            nav_inputs["gmap_vpids"] = nav_inputs.pop("gmap_vp_ids")
            no_vp_left = nav_inputs.pop("no_vp_left")
            with split("navigation"):
                logits = net(mode="navigation", txt_embeds=txt, txt_masks=lang["txt_masks"], **nav_inputs)["fused_logits"]
            with split("host_glue"):                    # stop scores, action choice, loss, move
                probs = F.softmax(logits, 1)
                for i in range(B):
                    stop_scores[i][cur_vp[i]] = probs[i, 0].data.item()
                if train:
                    teacher = torch.tensor([len(i) - 1 for i in nav_inputs["gmap_vpids"]], device=DEV)
                    loss = loss + F.cross_entropy(logits, teacher, reduction="sum")
                a = logits.argmax(dim=-1).cpu().numpy()
                for i in range(B):
                    prev[i] = (cur_vp[i], pos[i])
                    step = 0.5 if no_vp_left[i] else 1.0
                    pos[i] = tuple(np.add(pos[i], [step * np.sin(head[i]), 0.0, -step * np.cos(head[i])]))
                    head[i] = (head[i] + 0.3 * (int(a[i]) % 3 - 1)) % (2 * np.pi)
    if train:
        with split("backward"):
            net.vln_bert.zero_grad(set_to_none=True)
            loss.backward()


def bench_step(windows):
    net, wp = Policy(31, DEV), WC.predictor(31, DEV)
    graphs.install_ce_waypoint_step(net, waypoint_aug=True)
    graphs.install_ce_replay(net.vln_bert)
    tr = Trainer(net, DEV)
    graphs.install_ce_vp_features(tr)
    graphs.install_ce_gmap_features(tr)
    rows = []
    for train in (False, True):
        net.vln_bert.train(train)
        for B in (1, 4, 8):
            bev = C.LiftTrainer(B, DEV)
            graphs.install_ce_lift(bev)
            bev._nav_bev_variable = types.MethodType(agent_bev.ce_nav_bev_variable, bev)
            obs = WC.observations(B, 500 + B, DEV)
            lang = {k: v.to(DEV) for k, v in NC.lang_inputs(B).items()}
            for on in (False, True):                     # warm-up: graphs, allocator, pinned pool
                episode(tr, bev, wp, obs, lang, B, train, Split(on))
            total, parts = [], {p: [] for p in PARTS}
            for w in range(windows):
                for on in ((False, True) if w % 2 == 0 else (True, False)):
                    s = Split(on)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    episode(tr, bev, wp, obs, lang, B, train, s)
                    torch.cuda.synchronize()
                    if on:
                        for p in PARTS:
                            parts[p].append(s.ms[p] / STEPS)
                    else:
                        total.append((time.perf_counter() - t0) * 1e3 / STEPS)
            row = {"mode": "train" if train else "eval", "B": B, "step": [round(min(total), 2), round(max(total), 2)]}
            for p in PARTS:
                if train or p != "backward":
                    row[p] = [round(min(parts[p]), 2), round(max(parts[p]), 2)]
            rows.append(row)
            print("step %-5s B=%d  " % (row["mode"], B) + "  ".join(
                "%s %.2f-%.2f" % (k, *row[k]) for k in ("step",) + PARTS if k in row) + "  ms/step")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=6)
    ap.add_argument("--calls", type=int, default=500)
    ap.add_argument("--step-windows", type=int, default=4)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ce_lift.py needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    lift = bench_lift(a.windows, a.calls)
    step = bench_step(a.step_windows)
    print(json.dumps({"card": q, "lift_ms_per_call": lift, "step_ms": step}))


if __name__ == "__main__":
    main()
