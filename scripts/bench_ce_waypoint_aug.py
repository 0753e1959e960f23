"""Times the VLN-CE policy's `waypoint` call with waypoint augmentation (in_train=True, the trainer's IL.waypoint_aug
rollouts) plus the trainer's _vp_feature_variable per step, at B environments (12 B views of 224 x 224 rgb and cropped
256 x 256 depth), from CUDA events over alternating windows (min-max of the windows):

    (a) `per_module_replays`: the reference branch with in_train=True (oracle/ce_waypoint_aug_ref.py, the reference's
        own operations and sampling) and _vp_feature_variable around the three per-module replays
        (install_ce_rgb_encoder, install_ce_depth_encoder, install_ce_waypoint_predictor) with bb_waypoint_nms;
    (b) `reference_encoders`: the same branch around the reference's own encoders and predictor on PyTorch (the CLIP
        and depth towers as the fp16-autocast arms of oracle/ce_clip_ref.py and oracle/ce_depth_ref.py, the predictor
        module's own forward), which is what an in_train=True call runs under install_ce_waypoint_step's default;
    (c) `installed_step`: install_ce_waypoint_step(waypoint_aug=True) + install_ce_vp_features, one graph replay.

Per size it also reports the growth of allocated device memory over (c)'s first in_train=True call, made after the
in_train=False graph of the same size was captured (the second graph set), and the card's name and power limit, read
in the same run.

    python scripts/bench_ce_waypoint_aug.py [--sizes 1,4,8] [--iters 10] [--windows 6] [--out file.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import ce_waypoint_step_cases as C  # noqa: E402
from bench_ce_waypoint import card  # noqa: E402
from bevbert_b200 import graphs  # noqa: E402
from bevbert_b200.model import waypoint as WP  # noqa: E402
from oracle import ce_clip_ref as RC  # noqa: E402
from oracle import ce_depth_ref as RD  # noqa: E402
from oracle import ce_waypoint_aug_ref as RA  # noqa: E402
from oracle import ce_waypoint_step_ref as R  # noqa: E402

SEED = 31


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,4,8")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--windows", type=int, default=6)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ce_waypoint_aug.py measures on the GPU"
    name, pl = card()
    # each setup runs on its own twin modules with the same weights: the per-module installs and the step each keep
    # weight caches, and two caches over one module would move its packed biases back and forth between calls
    net, wp = C.Net(SEED, "cuda"), C.predictor(SEED, "cuda")
    net_b, wp_b = C.Net(SEED, "cuda"), C.predictor(SEED, "cuda")
    net_c, wp_c = C.Net(SEED, "cuda"), C.predictor(SEED, "cuda")
    graphs.install_ce_rgb_encoder(net.rgb_encoder)
    graphs.install_ce_depth_encoder(net.depth_encoder)
    graphs.install_ce_waypoint_predictor(wp)
    graphs.install_ce_waypoint_step(net_c, waypoint_aug=True)
    trainer = type("Trainer", (), {})()
    trainer._vp_feature_variable = lambda obs: R.vp_feature_variable(obs, "cuda")
    graphs.install_ce_vp_features(trainer)
    depth_enc = net.depth_encoder.visual_encoder
    vis_sd = {k: v.cpu() for k, v in net_b.rgb_encoder.model.visual.state_dict().items()}
    dep_sd = dict(net_b.depth_encoder.visual_encoder.state_dict())
    clip16 = RC.Fp16Tower(vis_sd).to("cuda")
    rows = []
    for B in [int(s) for s in a.sizes.split(",")]:
        obs = C.observations(B, 40 + B, "cuda", crop=True)

        def per_module():
            out = RA.waypoint_branch(obs, lambda o: depth_enc(o), net.rgb_encoder, wp, WP.nms, net.pano_angle_fts,
                                     net.pano_img_idxes, in_train=True)
            return out, R.vp_feature_variable(out, "cuda")

        def reference_encoders():
            out = RA.waypoint_branch(obs, lambda o: RD.forward_fp16(dep_sd, o["depth"]),
                                     lambda o: RC.forward_fp16(clip16, o["rgb"]), wp_b, WP.nms, net_b.pano_angle_fts,
                                     net_b.pano_img_idxes, in_train=True)
            return out, R.vp_feature_variable(out, "cuda")

        def installed():
            out = net_c(mode="waypoint", waypoint_predictor=wp_c, observations=obs, in_train=True)
            return out, trainer._vp_feature_variable(out)

        paths = {"per_module_replays": per_module, "reference_encoders": reference_encoders,
                 "installed_step": installed}
        with torch.no_grad():
            net_c(mode="waypoint", waypoint_predictor=wp_c, observations=obs, in_train=False)
            torch.cuda.synchronize()
            m0 = torch.cuda.memory_allocated()
            installed()
            torch.cuda.synchronize()
            growth = torch.cuda.memory_allocated() - m0
            got = installed()[0]
            # the reference branch fed the step's own noise around (a)'s towers picks the step's candidates
            ref = RA.waypoint_branch(obs, lambda o: depth_enc(o), net.rgb_encoder, wp, WP.nms, net.pano_angle_fts,
                                     net.pano_img_idxes, in_train=True, noise=got.noise)
            for _ in range(2):
                for f in paths.values():
                    f()
            torch.cuda.synchronize()
            times = {k: [] for k in paths}
            for w in range(a.windows):
                for k, f in (paths.items() if w % 2 == 0 else reversed(list(paths.items()))):
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    for _ in range(a.iters):
                        f()
                    e.record()
                    e.synchronize()
                    times[k].append(s.elapsed_time(e) / a.iters)
        row = {"B": B, "gpu": name, "power_limit": pl,
               "ms": {k: {"min": round(min(t), 3), "max": round(max(t), 3)} for k, t in times.items()},
               "same_candidates_given_noise": got["cand_angles"] == ref["cand_angles"]
               and got["cand_distances"] == ref["cand_distances"],
               "second_graph_memory_mb": round(growth / 2 ** 20, 1)}
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
