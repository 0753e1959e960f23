"""Times the VLN-CE policy's `waypoint` call plus the trainer's _vp_feature_variable per step, at B environments (12 B
views of 224 x 224 rgb and 256 x 256 depth), from CUDA events over alternating windows (min-max of the windows):

    (a) `per_module_replays`: the reference branch (oracle/ce_waypoint_step_ref.py, the reference's own operations)
        and _vp_feature_variable around the three per-module replays (install_ce_rgb_encoder, install_ce_depth_encoder,
        install_ce_waypoint_predictor) with bb_waypoint_nms;
    (c) `installed_step`: install_ce_waypoint_step + install_ce_vp_features, one graph replay per call.
    `replays_only`: the three per-module replays alone on pre-stacked views, so (a) minus it is the glue's cost.

The reference as shipped (fp16-autocast towers) is not timed here.  Per size it also reports whether (c) picked the
same candidates as (a), the memory the step's graphs hold, and the card's name and power limit, read in the same run.

    python scripts/bench_ce_waypoint_step.py [--sizes 1,4,8] [--iters 10] [--windows 6] [--out file.json]
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
from oracle import ce_waypoint_step_ref as R  # noqa: E402

SEED = 31


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,4,8")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--windows", type=int, default=6)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ce_waypoint_step.py measures on the GPU"
    name, pl = card()
    # (a) and (c) run on twin modules with the same weights: the per-module installs and the step each keep weight
    # caches, and two caches over one module would move its packed biases back and forth between calls
    net, wp = C.Net(SEED, "cuda"), C.predictor(SEED, "cuda")
    net_c, wp_c = C.Net(SEED, "cuda"), C.predictor(SEED, "cuda")
    graphs.install_ce_rgb_encoder(net.rgb_encoder)
    graphs.install_ce_depth_encoder(net.depth_encoder)
    graphs.install_ce_waypoint_predictor(wp)
    graphs.install_ce_waypoint_step(net_c)
    trainer = type("Trainer", (), {})()
    trainer._vp_feature_variable = lambda obs: R.vp_feature_variable(obs, "cuda")
    graphs.install_ce_vp_features(trainer)
    depth_enc = net.depth_encoder.visual_encoder
    rows = []
    for B in [int(s) for s in a.sizes.split(",")]:
        obs = C.observations(B, 40 + B, "cuda", crop=True)
        dep12 = torch.zeros_like(obs["depth"]).repeat(12, 1, 1, 1)
        rgb12 = torch.zeros_like(obs["rgb"]).repeat(12, 1, 1, 1)
        view12 = {"rgb": rgb12, "depth": dep12}

        def per_module():
            out = R.waypoint_branch(obs, lambda o: depth_enc(o), net.rgb_encoder, wp, WP.nms, net.pano_angle_fts,
                                    net.pano_img_idxes)
            return out, R.vp_feature_variable(out, "cuda")

        def installed():
            out = net_c(mode="waypoint", waypoint_predictor=wp_c, observations=obs, in_train=False)
            return out, trainer._vp_feature_variable(out)

        def replays_only():
            rgb_vec, _ = net.rgb_encoder(view12)
            return wp(rgb_vec, depth_enc(view12))

        paths = {"per_module_replays": per_module, "installed_step": installed, "replays_only": replays_only}
        with torch.no_grad():
            torch.cuda.synchronize()
            m0 = torch.cuda.memory_allocated()
            installed()
            torch.cuda.synchronize()
            pool = torch.cuda.memory_allocated() - m0
            ref, got = per_module()[0], installed()[0]
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
               "glue_ms": {"min": round(min(times["per_module_replays"]) - max(times["replays_only"]), 3),
                           "max": round(max(times["per_module_replays"]) - min(times["replays_only"]), 3)},
               "same_candidates": got["cand_angles"] == ref["cand_angles"]
               and got["cand_distances"] == ref["cand_distances"],
               "step_graph_memory_mb": round(pool / 2 ** 20, 1)}
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
