"""Times the VLN-CE policy's waypoint step per navigation step (Policy_ViewSelection_BEV.py:194-224 without the depth
and RGB encoders): the waypoint predictor, the softmax over each environment's 1440 cells, the wrap of one row at each
end and the heatmap NMS (max_predictions=5, sigma=(7, 5)), at B = 1, 4, 8 environments of 12 views.

Paths, on seeded weights (synth.waypoint_state) and seeded depth features:
  * fp32_reference / fp16_reference: the reference predictor's operations (oracle/ce_waypoint_ref.py) in fp32 eval
    mode, and under torch.autocast(float16) as the trainer calls it, then softmax, wrap and the reference nms's own
    torch operations on the device (ce_waypoint_ref.nms_device);
  * replay: the predictor routed through graphs.install_ce_waypoint_predictor (one CUDA graph per B), the same softmax
    and wrap, and bevbert_b200.model.waypoint.nms (bb_waypoint_nms).

    python scripts/bench_ce_waypoint.py [--sizes 1,4,8] [--iters 50] [--windows 6] [--out FILE]

ms per step from CUDA events over `iters` back-to-back steps; the paths are timed in alternating windows and the
min-max over windows is reported, with the predictor alone (no NMS) timed the same way.  Per size it also reports
whether the NMS maps of the replay path pick the same cells as those of the fp32 reference.  The card name and power
limit are read in the same run.  Prints one JSON line per size."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevbert_b200 import graphs, synth  # noqa: E402
from bevbert_b200.model import waypoint as WP  # noqa: E402
from oracle import ce_waypoint_ref as R  # noqa: E402

K_PRED, SIGMA = 5, (7.0, 5.0)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
    except Exception:
        name, pl = torch.cuda.get_device_name(0), "unknown"
    return name, pl


def heatmap(logits):
    """Policy_ViewSelection_BEV.py:212-220"""
    B = logits.shape[0]
    x = torch.softmax(logits.reshape(B, -1), dim=1).reshape(B, 120, 12)
    return torch.cat((x[:, -1:], x, x[:, :1]), dim=1).unsqueeze(1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,4,8")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--windows", type=int, default=6)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ce_waypoint.py measures on the GPU"
    name, pl = card()
    state = synth.waypoint_state(21)
    sd = {k: v.cuda() for k, v in state.items()}
    wp = WP.BinaryDistPredictor_TRM()
    wp.load_state_dict(state)
    wp = wp.cuda().requires_grad_(False).eval()
    graphs.install_ce_waypoint_predictor(wp)

    def ref32(rgb, dep):
        with torch.no_grad():
            return R._forward(sd, dep, torch.float32)

    def ref16(rgb, dep):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            return R._forward(sd, dep, torch.float32)

    def replay(rgb, dep):
        with torch.no_grad():
            return wp(rgb, dep)

    predictors = {"fp32_reference": ref32, "fp16_reference": ref16, "replay": replay}
    def step(predict, nms):
        return lambda rgb, dep: nms(heatmap(predict(rgb, dep).float()), K_PRED, SIGMA)

    steps = {k: step(f, WP.nms if k == "replay" else R.nms_device) for k, f in predictors.items()}
    rows = []
    for B in [int(s) for s in a.sizes.split(",")]:
        N = 12 * B
        dep = synth.det_uniform((N, 128, 4, 4), 100 + B, 5, 0.0, 1.0).cuda()
        rgb = torch.zeros(N, 512, device="cuda")
        maps = {k: f(rgb, dep) for k, f in steps.items()}
        for _ in range(3):
            for f in list(steps.values()) + list(predictors.values()):
                f(rgb, dep)
        torch.cuda.synchronize()
        row = {"B": B, "views": N, "gpu": name, "power_limit": pl}
        for label, table in (("step", steps), ("predictor_only", predictors)):
            times = {k: [] for k in table}
            for w in range(a.windows):
                for k, f in (table.items() if w % 2 == 0 else reversed(list(table.items()))):
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    for _ in range(a.iters):
                        f(rgb, dep)
                    e.record()
                    e.synchronize()
                    times[k].append(s.elapsed_time(e) / a.iters)
            row[label] = {k: {"ms_min": round(min(ts), 4), "ms_max": round(max(ts), 4)} for k, ts in times.items()}
        picked = {k: (m != 0).reshape(B, -1) for k, m in maps.items()}
        row["same_picks_as_fp32_reference"] = {k: int((picked[k] == picked["fp32_reference"]).all(dim=1).sum())
                                               for k in ("fp16_reference", "replay")}
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
