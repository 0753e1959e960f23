"""Times the VLN-CE policy's depth encoder at B = 1, 4, 8 environments (12 B depth images of 256 x 256): the restated
module (model/depth_resnet.py ResNetEncoder, the reference's PyTorch path) in fp32 eval and under fp16 autocast, against
the kernels (DepthTower), eager and graph-replayed (graphs.install_ce_depth_encoder).  CUDA events over back-to-back
calls in alternated windows, min-max over windows; the card name and power limit are read in the same run.  Every
timed size checks the outputs against the fp32 reference.  --profile instead reports, from torch.profiler, the split
of the kernels' time between convolution, GroupNorm and stem.

    python scripts/bench_ce_depth.py [--calls 20 --windows 5] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevbert_b200 import graphs, synth  # noqa: E402
from bevbert_b200.model import depth_resnet as D  # noqa: E402

GFLOP_PER_IMAGE = 0.699


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # noqa: BLE001
        return "%s (power limit unreadable: %s)" % (torch.cuda.get_device_name(), type(e).__name__)


class Wrapper(torch.nn.Module):
    def __init__(self, enc):
        super().__init__()
        self.visual_encoder = enc


def time_windows(fns, calls, windows):
    """{name: [ms per call, one per window]}, windows of the callables alternated"""
    res = {k: [] for k in fns}
    for _ in range(windows):
        for k, f in fns.items():
            f()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(calls):
                f()
            b.record()
            b.synchronize()
            res[k].append(a.elapsed_time(b) / calls)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    state = synth.depth_encoder_state(1)
    ref_mod = D.depth_encoder().cuda().eval().requires_grad_(False)
    ref_mod.load_state_dict(state)
    tower = D.DepthTower(ref_mod)
    kmod = D.depth_encoder().cuda().eval().requires_grad_(False)
    kmod.load_state_dict(state)
    wrap = Wrapper(kmod).eval()
    graphs.install_ce_depth_encoder(wrap)
    print("card: %s | cudnn.allow_tf32=%s" % (card(), torch.backends.cudnn.allow_tf32))
    if args.profile:
        depth = synth.depth_images(96, 2).cuda()
        tower.encode(depth)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                tower.encode(depth)
            torch.cuda.synchronize()
        split = {"conv": 0.0, "groupnorm": 0.0, "stem": 0.0, "other": 0.0}
        for ev in prof.key_averages():
            t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            name = ev.key
            kind = ("conv" if "conv_" in name else "groupnorm" if "gn_apply" in name else
                    "stem" if "depth_stem" in name else "other")
            split[kind] += t / 5 / 1000.0
        print(json.dumps({"profile_B8_ms_per_call": {k: round(v, 3) for k, v in split.items()}}))
        return
    rows = []
    with torch.no_grad():
        for B in (1, 4, 8):
            n = 12 * B
            depth = synth.depth_images(n, 10 + B).cuda()
            obs = {"depth": depth}
            ref = ref_mod(obs)

            def ref32():
                return ref_mod(obs)

            def ref16():
                with torch.autocast("cuda", dtype=torch.float16):
                    return ref_mod(obs)
            fns = {"ref_fp32": ref32, "ref_fp16_autocast": ref16, "kernels_eager": lambda: tower.encode(depth),
                   "kernels_replayed": lambda: kmod(obs)}
            errs = {k: float((f().float() - ref).norm() / ref.norm()) for k, f in fns.items()}
            t = time_windows(fns, args.calls, args.windows)
            row = {"B": B, "images": n}
            for k, v in t.items():
                row[k] = {"ms_min": round(min(v), 3), "ms_max": round(max(v), 3),
                          "tflops_best": round(GFLOP_PER_IMAGE * n / min(v), 2), "rel_err_vs_fp32": errs[k]}
            rows.append(row)
            print(json.dumps(row))
            assert errs["kernels_eager"] < 2e-2 and errs["kernels_replayed"] < 2e-2, errs


if __name__ == "__main__":
    main()
