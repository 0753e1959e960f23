"""Times the VLN-CE policy's CLIP ViT-B/16 RGB encoder per navigation step: the reference-shaped fp16 eager path
(oracle/ce_clip_ref.Fp16Tower: clip.load's dtypes, seq-first nn.MultiheadAttention, QuickGELU as written) against
the kernels (model/clip_visual.py), eager and replayed as a CUDA graph (graphs.install_ce_rgb_encoder), at B = 1, 2,
4, 8 environments of 12 views (12 to 96 images, uint8 224 x 224 observations, seeded weights).

    python scripts/bench_ce_clip.py [--sizes 1,2,4,8] [--iters 20] [--windows 5] [--out FILE]
    python scripts/bench_ce_clip.py --profile [--sizes 8]        # torch.profiler split, a run of its own

ms per call from CUDA events over `iters` back-to-back calls; the three paths are timed in alternating windows and
the min-max over windows is reported.  TFLOP/s counts 35.1 GFLOP per image (computed below from the shapes).  The
outputs of every timed size are compared (rel. L2 against the fp16 reference).  The card name and power limit are
read in the same run.  Prints one JSON line per size, and the profile table with --profile."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevbert_b200 import graphs, synth  # noqa: E402
from bevbert_b200.model import clip_visual as CV  # noqa: E402
from oracle import ce_clip_ref as R  # noqa: E402


def gflop_per_image(res=224, P=16, D=768, L=12, out=512):
    T, G = (res // P) ** 2 + 1, (res // P) ** 2
    block = 2 * T * D * 3 * D + 2 * T * D * D + 2 * 2 * T * D * 4 * D + 2 * 2 * T * T * D
    return (L * block + 2 * G * 3 * P * P * D + 2 * D * out) / 1e9


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
    except Exception:
        name, pl = torch.cuda.get_device_name(0), "unknown"
    return name, pl


class _Normalize(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.mean, self.std = list(R.MEAN), list(R.STD)


def encoder(state):
    enc = torch.nn.Module()
    enc.model = torch.nn.Module()
    enc.model.visual = CV.VisionTransformer(**synth.CLIP_B16)
    enc.model.visual.load_state_dict(state)
    for name, p in enc.model.visual.named_parameters():
        if name.endswith(R.FP16_KEYS):
            p.data = p.data.half()
    enc.rgb_transform = torch.nn.Sequential(torch.nn.Identity(), _Normalize())
    enc.requires_grad_(False)
    return enc.cuda().eval()


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,2,4,8")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ce_clip.py measures on the GPU"
    name, pl = card()
    state = synth.clip_visual_state(11)
    ref = R.Fp16Tower(state).cuda()
    enc = encoder(state)
    graphs.install_ce_rgb_encoder(enc)
    gf = gflop_per_image()

    def path_ref(rgb):
        return R.forward_fp16(ref, rgb)

    def path_eager(rgb):
        enc.train()
        try:
            with torch.no_grad():
                return enc({"rgb": rgb})
        finally:
            enc.eval()

    def path_replay(rgb):
        with torch.no_grad():
            return enc({"rgb": rgb})

    paths = {"fp16_reference": path_ref, "eager": path_eager, "replay": path_replay}
    rows = []
    for B in [int(s) for s in a.sizes.split(",")]:
        N = 12 * B
        rgb = synth.clip_images(N, 100 + B).cuda()
        outs = {k: f(rgb) for k, f in paths.items()}
        for _ in range(2):
            for f in paths.values():
                f(rgb)
        torch.cuda.synchronize()
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            table = {}
            for k, f in paths.items():
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(3):
                        f(rgb)
                    torch.cuda.synchronize()
                split = {"gemm": 0.0, "attention": 0.0, "row/other": 0.0}
                for e in prof.key_averages():
                    t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                    if t <= 0 or e.key.startswith(("ProfilerStep", "cuda", "Memcpy", "Memset")):
                        continue
                    n = e.key.lower()
                    if "flash" in n or "attn" in n or "attention" in n or "fmha" in n or "softmax" in n:
                        split["attention"] += t
                    elif any(s in n for s in ("gemm", "xmma", "cutlass", "sm90", "cublas", "nvjet")):
                        split["gemm"] += t
                    else:
                        split["row/other"] += t
                table[k] = {s: round(v / 3e3, 3) for s, v in split.items()}     # ms per call
            print(json.dumps({"B": B, "images": N, "profile_ms_per_call": table, "gpu": name, "power_limit": pl}))
            continue
        times = {k: [] for k in paths}
        for w in range(a.windows):
            for k, f in (paths.items() if w % 2 == 0 else reversed(list(paths.items()))):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(a.iters):
                    f(rgb)
                e.record()
                e.synchronize()
                times[k].append(s.elapsed_time(e) / a.iters)
        row = {"B": B, "images": N, "gpu": name, "power_limit": pl, "gflop_per_image": round(gf, 2)}
        for k, ts in times.items():
            row[k] = {"ms_min": round(min(ts), 3), "ms_max": round(max(ts), 3),
                      "tflops_at_min": round(gf * N / min(ts), 1)}
        row["rel_l2_vs_fp16_reference"] = {k: [round(rel(o, r), 5) for o, r in zip(outs[k], outs["fp16_reference"])]
                                           for k in ("eager", "replay")}
        row["replay_equals_eager"] = all(torch.equal(x, y) for x, y in zip(outs["eager"], outs["replay"]))
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
