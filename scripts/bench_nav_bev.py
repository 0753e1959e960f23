"""Agent-side BEV build per navigation step: the eager chain of the reference agents (torch.cat of the gathered node
clouds -> pad_sequence -> ego transform -> PointCloud.project_bev: cell_index_kernel + scatter_mean_f32_kernel) against
PointCloud.splat_nodes (one bb_bev_splat_nodes launch on the node clouds where they lie), alternated in one run.

Nodes are 2352-point panoramas (12 views of 14 x 14) with 768 fp32 features, views into batched PointCloud.forward
outputs as the agents' lift leaves them, distinct per sample.  For each shape: time per call from CUDA events and from
the host clock ending in a synchronise, two windows per variant; bytes per call computed from the shapes; the two
outputs compared bit for bit.  One shape above 21 nodes per sample runs the new path only (the eager chain's scatter
stages a sample's cell indices in shared memory and refuses more than 51,200 points).

    python scripts/bench_nav_bev.py [--calls 50] [--out DIR]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevbert_b200 import synth  # noqa: E402
from bevbert_b200.agent_bev import ego_frames  # noqa: E402
from bevbert_b200.model.bev_utils import PointCloud  # noqa: E402

D, RES, C, NPT = 21, 0.5, 768, 2352


def nodes_for(B, n, seed):
    """B x n distinct node clouds as views into one batched forward output (the agents' lift)"""
    pcl = PointCloud(math.radians(90), 1, 14, 14, D, RES)
    N = B * n
    depth = synth.det_uniform((N * 12, 1, 14, 14), seed, 1, 0.0, 0.6).cuda() * 10
    h = torch.arange(N * 12, dtype=torch.float64) * (math.pi / 6)
    T = torch.zeros(N * 12, 4, 4)
    T[:, 0, 0], T[:, 0, 2], T[:, 1, 1], T[:, 2, 0], T[:, 2, 2], T[:, 3, 3] = (
        h.cos().float(), h.sin().float(), -1.0, -h.sin().float(), h.cos().float(), 1.0)
    T[:, 0, 3] = synth.det_uniform((N * 12,), seed, 2, -3.0, 3.0)
    T[:, 2, 3] = synth.det_uniform((N * 12,), seed, 3, -3.0, 3.0)
    T[:, 1, 3] = 1.25
    pc, nod = pcl.forward(depth, T.cuda())
    pc, nod = pc.reshape(N, -1, 3), nod.reshape(N, -1)
    feat = torch.empty(N, NPT, C, device="cuda").uniform_(-1.7, 1.7, generator=torch.Generator("cuda").manual_seed(seed))
    return [[(pc[b * n + j], nod[b * n + j], feat[b * n + j]) for j in range(n)] for b in range(B)], pcl


def eager(clouds, S, T, pcl):
    pad = torch.nn.utils.rnn.pad_sequence
    pc = pad([torch.cat([x[0] for x in c]) for c in clouds], batch_first=True)
    nod = pad([torch.cat([x[1] for x in c]) for c in clouds], batch_first=True, padding_value=True)
    ft = pad([torch.cat([x[2] for x in c]) for c in clouds], batch_first=True)
    p = pc - S[:, None, :]
    e = []
    for j in range(3):
        acc = p[..., 0] * T[:, None, j, 0]
        acc = acc + p[..., 1] * T[:, None, j, 1]
        acc = acc + p[..., 2] * T[:, None, j, 2]
        acc = acc + T[:, None, j, 3]
        e.append(acc)
    bev, ob = pcl.project_bev(torch.stack(e, -1), nod, ft)
    return bev.reshape(len(clouds), D * D, -1), ob


def window(fn, calls):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls, (time.perf_counter() - t0) * 1e3 / calls


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    card, plim = torch.cuda.get_device_name(), power_limit()
    print("card: %s, power limit: %s" % (card, plim))
    rows = []
    shapes = [(B, n, True) for B in (4, 8, 16) for n in (1, 3, 6)] + [(4, 24, False)]
    for B, n, both in shapes:
        clouds, pcl = nodes_for(B, n, seed=B * 100 + n)
        obs = [{"position": [0.4 * b, -0.7 * b, 1.5], "heading": 0.9 * b - 1.0} for b in range(B)]
        s, t = ego_frames(obs)
        S, T = torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda()
        new = lambda: pcl.splat_nodes(clouds, S, T)          # noqa: E731
        old = lambda: eager(clouds, S, T, pcl)               # noqa: E731
        bn, obn = new()
        same = None
        if both:
            be, obe = old()
            same = bool(torch.equal(bn, be) and torch.equal(obn, obe.reshape(obn.shape)))
        for _ in range(3):
            new()
            if both:
                old()
        res = {"new": [], "eager": []}
        for _ in range(2):
            res["new"].append(window(new, args.calls))
            if both:
                res["eager"].append(window(old, args.calls))
        P = n * NPT
        feat, pts, out = B * P * C * 4, B * P * 13, B * D * D * (C * 4 + 1)
        # eager: cat (read + write) and pad (read + write) of features and points, the transform and cell index passes
        # over the points, the scatter's feature read; new: every feature row and point read once
        row = {"B": B, "nodes": n, "points_per_sample": P, "bit_identical": same,
               "bytes_new": feat + pts + out, "bytes_eager": 5 * feat + 8 * pts + out,
               "new_ms_events": [r[0] for r in res["new"]], "new_ms_host": [r[1] for r in res["new"]],
               "eager_ms_events": [r[0] for r in res["eager"]], "eager_ms_host": [r[1] for r in res["eager"]]}
        rows.append(row)
        fmt = lambda xs: "-".join("%.3f" % x for x in sorted(xs)) if xs else "n/a"     # noqa: E731
        print("B=%2d nodes=%2d  eager %s ms (host %s)  ->  new %s ms (host %s)  bit-identical=%s  GB/s new %.0f" % (
            B, n, fmt(row["eager_ms_events"]), fmt(row["eager_ms_host"]), fmt(row["new_ms_events"]),
            fmt(row["new_ms_host"]), same, row["bytes_new"] / min(row["new_ms_events"]) / 1e6), flush=True)
        del clouds, pcl
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_nav_bev.json"), "w") as f:
            json.dump({"card": card, "power_limit": plim, "calls_per_window": args.calls, "rows": rows}, f, indent=1)
    assert all(r["bit_identical"] is not False for r in rows), "outputs differ"


if __name__ == "__main__":
    main()
