"""Per-call time of the agents' per-step API (GlocalTextPathNavCMT.forward(mode, batch), full-depth model, eval mode,
no_grad) run eagerly against replayed as CUDA graphs (graphs.GraphedNavigation), alternated in one process.

Shapes: B in {4, 8, 16} (fine-tuning validates at 4, scripts/ft_r2r.bash), 21 x 21 BEV, G in {8, 20, 60} map nodes,
8 BEV candidates (stop included), 44-token instructions, 36 views, with and without 20 REVERIE object tokens.  Each
window is >= 200 calls of one mode with the same inputs; it is timed by CUDA events and by a host clock that ends in a
device synchronise.  Eager and graphed windows alternate, --reps times each, and min-max over the windows is printed.
Outputs of the two are compared at every timed shape (finite pattern, fused-logit argmax, relative L2, bit identity).
The GPU name and power limit are read in the same run.

    python scripts/bench_nav.py [--calls 200] [--reps 3] [--json out.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bevbert_b200 import synth  # noqa: E402
from bevbert_b200.config import make_config  # noqa: E402
from bevbert_b200.graphs import GraphedNavigation  # noqa: E402
from bevbert_b200.model.nav_vilmodel import GlocalTextPathNavCMT  # noqa: E402

L, V, KC, D, H, OBJ = 44, 36, 8, 21, 768, 20


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi not available"
    return "%s | power limit, max SM clock: %s" % (torch.cuda.get_device_name(), q)


def inputs(B, G, obj, seed=5):
    u = lambda shape, s, lo=-1.0, hi=1.0: synth.det_uniform(shape, seed, s, lo, hi).cuda()
    txt_lens = torch.tensor([L - 9 * (i % 3) for i in range(B)])
    txt_masks = (torch.arange(L)[None] < txt_lens[:, None]).cuda()
    lang = {"txt_ids": synth.det_randint((B, L), seed, 1, 1000, 1999).cuda() * txt_masks, "txt_masks": txt_masks}
    obj_lens = torch.tensor([OBJ - 4 * (i % 3) for i in range(B)]).cuda() if obj else None
    Vt = V + (OBJ if obj else 0)
    pano = {"view_img_fts": u((B, V, H), 2), "obj_img_fts": u((B, OBJ, H), 3) if obj else None,
            "loc_fts": u((B, Vt, 7), 4), "nav_types": synth.det_randint((B, Vt), seed, 5, 0, 1).cuda(),
            "view_lens": torch.full((B,), V).cuda(), "obj_lens": obj_lens}
    gl = torch.tensor([max(G - 2 * (i % 3), 2) for i in range(B)])
    gmask = torch.arange(G)[None] < gl[:, None]
    vpids = [[None] + ["s%dn%d" % (i, j) for j in range(1, int(gl[i]))] for i in range(B)]
    visited = torch.zeros(B, G, dtype=torch.bool)
    visited[:, 1:max(G // 2, 2)] = True
    cands = [[None] + [vpids[i][1 + (3 * k) % (len(vpids[i]) - 1)] for k in range(KC - 1)] for i in range(B)]
    n = D * D
    cidx = torch.tensor([[(n - 1) // 2] + [(7 + i + 11 * k) % n for k in range(KC - 1)] for i in range(B)])
    navm = torch.zeros(B, n, dtype=torch.bool)
    navm[torch.arange(B)[:, None], cidx] = True
    pd = synth.det_uniform((B, G, G), seed, 6, 0.0, 3.0)
    pd = (pd + pd.transpose(1, 2)) * gmask[:, :, None] * gmask[:, None, :]
    nav = {"txt_masks": txt_masks, "gmap_img_embeds": u((B, G, H), 7) * gmask[:, :, None].cuda(),
           "gmap_step_ids": (synth.det_randint((B, G), seed, 8, 0, 15) * gmask).cuda(), "gmap_pos_fts": u((B, G, 7), 9),
           "gmap_masks": gmask.cuda(), "gmap_pair_dists": pd.cuda(), "gmap_visited_masks": visited.cuda(),
           "gmap_vpids": vpids, "bev_fts": u((B, n, H), 10), "bev_pos_fts": u((B, n, 10), 11),
           "bev_masks": torch.ones(B, n, dtype=torch.bool).cuda(), "bev_nav_masks": navm.cuda(),
           "bev_cand_idxs": cidx.cuda(), "bev_cand_vpids": cands, "obj_embeds": None, "obj_masks": None}
    return lang, pano, nav


def window(fn, calls):
    """(device ms per call from events, host ms per call ending in a synchronise) over `calls` calls"""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls, (time.perf_counter() - t0) * 1e3 / calls


def compare(a, b):
    """(finite patterns equal, fused argmax equal, max relative L2 over outputs, bit-identical)"""
    if torch.is_tensor(a):
        a, b = {"out": a}, {"out": b}
    elif isinstance(a, tuple):
        a, b = dict(enumerate(a)), dict(enumerate(b))
    fin, rel, same = True, 0.0, True
    for k in a:
        if a[k] is None:
            continue
        x, y = a[k].float(), b[k].float()
        f = torch.isfinite(y)
        fin = fin and torch.equal(torch.isfinite(x), f)
        if f.any():
            rel = max(rel, float((x[f] - y[f]).norm() / (y[f].norm() + 1e-30)))
        same = same and torch.equal(a[k], b[k])
    am = torch.equal(a["fused_logits"].argmax(1), b["fused_logits"].argmax(1)) if "fused_logits" in a else None
    return fin, am, rel, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_nav needs a GPU"
    print("before: " + card())
    rows = []
    for obj in (0, 1):
        cfg = make_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, feat_dropout=0.0,
                          **(dict(obj_feat_size=768) if obj else {}))
        model = synth.det_init_(GlocalTextPathNavCMT(cfg), seed=4).cuda().eval()
        nav = GraphedNavigation(model)
        for B in (4, 8, 16):
            for G in (8, 20, 60):
                lang, pano, navb = inputs(B, G, obj)
                with torch.no_grad():
                    t = model("language", lang)
                    pe, pm = model("panorama", pano)
                    navb["txt_embeds"] = t
                    if obj:
                        navb["obj_embeds"], navb["obj_masks"] = pe[:, V:V + OBJ], pm[:, V:V + OBJ]
                    # language / panorama do not depend on G: timed once per B
                    modes = (("language", lang), ("panorama", pano), ("navigation", navb)) if G == 8 else \
                        (("navigation", navb),)
                    for mode, b in modes:
                        eager, graphed = (lambda: model(mode, b)), (lambda: nav(mode, b))
                        check = compare(graphed(), eager())
                        assert check[0] and check[1] in (None, True) and check[2] < 1e-2, (mode, B, G, obj, check)
                        for _ in range(3):
                            eager(), graphed()
                        res = {"eager": [], "graphed": []}
                        for _ in range(args.reps):
                            res["eager"].append(window(eager, args.calls))
                            res["graphed"].append(window(graphed, args.calls))
                        row = {"mode": mode, "B": B, "G": G if mode == "navigation" else None, "objects": bool(obj),
                               "launches_per_replay": nav.launches(mode, b), "bit_identical": check[3],
                               "rel_l2": check[2]}
                        for k, v in res.items():
                            row[k + "_device_ms"] = [round(min(x[0] for x in v), 4), round(max(x[0] for x in v), 4)]
                            row[k + "_host_ms"] = [round(min(x[1] for x in v), 4), round(max(x[1] for x in v), 4)]
                        rows.append(row)
                        print("%-10s B=%2d G=%-4s obj=%d | eager: events %.3f-%.3f ms, host %.3f-%.3f ms | graphed: events "
                              "%.3f-%.3f ms, host %.3f-%.3f ms | launches/replay %s, bit-identical %s, rel_l2 %.1e" % (
                                  mode, B, row["G"], obj, *row["eager_device_ms"], *row["eager_host_ms"],
                                  *row["graphed_device_ms"], *row["graphed_host_ms"], row["launches_per_replay"],
                                  check[3], check[2]), flush=True)
        del nav, model
        torch.cuda.empty_cache()
    print("after: " + card())
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(json.dumps({"card": card()}) + "\n")
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
