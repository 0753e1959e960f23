"""Per-call time of the VLN-CE policy's calls on the CE navigation network (model/ce_nav.py, full depth: 9 language, 2
panorama, 4 cross-modal layers; depth embedding and graph sprels on; eval mode, no_grad) run eagerly against replayed
as CUDA graphs (graphs.install_ce_replay), and of the trainer-side BEV build, eager chain against
agent_bev.ce_nav_bev_variable; alternated in one process.

Shapes: B in {1, 4, 8}; 200-token instructions (VLN-CE pads every instruction to 200); 12 views; an 11 x 11 BEV; G in
{10, 40} map nodes; 6 BEV candidates.  Each window is >= --calls calls of one shape with the same inputs, timed by CUDA
events and by a host clock that ends in a device synchronise; eager and graphed windows alternate --reps times each and
min-max over the windows is printed.  Replayed outputs are compared with eager ones at every timed shape.  The BEV
eager chain is the trainer's: torch.cat of the gathered clouds, pad_sequence, the ego transform and a scatter-mean per
sample (index_add_), on the device.  The GPU name and power limit are read in the same run.

    python scripts/bench_ce_nav.py [--calls 100] [--reps 3] [--json out.jsonl]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
import torch  # noqa: E402
from torch.nn.utils.rnn import pad_sequence  # noqa: E402

import ce_nav_bev_cases as BC  # noqa: E402
import ce_nav_cases as C  # noqa: E402
from bench_nav import card, compare, window  # noqa: E402
from bevbert_b200 import synth  # noqa: E402
from bevbert_b200.agent_bev import ce_nav_bev_variable  # noqa: E402
from bevbert_b200.config import make_ce_nav_config  # noqa: E402
from bevbert_b200.graphs import install_ce_replay  # noqa: E402
from bevbert_b200.model.ce_nav import GlocalTextPathNavCMT  # noqa: E402

L, V, KC = 200, 12, 6


def _cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in d.items()}


def eager_bev(tr, cur_vp, cur_pos, cur_ori):
    """the trainer's chain on the device (ss_trainer_BEV.py:477-532 + splat + project_bev), features only"""
    import numpy as np
    D = tr.bev_dim
    pcs, nods, fts = [], [], []
    for gm, vp in zip(tr.gmaps, cur_vp):
        nodes = [gm.node_pc[c] for c in gm.node_pc if len(gm.shortest_path[vp][c]) <= 1]
        pcs.append(torch.cat([n[0] for n in nodes]))
        nods.append(torch.cat([n[1] for n in nodes]))
        fts.append(torch.cat([n[2] for n in nodes]))
    pc = pad_sequence(pcs, batch_first=True)
    nod = pad_sequence(nods, batch_first=True, padding_value=True)
    ft = pad_sequence(fts, batch_first=True)
    S = torch.from_numpy(np.array(cur_pos, dtype=np.float32)).cuda()
    h = -np.array([BC.heading_from_quaternion(o) for o in cur_ori])
    c, s = np.cos(h), np.sin(h)
    T = np.zeros((len(h), 4, 4))
    T[:, 0, 0], T[:, 0, 2], T[:, 1, 1], T[:, 2, 0], T[:, 2, 2], T[:, 3, 3] = c, s, 1, -s, c, 1
    T = torch.from_numpy(T.astype(np.float32)).cuda()
    p = pc - S[:, None]
    ego = torch.cat([p, torch.ones_like(p[..., :1])], -1) @ T.transpose(1, 2)
    g = (ego[..., [0, 2]] / tr.bev_res + (D - 1) / 2).round()
    bad = nod | (g >= D).any(-1) | (g < 0).any(-1) | (ego[..., 1] > 0.5)
    idx = (D * g[..., 1] + g[..., 0]).long()
    out = []
    for b in range(len(pcs)):
        k = ~bad[b]
        acc = torch.zeros(D * D, ft.shape[-1], device="cuda").index_add_(0, idx[b][k], ft[b][k])
        cnt = torch.zeros(D * D, device="cuda").index_add_(0, idx[b][k], torch.ones(int(k.sum()), device="cuda"))
        out.append(acc / cnt.clamp(min=1)[:, None])
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ce_nav needs a GPU"
    print("before: " + card())
    rows = []
    cfg = make_ce_nav_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, feat_dropout=0.0)
    model = synth.det_init_(GlocalTextPathNavCMT(cfg), seed=4).cuda().eval()
    eager_net = GlocalTextPathNavCMT
    replay = install_ce_replay(model)
    calls = {"language": lambda b: model.forward_txt(b["txt_ids"], b["txt_masks"]),
             "panorama": lambda b: model.forward_panorama(*[b[k] for k in C.PANO_ARGS]),
             "navigation": lambda b: model.forward_navigation(*[b[k] for k in C.NAV_ARGS])}
    eager = {"language": lambda b: eager_net.forward_txt(model, b["txt_ids"], b["txt_masks"]),
             "panorama": lambda b: eager_net.forward_panorama(model, *[b[k] for k in C.PANO_ARGS]),
             "navigation": lambda b: eager_net.forward_navigation(model, *[b[k] for k in C.NAV_ARGS])}
    for B in (1, 4, 8):
        for G in (10, 40):
            lang = _cuda(C.lang_inputs(B, L))
            pano = _cuda(C.pano_inputs(B, V))
            nav = _cuda(C.nav_inputs(B, G, KC))
            with torch.no_grad():
                t = eager["language"](lang)
                pe, pm = eager["panorama"](pano)
                nav.update(txt_embeds=t, txt_masks=lang["txt_masks"],
                           gmap_img_fts=torch.cat([pe, pe, pe, pe], 1)[:, :G] * nav["gmap_masks"][..., None])
                modes = (("language", lang), ("panorama", pano), ("navigation", nav)) if G == 10 else \
                    (("navigation", nav),)
                for mode, b in modes:
                    e, g = (lambda: eager[mode](b)), (lambda: calls[mode](b))
                    check = compare(g(), e())
                    assert check[0] and check[1] in (None, True) and check[2] < 1e-2, (mode, B, G, check)
                    for _ in range(3):
                        e(), g()
                    res = {"eager": [], "graphed": []}
                    for _ in range(args.reps):
                        res["eager"].append(window(e, args.calls))
                        res["graphed"].append(window(g, args.calls))
                    row = {"mode": mode, "B": B, "G": G if mode == "navigation" else None,
                           "launches_per_replay": replay.launches(mode, b), "bit_identical": check[3],
                           "rel_l2": check[2]}
                    for k, v in res.items():
                        row[k + "_device_ms"] = [round(min(x[0] for x in v), 4), round(max(x[0] for x in v), 4)]
                        row[k + "_host_ms"] = [round(min(x[1] for x in v), 4), round(max(x[1] for x in v), 4)]
                    rows.append(row)
                    print("%-10s B=%d G=%-4s | eager: events %.3f-%.3f ms, host %.3f-%.3f ms | graphed: events "
                          "%.3f-%.3f ms, host %.3f-%.3f ms | launches/replay %s, bit-identical %s, rel_l2 %.1e" % (
                              mode, B, row["G"], *row["eager_device_ms"], *row["eager_host_ms"],
                              *row["graphed_device_ms"], *row["graphed_host_ms"], row["launches_per_replay"],
                              check[3], check[2]), flush=True)
    # BEV: one node cloud of 12 views x 14 x 14 points per sample (the CE trainer's lift at order 1)
    for B in (1, 4, 8):
        for tr, vp, pos, ori in BC.episode(B=B, steps=3, device="cuda", n=12 * 14 * 14):
            pass
        ref = ce_nav_bev_variable(tr, vp, pos, ori)["bev_fts"]
        rel = float((eager_bev(tr, vp, pos, ori) - ref).norm() / ref.norm())
        assert rel < 1e-5, rel
        e, g = (lambda: eager_bev(tr, vp, pos, ori)), (lambda: ce_nav_bev_variable(tr, vp, pos, ori))
        for _ in range(3):
            e(), g()
        res = {"eager": [], "kernel": []}
        for _ in range(args.reps):
            res["eager"].append(window(e, args.calls))
            res["kernel"].append(window(g, args.calls))
        row = {"mode": "bev", "B": B, "rel_l2": rel}
        for k, v in res.items():
            row[k + "_device_ms"] = [round(min(x[0] for x in v), 4), round(max(x[0] for x in v), 4)]
            row[k + "_host_ms"] = [round(min(x[1] for x in v), 4), round(max(x[1] for x in v), 4)]
        rows.append(row)
        print("bev        B=%d | eager chain: events %.3f-%.3f ms, host %.3f-%.3f ms | ce_nav_bev_variable: events "
              "%.3f-%.3f ms, host %.3f-%.3f ms | rel_l2 %.1e" % (B, *row["eager_device_ms"], *row["eager_host_ms"],
                                                                 *row["kernel_device_ms"], *row["kernel_host_ms"], rel),
              flush=True)
    print("after: " + card())
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(json.dumps({"card": card()}) + "\n")
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
