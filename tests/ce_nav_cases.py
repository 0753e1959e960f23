"""Inputs and one teacher-forced rollout for the VLN-CE navigation network (model/ce_nav.py), shared by the golden
generator (tests/golden/make_ce_nav_golden.py, which runs the unmodified CE reference), the CPU tests and the GPU tests.

A network is anything with the CE policy's three methods: the reference class, model/ce_nav.py or the oracle
(oracle/ce_nav_ref.py).  The inputs are shaped like the CE trainer's `_language_variable`, `_panorama_feature_variable`
and `_nav_*_variable` (ss_trainer_BEV.py:340-580): ragged instructions and view counts, 512-d RGB and 128-d depth view
features, 4 angle columns, an 11 x 11 BEV with candidate cells, visited nodes and back-track candidates."""
import torch
import torch.nn.functional as F

from bevbert_b200 import synth
from bevbert_b200.config import make_ce_nav_config

H, D = 768, 11
# (use_depth_embedding, graph_sprels): the four constructor branches the golden covers
VARIANTS = [(True, True), (True, False), (False, True), (False, False)]
WEIGHT_SEED, INPUT_SEED, STEPS = 5, 9, 3


def config(depth=True, sprels=True, **kw):
    return make_ce_nav_config(small=True, use_depth_embedding=depth, graph_sprels=sprels, **kw)


def lang_inputs(B, L=16, seed=INPUT_SEED):
    lens = torch.tensor([L - 5 * (i % 3) for i in range(B)])
    masks = torch.arange(L)[None] < lens[:, None]
    return {"txt_ids": synth.det_randint((B, L), seed, 1, 1000, 1999) * masks, "txt_masks": masks}


def pano_inputs(B, V=14, seed=INPUT_SEED, step=0):
    u = lambda shape, s, lo=-1.0, hi=1.0: synth.det_uniform(shape, seed + 100 * step, s, lo, hi)
    lens = torch.tensor([V - (i + step) % 4 for i in range(B)])
    lens[0] = V                                    # the padded width is max(view_lens), as pad_sequence makes it
    vm = (torch.arange(V)[None] < lens[:, None])
    nav_types = torch.zeros(B, V, dtype=torch.long)
    nav_types[:, :3 + step % 2] = 1                # candidate views first
    return {"rgb_fts": u((B, V, 512), 1, -1.7, 1.7) * vm[..., None], "dep_fts": u((B, V, 128), 2) * vm[..., None],
            "loc_fts": u((B, V, 4), 3) * vm[..., None], "nav_types": nav_types * vm, "view_lens": lens}


def nav_inputs(B, G=9, Kc=4, seed=INPUT_SEED, step=0):
    """everything of forward_navigation but txt_embeds and gmap_img_fts (those come from the other calls)"""
    u = lambda shape, s, lo=-1.0, hi=1.0: synth.det_uniform(shape, seed + 100 * step, s, lo, hi)
    n = D * D
    glens = torch.tensor([max(G - i % 3, 5) for i in range(B)])
    gmask = torch.arange(G)[None] < glens[:, None]
    vpids = [[None] + ["s%dn%d" % (i, j) for j in range(1, int(glens[i]))] for i in range(B)]
    visited = torch.zeros(B, G, dtype=torch.bool)
    visited[:, 1:3] = True
    cand_vpids = [[None] + [vpids[i][1 + (2 * k + step) % (len(vpids[i]) - 1)] for k in range(Kc - 1)]
                  for i in range(B)]
    cand_idx = torch.tensor([[(n - 1) // 2] + [(5 + i + 3 * k + 7 * step) % n for k in range(Kc - 1)]
                             for i in range(B)])
    navm = torch.zeros(B, n, dtype=torch.bool)
    navm[torch.arange(B)[:, None], cand_idx] = True
    pd = u((B, G, G), 6, 0.0, 3.0)
    pd = (pd + pd.transpose(1, 2)) * gmask[:, :, None] * gmask[:, None, :]
    return {"gmap_vpids": vpids, "gmap_step_ids": synth.det_randint((B, G), seed, 8, 0, 5) * gmask,
            "gmap_pos_fts": u((B, G, 7), 9) * gmask[..., None], "gmap_masks": gmask, "gmap_visited_masks": visited,
            "gmap_pair_dists": pd, "bev_fts": u((B, n, H), 10, -1.7, 1.7), "bev_pos_fts": u((B, n, 10), 11),
            "bev_masks": torch.ones(B, n, dtype=torch.bool), "bev_nav_masks": navm, "bev_cand_idxs": cand_idx,
            "bev_cand_vpids": cand_vpids}


NAV_ARGS = ("txt_embeds", "txt_masks", "gmap_vpids", "gmap_step_ids", "gmap_img_fts", "gmap_pos_fts", "gmap_masks",
            "gmap_visited_masks", "gmap_pair_dists", "bev_fts", "bev_pos_fts", "bev_masks", "bev_nav_masks",
            "bev_cand_idxs", "bev_cand_vpids")
PANO_ARGS = ("rgb_fts", "dep_fts", "loc_fts", "nav_types", "view_lens")


def embed_pin(x, k=16):
    """what the golden keeps of an embedding tensor (..., H): its first k channels and its row norms (fp64)"""
    return {"head": x[..., :k].detach().clone(), "norm": x.detach().double().norm(dim=-1)}


def node_embeds(pe, pm, gmask):
    """host-side node memory of one step: [stop] zero, the current node the masked panorama average, the others
    panorama views (differentiable, so the rollout's gradient reaches the panorama encoder)"""
    G = gmask.shape[1]
    avg = (pe * pm[:, :, None]).sum(1) / pm.sum(1, keepdim=True)
    g = torch.cat([pe.new_zeros(pe.shape[0], 1, pe.shape[2]), avg[:, None], pe[:, :G - 2]], 1)
    return g * gmask[:, :, None]


def targets(nav):
    """teacher action per sample: its last map node (unvisited, so its fused logit is finite)"""
    return nav["gmap_masks"].sum(1) - 1


def rollout(net, B, steps=STEPS, prep=lambda x: x, G=9, Kc=4, L=16, V=14):
    """language once, then per step panorama -> node memory -> navigation, the fused-logit cross-entropy summed over
    steps, over B, like the CE trainer's teacher forcing (ss_trainer_BEV.py:1094).  -> (loss, per-step outputs)"""
    P = lambda d: {k: prep(v) for k, v in d.items()}
    lang = P(lang_inputs(B, L))
    txt = net.forward_txt(lang["txt_ids"], lang["txt_masks"])
    loss, outs = 0.0, []
    for t in range(steps):
        pano = P(pano_inputs(B, V, step=t))
        pe, pm = net.forward_panorama(*[pano[k] for k in PANO_ARGS])
        nav = P(nav_inputs(B, G, Kc, step=t))
        nav.update(txt_embeds=txt, txt_masks=lang["txt_masks"], gmap_img_fts=node_embeds(pe, pm, nav["gmap_masks"]))
        out = net.forward_navigation(*[nav[k] for k in NAV_ARGS])
        loss = loss + F.cross_entropy(out["fused_logits"], targets(nav), reduction="sum")
        outs.append({"txt": txt, "pano": (pe, pm), "nav": out})
    return loss / B, outs
