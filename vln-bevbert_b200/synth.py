"""Synthetic R2R / REVERIE pre-training batches in the reference's collate layout.

The reference's data pipeline (pretrain_src/data/dataset.py, tasks.py) needs Matterport features, HDF5
stores and the MatterSim simulator, none of which exist offline; batches are therefore synthetic but laid
out exactly as `mlm_collate` / `sap_collate` / ... produce them (pretrain_src/data/tasks.py:118-160,
362-411; SURVEY.md 8a-0).  All random values come from a counter-based integer hash evaluated with exact
int64 torch ops, so a (seed, config) pair yields bit-identical batches on every machine and torch
version -- golden fixtures only need to store outputs.
"""
from dataclasses import dataclass, field
import math
from typing import List, Optional

import torch

_MASK64 = (1 << 64) - 1


def _to_signed(v: int) -> int:
    v &= _MASK64
    return v - (1 << 64) if v >= (1 << 63) else v


_C1 = _to_signed(0x9E3779B97F4A7C15)
_C2 = _to_signed(0xBF58476D1CE4E5B9)
_C3 = _to_signed(0x94D049BB133111EB)


def _lsr(z: torch.Tensor, s: int) -> torch.Tensor:
    """logical shift right on int64 (torch's >> is arithmetic)."""
    return (z >> s) & ((1 << (64 - s)) - 1)


def det_bits(n: int, seed: int, stream: int = 0) -> torch.Tensor:
    """n pseudo-random 24-bit integers (int64 tensor); splitmix64 finaliser over (seed, stream, index)."""
    idx = torch.arange(n, dtype=torch.int64)
    z = idx * _C1 + _to_signed((seed * 0x632BE59BD9B4E019 + stream * 0xD1342543DE82EF95 + 0x1234567) & _MASK64)
    z = (z ^ _lsr(z, 30)) * _C2
    z = (z ^ _lsr(z, 27)) * _C3
    z = z ^ _lsr(z, 31)
    return _lsr(z, 40)


def det_uniform(shape, seed: int, stream: int = 0, lo: float = 0.0, hi: float = 1.0) -> torch.Tensor:
    """float32 uniform in [lo, hi), exactly reproducible."""
    n = 1
    for s in shape:
        n *= int(s)
    u = det_bits(n, seed, stream).to(torch.float32) / float(1 << 24)
    return (u * (hi - lo) + lo).reshape(*shape)


def det_randint(shape, seed: int, stream: int, lo: int, hi: int) -> torch.Tensor:
    """int64 uniform integers in [lo, hi] inclusive."""
    n = 1
    for s in shape:
        n *= int(s)
    return (det_bits(n, seed, stream) % (hi - lo + 1) + lo).reshape(*shape)


def pose_matrices(xyzhe: torch.Tensor) -> torch.Tensor:
    """(N,5) x,y,z,heading,elevation -> (N,4,4) float32 rigid transforms.

    Same convention as `transfrom3D` in pretrain_src/model/bev_utils.py:7-36 (rotation about y by heading
    composed with rotation about x by elevation, translation in the last column); evaluated in float64
    and rounded to float32 like the numpy reference.
    """
    p = xyzhe.to(torch.float64)
    ce, se = torch.cos(p[:, 4]), torch.sin(p[:, 4])
    ch, sh = torch.cos(p[:, 3]), torch.sin(p[:, 3])
    T = torch.zeros(p.shape[0], 4, 4, dtype=torch.float64)
    T[:, 0, 0], T[:, 0, 1], T[:, 0, 2], T[:, 0, 3] = ch, se * sh, ce * sh, p[:, 0]
    T[:, 1, 1], T[:, 1, 2], T[:, 1, 3] = ce, -se, p[:, 1]
    T[:, 2, 0], T[:, 2, 1], T[:, 2, 2], T[:, 2, 3] = -sh, ch * se, ch * ce, p[:, 2]
    T[:, 3, 3] = 1.0
    return T.to(torch.float32)


@dataclass
class SynthConfig:
    """Shape of a synthetic batch. Defaults = BASELINE.json config 2 (R2R, 21x21 BEV)."""
    batch_size: int = 32
    txt_len: int = 80
    vocab_lo: int = 1000
    vocab_hi: int = 2000
    bev_dim: int = 21
    bev_res: float = 0.5
    image_feat_size: int = 768
    n_views: int = 36
    pano_min: int = 3
    pano_max: int = 8
    gmap_min: int = 8
    gmap_max: int = 20
    cand_min: int = 2     # candidate views at the last viewpoint (local action space, excluding [stop])
    cand_max: int = 6
    n_mask_tokens: int = 12
    obj_feat_size: int = 0      # >0: REVERIE-style object tokens
    obj_max: int = 0
    obj_prob_size: int = 1000
    depth_zero_frac: float = 0.05
    ragged_txt: bool = False     # variable instruction lengths (txt_lens < txt_len)
    depth_feat_size: int = 0     # >0: VLN-CE batch (traj_view_dep_fts, 4 location columns, no semantic labels)


def make_batch(cfg: SynthConfig, seed: int = 1234, task: str = "sap") -> dict:
    """One collated batch (CPU tensors + host lists) for `task` in {mlm, sap, masksem, sem, mrc, og}.  With
    cfg.depth_feat_size > 0 it is laid out as the VLN-CE collate gives it (bevbert_ce/pretrain/pretrain_src/data): depth
    features per view, location features of 4 angle columns and no `sems`; everything else is drawn as for R2R."""
    B, L, D = cfg.batch_size, cfg.txt_len, cfg.bev_dim
    ncell = D * D
    s = [0]

    def stream():
        s[0] += 1
        return s[0]

    batch = {}
    # ---------------------------------------------------------------- text
    if cfg.ragged_txt:
        txt_lens = det_randint((B,), seed, stream(), max(4, L // 2), L)
        txt_lens[0] = L
    else:
        txt_lens = torch.full((B,), L, dtype=torch.int64)
        stream()
    txt_ids = det_randint((B, L), seed, stream(), cfg.vocab_lo, cfg.vocab_hi - 1)
    txt_ids[:, 0] = 101
    ar = torch.arange(L)[None, :]
    txt_ids = torch.where(ar < txt_lens[:, None], txt_ids, torch.zeros_like(txt_ids))
    batch["txt_ids"] = txt_ids
    batch["txt_lens"] = txt_lens
    if task.startswith("mlm"):
        labels = torch.full((B, L), -1, dtype=torch.int64)
        for i in range(B):
            n = int(txt_lens[i])
            step = max(1, n // max(1, cfg.n_mask_tokens))
            pos = list(range(1, n, step))[: cfg.n_mask_tokens]
            for p_ in pos:
                labels[i, p_] = txt_ids[i, p_]
                txt_ids[i, p_] = 103
        batch["txt_labels"] = labels

    # ---------------------------------------------------------------- trajectory / topological map (host graph)
    n_pano = det_randint((B,), seed, stream(), cfg.pano_min, cfg.pano_max).tolist()
    gmap_target = det_randint((B,), seed, stream(), cfg.gmap_min, cfg.gmap_max).tolist()
    last_cands = det_randint((B,), seed, stream(), cfg.cand_min, cfg.cand_max).tolist()
    traj_step_lens: List[int] = []
    traj_vpids, traj_cand_vpids, gmap_vpids = [], [], []
    gmap_lens, gmap_step_ids, gmap_visited = [], [], []
    vp_view_lens, vp_obj_lens, nav_types_rows = [], [], []
    V = cfg.n_views
    O = cfg.obj_max if cfg.obj_feat_size > 0 else 0
    obj_counts_all = det_randint((sum(n_pano),), seed, stream(), 0, max(O, 0)).tolist() if O > 0 else None
    k_pano = 0
    for i in range(B):
        P = n_pano[i]
        path = [f"s{i}v{t}" for t in range(P)]
        n_unvisited = max(1, gmap_target[i] - 1 - P)
        # spread the unvisited nodes over the panoramas; the last panorama gets `last_cands[i]` candidates
        per_step = [[] for _ in range(P)]
        u = 0
        for t in range(P):
            if t + 1 < P:
                per_step[t].append(path[t + 1])          # next node on the path
            if t > 0:
                per_step[t].append(path[t - 1])          # way back
        t = 0
        while u < n_unvisited:
            per_step[t % P].append(f"s{i}u{u}")
            u += 1
            t += 1
        # last step: trim / extend to the requested number of candidates (keep >=1 unvisited)
        want = max(2, last_cands[i])
        extra = 0
        while len(per_step[-1]) < want:
            per_step[-1].append(f"s{i}u{n_unvisited + extra}")
            extra += 1
        per_step[-1] = per_step[-1][: max(want, 1)]
        if not any(v.startswith(f"s{i}u") for v in per_step[-1]):
            per_step[-1][-1] = f"s{i}u{n_unvisited + extra}"
            extra += 1
        # unvisited set in first-seen order (dataset.py:330-342)
        visited = set(path)
        seen_unvisited = []
        for t in range(P):
            for vp in per_step[t]:
                if vp not in visited and vp not in seen_unvisited:
                    seen_unvisited.append(vp)
        gm = [None] + path + seen_unvisited
        traj_step_lens.append(P)
        traj_vpids.append(path)
        traj_cand_vpids.append(per_step)
        gmap_vpids.append(gm)
        gmap_lens.append(len(gm))
        gmap_step_ids.append([0] + list(range(1, P + 1)) + [0] * len(seen_unvisited))
        gmap_visited.append([0] + [1] * P + [0] * len(seen_unvisited))
        for t in range(P):
            nobj = obj_counts_all[k_pano] if O > 0 else 0
            vp_view_lens.append(V)
            vp_obj_lens.append(nobj)
            ncand = len(per_step[t])
            nav_types_rows.append([1] * ncand + [0] * (V - ncand) + [2] * nobj)
            k_pano += 1
    sumP = sum(traj_step_lens)
    G = max(gmap_lens)
    batch["traj_step_lens"] = traj_step_lens
    batch["traj_vpids"] = traj_vpids
    batch["traj_cand_vpids"] = traj_cand_vpids
    batch["gmap_vpids"] = gmap_vpids
    batch["gmap_lens"] = torch.tensor(gmap_lens, dtype=torch.int64)
    gsi = torch.zeros(B, G, dtype=torch.int64)
    gvm = torch.zeros(B, G, dtype=torch.bool)
    for i in range(B):
        gsi[i, : gmap_lens[i]] = torch.tensor(gmap_step_ids[i])
        gvm[i, : gmap_lens[i]] = torch.tensor(gmap_visited[i], dtype=torch.bool)
    batch["gmap_step_ids"] = gsi
    batch["gmap_visited_masks"] = gvm
    gpos = det_uniform((B, G, 7), seed, stream(), -1.0, 1.0)
    gmask = (torch.arange(G)[None, :] < batch["gmap_lens"][:, None])
    gpos = gpos * gmask[:, :, None]
    gpos[:, 0] = 0.0
    batch["gmap_pos_fts"] = gpos
    pd = det_uniform((B, G, G), seed, stream(), 0.0, 1.0)
    pd = torch.triu(pd, diagonal=1)
    pd = pd + pd.transpose(1, 2)
    pd = pd * gmask[:, :, None] * gmask[:, None, :]
    pd[:, 0, :] = 0.0
    pd[:, :, 0] = 0.0
    batch["gmap_pair_dists"] = pd

    ft = cfg.image_feat_size
    batch["traj_view_img_fts"] = det_uniform((sumP, V, ft), seed, stream(), -1.7320508, 1.7320508)
    maxobj = max(vp_obj_lens) if O > 0 else 0
    Vtot = V + maxobj
    if O > 0:
        ofts = det_uniform((sumP, max(maxobj, 1), cfg.obj_feat_size), seed, stream(), -1.7320508, 1.7320508)
        omask = torch.arange(max(maxobj, 1))[None, :] < torch.tensor(vp_obj_lens)[:, None]
        batch["traj_obj_img_fts"] = ofts * omask[:, :, None]
        batch["traj_vp_obj_lens"] = torch.tensor(vp_obj_lens, dtype=torch.int64)
    else:
        stream()
    loc = det_uniform((sumP, Vtot, 7), seed, stream(), -1.0, 1.0)
    loc[:, :V, 4:] = 1.0                        # view box features are (1,1,1) (dataset.py get_traj_pano_fts)
    tot_lens = torch.tensor([a + b for a, b in zip(vp_view_lens, vp_obj_lens)])
    loc = loc * (torch.arange(Vtot)[None, :] < tot_lens[:, None])[:, :, None]
    batch["traj_loc_fts"] = loc
    nt = torch.zeros(sumP, Vtot, dtype=torch.int64)
    for r, row in enumerate(nav_types_rows):
        nt[r, : len(row)] = torch.tensor(row)
    batch["traj_nav_types"] = nt
    batch["traj_vp_view_lens"] = torch.tensor(vp_view_lens, dtype=torch.int64)

    # ---------------------------------------------------------------- BEV lift-splat inputs
    batch["rgbs"] = det_uniform((B, 12, 14, 14, 768), seed, stream(), -1.7320508, 1.7320508)
    depths = det_uniform((B, 12, 1, 14, 14), seed, stream(), 0.0, 0.5)
    zero = det_uniform((B, 12, 1, 14, 14), seed, stream(), 0.0, 1.0) < cfg.depth_zero_frac
    depths = torch.where(zero, torch.zeros_like(depths), depths)
    batch["depths"] = depths
    sem_ids = det_randint((B, 12 * 14 * 14), seed, stream(), 0, 39)
    batch["sems"] = torch.nn.functional.one_hot(sem_ids, 40).to(torch.float64)
    fan = torch.zeros(12, 5, dtype=torch.float32)
    fan[:, 3] = -torch.arange(12, dtype=torch.float32) * math.radians(30)      # dataset.py:405-411
    fan[:, 4] = math.pi
    batch["T_c2w"] = pose_matrices(fan)[None].repeat(B, 1, 1, 1).contiguous()
    head = torch.zeros(B, 5, dtype=torch.float32)
    head[:, 3] = det_uniform((B,), seed, stream(), 0.0, 2 * math.pi)
    batch["T_w2c"] = pose_matrices(head)[:, None].contiguous()
    batch["S_w2c"] = torch.zeros(B, 1, 3, dtype=torch.float32)
    batch["bev_gpos_fts"] = det_uniform((B, 1, 7), seed, stream(), -1.0, 1.0)
    batch["bev_masks"] = torch.ones(B, ncell, dtype=torch.bool)
    # candidate cells: [centre] + one distinct non-zero cell per candidate view of the last panorama
    Ks = [1 + len(traj_cand_vpids[i][-1]) for i in range(B)]
    K = max(Ks)
    cand = torch.zeros(B, K, dtype=torch.int64)
    navm = torch.zeros(B, ncell, dtype=torch.bool)
    centre = (ncell - 1) // 2
    raw = det_randint((B, K), seed, stream(), 1, ncell - 1)
    for i in range(B):
        used = {centre}
        cand[i, 0] = centre
        for j in range(1, Ks[i]):
            c = int(raw[i, j])
            while c in used or c == 0:
                c = (c + 7) % ncell
            used.add(c)
            cand[i, j] = c
        navm[i, cand[i, : Ks[i]]] = True
    batch["bev_cand_idxs"] = cand
    batch["bev_nav_masks"] = navm

    # ---------------------------------------------------------------- task labels
    if task.startswith("sap"):
        gl, ll = [], []
        pick = det_randint((B,), seed, stream(), 0, 1 << 20).tolist()
        for i in range(B):
            cands = traj_cand_vpids[i][-1]
            unv = [j for j, vp in enumerate(cands) if vp not in set(traj_vpids[i])]
            j = unv[pick[i] % len(unv)]
            if pick[i] % 5 == 0:                       # some [stop] actions
                gl.append(0)
                ll.append(0)
            else:
                ll.append(j + 1)
                gl.append(gmap_vpids[i].index(cands[j]))
        batch["global_act_labels"] = torch.tensor(gl, dtype=torch.int64)
        batch["local_act_labels"] = torch.tensor(ll, dtype=torch.int64)
    if task.startswith("masksem"):
        batch["bev_mrc_masks"] = det_uniform((B, ncell), seed, stream(), 0.0, 1.0) < 0.15
        batch["bev_mrc_masks"][:, 0] = True
    if task.startswith("mrc") or task.startswith("og"):
        assert O > 0, "mrc / og need object tokens (obj_feat_size > 0)"
        last_obj = []
        k = 0
        for i in range(B):
            k += traj_step_lens[i]
            last_obj.append(vp_obj_lens[k - 1])
        mo = max(max(last_obj), 1)
        if task.startswith("mrc"):
            probs = det_uniform((B, mo, cfg.obj_prob_size), seed, stream(), 0.0, 1.0)
            probs = probs / probs.sum(-1, keepdim=True)
            om = torch.arange(mo)[None, :] < torch.tensor(last_obj)[:, None]
            mm = (det_uniform((B, mo), seed, stream(), 0.0, 1.0) < 0.3) & om
            for i in range(B):
                if last_obj[i] > 0 and not mm[i].any():
                    mm[i, 0] = True
            batch["vp_obj_probs"] = probs * om[:, :, None]
            batch["vp_obj_mrc_masks"] = mm
        else:
            lab = det_randint((B,), seed, stream(), 0, 1 << 20)
            batch["obj_labels"] = torch.tensor(
                [int(lab[i]) % last_obj[i] if last_obj[i] > 0 else -100 for i in range(B)], dtype=torch.int64)
    if cfg.depth_feat_size > 0:
        # drawn last, so that every other tensor matches the R2R batch of the same seed
        batch["traj_view_dep_fts"] = det_uniform((sumP, V, cfg.depth_feat_size), seed, stream(), -1.7320508, 1.7320508)
        batch["traj_loc_fts"] = batch["traj_loc_fts"][:, :, :4].contiguous()
        del batch["sems"]
    return batch


def ce_synth_config(**kw) -> SynthConfig:
    """SynthConfig of a VLN-CE batch: 512-d view and 128-d depth features, nav types {0, 1}, an 11 x 11 BEV at 1 m."""
    d = dict(image_feat_size=512, depth_feat_size=128, bev_dim=11, bev_res=1.0)
    d.update(kw)
    return SynthConfig(**d)


def batch_to(batch: dict, device, non_blocking: bool = False) -> dict:
    """Move tensor entries to `device` (host lists stay), like PrefetchLoader (data/loader.py:78-87)."""
    out = {}
    for k, v in batch.items():
        out[k] = v.to(device, non_blocking=non_blocking) if torch.is_tensor(v) else v
    return out


def clone_batch(batch: dict) -> dict:
    """Shallow copy with cloned tensors; forward() pops / adds keys (pretrain_cmt.py:115-165)."""
    return {k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}


def det_init_(model, seed: int = 0, std: float = 0.02):
    """Deterministic, machine-independent parameter init for tests / benchmarks: every tensor is filled from the
    counter-based generator (uniform with the given std; LayerNorm weights around 1).  Tied parameters are
    filled once.  Returns the model."""
    ln_w = set()
    for m in model.modules():
        if isinstance(m, torch.nn.LayerNorm):
            ln_w.add(id(m.weight))
    a = std * math.sqrt(3.0)
    seen = set()
    with torch.no_grad():
        for i, (name, p) in enumerate(sorted(model.named_parameters(), key=lambda kv: kv[0])):
            if id(p) in seen:
                continue
            seen.add(id(p))
            v = det_uniform(tuple(p.shape), seed, 1000 + i, -a, a)
            if id(p) in ln_w:
                v = v + 1.0
            p.copy_(v.to(p.device))
    return model


_PANO_KEYS = ("traj_view_img_fts", "traj_view_dep_fts", "traj_obj_img_fts", "traj_vp_obj_lens", "traj_loc_fts",
              "traj_nav_types", "traj_vp_view_lens")


def split_batch(batch: dict, parts: int):
    """Splits a collated batch into `parts` equal per-sample shards (what DistributedSampler would give each
    rank): per-sample tensors / lists are sliced on dim 0, per-panorama tensors by `traj_step_lens`."""
    B = len(batch["traj_step_lens"])
    assert B % parts == 0
    n = B // parts
    pano_off = [0]
    for s in batch["traj_step_lens"]:
        pano_off.append(pano_off[-1] + s)
    out = []
    for r in range(parts):
        lo, hi = r * n, (r + 1) * n
        sub = {}
        for k, v in batch.items():
            if k in _PANO_KEYS:
                sub[k] = v[pano_off[lo]:pano_off[hi]]
            else:
                sub[k] = v[lo:hi]
        out.append(sub)
    return out


CLIP_B16 = dict(input_resolution=224, patch_size=16, width=768, layers=12, heads=12, output_dim=512)
_CLIP_FP16 = ("conv1.weight", "proj", "in_proj_weight", "in_proj_bias", "out_proj.weight", "out_proj.bias",
              "c_fc.weight", "c_fc.bias", "c_proj.weight", "c_proj.bias")


def clip_visual_state(seed: int = 0, input_resolution=224, patch_size=16, width=768, layers=12, heads=12,
                      output_dim=512):
    """Seeded state_dict of CLIP's ViT image tower (clip/model.py VisionTransformer keys, in its state_dict order),
    machine-independent (det_uniform).  Scales follow CLIP's own: embeddings and proj width^-0.5 (VisionTransformer's
    constructor); in_proj / out_proj / c_fc / c_proj with initialize_parameters' attn_std, proj_std and fc_std; conv1
    (3 P^2)^-0.5.  Biases are small but non-zero and LayerNorms are perturbed around (1, 0), so that every term of the
    forward is exercised.  Tensors are fp32, rounded to fp16 where clip's convert_weights stores fp16."""
    D, P, L = width, patch_size, layers
    attn_std, proj_std, fc_std = D ** -0.5, D ** -0.5 * (2 * L) ** -0.5, (2 * D) ** -0.5
    shapes = [("class_embedding", (D,), D ** -0.5), ("positional_embedding", ((input_resolution // P) ** 2 + 1, D),
                                                      D ** -0.5),
              ("proj", (D, output_dim), D ** -0.5), ("conv1.weight", (D, 3, P, P), (3 * P * P) ** -0.5),
              ("ln_pre.weight", (D,), "ln"), ("ln_pre.bias", (D,), 0.05)]
    for i in range(L):
        b = "transformer.resblocks.%d." % i
        shapes += [(b + "attn.in_proj_weight", (3 * D, D), attn_std), (b + "attn.in_proj_bias", (3 * D,), 0.02),
                   (b + "attn.out_proj.weight", (D, D), proj_std), (b + "attn.out_proj.bias", (D,), 0.02),
                   (b + "ln_1.weight", (D,), "ln"), (b + "ln_1.bias", (D,), 0.05),
                   (b + "mlp.c_fc.weight", (4 * D, D), fc_std), (b + "mlp.c_fc.bias", (4 * D,), 0.02),
                   (b + "mlp.c_proj.weight", (D, 4 * D), proj_std), (b + "mlp.c_proj.bias", (D,), 0.02),
                   (b + "ln_2.weight", (D,), "ln"), (b + "ln_2.bias", (D,), 0.05)]
    shapes += [("ln_post.weight", (D,), "ln"), ("ln_post.bias", (D,), 0.05)]
    sd = {}
    for j, (k, shape, std) in enumerate(shapes):
        a = (0.1 if std == "ln" else std) * math.sqrt(3.0)
        v = det_uniform(shape, seed, 7000 + j, -a, a) + (1.0 if std == "ln" else 0.0)
        sd[k] = v.half().float() if k.endswith(_CLIP_FP16) else v
    return sd


def clip_images(n: int, seed: int = 0, res: int = 224) -> torch.Tensor:
    """n seeded uint8 RGB observations (n, res, res, 3), as habitat delivers observations["rgb"]"""
    return det_randint((n, res, res, 3), seed, 7999, 0, 255).to(torch.uint8)


def waypoint_state(seed: int = 0):
    """Seeded state_dict of the VLN-CE waypoint predictor (waypoint_pred/TRM_net.py BinaryDistPredictor_TRM keys, in its
    state_dict order, the unused visual_merge / mergefeats_LayerNorm included), machine-independent (det_uniform).
    Linear weights are uniform with standard deviation fan_in^-0.5, biases small but non-zero, LayerNorms perturbed
    around (1, 0), so that logits stay O(1) and every term of the forward is exercised."""
    D, F = 768, 3072
    shapes = [("visual_fc_depth.1.weight", (D, 2048), 2048 ** -0.5), ("visual_fc_depth.1.bias", (D,), 0.02),
              ("visual_merge.0.weight", (D, 2 * D), (2 * D) ** -0.5), ("visual_merge.0.bias", (D,), 0.02)]
    for i in range(2):
        b = "waypoint_TRM.bert.encoder.layer.%d." % i
        for name in ("query", "key", "value"):
            shapes += [(b + "attention.self.%s.weight" % name, (D, D), D ** -0.5),
                       (b + "attention.self.%s.bias" % name, (D,), 0.02)]
        shapes += [(b + "attention.output.dense.weight", (D, D), D ** -0.5),
                   (b + "attention.output.dense.bias", (D,), 0.02),
                   (b + "attention.output.LayerNorm.weight", (D,), "ln"),
                   (b + "attention.output.LayerNorm.bias", (D,), 0.05),
                   (b + "intermediate.dense.weight", (F, D), D ** -0.5), (b + "intermediate.dense.bias", (F,), 0.02),
                   (b + "output.dense.weight", (D, F), F ** -0.5), (b + "output.dense.bias", (D,), 0.02),
                   (b + "output.LayerNorm.weight", (D,), "ln"), (b + "output.LayerNorm.bias", (D,), 0.05)]
    shapes += [("mergefeats_LayerNorm.weight", (D,), "ln"), ("mergefeats_LayerNorm.bias", (D,), 0.05),
               ("vis_classifier.0.weight", (D, D), D ** -0.5), ("vis_classifier.0.bias", (D,), 0.02),
               ("vis_classifier.2.weight", (120, D), D ** -0.5), ("vis_classifier.2.bias", (120,), 0.02)]
    sd = {}
    for j, (k, shape, std) in enumerate(shapes):
        a = (0.1 if std == "ln" else std) * math.sqrt(3.0)
        sd[k] = det_uniform(shape, seed, 8000 + j, -a, a) + (1.0 if std == "ln" else 0.0)
    return sd


def depth_encoder_state(seed: int = 0, height=256, width=256):
    """Seeded state_dict of the VLN-CE policy's depth encoder (model.depth_resnet.depth_encoder(): habitat-lab's
    ResNetEncoder over resnet50 with 32 base planes and GroupNorm(16); keys in its state_dict order),
    machine-independent (det_uniform).  Conv weights are uniform with He's standard deviation (2 / fan_in)^0.5;
    GroupNorm weights are perturbed around 1 and biases around 0, so that every term of the forward is exercised."""
    from .model.depth_resnet import depth_encoder
    sd = {}
    for j, (k, v) in enumerate(depth_encoder(height, width).state_dict().items()):
        if v.dim() == 4:
            a = (2.0 / (v[0].numel())) ** 0.5 * math.sqrt(3.0)
            sd[k] = det_uniform(tuple(v.shape), seed, 9000 + j, -a, a)
        elif k.endswith("weight"):
            a = 0.1 * math.sqrt(3.0)
            sd[k] = det_uniform(tuple(v.shape), seed, 9000 + j, 1.0 - a, 1.0 + a)
        else:
            a = 0.05 * math.sqrt(3.0)
            sd[k] = det_uniform(tuple(v.shape), seed, 9000 + j, -a, a)
    return sd


def ddppo_checkpoint(seed: int = 0):
    """A DD-PPO checkpoint as VlnResnetDepthEncoder loads it (resnet_encoders.py:38-47): {"state_dict": ...} with the
    depth_encoder_state(seed) weights under `actor_critic.net.visual_encoder.*`, plus keys of the policy's other parts
    that the loader must skip."""
    sd = {"actor_critic.net.prev_action_embedding.weight": det_uniform((5, 32), seed, 9900, -1.0, 1.0)}
    for k, v in depth_encoder_state(seed).items():
        sd["actor_critic.net.visual_encoder." + k] = v
    sd["actor_critic.net.visual_fc.1.weight"] = det_uniform((512, 2048), seed, 9901, -0.01, 0.01)
    sd["actor_critic.net.state_encoder.rnn.weight_ih_l0"] = det_uniform((2048, 544), seed, 9902, -0.01, 0.01)
    sd["actor_critic.net.state_encoder.rnn.bias_ih_l0"] = det_uniform((2048,), seed, 9903, -0.01, 0.01)
    sd["actor_critic.action_distribution.linear.weight"] = det_uniform((4, 512), seed, 9904, -0.01, 0.01)
    sd["actor_critic.action_distribution.linear.bias"] = torch.zeros(4)
    sd["actor_critic.critic.fc.weight"] = det_uniform((1, 512), seed, 9905, -0.01, 0.01)
    return {"state_dict": sd, "extra_state": {"step": 0}}


def depth_images(n: int, seed: int = 0, height=256, width=256) -> torch.Tensor:
    """n seeded depth observations (n, height, width, 1) in [0, 1], as habitat delivers observations["depth"]"""
    return det_uniform((n, height, width, 1), seed, 9999, 0.0, 1.0)
