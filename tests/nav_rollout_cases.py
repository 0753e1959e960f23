"""Fine-tuning episodes of the navigation agents and one rollout driver for both the model and the oracle.

An agent trains `GlocalTextPathNavCMT` through `forward(mode, batch)` (map_nav_src/r2r/agent.py:470-633): `language`
once, then per step `panorama`, a host-side masked average into the node memory of its topological map, and
`navigation` on inputs assembled from that memory; the cross-entropy losses of all steps are summed and there is ONE
backward.  Gradients reach the language encoder from every step and the panorama encoder through the node embeddings,
and the model's step arenas are carved by every `Runtime.begin()` before that single backward.

`make_episode` builds deterministic episodes (`synth.det_*`) with what the agents produce: ragged instruction, view,
object and candidate counts; a sample whose only candidate is [stop] (Kc = 1); padded candidate slots (cell 0, mask
False) as `pad_tensors` makes them; two candidates in one BEV cell; a candidate clamped to cell 0; revisited nodes;
candidates leading back to visited nodes (the fusion back-track term); unvisited nodes seen from two steps (a running
mean of two embeddings); samples that stop early (target -100 afterwards); and a graph of G = 2 + 4T nodes
(26 at T = 6, so G % 8 != 0).  BEV inputs are synthetic.

`rollout(call, episode, fusion, obj)` runs one episode through `call` -- `ModelCall` (the model on its device) or
`OracleCall` (oracle.bevbert_ref.nav_forward on CPU, in fp64 or under bf16 autocast) -- and returns the per-step
outputs, the loss and, in training, every parameter gradient.

Known semantic difference, not exercised: our fused logits add 0 for a MASKED candidate where the reference would add
-inf.  The agents never mask a real candidate and padded slots carry no viewpoint id, so it cannot arise; the padded
slots here pin the behaviour that does arise (including a padded slot whose cell 0 is a navigable cell, so its local
logit is finite on both sides).
"""
import torch
import torch.nn.functional as F

from bevbert_b200 import synth
from oracle import bevbert_ref as R

H = 768


# ------------------------------------------------------------------------------------------------- episodes
def _walk(role, i, T, n, seed):
    """Host plan of sample i: one record per step.  Roles: 0 explores (4 new nodes per step, back-track candidate,
    a node seen again, two candidates in one cell), 1 stands at a dead end (only [stop], stops at step 0),
    2 walks back and forth (revisits, a candidate clamped to cell 0), 3 stops after two steps."""
    centre = (n - 1) // 2
    count = [0]

    def new():
        count[0] += 1
        return "s%dn%d" % (i, count[0] - 1)

    def cell(t, j):
        c = (centre + 1 + 7 * j + 13 * t + 29 * i + int(synth.det_randint((1,), seed, 100 + 8 * t + i, 0, 3))) % n
        return 1 if c in (0, centre) else c

    cur, nodes, visited, step_ids = new(), [], set(), {}
    nodes.append(cur)
    recs, prev, seen_later, back = [], None, None, None
    for t in range(T):
        if recs and (recs[-1]["ended"] or recs[-1]["nxt"] is None):
            recs.append(dict(recs[-1], ended=True))
            continue
        visited.add(cur)
        step_ids[cur] = t + 1
        if role == 0:
            fresh = [new() for _ in range(4)]
            cands = ([prev] if prev is not None else []) + ([seen_later] if seen_later else []) + fresh
            seen_later, nxt = fresh[-1], fresh[0]
        elif role == 1:
            cands, nxt = [], None
        elif role == 2:
            if t % 2 == 0:
                back = back or [new(), new()]
                cands = list(back)
                nxt = back[0] if t == 0 else next((c for c in cands if c not in visited), back[1])
            else:
                cands = [prev, new()]
                nxt = prev                       # walk back: a revisit
            if t == T - 1 and T > 1:
                nxt = None
        else:
            cands = [new() for _ in range(1 + t % 3)]
            nxt = cands[0] if t < min(2, T - 1) else None
        for c in cands:
            if c not in nodes:
                nodes.append(c)
        cells = [cell(t, j) for j in range(len(cands))]
        if role == 0 and len(cands) >= 4:
            cells[3] = cells[2]                  # two candidates in the same BEV cell
        if role == 2 and t == 0:
            cells[0] = 0                         # a far candidate clamped to cell 0
        recs.append({"cur": cur, "cands": list(cands), "cells": cells, "nxt": nxt, "ended": False,
                     "nodes": list(nodes), "visited": set(visited), "step_ids": dict(step_ids)})
        if nxt is not None:
            prev, cur = cur, nxt
    return recs


def _targets(r):
    """(local, global/fused) action targets of one sample at one step; -100 once the sample has stopped.  A global
    target always names an unvisited node (the teacher of the global / fused policies picks among those)."""
    if r["ended"]:
        return -100, -100
    if r["nxt"] is None:
        return 0, 0
    loc = r["cands"].index(r["nxt"]) + 1
    if r["nxt"] not in r["visited"]:
        return loc, 1 + r["nodes"].index(r["nxt"])
    free = [k for k, vp in enumerate(r["nodes"]) if vp not in r["visited"]]
    return loc, (1 + free[0]) if free else 0


def make_episode(B, T, D, seed=0, obj=False):
    n = D * D
    centre = (n - 1) // 2
    u = lambda shape, s, lo=-1.0, hi=1.0: synth.det_uniform(shape, seed, s, lo, hi)
    walks = [_walk(i % 4, i, T, n, seed) for i in range(B)]
    L = 44
    txt_lens = torch.tensor([L, 29, 37, 12][:B] if B > 1 else [23])
    txt_masks = torch.arange(L)[None] < txt_lens[:, None]
    ep = {"B": B, "T": T, "D": D, "obj": obj,
          "lang": {"txt_ids": synth.det_randint((B, L), seed, 1, 1000, 1999) * txt_masks, "txt_masks": txt_masks},
          "steps": []}
    for t in range(T):
        recs = [w[t] for w in walks]
        s0 = 1000 * (t + 1)
        # panorama: candidate views first, then the other views (ragged counts), then objects
        vl = torch.tensor([max(len(r["cands"]), 31 + (5 * i + 3 * t) % 8) for i, r in enumerate(recs)])
        ol = torch.tensor([0 if i % 4 == 1 else 1 + (i + t) % 4 for i in range(B)]) if obj else None
        V = int(vl.max())
        tot = vl + (ol if obj else 0)
        Vt = int(tot.max())
        vmask = torch.arange(V)[None] < vl[:, None]
        tmask = torch.arange(Vt)[None] < tot[:, None]
        nav_types = torch.zeros(B, Vt, dtype=torch.long)
        for i, r in enumerate(recs):
            nav_types[i, :len(r["cands"])] = 1
            if obj:
                nav_types[i, int(vl[i]):int(tot[i])] = 2
        pano = {"view_img_fts": u((B, V, H), s0 + 1, -1.7, 1.7) * vmask[:, :, None],
                "obj_img_fts": None, "loc_fts": u((B, Vt, 7), s0 + 2) * tmask[:, :, None], "nav_types": nav_types,
                "view_lens": vl, "obj_lens": ol}
        if obj:
            Om = int(ol.max())
            pano["obj_img_fts"] = u((B, Om, H), s0 + 3) * (torch.arange(Om)[None] < ol[:, None])[:, :, None]
        # navigation: everything but the node embeddings (those come from the node memory)
        G = 1 + max(len(r["nodes"]) for r in recs)
        Kc = 1 + max(len(r["cands"]) for r in recs)
        gmask = torch.zeros(B, G, dtype=torch.bool)
        visited = torch.zeros(B, G, dtype=torch.bool)
        step_ids = torch.zeros(B, G, dtype=torch.long)
        xy = torch.zeros(B, G, 2)
        cand_idx = torch.zeros(B, Kc, dtype=torch.long)
        navm = torch.zeros(B, n, dtype=torch.bool)
        bevm = torch.ones(B, n, dtype=torch.bool)
        for i, r in enumerate(recs):
            gmask[i, :1 + len(r["nodes"])] = True
            for k, vp in enumerate(r["nodes"]):
                visited[i, k + 1] = vp in r["visited"]
                step_ids[i, k + 1] = r["step_ids"].get(vp, 0)
                xy[i, k + 1] = synth.det_uniform((2,), seed, 7000 + 64 * i + int(vp.split("n")[-1]), -6.0, 6.0)
            cand_idx[i, :1 + len(r["cands"])] = torch.tensor([centre] + r["cells"])
            navm[i, cand_idx[i, :1 + len(r["cands"])]] = True
            if i % 4 == 3:
                bevm[i, n - 7:] = navm[i, n - 7:]   # a few cells without points (attention key mask)
        pd = (xy[:, :, None] - xy[:, None, :]).norm(dim=-1) * (gmask[:, :, None] & gmask[:, None, :])
        pd[:, 0] = 0
        pd[:, :, 0] = 0
        nav = {"txt_masks": txt_masks, "gmap_step_ids": step_ids,
               "gmap_pos_fts": u((B, G, 7), s0 + 4) * gmask[:, :, None], "gmap_masks": gmask, "gmap_pair_dists": pd, "gmap_visited_masks": visited,
               "gmap_vpids": [[None] + r["nodes"] for r in recs],
               "bev_fts": u((B, n, H), s0 + 5, -1.7, 1.7), "bev_pos_fts": u((B, n, 10), s0 + 6), "bev_masks": bevm,
               "bev_nav_masks": navm, "bev_cand_idxs": cand_idx, "bev_cand_vpids": [[None] + r["cands"] for r in recs]}
        tl, tg = zip(*[_targets(r) for r in recs])
        og = [-100 if (r["ended"] or int(ol[i]) == 0) else (t + i) % int(ol[i]) for i, r in enumerate(recs)] if obj \
            else None
        ep["steps"].append({"recs": recs, "pano": pano, "nav": nav, "G": G,
                            "targets": {"local": torch.tensor(tl), "global": torch.tensor(tg),
                                        "fused": torch.tensor(tg)},
                            "og": torch.tensor(og) if obj else None})
    return ep


def describe(ep):
    """The edges an episode reaches (the CPU test asserts them on the shared episodes)."""
    d = {"G": max(s["G"] for s in ep["steps"]), "kc1": False, "padded": False, "dup_cell": False, "cell0": False,
         "revisit": False, "backtrack": False, "ended": False, "two_views": False}
    been = [set() for _ in range(ep["B"])]
    seen = [{} for _ in range(ep["B"])]
    for s in ep["steps"]:
        kc = s["nav"]["bev_cand_idxs"].shape[1]
        for i, r in enumerate(s["recs"]):
            d["ended"] |= r["ended"]
            if r["ended"]:
                continue
            d["kc1"] |= not r["cands"]
            d["padded"] |= len(r["cands"]) + 1 < kc
            d["dup_cell"] |= len(set(r["cells"])) < len(r["cells"])
            d["cell0"] |= 0 in r["cells"]
            d["revisit"] |= r["cur"] in been[i]
            been[i].add(r["cur"])
            d["backtrack"] |= any(c in r["visited"] for c in r["cands"])
            for c in r["cands"]:
                if c not in r["visited"]:
                    seen[i][c] = seen[i].get(c, 0) + 1
                    d["two_views"] |= seen[i][c] > 1
    return d


# ------------------------------------------------------------------------------------------------- backends
class ModelCall:
    """`model(mode, batch)` with float inputs moved to `device` in fp32 (the API's dtype)."""

    def __init__(self, model, device):
        self.model, self.device, self.dtype = model, device, torch.float32

    def prep(self, x):
        if not torch.is_tensor(x):
            return x
        return x.to(self.device, torch.float32) if x.is_floating_point() else x.to(self.device)

    def __call__(self, mode, batch):
        return self.model(mode, batch)

    def params(self):
        return dict(self.model.named_parameters())


class OracleCall:
    """oracle.nav_forward on CPU over a copy of `model`'s state dict in `dtype` (fp64), or in fp32 under bf16 autocast
    (the precision class of the product path).  Only the parameters the model trains require grad, so gradient
    presence can be compared."""

    def __init__(self, model, cfg, dtype=torch.float64, autocast=False):
        train = {n for n, p in model.named_parameters() if p.requires_grad}
        self.sd = {k: (v.detach().cpu().to(dtype).clone().requires_grad_(k in train) if v.is_floating_point()
                       else v.detach().cpu().clone()) for k, v in model.state_dict().items()}
        self.ocfg = R.OracleConfig(cfg)
        self.dtype, self.autocast = dtype, autocast

    def prep(self, x):
        if not torch.is_tensor(x):
            return x
        return x.to("cpu", self.dtype) if x.is_floating_point() else x.cpu()

    def __call__(self, mode, batch):
        if self.autocast:
            with torch.autocast("cpu", dtype=torch.bfloat16):
                out = R.nav_forward(self.sd, mode, batch, self.ocfg)
        else:
            out = R.nav_forward(self.sd, mode, batch, self.ocfg)
        cast = lambda x: x.to(self.dtype) if torch.is_tensor(x) and x.is_floating_point() else x
        if isinstance(out, dict):
            return {k: cast(v) for k, v in out.items()}
        if isinstance(out, tuple):
            return tuple(cast(v) for v in out)
        return cast(out)

    def params(self):
        return self.sd


# ------------------------------------------------------------------------------------------------- the driver
def rollout(call, ep, fusion="fused", obj=None, train=True, detach_avg_step=None, drop_loss_step=None):
    """One agent episode through `call`.  -> {"txt", "pano": [(embeds, masks)], "nav": [outputs], "loss",
    "grads": {name: grad or None} (training only)}.  `detach_avg_step` / `drop_loss_step` break the rollout at one
    step (negative controls)."""
    obj = ep["obj"] if obj is None else obj
    P = lambda d: {k: call.prep(v) for k, v in d.items()}
    B = ep["B"]
    if train:
        for p in call.params().values():
            p.grad = None
    txt = call("language", P(ep["lang"]))
    mem = [{} for _ in range(B)]         # vp -> [sum of embeddings, count] (GraphMap.update_node_embed)
    res = {"txt": txt, "pano": [], "nav": []}
    loss = 0.0
    for t, st in enumerate(ep["steps"]):
        pe, pm = call("panorama", P(st["pano"]))
        res["pano"].append((pe, pm))
        avg = (pe * pm[:, :, None]).sum(1) / pm.sum(1, keepdim=True)
        if detach_avg_step == t:
            avg = avg.detach()
        for i, r in enumerate(st["recs"]):
            if r["ended"]:
                continue
            mem[i][r["cur"]] = [avg[i], 1]                       # the visited node is rewritten
            for j, c in enumerate(r["cands"]):
                if c not in r["visited"]:                        # unvisited: running mean of what it was seen as
                    m = mem[i].get(c)
                    mem[i][c] = [pe[i, j], 1] if m is None else [m[0] + pe[i, j], m[1] + 1]
        G = st["G"]
        rows = []
        for i, r in enumerate(st["recs"]):
            e = torch.stack([pe.new_zeros(H)] + [mem[i][vp][0] / mem[i][vp][1] for vp in r["nodes"]])
            rows.append(F.pad(e, (0, 0, 0, G - e.shape[0])))
        nav = P(st["nav"])
        nav["txt_embeds"], nav["gmap_img_embeds"] = txt, torch.stack(rows)
        nav["obj_embeds"] = nav["obj_masks"] = None
        if obj:
            vl, ol = st["pano"]["view_lens"], st["pano"]["obj_lens"]
            Om = int(ol.max())
            nav["obj_embeds"] = torch.stack([F.pad(pe[i, int(vl[i]):int(vl[i] + ol[i])], (0, 0, 0, Om - int(ol[i])))
                                             for i in range(B)])
            nav["obj_masks"] = call.prep(torch.arange(Om)[None] < ol[:, None])
        out = call("navigation", nav)
        res["nav"].append(out)
        if train and t != drop_loss_step:
            tgt = call.prep(st["targets"][fusion])
            loss = loss + F.cross_entropy(out[fusion + "_logits"], tgt, ignore_index=-100, reduction="sum")
            if obj:
                og = st["og"]
                sel = og >= 0                   # a sample without objects has no finite object logit
                if bool(sel.any()):
                    loss = loss + F.cross_entropy(out["obj_logits"][call.prep(sel)], call.prep(og[sel]),
                                                  reduction="sum")
    if train:
        loss = loss / B
        loss.backward()
        res["grads"] = {n: p.grad for n, p in call.params().items()}
        res["loss"] = loss.detach()
    return res


# ------------------------------------------------------------------------------------------------- comparison
def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def errors(got, ref, ep, train=True):
    """Worst relative L2 errors of a rollout against a reference rollout of the same episode, by kind: "txt" (valid
    tokens), "pano" (valid panorama tokens, worst step), "gmap" (valid nodes), "logits" (finite entries of the global,
    local, fused and object logits), "loss", "grad" (all parameter gradients together) and "param" (worst single
    parameter, measured against max(its norm, 1e-2 x the largest reference norm); its name is under "param_name").
    Asserts that panorama masks are bit-equal, that finite-logit patterns are equal and that gradient presence
    agrees."""
    from helpers import grad_errors
    tm = ep["lang"]["txt_masks"]
    e = {"txt": _rel(got["txt"].cpu()[tm], ref["txt"].cpu()[tm]), "pano": 0.0, "gmap": 0.0, "logits": 0.0}
    for t, ((pe, pm), (rpe, rpm)) in enumerate(zip(got["pano"], ref["pano"])):
        pm, rpm = pm.cpu(), rpm.cpu()
        assert torch.equal(pm, rpm), "panorama masks differ at step %d" % t
        e["pano"] = max(e["pano"], _rel(pe.cpu()[pm], rpe.cpu()[rpm]))
    for t, (o, r) in enumerate(zip(got["nav"], ref["nav"])):
        gm = ep["steps"][t]["nav"]["gmap_masks"]
        e["gmap"] = max(e["gmap"], _rel(o["gmap_embeds"].cpu()[gm], r["gmap_embeds"].cpu()[gm]))
        for k in ("global_logits", "local_logits", "fused_logits", "obj_logits"):
            assert (o[k] is None) == (r[k] is None), k
            if r[k] is None:
                continue
            a, b = o[k].detach().cpu(), r[k].detach().cpu()
            fin = torch.isfinite(b)
            assert torch.equal(torch.isfinite(a), fin), "finite pattern of %s differs at step %d" % (k, t)
            e["logits"] = max(e["logits"], _rel(a[fin], b[fin]))
    if train:
        e["loss"] = _rel(got["loss"].reshape(1), ref["loss"].reshape(1))
        errs, e["grad"] = grad_errors(got["grads"], {n: ref["grads"].get(n) for n in got["grads"]})
        e["param_name"], e["param"] = max(errs.items(), key=lambda kv: kv[1])
    return e
