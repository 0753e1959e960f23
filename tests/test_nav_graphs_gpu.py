"""CUDA-graph replay of the agents' per-step API (bevbert_b200.graphs.GraphedNavigation): replay equals the eager model
on the same padded inputs bit for bit, padding is invisible against the fp32 oracle, outputs the agent keeps survive
later replays, weight changes between episodes are seen, and the calls really replay.

`python tests/test_nav_graphs_gpu.py det` runs the deterministic-mode case directly (it needs CUBLAS_WORKSPACE_CONFIG
before CUDA initialises, so the test runs it in a fresh interpreter)."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [p for p in (ROOT, os.path.join(ROOT, "tests")) if p not in sys.path]

from bevbert_b200 import kernels as K  # noqa: E402
from bevbert_b200 import synth  # noqa: E402
from bevbert_b200.graphs import GraphedNavigation, nav_forward_padded, nav_pad, nav_slice  # noqa: E402
from bevbert_b200.model.nav_vilmodel import GlocalTextPathNavCMT  # noqa: E402
from helpers import rel_l2  # noqa: E402
from test_nav_api_cpu import nav_batches, nav_config  # noqa: E402

NAV_KEYS = ("gmap_embeds", "global_logits", "local_logits", "fused_logits", "obj_logits")


def _to(d, dev="cuda"):
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in d.items()}


def _model(obj, seed=4):
    cfg = nav_config(**(dict(obj_feat_size=768) if obj else {}))
    return synth.det_init_(GlocalTextPathNavCMT(cfg), seed=seed).cuda().eval()


def _eager_padded(model, mode, batch):
    """the eager model on the padded inputs a replay computes on, sliced back"""
    host = (batch["gmap_vpids"], batch["bev_cand_vpids"]) if mode == "navigation" else None
    return nav_slice(mode, nav_forward_padded(model, mode, nav_pad(mode, batch, "cuda"), host), batch)


def _inputs(B, G, K_, L=30, obj=0, D=11, H=768, seed=3, step=0):
    """per-step inputs shaped like map_nav_src/r2r/agent.py:_nav_*_variable (the layout of nav_batches) for any B, G,
    K and instruction length; sample i has G - i % 3 nodes, L - 7 * (i % 2) tokens and a candidate list that points at
    map nodes (repeats included: the last view wins in the fusion)."""
    u = lambda shape, s, lo=-1.0, hi=1.0: synth.det_uniform(shape, seed + 100 * step, s, lo, hi)
    txt_lens = torch.tensor([L - 7 * (i % 2) for i in range(B)])
    txt_masks = torch.arange(L)[None] < txt_lens[:, None]
    lang = {"txt_ids": synth.det_randint((B, L), seed, 1, 1000, 1999) * txt_masks, "txt_masks": txt_masks}
    V = 36
    obj_lens = torch.tensor([max(obj - i % 3, 0) for i in range(B)]) if obj else None
    Vt = V + obj
    pano = {"view_img_fts": u((B, V, H), 2, -1.7, 1.7), "obj_img_fts": u((B, obj, H), 3) if obj else None,
            "loc_fts": u((B, Vt, 7), 4), "nav_types": synth.det_randint((B, Vt), seed + step, 5, 0, 1),
            "view_lens": torch.full((B,), V), "obj_lens": obj_lens}
    gmap_lens = torch.tensor([max(G - i % 3, 3) for i in range(B)])
    gmask = torch.arange(G)[None] < gmap_lens[:, None]
    vpids = [[None] + ["s%dn%d" % (i, j) for j in range(1, int(gmap_lens[i]))] for i in range(B)]
    visited = torch.zeros(B, G, dtype=torch.bool)
    visited[:, 1:3] = True
    cand_vpids = [[None] + [vpids[i][1 + (k * 2 + step) % (len(vpids[i]) - 1)] for k in range(K_ - 1)] for i in range(B)]
    n = D * D
    cand_idx = torch.tensor([[(n - 1) // 2] + [(5 + i + 3 * k + step) % n for k in range(K_ - 1)] for i in range(B)])
    navm = torch.zeros(B, n, dtype=torch.bool)
    navm[torch.arange(B)[:, None], cand_idx] = True
    pd = u((B, G, G), 6, 0.0, 1.0)
    pd = (pd + pd.transpose(1, 2)) * gmask[:, :, None] * gmask[:, None, :]
    nav = {"txt_masks": txt_masks, "gmap_img_embeds": u((B, G, H), 7) * gmask[:, :, None],
           "gmap_step_ids": synth.det_randint((B, G), seed, 8, 0, 5) * gmask, "gmap_pos_fts": u((B, G, 7), 9),
           "gmap_masks": gmask, "gmap_pair_dists": pd, "gmap_visited_masks": visited, "gmap_vpids": vpids,
           "bev_fts": u((B, n, H), 10, -1.7, 1.7), "bev_pos_fts": u((B, n, 10), 11),
           "bev_masks": torch.ones(B, n, dtype=torch.bool), "bev_nav_masks": navm, "bev_cand_idxs": cand_idx,
           "bev_cand_vpids": cand_vpids, "obj_embeds": None, "obj_masks": None}
    return _to(lang), _to(pano), _to(nav)


def _with_objects(nav, pe, pm, obj):
    if obj:
        nav["obj_embeds"], nav["obj_masks"] = pe[:, 36:36 + obj], pm[:, 36:36 + obj]
    return nav


def _episode(run, lang, pano, nav, obj):
    """language, panorama, navigation through `run(mode, batch)` -> (txt_embeds, (pano_embeds, masks), nav outputs)"""
    t = run("language", lang)
    pe, pm = run("panorama", pano)
    nav = _with_objects(dict(nav, txt_embeds=t), pe, pm, obj)
    return t, (pe, pm), run("navigation", nav)


def _equal(a, b, what):
    if isinstance(a, dict):
        for k in NAV_KEYS:
            assert (a[k] is None) == (b[k] is None), (what, k)
            if a[k] is not None:
                _equal(a[k], b[k], (what, k))
        return
    assert a.shape == b.shape and torch.equal(a, b), (what, float((a.float() - b.float()).abs().nan_to_num().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("obj", [0, 5])
@pytest.mark.parametrize("B", [1, 4, 8])
def test_replay_equals_padded_eager_bit_for_bit(B, obj):
    model = _model(obj)
    nav = GraphedNavigation(model)
    # (G, K) on both sides of the bucket edges at 8 and 16, and a repeat of a bucket with smaller real sizes
    for G, K_ in [(8, 8), (9, 9), (16, 3), (12, 6)]:
        lang, pano, navb = _inputs(B, G, K_, obj=obj, L=24 + G)
        with torch.no_grad():
            t, (pe, pm), out = _episode(nav, lang, pano, navb, obj)
            te, (pee, pme), oute = _episode(lambda m, b: _eager_padded(model, m, b), lang, pano, navb, obj)
        _equal(t, te, "language")
        _equal(pe, pee, "panorama")
        _equal(pm, pme, "panorama masks")
        _equal(out, oute, "navigation")
        for mode, b in (("language", lang), ("panorama", pano)):
            assert nav.launches(mode, b), (mode, G, K_)
        nb = _with_objects(dict(navb, txt_embeds=t), pe, pm, obj)
        assert nav.launches("navigation", nb), (G, K_)
        # a replay launches nothing of the library eagerly
        with torch.no_grad():
            n0 = K.launch_count()
            nav("navigation", nb)
            assert K.launch_count() == n0
    assert not any(e["failed"] for e in nav.entries.values())


@pytest.mark.gpu
@pytest.mark.parametrize("obj", [0, 5])
def test_padding_is_invisible(obj):
    """replay on unpadded inputs against the fp32 oracle with test_nav_gpu's bars; finite pattern and argmax of the fused
    logits as eager's.  Whether the values are also bit-identical to unpadded eager is printed (`pytest -s`)."""
    from oracle import bevbert_ref as R
    model = _model(obj)
    nav = GraphedNavigation(model)
    sd = {k: v.detach().float().cpu().clone() for k, v in model.state_dict().items()}
    ocfg = R.OracleConfig(model.config)
    lang, pano, navb = nav_batches(obj=obj)
    with torch.no_grad():
        t, (pe, pm), _ = _episode(nav, _to(lang), _to(pano), _to(navb), obj)
        te, (pee, pme), _ = _episode(model, _to(lang), _to(pano), _to(navb), obj)
        rt_ = R.nav_forward(sd, "language", lang, ocfg)
        rpe, rpm = R.nav_forward(sd, "panorama", pano, ocfg)
        assert rel_l2(t, rt_) < 1e-2 and rel_l2(pe, rpe) < 1e-2 and torch.equal(pm.cpu(), rpm)
        navb["txt_embeds"] = rt_
        if obj:
            navb["obj_embeds"], navb["obj_masks"] = rpe[:, 36:36 + obj], rpm[:, 36:36 + obj]
        ref = R.nav_forward(sd, "navigation", navb, ocfg)
        out = nav("navigation", _to(navb))
        oute = model("navigation", _to(navb))
    for k in ("gmap_embeds", "global_logits", "local_logits", "fused_logits"):
        fin = torch.isfinite(ref[k])
        assert torch.equal(torch.isfinite(out[k].cpu()), fin), k
        assert torch.equal(torch.isfinite(out[k]), torch.isfinite(oute[k])), k
        assert rel_l2(out[k].cpu()[fin], ref[k][fin]) < 2e-2, (k, rel_l2(out[k].cpu()[fin], ref[k][fin]))
    assert torch.equal(out["fused_logits"].argmax(1), oute["fused_logits"].argmax(1))
    same = {"language": torch.equal(t, te), "panorama": torch.equal(pe, pee)}
    same.update({k: torch.equal(out[k], oute[k]) for k in NAV_KEYS if out[k] is not None})
    print("obj=%d replay bit-identical to unpadded eager: %s" % (obj, same))


@pytest.mark.gpu
def test_rollout_keeps_earlier_outputs():
    """15 navigation steps at B = 4 with G growing across bucket edges, K varying and episodes ending (an ended sample
    keeps its last map); every output kept from earlier steps must still equal its step's eager result at the end."""
    obj = 5
    model = _model(obj)
    nav = GraphedNavigation(model)
    B = 4
    lang, _, _ = _inputs(B, 4, 3, obj=obj)
    kept = []
    with torch.no_grad():
        t = nav("language", lang)
        kept.append((t, _eager_padded(model, "language", lang)))
        ended_at = [15, 6, 11, 15]
        for s in range(15):
            G, K_ = 3 + s, 2 + (s * 5) % 7
            _, pano, navb = _inputs(B, G, K_, obj=obj, step=s)
            pe, pm = nav("panorama", pano)
            kept.append((pe[1, 3], _eager_padded(model, "panorama", pano)[0][1, 3]))      # gmap.update_node_embed view
            navb = _with_objects(dict(navb, txt_embeds=t), pe, pm, obj)
            for i, e in enumerate(ended_at):       # ended samples: the map stops growing
                if s >= e:
                    navb["gmap_masks"][i, 3 + e:] = False
                    navb["gmap_img_embeds"][i, 3 + e:] = 0
                    navb["gmap_pair_dists"][i, 3 + e:] = 0
                    navb["gmap_pair_dists"][i, :, 3 + e:] = 0
                    navb["gmap_vpids"][i] = navb["gmap_vpids"][i][:3 + e]
            out = nav("navigation", navb)
            kept.append((out, _eager_padded(model, "navigation", navb)))
            assert nav.launches("navigation", navb)
    for i, (a, b) in enumerate(kept):
        _equal(a, b, "kept output %d" % i)


@pytest.mark.gpu
def test_weight_changes_are_seen_by_the_next_episode():
    model = _model(0)
    nav = GraphedNavigation(model)
    lang, pano, navb = _inputs(4, 10, 5)
    run_e = lambda m, b: _eager_padded(model, m, b)
    with torch.no_grad():
        first = _episode(nav, lang, pano, navb, 0)
        _equal(first[2], _episode(run_e, lang, pano, navb, 0)[2], "initial weights")
    # load_state_dict between validations
    other = synth.det_init_(GlocalTextPathNavCMT(model.config), seed=9)
    model.load_state_dict(other.state_dict())
    with torch.no_grad():
        second = _episode(nav, lang, pano, navb, 0)
        _equal(second[2], _episode(run_e, lang, pano, navb, 0)[2], "after load_state_dict")
    assert not torch.equal(first[2]["fused_logits"], second[2]["fused_logits"])
    # a foreign optimizer's step between validations
    model.train()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    out = model("navigation", dict(navb, txt_embeds=second[0]))
    out["fused_logits"][torch.isfinite(out["fused_logits"])].sum().backward()
    opt.step()
    model.eval()
    with torch.no_grad():
        third = _episode(nav, lang, pano, navb, 0)
        _equal(third[2], _episode(run_e, lang, pano, navb, 0)[2], "after an AdamW step")
    assert not torch.equal(second[2]["fused_logits"], third[2]["fused_logits"])
    assert not any(e["failed"] for e in nav.entries.values())


@pytest.mark.gpu
def test_grad_and_training_calls_run_eagerly():
    model = _model(0)
    nav = GraphedNavigation(model)
    lang, _, _ = _inputs(2, 8, 4)
    t = nav("language", lang)                   # grad enabled: the model itself
    assert not nav.entries
    with torch.no_grad():
        _equal(t, model("language", lang), "grad-enabled call")


@pytest.mark.gpu
def test_deterministic_replays_are_bit_identical():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] +
                                        ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, "-s", os.path.abspath(__file__), "det"], env=env, capture_output=True,
                       text=True, timeout=1800)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stderr[-6000:]


def _det_case():
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    model = _model(5)
    nav = GraphedNavigation(model)
    lang, pano, navb = _inputs(4, 13, 6, obj=5)
    with torch.no_grad():
        runs = [_episode(nav, lang, pano, navb, 5) for _ in range(3)]
        nb = _with_objects(dict(navb, txt_embeds=runs[0][0]), runs[0][1][0], runs[0][1][1], 5)
        assert nav.launches("navigation", nb) and nav.launches("language", lang)
        assert all(k[1] for k in nav.entries)              # captured in deterministic mode
    torch.cuda.synchronize()
    for r in runs[2:]:
        _equal(r[0], runs[1][0], "language")
        _equal(r[1][0], runs[1][1][0], "panorama")
        _equal(r[2], runs[1][2], "navigation")
    print("deterministic replays identical; launches per navigation replay: %d" % nav.launches("navigation", nb))


if __name__ == "__main__":
    if sys.argv[1:] == ["det"]:
        _det_case()
