"""The VLN-CE navigation network (model/ce_nav.py), its graph-replay surface and its BEV adapter on CPU: the fp32 oracle
(oracle/ce_nav_ref.py) against the golden outputs and gradients of the unmodified CE reference, the reference's
state_dict surface and from_pretrained remap, the host logic with the kernels emulated, padded against unpadded eager
calls, and the BEV oracle and adapter host logic against the reference's gather / transform / pooling."""
import os
import sys

import numpy as np
import pytest
import torch

import ce_cases
import ce_nav_bev_cases as BC
import ce_nav_bev_oracle as BO
import ce_nav_cases as C
from bevbert_b200 import synth
from bevbert_b200.config import make_ce_config
from bevbert_b200.graphs import (CE_NAV_CALLS, ce_nav_bucket, ce_nav_forward_padded, ce_nav_pad, ce_nav_slice,
                                 install_ce_replay)
from bevbert_b200.model.ce_nav import GlocalTextPathNavCMT
from bevbert_b200.model.ce_pretrain import GlocalTextPathCMTPreTraining
from oracle import ce_nav_ref as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden():
    sys.path.insert(0, GOLD)
    import make_ce_golden
    return make_ce_golden, torch.load(os.path.join(GOLD, "small_ce_nav.pt"), weights_only=False)


@pytest.fixture
def ce_emu(emu, monkeypatch):
    import bevbert_b200.kernels as K
    monkeypatch.setattr(K, "add_rows", ce_cases.emu_add_rows(emu.add_rows))
    return emu


def _model(depth=True, sprels=True, **kw):
    return synth.det_init_(GlocalTextPathNavCMT(C.config(depth, sprels, **kw)), seed=C.WEIGHT_SEED)


def _pin_close(got, pin, tol=1e-5):
    p = C.embed_pin(got)
    assert torch.allclose(p["head"], pin["head"], rtol=tol, atol=tol), float((p["head"] - pin["head"]).abs().max())
    assert torch.allclose(p["norm"], pin["norm"], rtol=tol, atol=0), float(((p["norm"] - pin["norm"]) / pin["norm"]).abs().max())


def _logits_close(a, r, tol=1e-5):
    fin = torch.isfinite(r)
    assert torch.equal(torch.isfinite(a), fin)
    assert torch.allclose(a[fin], r[fin], rtol=tol, atol=tol), float((a[fin] - r[fin]).abs().max())


def _check_calls(o, g, tol=1e-5):
    _pin_close(o["txt"], g["txt"], tol)
    _pin_close(o["pano"][0], g["pano"][0], tol)
    assert torch.equal(o["pano"][1], g["pano"][1])
    _pin_close(o["nav"]["gmap_embeds"], g["nav"]["gmap_embeds"], tol)
    assert set(o["nav"]) == set(g["nav"])
    for k in ("global_logits", "local_logits", "fused_logits"):
        _logits_close(o["nav"][k], g["nav"][k], tol)


def _grads_close(grads, v, mk, tol=1e-3):
    assert set(grads) == set(v["grad_norms"]), set(grads) ^ set(v["grad_norms"])
    top = max(v["grad_norms"].values())
    for n, gn in v["grad_norms"].items():
        g = grads[n].detach().double()
        assert abs(float(g.norm()) - gn) <= tol * max(gn, 1e-4 * top), (n, float(g.norm()), gn)
        pr = mk.grad_projections(n, g)
        scale = max(gn, 1e-4 * top) * float(mk.grad_probes(n, tuple(g.shape)).reshape(2, -1).norm(dim=1).max())
        assert ((pr - v["grad_proj"][n]).abs() <= tol * scale).all(), n


@pytest.mark.parametrize("variant", C.VARIANTS)
def test_oracle_reproduces_ce_nav_reference(variant):
    mk, gold = _golden()
    v = gold["variants"][variant]
    model = _model(*variant)
    sd = {k: t.detach().clone() for k, t in model.state_dict().items()}
    ocfg = O.OracleConfig(model.config)
    with torch.no_grad():
        _, outs = C.rollout(O.GlocalTextPathNavCMT(sd, ocfg), gold["B"], steps=1)
    _check_calls(outs[0], v["calls"])
    train = {n for n, p in model.named_parameters() if p.requires_grad}
    sd = {k: (t.requires_grad_(True) if k in train else t) for k, t in sd.items()}
    loss, _ = C.rollout(O.GlocalTextPathNavCMT(sd, ocfg), gold["B"])
    loss.backward()
    assert abs(float(loss.detach()) - v["loss"]) <= 1e-5 * abs(v["loss"])
    _grads_close({k: t.grad for k, t in sd.items() if t.grad is not None}, v, mk)


@pytest.mark.parametrize("variant", C.VARIANTS)
def test_state_dict_keys_shapes_and_parameter_order(variant):
    _, gold = _golden()
    v = gold["variants"][variant]
    model = GlocalTextPathNavCMT(C.config(*variant))
    assert list(model.state_dict()) == list(v["shapes"])
    assert {k: tuple(t.shape) for k, t in model.state_dict().items()} == v["shapes"]
    assert [n for n, _ in model.named_parameters()] == v["param_order"]


def test_fix_flags_freeze_the_reference_modules():
    model = GlocalTextPathNavCMT(C.config(fix_lang_embedding=True, fix_pano_embedding=True))
    frozen = {n for n, p in model.named_parameters() if not p.requires_grad}
    assert frozen == {n for n, _ in model.named_parameters()
                      if n.startswith(("embeddings.", "lang_encoder.", "img_embeddings."))}


def test_from_pretrained_loads_what_the_reference_loads():
    """a CE pre-training model's state_dict, remapped as get_vlnbert_models remaps it (vlnbert_init.py:21-30)"""
    sys.path.insert(0, GOLD)
    import make_ce_nav_golden as G
    _, gold = _golden()
    pt = synth.det_init_(GlocalTextPathCMTPreTraining(make_ce_config(small=True)), seed=2)
    remapped = G.pretrain_remap(pt.state_dict())
    assert sorted(remapped) == gold["pretrain_keys"]
    cfg = C.config()
    fresh = GlocalTextPathNavCMT(cfg).state_dict()
    model = GlocalTextPathNavCMT.from_pretrained(None, config=cfg, state_dict=remapped)
    sd = model.state_dict()
    loaded = sorted(k for k in sd if any(torch.equal(sd[k], remapped[p + k]) for p in ("", "bert.") if p + k in remapped)
                    and not torch.equal(sd[k], fresh[k]))
    assert loaded == gold["pretrain_loaded"]
    # every encoder weight of the pre-training model lands, and the SAP heads too
    enc = {k[5:] for k in pt.state_dict() if k.startswith("bert.")} & set(sd)
    assert enc and all(torch.equal(sd[k], pt.state_dict()["bert." + k]) for k in enc)
    for h in ("global_sap_head", "local_sap_head", "sap_fuse_linear"):
        assert torch.equal(sd[h + ".net.0.weight"], pt.state_dict()[h + ".net.0.weight"])


def test_forward_mode_batch_raises():
    model = GlocalTextPathNavCMT(C.config())
    with pytest.raises(NotImplementedError, match="forward_txt, forward_panorama and forward_navigation"):
        model("language", {})


@pytest.mark.parametrize("variant", C.VARIANTS)
def test_host_logic_matches_oracle(ce_emu, variant):
    model = _model(*variant).train()
    sd = {k: t.detach().clone().requires_grad_(t.requires_grad) if t.is_floating_point() else t.detach().clone()
          for k, t in dict(model.named_parameters(), **dict(model.named_buffers())).items()}
    ocfg = O.OracleConfig(model.config)
    loss, outs = C.rollout(model, 3)
    loss.backward()
    rloss, routs = C.rollout(O.GlocalTextPathNavCMT(sd, ocfg), 3)
    rloss.backward()
    assert abs(float(loss) - float(rloss)) <= 1e-5 * abs(float(rloss))
    for o, r in zip(outs, routs):
        assert torch.allclose(o["pano"][0], r["pano"][0], rtol=1e-4, atol=1e-5)
        assert torch.equal(o["pano"][1], r["pano"][1])
        for k in ("gmap_embeds", "global_logits", "local_logits", "fused_logits"):
            _logits_close(o["nav"][k].detach(), r["nav"][k].detach(), 1e-4)
        assert "obj_logits" not in o["nav"]
    from helpers import grad_report
    got = {n: p.grad for n, p in model.named_parameters() if p.grad is not None}
    ref = {n: t.grad for n, t in sd.items() if t.grad is not None}
    assert set(got) == set(ref)
    worst, name = grad_report(got, ref)
    assert worst < 1e-4, (name, worst)


def _batches(B, G, Kc, L, V, step=0):
    lang = C.lang_inputs(B, L)
    pano = C.pano_inputs(B, V, step=step)
    nav = C.nav_inputs(B, G, Kc, step=step)
    return lang, pano, nav


@pytest.mark.parametrize("depth", [True, False])
@pytest.mark.parametrize("G,Kc,L,V", [(9, 4, 16, 14), (8, 3, 13, 12), (11, 9, 24, 16)])
def test_padded_eager_equals_unpadded_eager(ce_emu, depth, G, Kc, L, V):
    model = _model(depth).eval()
    lang, pano, nav = _batches(3, G, Kc, L, V)
    with torch.no_grad():
        t = model.forward_txt(lang["txt_ids"], lang["txt_masks"])
        tp = ce_nav_slice("language", ce_nav_forward_padded(model, "language", ce_nav_pad("language", lang, "cpu")), lang)
        assert torch.allclose(tp, t, rtol=1e-5, atol=1e-5)
        pe, pm = model.forward_panorama(*[pano[k] for k in C.PANO_ARGS])
        qe, qm = ce_nav_slice("panorama", ce_nav_forward_padded(model, "panorama", ce_nav_pad("panorama", pano, "cpu")),
                              pano)
        assert torch.equal(qm, pm) and torch.allclose(qe, pe, rtol=1e-5, atol=1e-5)
        nav.update(txt_embeds=t, txt_masks=lang["txt_masks"], gmap_img_fts=C.node_embeds(pe, pm, nav["gmap_masks"]))
        ref = model.forward_navigation(*[nav[k] for k in C.NAV_ARGS])
        got = ce_nav_slice("navigation", ce_nav_forward_padded(model, "navigation", ce_nav_pad("navigation", nav, "cpu"),
                                                               (nav["gmap_vpids"], nav["bev_cand_vpids"])), nav)
    assert set(got) == set(ref)
    for k in ref:
        _logits_close(got[k], ref[k])


def test_bucket_keys():
    lang, pano, nav = _batches(3, 9, 4, 16, 14)
    nav["txt_embeds"] = torch.zeros(3, 16, 768)
    nav["gmap_img_fts"] = torch.zeros(3, 9, 768)
    k = dict(zip(["txt_embeds", "txt_masks", "gmap_step_ids", "gmap_img_fts", "gmap_pos_fts", "gmap_masks",
                  "gmap_visited_masks", "gmap_pair_dists", "bev_fts", "bev_pos_fts", "bev_masks", "bev_nav_masks",
                  "bev_cand_idxs"], ce_nav_bucket("navigation", nav)[2:]))
    assert k["txt_embeds"] == ((3, 16, 768), torch.float32) and k["gmap_pair_dists"][0] == (3, 16, 16)
    assert k["gmap_img_fts"][0] == (3, 16, 768) and k["bev_fts"][0] == (3, 121, 768) and k["bev_cand_idxs"][0] == (3, 8)
    kp = ce_nav_bucket("panorama", pano)
    assert kp[2][0] == (3, 16, 512) and kp[3][0] == (3, 16, 128) and kp[6][0] == (3,)
    # B is exact: the rollout drops finished episodes
    assert ce_nav_bucket("language", C.lang_inputs(3)) != ce_nav_bucket("language", C.lang_inputs(2))
    assert ce_nav_bucket("language", C.lang_inputs(3, 9)) == ce_nav_bucket("language", C.lang_inputs(3, 16))


def test_installed_replay_runs_grad_enabled_calls_on_the_network(ce_emu):
    model = _model().train()
    lang, pano, _ = _batches(3, 9, 4, 16, 14)
    ref = model.forward_txt(lang["txt_ids"], lang["txt_masks"])
    rpe, _ = model.forward_panorama(*[pano[k] for k in C.PANO_ARGS])
    replay = install_ce_replay(model)
    assert set(CE_NAV_CALLS) <= set(vars(model))
    got = model.forward_txt(lang["txt_ids"], txt_masks=lang["txt_masks"])
    pe, _ = model.forward_panorama(*[pano[k] for k in C.PANO_ARGS])
    assert got.requires_grad and torch.equal(got, ref) and torch.equal(pe, rpe)
    assert not replay.entries
    assert "forward_txt" not in model.state_dict() and list(model.state_dict()) == list(_model().state_dict())


# ------------------------------------------------------------------------------------------------------------- BEV
def test_bev_oracle_matches_reference_golden():
    _, gold = _golden()
    bev = gold["bev"]
    import networkx as nx

    class GM:
        pass
    gm = GM()
    g = nx.Graph()
    g.add_weighted_edges_from([("a", "b", 1.0), ("b", "c", 1.0), ("c", "d", 1.0), ("b", "e", 2.0)])
    gm.shortest_path = dict(nx.all_pairs_dijkstra_path(g))
    gm.node_pc = {vp: (torch.full((k + 1, 3), float(k)),) for k, vp in enumerate(["c", "a", "e", "b", "d"])}
    from bevbert_b200.agent_bev import gathered_nodes
    for (vp, order), want in bev["gather"].items():
        got = [float(v) for c in BO.gather_nodes(gm, vp, order) for v in gm.node_pc[c][0][:, 0]]
        assert got == want, (vp, order)
        assert gathered_nodes(gm, vp, order, lambda a, b: gm.shortest_path[a][b]) == BO.gather_nodes(gm, vp, order)
    xyzhe = np.zeros((len(bev["headings"]), 5))
    xyzhe[:, 3] = bev["headings"].numpy()
    assert torch.equal(torch.from_numpy(BO.transfrom3D(xyzhe)), bev["T"])
    # the adapter's frames are transfrom3D's (equal as numbers: a few zeros differ in sign only)
    from bevbert_b200.agent_bev import heading_frames
    _, T = heading_frames(np.zeros((len(xyzhe), 3)), xyzhe[:, 3])
    assert torch.equal(torch.from_numpy(T), bev["T"])
    p = bev["project"]
    sys.path.insert(0, GOLD)
    import make_ce_nav_golden as G
    feat = G.project_feats(p["pc"].shape[1])
    eye = torch.eye(4)[None].expand(2, -1, -1)
    clouds = [[(p["pc"][b], p["no_depth"][b], feat[b])] for b in range(2)]
    got, ob = BO.splat(clouds, torch.zeros(2, 3), eye, 11, 1)
    assert torch.equal(got[..., :8], p["bev8"]) and torch.equal(ob, p["ob"])


def _splat_nodes_cpu(clouds, S_w2c, T_w2c, map_dim, map_res, y_clip=0.5, C=None):
    return BO.splat(clouds, S_w2c, T_w2c, map_dim, map_res, y_clip)


@pytest.fixture
def splat_cpu(monkeypatch):
    from bevbert_b200 import bev_nodes
    calls = []

    def spy(clouds, S, T, *a, **k):
        calls.append((clouds, S, T, a))
        return _splat_nodes_cpu(clouds, S, T, *a, **k)
    monkeypatch.setattr(bev_nodes, "bev_splat_nodes", spy)
    return calls


def test_adapter_host_logic_equals_oracle(splat_cpu):
    from bevbert_b200.agent_bev import ce_nav_bev_variable
    for tr, vp, pos, ori in BC.episode(B=3, steps=6):
        got = ce_nav_bev_variable(tr, vp, pos, ori)
        ref = BO.ce_nav_bev_variable(tr.gmaps, vp, pos, ori, [BC.heading_from_quaternion(o) for o in ori], BC.D,
                                     BC.RES, tr._discretize_polar_relpos, tr.bev_pos)
        assert set(got) == set(ref)
        for k in ("bev_fts", "bev_pos_fts", "bev_masks", "bev_nav_masks", "bev_cand_idxs"):
            assert got[k].dtype == ref[k].dtype and torch.equal(got[k], ref[k]), k
        assert got["bev_cand_vpids"] == ref["bev_cand_vpids"]
        clouds, S, T, a = splat_cpu[-1]
        assert a[:2] == (BC.D, BC.RES)
        # the node set at order 1 is the current node alone; the frames are splat's
        assert [len(c) for c in clouds] == [1, 1, 1]
        S_ref, T_ref = BO.splat_frames(pos, [BC.heading_from_quaternion(o) for o in ori])
        assert torch.equal(S, S_ref) and torch.equal(T, T_ref)
    assert any(len(v) > 2 for v in got["bev_cand_vpids"])


def test_from_pretrained_reads_the_prefixed_keys_and_rejects_shape_mismatches():
    """transformers' start_prefix rule, as the reference loads: with any `bert` key, only `bert.` keys are read"""
    cfg = C.config()
    src = _model().state_dict()
    k = "global_sap_head.net.0.bias"
    prefixed = {"bert." + n: v for n, v in src.items() if n != k}
    prefixed[k] = torch.full_like(src[k], 7.0)                  # unprefixed: ignored while prefixed keys exist
    sd = GlocalTextPathNavCMT.from_pretrained(None, config=cfg, state_dict=prefixed).state_dict()
    assert all(torch.equal(sd[n], src[n]) for n in src if n != k) and not torch.equal(sd[k], prefixed[k])
    plain = GlocalTextPathNavCMT.from_pretrained(None, config=cfg, state_dict=src).state_dict()
    assert all(torch.equal(plain[n], src[n]) for n in src)
    bad = dict(src, **{"img_embeddings.loc_linear.weight": torch.zeros(768, 7)})
    with pytest.raises(RuntimeError, match="img_embeddings.loc_linear.weight"):
        GlocalTextPathNavCMT.from_pretrained(None, config=cfg, state_dict=bad)


class _TrainerSubclass(BC.StubTrainer):
    """a trainer subclass whose module (this one) does not import heading_from_quaternion"""


def test_heading_function_is_the_trainers_own(monkeypatch):
    import types
    from bevbert_b200.agent_bev import _trainer_heading_fn
    assert "heading_from_quaternion" not in globals()
    assert _trainer_heading_fn(_TrainerSubclass(1)) is BC.heading_from_quaternion       # the base class's module
    # no module on the class chain has it: graph_utils' (where the CE trainer imports it from)
    mod = types.ModuleType("vlnce_baselines.models.graph_utils")
    mod.heading_from_quaternion = lambda q: 0.25
    monkeypatch.setitem(sys.modules, "vlnce_baselines.models.graph_utils", mod)
    assert _trainer_heading_fn(object()) is mod.heading_from_quaternion
