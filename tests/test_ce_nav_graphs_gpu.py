"""CUDA-graph replay of the VLN-CE policy's calls (bevbert_b200.graphs.install_ce_replay on model/ce_nav.py): replay
equals the eager network on the same padded inputs bit for bit on both sides of the bucket edges, while B shrinks as
episodes finish, outputs kept over a 15-step rollout stay their own step's, weight changes between episodes are seen,
and a replay launches nothing of the library eagerly.  Deterministic-mode replays are in tests/test_ce_nav_gpu.py."""
import pytest
import torch

import ce_nav_cases as C
from bevbert_b200 import kernels as K
from bevbert_b200 import synth
from bevbert_b200.graphs import ce_nav_forward_padded, ce_nav_pad, ce_nav_slice, install_ce_replay
from bevbert_b200.model.ce_nav import GlocalTextPathNavCMT

pytestmark = pytest.mark.gpu
KEYS = ("gmap_embeds", "global_logits", "local_logits", "fused_logits")


def _to(d):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in d.items()}


def _model(depth=True, seed=C.WEIGHT_SEED):
    return synth.det_init_(GlocalTextPathNavCMT(C.config(depth)), seed=seed).cuda().eval()


class PaddedEager:
    """the network's own methods on the padded inputs a replay computes on, sliced back"""

    def __init__(self, model):
        self.m = model

    def _run(self, mode, batch):
        host = (batch["gmap_vpids"], batch["bev_cand_vpids"]) if mode == "navigation" else None
        return ce_nav_slice(mode, ce_nav_forward_padded(self.m, mode, ce_nav_pad(mode, batch, "cuda"), host), batch)

    def forward_txt(self, txt_ids, txt_masks):
        return self._run("language", {"txt_ids": txt_ids, "txt_masks": txt_masks})

    def forward_panorama(self, *a):
        return self._run("panorama", dict(zip(C.PANO_ARGS, a)))

    def forward_navigation(self, *a):
        return self._run("navigation", dict(zip(C.NAV_ARGS, a)))


def _equal(a, b, what):
    assert a.shape == b.shape and torch.equal(a, b), (what, float((a.float() - b.float()).abs().nan_to_num().max()))


def _same(outs, refs):
    for t, (o, r) in enumerate(zip(outs, refs)):
        _equal(o["txt"], r["txt"], "language")
        _equal(o["pano"][0], r["pano"][0], ("panorama", t))
        _equal(o["pano"][1], r["pano"][1], ("panorama masks", t))
        assert set(o["nav"]) == set(KEYS)
        for k in KEYS:
            _equal(o["nav"][k], r["nav"][k], (k, t))


@pytest.mark.parametrize("depth", [True, False])
@pytest.mark.parametrize("B", [1, 4, 8])
def test_replay_equals_padded_eager_bit_for_bit(B, depth):
    model = _model(depth)
    eager = PaddedEager(model)
    replay = install_ce_replay(model)
    # (G, Kc, L, V) on both sides of the bucket edges at 8 and 16, and a repeat of a bucket with smaller real sizes
    for G, Kc, L, V in [(8, 8, 16, 12), (9, 9, 17, 14), (16, 3, 24, 16), (12, 6, 9, 12)]:
        with torch.no_grad():
            outs = C.rollout(model, B, steps=2, prep=_cuda, G=G, Kc=Kc, L=L, V=V)[1]
            refs = C.rollout(eager, B, steps=2, prep=_cuda, G=G, Kc=Kc, L=L, V=V)[1]
        _same(outs, refs)
        # a replay launches nothing of the library eagerly; the language call re-casts the weight shadows first
        # (GraphedNavigation.refresh, once per episode) and launches nothing beyond that.  Counted on a second episode:
        # in the first, the packed-bias re-homing of a later mode's first call moves parameters, and the graphs
        # captured before it are captured again at their next call (see GraphedNavigation)
        lang, pano, nav = _to(C.lang_inputs(B, L)), _to(C.pano_inputs(B, V, step=1)), _to(C.nav_inputs(B, G, Kc, step=1))
        with torch.no_grad():
            C.rollout(model, B, steps=1, prep=_cuda, G=G, Kc=Kc, L=L, V=V)
            n0 = K.launch_count()
            replay.refresh()
            n_refresh = K.launch_count() - n0
            n0 = K.launch_count()
            txt = model.forward_txt(lang["txt_ids"], lang["txt_masks"])
            assert K.launch_count() - n0 == n_refresh, ("language", K.launch_count() - n0, n_refresh)
            n0 = K.launch_count()
            pe, pm = model.forward_panorama(*[pano[k] for k in C.PANO_ARGS])
            assert K.launch_count() == n0, "panorama"
            nav.update(txt_embeds=txt, txt_masks=lang["txt_masks"], gmap_img_fts=C.node_embeds(pe, pm, nav["gmap_masks"]))
            n0 = K.launch_count()
            model.forward_navigation(*[nav[k] for k in C.NAV_ARGS])
            assert K.launch_count() == n0, "navigation"
    assert replay.entries and not any(e["failed"] for e in replay.entries.values())
    assert all(e["launches"] for e in replay.entries.values())


def _cuda(x):
    return x.cuda() if torch.is_tensor(x) else x


def test_shrinking_batch_and_kept_outputs_over_15_steps():
    """the CE rollout drops finished episodes (ss_trainer_BEV.py:1015-1016): B goes 8 -> 5 -> 2 while the map grows;
    every step's outputs, kept by the caller, still equal that step's padded eager results at the end"""
    model = _model()
    eager = PaddedEager(model)
    install_ce_replay(model)
    kept, refs = [], []
    with torch.no_grad():
        lang = _to(C.lang_inputs(8, 20))
        txt = model.forward_txt(lang["txt_ids"], lang["txt_masks"])
        rtxt = eager.forward_txt(lang["txt_ids"], lang["txt_masks"])
        _equal(txt, rtxt, "language")
        for t in range(15):
            B = 8 if t < 5 else (5 if t < 10 else 2)
            keep = torch.arange(B, device="cuda")
            pano = _to(C.pano_inputs(B, 20, step=t))
            nav = _to(C.nav_inputs(B, 5 + t, 4, step=t))
            for net, store, tx in ((model, kept, txt), (eager, refs, rtxt)):
                pe, pm = net.forward_panorama(*[pano[k] for k in C.PANO_ARGS])
                n = dict(nav, txt_embeds=tx[keep], txt_masks=lang["txt_masks"][keep],
                         gmap_img_fts=C.node_embeds(pe, pm, nav["gmap_masks"]))
                store.append({"txt": tx, "pano": (pe, pm), "nav": net.forward_navigation(*[n[k] for k in C.NAV_ARGS])})
    _same(kept, refs)


def test_weight_changes_between_episodes_are_seen():
    model = _model()
    install_ce_replay(model)
    with torch.no_grad():
        before = C.rollout(model, 4, steps=1, prep=_cuda)[1]
        model.load_state_dict(_model(seed=C.WEIGHT_SEED + 1).state_dict())
        after = C.rollout(model, 4, steps=1, prep=_cuda)[1]
        refs = C.rollout(PaddedEager(model), 4, steps=1, prep=_cuda)[1]
    assert not torch.equal(before[0]["nav"]["fused_logits"], after[0]["nav"]["fused_logits"])
    _same(after, refs)


def test_training_and_grad_enabled_calls_run_the_network():
    model = _model().train()
    replay = install_ce_replay(model)
    loss, _ = C.rollout(model, 2, prep=_cuda)
    loss.backward()
    assert not replay.entries and model.local_sap_head.net[0].weight.grad is not None


@pytest.mark.parametrize("replayed", [False, True])
def test_navigation_takes_the_bev_adapters_dict(replayed):
    """the dict of agent_bev.ce_nav_bev_variable goes into forward_navigation as the trainer passes it, with
    bev_cand_idxs on the host (ss_trainer_BEV.py:511, 1070-1076): eager and replayed calls equal the same call with
    every input on the device"""
    import ce_nav_bev_cases as BC
    from bevbert_b200.agent_bev import ce_nav_bev_variable
    model = _model()
    if replayed:
        install_ce_replay(model)
    B, G = 3, 9
    for t, (tr, vp, pos, ori) in enumerate(BC.episode(B=B, steps=4, device="cuda")):
        bev = ce_nav_bev_variable(tr, vp, pos, ori)
        assert not bev["bev_cand_idxs"].is_cuda
        lang = _to(C.lang_inputs(B))
        pano = _to(C.pano_inputs(B, step=t))
        nav = _to(C.nav_inputs(B, G, step=t))
        with torch.no_grad():
            txt = model.forward_txt(lang["txt_ids"], lang["txt_masks"])
            pe, pm = model.forward_panorama(*[pano[k] for k in C.PANO_ARGS])
            nav.update(bev, txt_embeds=txt, txt_masks=lang["txt_masks"],
                       gmap_img_fts=C.node_embeds(pe, pm, nav["gmap_masks"]))
            got = model.forward_navigation(*[nav[k] for k in C.NAV_ARGS])
            on_dev = dict(nav, bev_cand_idxs=nav["bev_cand_idxs"].cuda())
            if replayed:
                ref = PaddedEager(model).forward_navigation(*[on_dev[k] for k in C.NAV_ARGS])
            else:
                ref = type(model).forward_navigation(model, *[on_dev[k] for k in C.NAV_ARGS])
        assert set(got) == set(KEYS)
        for k in KEYS:
            _equal(got[k], ref[k], (k, t))
