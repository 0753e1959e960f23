"""Fine-tuning rollouts of GlocalTextPathNavCMT (tests/nav_rollout_cases.py) on CPU with the emulated kernels against
the fp64 oracle: the host logic of a multi-call episode with one backward (node memory, many Runtime.begin() before
it), and the bf16 weight shadows after an optimizer step that bumps no tensor version."""
import pytest
import torch

from bevbert_b200 import synth
from bevbert_b200.model.nav_vilmodel import GlocalTextPathNavCMT
from nav_rollout_cases import ModelCall, OracleCall, describe, errors, make_episode, rollout
from test_nav_api_cpu import nav_config

# the emulation is fp32 torch: what is left against fp64 is fp32 rounding
BAR = {"txt": 1e-5, "pano": 1e-5, "gmap": 1e-5, "logits": 1e-4, "loss": 1e-5, "grad": 1e-4, "param": 1e-3}


def _check(e, bar=BAR):
    bad = {k: (e[k], b) for k, b in bar.items() if k in e and not e[k] <= b}
    assert not bad, (bad, e.get("param_name"))


def _model(obj):
    cfg = nav_config(obj_feat_size=768) if obj else nav_config()
    return cfg, synth.det_init_(GlocalTextPathNavCMT(cfg), seed=4).train()


def test_episodes_reach_every_edge():
    ep = make_episode(4, 6, 11)
    d = describe(ep)
    assert d.pop("G") >= 20 and ep["steps"][-1]["G"] % 8 != 0
    assert all(d.values()), d
    lens = ep["lang"]["txt_masks"].sum(1)
    assert len(set(lens.tolist())) == 4
    vl = torch.stack([s["pano"]["view_lens"] for s in ep["steps"]])
    assert len(set(vl.flatten().tolist())) > 3
    kc = [len(r["cands"]) for s in ep["steps"] for r in s["recs"] if not r["ended"]]
    assert 0 in kc and len(set(kc)) > 3
    ob = make_episode(4, 3, 11, obj=True)
    ol = torch.stack([s["pano"]["obj_lens"] for s in ob["steps"]])
    assert 0 in ol.tolist()[0] and len(set(ol.flatten().tolist())) > 2
    for s in ep["steps"]:
        for k in ("local", "fused"):
            assert bool((s["targets"][k] == -100).any()) == any(r["ended"] for r in s["recs"])


@pytest.mark.parametrize("obj,fusion", [(False, "fused"), (False, "local"), (True, "fused"), (True, "global")])
def test_rollout_matches_fp64(emu, obj, fusion):
    cfg, model = _model(obj)
    ep = make_episode(4, 4, 11, seed=1, obj=obj)
    got = rollout(ModelCall(model, "cpu"), ep, fusion)
    ref = rollout(OracleCall(model, cfg), ep, fusion)
    e = errors(got, ref, ep)
    print(obj, fusion, {k: ("%.2e" % v if isinstance(v, float) else v) for k, v in e.items()})
    _check(e)
    # every call reaches the gradients: the panorama encoder through the node memory, the language encoder and the
    # object head (REVERIE)
    g = got["grads"]
    heads = {"fused": ("global_sap_head", "local_sap_head"), "global": ("global_sap_head",),
             "local": ("local_sap_head",)}[fusion] + (("og_head",) if obj else ())
    for name in ("img_embeddings.img_linear.weight", "lang_encoder.layer.0.attention.self.query.weight",
                 "sap_fuse_linear.net.0.weight") + tuple(h + ".net.0.weight" for h in heads):
        assert g[name] is not None and float(g[name].abs().sum()) > 0, name


def _update(kind, model):
    """One optimizer step after a training rollout's backward."""
    params = [p for p in model.parameters() if p.grad is not None]
    if kind == "pdata":
        with torch.no_grad():
            for p in params:
                p.data.add_(p.grad.sign(), alpha=-1e-2)
        return
    torch.optim.AdamW(params, lr=1e-2, fused=(kind == "fused")).step()


def freshness(kind, model, cfg, call, update=_update, bar=BAR):
    """Train, step with `kind`, then evaluate and train again; both must match the fp64 oracle on the NEW weights."""
    ep = make_episode(2, 2, cfg.bev_dim, seed=5, obj=cfg.obj_feat_size > 0)
    model.train()
    rollout(call, ep, "fused")
    update(kind, model)
    model.eval()
    with torch.no_grad():
        got = rollout(call, ep, "fused", train=False)
        ref = rollout(OracleCall(model, cfg), ep, "fused", train=False)
    e_eval = errors(got, ref, ep, train=False)
    model.train()
    got = rollout(call, ep, "fused")
    ref = rollout(OracleCall(model, cfg), ep, "fused")
    e_train = errors(got, ref, ep)
    print("%s: eval %s | train %s" % (kind, {k: "%.2e" % e_eval[k] for k in ("txt", "pano", "gmap", "logits")},
                                       {k: ("%.2e" % v if isinstance(v, float) else v) for k, v in e_train.items()}))
    if bar is not None:
        _check(e_eval, bar)
        _check(e_train, bar)
    return e_eval, e_train


@pytest.mark.parametrize("kind", ["default", "fused", "pdata"])
def test_eval_after_optimizer_step_uses_new_weights(emu, kind):
    cfg, model = _model(False)
    freshness(kind, model, cfg, ModelCall(model, "cpu"))
