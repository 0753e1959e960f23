"""Fine-tuning rollouts of GlocalTextPathNavCMT on the CUDA kernels against fp64 autograd of the oracle.

An agent episode (tests/nav_rollout_cases.py): `language` once, T rounds of `panorama` -> node memory -> `navigation`,
the summed action (and REVERIE object-grounding) cross-entropies, ONE backward.  Compared at every step: text,
panorama embeddings (masks bit-equal), global-map embeddings, the global / local / fused / object logits (finite
patterns equal), then the loss and every parameter gradient (presence equal: frozen parameters are None on both sides).

  * fp32 verification arm (kernels.set_precision(True)): the same host logic and kernels with fp32 storage; bars in
    BARS at about 3x the floor measured on an H100, never above the pre-training fp32 arm's 1e-3 (global) / 5e-3
    (per parameter).
  * bf16 product path: the fixed bars in BARS and, as in test_model_gpu._compare, the global gradient error within
    2.5x (each parameter within 3x) the error of the oracle run under CPU bf16 autocast on the same inputs.
  * negative controls: detaching one step's panorama average before the node memory, or dropping one step's loss, in
    the model's rollout only, must push some gradient error to 5x its bar.
  * weight freshness: after a training rollout and one update by torch's AdamW (default and fused), a `p.data` update
    or bevbert_b200.optim.AdamW, eval-mode calls and a second training rollout match the oracle on the new weights.

The fused-logit semantics for masked candidates are recorded in nav_rollout_cases."""
import pytest
import torch

from bevbert_b200 import synth
from bevbert_b200.config import make_config
from bevbert_b200.model.nav_vilmodel import GlocalTextPathNavCMT
from helpers import grad_errors, small_config
from nav_rollout_cases import ModelCall, OracleCall, errors, make_episode, rollout
from test_nav_rollout_cpu import _update, freshness

pytestmark = pytest.mark.gpu

NOFIX = dict(fix_lang_embedding=False, fix_pano_embedding=False, fix_local_branch=False)

# name: model config overrides, fusion, objects, B, T, D, full depth
CASES = {
    "r2r_fused_b4_t6": dict(fusion="fused", B=4, T=6),
    "reverie_fused_b4_t6": dict(fusion="fused", obj=True, B=4, T=6),
    "r2r_global_nofuse_b1_t1": dict(fusion="global", B=1, T=1, cfg=dict(glocal_fuse=False)),
    "r2r_local_b4_t3": dict(fusion="local", B=4, T=3),
    "reverie_global_nofuse_b4_t3": dict(fusion="global", obj=True, B=4, T=3, cfg=dict(glocal_fuse=False)),
    "fix_lang_b4_t3": dict(fusion="fused", B=4, T=3, cfg=dict(fix_lang_embedding=True)),
    "fix_pano_b4_t3": dict(fusion="fused", B=4, T=3, cfg=dict(fix_pano_embedding=True)),
    "reverie_fix_local_b4_t3": dict(fusion="fused", obj=True, B=4, T=3, cfg=dict(fix_local_branch=True)),
    "d21_b4_t2": dict(fusion="fused", B=4, T=2, D=21),
    "full_d21_b2_t3": dict(fusion="fused", B=2, T=3, D=21, full=True),
}
KINDS = ("txt", "pano", "gmap", "logits", "loss", "grad", "param")
CAP = {"fp32": dict({k: 1e-3 for k in KINDS}, param=5e-3)}

# (floor, bar) per case and arm, for each of KINDS in order (see nav_rollout_cases.errors).  The floors were measured on
# an H100 80GB HBM3 at 700 W with these inputs; each bar is about 3x its floor.  "freshness" is the episode of the
# weight-freshness tests (fp32 arm; worst of the four updates, eval and training).  The negative controls measured
# 2e3 x (detached average) and 1e5 x (dropped step loss) the gradient bar.
BARS = {
    "r2r_fused_b4_t6": {
        "fp32": ((5.76e-07, 1.7e-06), (5.45e-07, 1.6e-06), (6.66e-07, 2e-06), (1.68e-06, 5e-06),
                 (4.37e-08, 1.3e-07), (1.06e-06, 3.2e-06), (2.32e-06, 7e-06)),
        "bf16": ((0.00411, 0.012), (0.00506, 0.015), (0.006, 0.018), (0.0109, 0.033),
                 (0.000329, 0.00099), (0.0582, 0.17), (0.109, 0.33)),
    },
    "reverie_fused_b4_t6": {
        "fp32": ((5.76e-07, 1.7e-06), (5.44e-07, 1.6e-06), (6.64e-07, 2e-06), (1.79e-06, 5.4e-06),
                 (5.05e-08, 1.5e-07), (1.02e-06, 3.1e-06), (2.24e-06, 6.7e-06)),
        "bf16": ((0.00411, 0.012), (0.00505, 0.015), (0.00601, 0.018), (0.0205, 0.061),
                 (0.000278, 0.00083), (0.0571, 0.17), (0.103, 0.31)),
    },
    "r2r_global_nofuse_b1_t1": {
        "fp32": ((5.85e-07, 1.8e-06), (5.34e-07, 1.6e-06), (6.77e-07, 2e-06), (1.9e-06, 5.7e-06),
                 (1.76e-07, 5.3e-07), (9.55e-07, 2.9e-06), (1.89e-06, 5.7e-06)),
        "bf16": ((0.00415, 0.012), (0.00504, 0.015), (0.00594, 0.018), (0.00616, 0.018),
                 (0.000132, 0.0004), (0.0523, 0.16), (0.0826, 0.25)),
    },
    "r2r_local_b4_t3": {
        "fp32": ((5.76e-07, 1.7e-06), (5.44e-07, 1.6e-06), (6.66e-07, 2e-06), (1.68e-06, 5e-06),
                 (7.03e-09, 2.1e-08), (9.76e-07, 2.9e-06), (1.82e-06, 5.5e-06)),
        "bf16": ((0.00411, 0.012), (0.00506, 0.015), (0.006, 0.018), (0.0109, 0.033),
                 (0.000161, 0.00048), (0.0757, 0.23), (0.125, 0.38)),
    },
    "reverie_global_nofuse_b4_t3": {
        "fp32": ((5.76e-07, 1.7e-06), (5.43e-07, 1.6e-06), (6.64e-07, 2e-06), (1.63e-06, 4.9e-06),
                 (8e-08, 2.4e-07), (9.55e-07, 2.9e-06), (1.81e-06, 5.4e-06)),
        "bf16": ((0.00411, 0.012), (0.00502, 0.015), (0.006, 0.018), (0.0205, 0.061),
                 (0.000552, 0.0017), (0.0556, 0.17), (0.112, 0.34)),
    },
    "fix_lang_b4_t3": {
        "fp32": ((5.76e-07, 1.7e-06), (5.44e-07, 1.6e-06), (6.66e-07, 2e-06), (1.68e-06, 5e-06),
                 (5.81e-08, 1.7e-07), (1.03e-06, 3.1e-06), (2.18e-06, 6.5e-06)),
        "bf16": ((0.00411, 0.012), (0.00506, 0.015), (0.006, 0.018), (0.0109, 0.033),
                 (0.000734, 0.0022), (0.0584, 0.18), (0.128, 0.38)),
    },
    "fix_pano_b4_t3": {
        "fp32": ((5.76e-07, 1.7e-06), (5.44e-07, 1.6e-06), (6.66e-07, 2e-06), (1.68e-06, 5e-06),
                 (5.81e-08, 1.7e-07), (1.03e-06, 3.1e-06), (2.18e-06, 6.5e-06)),
        "bf16": ((0.00411, 0.012), (0.00506, 0.015), (0.006, 0.018), (0.0109, 0.033),
                 (0.000734, 0.0022), (0.0594, 0.18), (0.128, 0.38)),
    },
    "reverie_fix_local_b4_t3": {
        "fp32": ((5.76e-07, 1.7e-06), (5.43e-07, 1.6e-06), (6.64e-07, 2e-06), (1.63e-06, 4.9e-06),
                 (1.02e-07, 3.1e-07), (1.03e-06, 3.1e-06), (1.84e-06, 5.5e-06)),
        "bf16": ((0.00411, 0.012), (0.00502, 0.015), (0.006, 0.018), (0.0205, 0.061),
                 (0.000552, 0.0017), (0.065, 0.2), (0.107, 0.32)),
    },
    "d21_b4_t2": {
        "fp32": ((5.76e-07, 1.7e-06), (5.44e-07, 1.6e-06), (6.66e-07, 2e-06), (1.89e-06, 5.7e-06),
                 (6.82e-08, 2e-07), (1.21e-06, 3.6e-06), (2.84e-06, 8.5e-06)),
        "bf16": ((0.00411, 0.012), (0.00502, 0.015), (0.006, 0.018), (0.0118, 0.035),
                 (0.000745, 0.0022), (0.0621, 0.19), (0.111, 0.33)),
    },
    "full_d21_b2_t3": {
        "fp32": ((1.17e-06, 3.5e-06), (6.52e-07, 2e-06), (9.01e-07, 2.7e-06), (3.61e-06, 1.1e-05),
                 (1.81e-07, 5.4e-07), (1.38e-06, 4.1e-06), (5.06e-06, 1.5e-05)),
        "bf16": ((0.00797, 0.024), (0.00562, 0.017), (0.00739, 0.022), (0.0175, 0.053),
                 (0.00127, 0.0038), (0.0756, 0.23), (0.143, 0.43)),
    },
    "freshness": {
        "fp32": ((6.28e-07, 1.9e-06), (5.06e-07, 1.5e-06), (5.78e-07, 1.7e-06), (8.6e-06, 2.6e-05),
                 (1.84e-06, 5.5e-06), (2.6e-06, 7.8e-06), (5.99e-06, 1.8e-05)),
    },
}


def _cfg(c):
    kw = dict(NOFIX, **c.get("cfg", {}))
    if c.get("obj"):
        kw["obj_feat_size"] = 768
    D = c.get("D", 11)
    if c.get("full"):
        return make_config(bev_dim=D, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, feat_dropout=0.0, **kw)
    return small_config(bev_dim=D, **kw)


def _model(cfg):
    return synth.det_init_(GlocalTextPathNavCMT(cfg), seed=4)


_REF = {}


def _case(name):
    c = CASES[name]
    cfg = _cfg(c)
    ep = make_episode(c["B"], c["T"], c.get("D", 11), seed=2, obj=c.get("obj", False))
    if name not in _REF:
        _REF[name] = rollout(OracleCall(_model(cfg), cfg), ep, c["fusion"])
    return c, cfg, ep, _REF[name]


def _run_model(cfg, ep, fusion, arm, **kw):
    from bevbert_b200 import kernels as K
    prev = K.set_precision(arm == "fp32")
    try:
        model = _model(cfg).cuda().train()
        got = rollout(ModelCall(model, "cuda"), ep, fusion, **kw)
        torch.cuda.synchronize()
    finally:
        K.set_precision(prev)
    return got


def _report(name, arm, e, extra=""):
    print("%s/%s: %s worst param %s%s" % (name, arm, " ".join("%s %.3g" % (k, e[k]) for k in KINDS), e["param_name"],
                                         extra))


def _bars(name, arm):
    bars = {k: fb[1] for k, fb in zip(KINDS, BARS[name][arm])}
    for k, cap in CAP.get(arm, {}).items():
        assert bars[k] <= cap, (name, arm, k)
    return bars


def _assert_within(e, bars):
    bad = {k: (e[k], bars[k]) for k in KINDS if not e[k] <= bars[k]}
    assert not bad, (bad, e["param_name"])


@pytest.mark.parametrize("name", list(CASES))
def test_rollout_fp32_arm_matches_fp64(name):
    c, cfg, ep, ref = _case(name)
    e = errors(_run_model(cfg, ep, c["fusion"], "fp32"), ref, ep)
    _report(name, "fp32", e)
    _assert_within(e, _bars(name, "fp32"))


@pytest.mark.parametrize("name", list(CASES))
def test_rollout_bf16_matches_fp64(name):
    c, cfg, ep, ref = _case(name)
    got = _run_model(cfg, ep, c["fusion"], "bf16")
    e = errors(got, ref, ep)
    ac = rollout(OracleCall(_model(cfg), cfg, dtype=torch.float32, autocast=True), ep, c["fusion"])
    e_ac = errors(ac, ref, ep)
    names = list(got["grads"])
    errs, _ = grad_errors(got["grads"], {n: ref["grads"].get(n) for n in names})
    errs_ac, _ = grad_errors({n: ac["grads"].get(n) for n in names}, {n: ref["grads"].get(n) for n in names})
    _report(name, "bf16", e, " | autocast grad %.3g param %.3g loss %.3g" % (e_ac["grad"], e_ac["param"], e_ac["loss"]))
    bars = _bars(name, "bf16")
    _assert_within({k: v for k, v in e.items() if k != "param"} | {"param": 0.0}, bars)
    assert e["grad"] <= max(1e-2, 2.5 * e_ac["grad"]), (e["grad"], e_ac["grad"])
    bad = {n: (x, errs_ac[n]) for n, x in errs.items() if x > max(bars["param"], 3.0 * errs_ac[n])}
    assert not bad, bad


@pytest.mark.parametrize("control", ["detach_avg_step", "drop_loss_step"])
def test_negative_controls_are_seen(control):
    """The model's rollout broken at step 2 (index 1) only: a detached panorama average, or a missing step loss."""
    name = "r2r_fused_b4_t6"
    c, cfg, ep, ref = _case(name)
    e = errors(_run_model(cfg, ep, c["fusion"], "fp32", **{control: 1}), ref, ep)
    bars = _bars(name, "fp32")
    _report(name, "fp32 " + control, e, " | x bar: grad %.3g param %.3g" % (e["grad"] / bars["grad"],
                                                                             e["param"] / bars["param"]))
    assert max(e["grad"] / bars["grad"], e["param"] / bars["param"]) >= 5.0


def _update_gpu(kind, model):
    if kind == "bevbert":
        from bevbert_b200.optim import AdamW
        AdamW([p for p in model.parameters() if p.grad is not None], lr=1e-2, runtime=model.rt).step()
    else:
        _update(kind, model)


@pytest.mark.parametrize("kind", ["default", "fused", "pdata", "bevbert"])
def test_eval_after_optimizer_step_uses_new_weights(kind):
    from bevbert_b200 import kernels as K
    cfg = _cfg({})
    prev = K.set_precision(True)
    try:
        model = _model(cfg).cuda()
        bars = _bars("freshness", "fp32")
        e_eval, e_train = freshness(kind, model, cfg, ModelCall(model, "cuda"), update=_update_gpu, bar=None)
    finally:
        K.set_precision(prev)
    _report("freshness " + kind, "fp32", e_train, " | eval " + " ".join("%s %.3g" % (k, e_eval[k]) for k in KINDS[:4]))
    _assert_within({k: e_eval.get(k, 0.0) for k in KINDS} | {"param_name": ""}, bars)
    _assert_within(e_train, bars)
