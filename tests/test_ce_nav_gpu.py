"""The VLN-CE navigation network (model/ce_nav.py) on the H100 against its oracle (oracle/ce_nav_ref.py, pinned to the
unmodified CE reference by tests/golden/small_ce_nav.pt): a teacher-forced rollout of the three calls on the fp32
verification arm and on the bf16 path, bit-identical results with autocast on and off, the GradScaler step, graph
replay of the installed calls (tests/test_ce_nav_graphs_gpu.py has the bucket cases), and the trainer-side BEV adapter.

`python tests/test_ce_nav_gpu.py det` runs the deterministic-mode cases directly (they need CUBLAS_WORKSPACE_CONFIG
before CUDA initialises, so the test runs them in a fresh interpreter)."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [p for p in (ROOT, os.path.join(ROOT, "tests")) if p not in sys.path]

import ce_nav_bev_cases as BC  # noqa: E402
import ce_nav_bev_oracle as BO  # noqa: E402
import ce_nav_cases as C  # noqa: E402
from bevbert_b200 import kernels as K  # noqa: E402
from bevbert_b200 import synth  # noqa: E402
from bevbert_b200.model.ce_nav import GlocalTextPathNavCMT  # noqa: E402
from helpers import grad_errors, grad_report  # noqa: E402
from oracle import ce_nav_ref as O  # noqa: E402

LOGIT_BAR, SAP_GRAD_BAR = 1e-2, 1.3e-1      # the bf16 bars of tests/test_ce_model_gpu.py (logits; SAP global gradient)
KEYS = ("gmap_embeds", "global_logits", "local_logits", "fused_logits")


def _cuda(x):
    return x.cuda() if torch.is_tensor(x) else x


def _model(variant=(True, True), fp32=False, seed=C.WEIGHT_SEED):
    prev = K.set_precision(fp32)
    try:
        return synth.det_init_(GlocalTextPathNavCMT(C.config(*variant)), seed=seed).cuda()
    finally:
        K.set_precision(prev)


def _model_rollout(model, B, fp32=False, autocast=False, steps=C.STEPS):
    prev = K.set_precision(fp32)
    try:
        model.zero_grad(set_to_none=True)
        with torch.autocast("cuda", enabled=autocast):
            loss, outs = C.rollout(model, B, steps=steps, prep=_cuda)
        loss.backward()
        torch.cuda.synchronize()
    finally:
        K.set_precision(prev)
    # clones: parameter gradients may live in the per-step arena the next rollout reuses
    return loss.detach(), outs, {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}


def _oracle_rollout(model, B, dtype=torch.float64, autocast=False):
    train = {n for n, p in model.named_parameters() if p.requires_grad}
    sd = {k: (v.detach().cpu().to(dtype).clone().requires_grad_(k in train) if v.is_floating_point() else v.detach().cpu())
          for k, v in model.state_dict().items()}
    prep = lambda x: x.to(dtype) if torch.is_tensor(x) and x.is_floating_point() else x
    if autocast:
        with torch.autocast("cpu", dtype=torch.bfloat16):
            loss, outs = C.rollout(O.GlocalTextPathNavCMT(sd, O.OracleConfig(model.config)), B, prep=prep)
    else:
        loss, outs = C.rollout(O.GlocalTextPathNavCMT(sd, O.OracleConfig(model.config)), B, prep=prep)
    loss.backward()
    return loss.detach(), outs, {n: v.grad for n, v in sd.items() if v.grad is not None}


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def _out_errors(outs, routs):
    """worst relative L2 error of the text, panorama (valid tokens) and navigation outputs (finite entries) over the
    steps; finite patterns and panorama masks must agree"""
    e = {"txt": _rel(outs[0]["txt"], routs[0]["txt"]), "pano": 0.0, "nav": 0.0}
    for o, r in zip(outs, routs):
        pm = r["pano"][1]
        assert torch.equal(o["pano"][1].cpu(), pm)
        e["pano"] = max(e["pano"], _rel(o["pano"][0].cpu()[pm], r["pano"][0][pm]))
        for k in KEYS:
            a, b = o["nav"][k].detach().cpu(), r["nav"][k].detach()
            fin = torch.isfinite(b)
            assert torch.equal(torch.isfinite(a), fin), k
            e["nav"] = max(e["nav"], _rel(a[fin], b[fin]))
    return e


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 4, 8])
@pytest.mark.parametrize("variant", C.VARIANTS)
def test_fp32_arm_matches_oracle(variant, B):
    model = _model(variant, fp32=True).train()
    loss, outs, grads = _model_rollout(model, B, fp32=True)
    rloss, routs, rgrads = _oracle_rollout(model, B)
    e = _out_errors(outs, routs)
    worst, name = grad_report(grads, rgrads)
    print("fp32 arm", variant, "B", B, e, "loss %.2e" % _rel(loss.reshape(1), rloss.reshape(1)), "grad %.2e" % worst, name)
    assert max(e.values()) < 1e-3
    assert _rel(loss.reshape(1), rloss.reshape(1)) < 1e-3
    assert set(grads) == set(rgrads) and worst < 1e-3, (name, worst)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", C.VARIANTS)
def test_bf16_within_bars(variant):
    B = 4
    model = _model(variant).train()
    loss, outs, grads = _model_rollout(model, B)
    rloss, routs, rgrads = _oracle_rollout(model, B)
    _, aouts, agrads = _oracle_rollout(model, B, dtype=torch.float32, autocast=True)
    e, ea = _out_errors(outs, routs), _out_errors(aouts, routs)
    _, g = grad_errors(grads, rgrads)
    _, ga = grad_errors(agrads, rgrads)
    print("bf16", variant, e, "autocast", ea, "global grad %.3g (autocast %.3g)" % (g, ga))
    for k in e:
        assert e[k] <= max(LOGIT_BAR, 2.5 * ea[k]), k
    assert g <= SAP_GRAD_BAR and g <= 2.5 * ga


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [(True, True), (False, False)])
def test_autocast_on_and_off_bit_identical(variant):
    """outputs and loss; the gradients are compared in deterministic mode (test_deterministic_cases), where repeated
    backward passes are bit-identical to begin with"""
    model = _model(variant).train()
    loss, outs, _ = _model_rollout(model, 4)
    aloss, aouts, _ = _model_rollout(model, 4, autocast=True)
    assert torch.equal(loss, aloss)
    for o, a in zip(outs, aouts):
        assert torch.equal(o["txt"], a["txt"]) and torch.equal(o["pano"][0], a["pano"][0])
        for k in KEYS:
            assert o["nav"][k].dtype == torch.float32 and torch.equal(o["nav"][k], a["nav"][k]), k


@pytest.mark.gpu
def test_forward_mode_batch_raises():
    with pytest.raises(NotImplementedError):
        _model()("navigation", {})


# ------------------------------------------------------------------------------------------------------------- BEV
@pytest.mark.gpu
@pytest.mark.parametrize("feat_dtype", [torch.float32, torch.bfloat16])
def test_bev_adapter_matches_oracle_bit_for_bit(feat_dtype):
    from bevbert_b200.agent_bev import ce_nav_bev_variable
    n = 0
    for tr, vp, pos, ori in BC.episode(B=3, steps=6, device="cuda", feat_dtype=feat_dtype):
        got = ce_nav_bev_variable(tr, vp, pos, ori)
        ref = BO.ce_nav_bev_variable(tr.gmaps, vp, pos, ori, [BC.heading_from_quaternion(o) for o in ori], BC.D,
                                     BC.RES, tr._discretize_polar_relpos, tr.bev_pos)
        for k in ("bev_fts", "bev_pos_fts", "bev_masks", "bev_nav_masks", "bev_cand_idxs"):
            assert torch.equal(got[k].cpu(), ref[k]), k
        assert got["bev_fts"].is_cuda and got["bev_cand_vpids"] == ref["bev_cand_vpids"]
        n += int((ref["bev_fts"].abs().sum(-1) == 0).sum())
    assert n > 0          # cells without a point (outside, above the clip, no depth) are zero on both sides


# ------------------------------------------------------------------------------------------------ deterministic mode
@pytest.mark.gpu
def test_deterministic_cases():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] +
                                        ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, "-s", os.path.abspath(__file__), "det"], env=env, capture_output=True,
                       text=True, timeout=1800)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stderr[-6000:]


def _det_cases():
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    # a GradScaler step (power-of-two scale, nothing overflows) updates the parameters exactly as an unscaled step
    params = []
    for scaled in (False, True):
        model = _model().train()
        opt = torch.optim.AdamW(model.parameters(), lr=1e-4)
        scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12)
        for _ in range(2):
            opt.zero_grad(set_to_none=True)
            with torch.autocast("cuda"):
                loss, _ = C.rollout(model, 4, prep=_cuda)
            if scaled:
                scaler.scale(loss).backward()
                scaler.step(opt)
                scaler.update()
            else:
                loss.backward()
                opt.step()
        params.append([p.detach().clone() for p in model.parameters()])
        if scaled:
            assert scaler.get_scale() == 2.0 ** 12      # no step was skipped
    assert all(torch.equal(a, b) for a, b in zip(*params)), "GradScaler step differs from the unscaled step"
    # deterministic rollouts, autocast off and on: identical gradients
    for variant in ((True, True), (False, False)):
        model = _model(variant).train()
        g1 = _model_rollout(model, 4)[2]
        g2 = _model_rollout(model, 4, autocast=True)[2]
        assert set(g1) == set(g2) and all(torch.equal(g1[n], g2[n]) for n in g1), variant
    # replays of the installed calls are bit-identical
    from bevbert_b200.graphs import install_ce_replay
    model = _model().eval()
    replay = install_ce_replay(model)
    with torch.no_grad():
        runs = [C.rollout(model, 4, prep=_cuda)[1] for _ in range(3)]
    assert all(k[1] for k in replay.entries) and not any(e["failed"] for e in replay.entries.values())
    for r in runs[2:]:
        for a, b in zip(r, runs[1]):
            assert torch.equal(a["txt"], b["txt"]) and torch.equal(a["pano"][0], b["pano"][0])
            assert all(torch.equal(a["nav"][k], b["nav"][k]) for k in KEYS)
    print("deterministic: GradScaler step exact, gradients with autocast on and off and replays bit-identical")


if __name__ == "__main__":
    if sys.argv[1:] == ["det"]:
        _det_cases()
