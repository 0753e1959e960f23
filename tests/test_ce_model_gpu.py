"""The VLN-CE pre-training model (model/ce_pretrain.py) on the H100 against its fp32 oracle (oracle/ce_ref.py, pinned to
the unmodified CE reference by tests/golden/small_ce.pt): BEV tensors bit-exact, the fp32 verification arm within 1e-3,
the bf16 path within the bars of tests/test_model_gpu.py, compute_loss=False logits, CUDA-graph replay, deterministic
mode, and the tasks the CE reference cannot run."""
import pytest
import torch

import ce_cases as C
from bevbert_b200 import kernels as K
from bevbert_b200 import synth
from bevbert_b200.config import make_ce_config
from bevbert_b200.model.ce_pretrain import GlocalTextPathCMTPreTraining
from helpers import grad_errors, rel_l2
from oracle import bevbert_ref as R
from oracle import ce_ref as CR

pytestmark = pytest.mark.gpu

GLOBAL_GRAD_BAR = {"mlm": 3e-2, "sap": 1.3e-1}       # the per-task bars of tests/test_model_gpu.py


def _case():
    return make_ce_config(small=True), synth.ce_synth_config(batch_size=2, pano_min=4, pano_max=6, gmap_min=8, gmap_max=8)


def _oracle(sd, b, task, cfg, autocast=False):
    for v in sd.values():
        v.grad = None
    if autocast:
        with torch.autocast("cpu", dtype=torch.bfloat16):
            out = CR.forward(sd, synth.clone_batch(b), task, CR.OracleConfig(cfg))
    else:
        out = CR.forward(sd, synth.clone_batch(b), task, CR.OracleConfig(cfg))
    out.float().mean().backward()
    return out.detach().float(), {n: v.grad.clone() for n, v in sd.items() if v.grad is not None}


def _model_step(cfg, b, task, fp32):
    prev = K.set_precision(fp32)
    try:
        model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).cuda().train()
        out = model(synth.batch_to(b, "cuda"), task, compute_loss=True)
        out.mean().backward()
        torch.cuda.synchronize()
    finally:
        K.set_precision(prev)
    return model, out


def test_bev_cells_and_features_bit_exact():
    cfg, scfg = _case()
    model = GlocalTextPathCMTPreTraining(cfg).cuda().eval()
    b = synth.make_batch(scfg, seed=11, task="sap")
    bb = model.lift_splat(dict(synth.batch_to(b, "cuda")))
    rb = CR.lift_splat(dict(synth.clone_batch(b)))
    for k in ("bev_cell_idx", "bev_fts", "bev_pos_fts", "bev_masks"):
        assert torch.equal(bb[k].cpu().to(rb[k].dtype), rb[k]), k
    assert "bev_sems" not in bb
    # known-answer points: round-half-even boundaries at +-0.5 m / +-1.5 m, the height clip, cells 0 / 60 / 120
    pts, nod, want = C.lift_kat_points()
    got = K.bev_cell_index(pts.cuda(), nod.cuda(), C.D_CE, C.RES_CE)
    assert torch.equal(got.cpu().long()[0], want)
    # scatter-mean over 121 cells: 15 full blocks of 8 cells and a partial last block holding cell 120 alone
    g = torch.Generator().manual_seed(4)
    cells = torch.cat([torch.arange(121), torch.randint(100, 121, (300,), generator=g), torch.full((40,), -1)])
    cells = cells[torch.randperm(cells.numel(), generator=g)].to(torch.int32)[None]
    feats = torch.randn(1, cells.shape[1], 768, generator=g)
    o32, _, ob, cnt = K.bev_scatter_mean(feats.cuda(), cells.cuda(), 121, True, False)
    want = R.scatter_mean(feats[0], cells[0].long(), 121)
    assert torch.equal(o32.cpu()[0], want)
    assert torch.equal(cnt.cpu()[0].long(), torch.bincount(cells[0][cells[0] >= 0].long(), minlength=121))


@pytest.mark.parametrize("task", ["mlm", "sap"])
def test_fp32_verification_arm_holds_1e3(task):
    cfg, scfg = _case()
    b = synth.make_batch(scfg, seed=7, task=task)
    model, out = _model_step(cfg, b, task, fp32=True)
    sd = {k: v.detach().float().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    ref, rg = _oracle(sd, b, task, cfg)
    names = [n for n, _ in model.named_parameters()]
    errs, glob = grad_errors({n: p.grad for n, p in model.named_parameters()}, {n: rg.get(n) for n in names})
    le = rel_l2(out, ref)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:3]
    print("CE fp32 arm task=%s loss rel-L2 %.3e | all-grads rel-L2 %.3e | worst %s" % (task, le, glob, worst))
    assert le < 1e-3 and glob < 1e-3, (le, glob)
    assert all(e < 1e-3 for e in errs.values()), worst


@pytest.mark.parametrize("task", ["mlm", "sap"])
def test_bf16_path_matches_oracle(task):
    cfg, scfg = _case()
    b = synth.make_batch(scfg, seed=7, task=task)
    model, out = _model_step(cfg, b, task, fp32=False)
    sd = {k: v.detach().float().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    ref, rg = _oracle(sd, b, task, cfg)
    ac, ag = _oracle(sd, b, task, cfg, autocast=True)
    names = [n for n, _ in model.named_parameters()]
    errs, glob = grad_errors({n: p.grad for n, p in model.named_parameters()}, {n: rg.get(n) for n in names})
    errs_ac, glob_ac = grad_errors({n: ag.get(n) for n in names}, {n: rg.get(n) for n in names})
    le = rel_l2(out, ref)
    print("CE bf16 task=%s loss rel-L2 %.3e (autocast %.3e) | all-grads rel-L2 %.3e (autocast %.3e)" % (
        task, le, rel_l2(ac, ref), glob, glob_ac))
    bar = GLOBAL_GRAD_BAR[task]
    assert le < 1e-2, le
    assert glob < bar and glob < max(1e-2, 2.5 * glob_ac), (glob, glob_ac)
    bad = {n: (e, errs_ac[n]) for n, e in errs.items() if e > max(2 * bar, 3.0 * errs_ac[n])}
    assert not bad, bad
    # compute_loss=False: the logits against the oracle's, within 1e-2 or, for the ill-conditioned SAP heads, within
    # 2.5x the error of PyTorch's bf16 autocast of the oracle on the same inputs (the gradient rule above)
    sd0 = {k: v.detach() for k, v in sd.items()}
    with torch.no_grad():
        mine = model(synth.batch_to(b, "cuda"), task, compute_loss=False)
        theirs = CR.forward(sd0, synth.clone_batch(b), task, CR.OracleConfig(cfg), compute_loss=False)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            auto = CR.forward(sd0, synth.clone_batch(b), task, CR.OracleConfig(cfg), compute_loss=False)
    tup = lambda x: x if isinstance(x, tuple) else (x,)
    mine, theirs, auto = tup(mine), tup(theirs), tup(auto)
    for a, r, ac in zip(mine[:3], theirs[:3], auto[:3]):
        fin = torch.isfinite(r)
        assert torch.equal(torch.isfinite(a.cpu()), fin)
        e, e_ac = rel_l2(a.cpu()[fin], r[fin]), rel_l2(ac.float()[fin], r[fin])
        print("    logits rel-L2 %.3e (autocast %.3e)" % (e, e_ac))
        assert e < max(1e-2, 2.5 * e_ac), (e, e_ac)
    for a, r in zip(mine[3:], theirs[3:]):
        assert torch.equal(a.cpu(), r)


def _train(graphed, lr, seq):
    from bevbert_b200.graphs import GraphedTrainStep
    from bevbert_b200.model.ops import prepare_batch
    from bevbert_b200.optim import AdamW, build_param_groups
    from bevbert_b200.parallel import direct_param_grads
    cfg, scfg = _case()
    batches = {t: synth.batch_to(prepare_batch(synth.make_batch(scfg, seed=40 + i, task=t), wire_dtype=torch.bfloat16),
                                 "cuda") for i, t in enumerate(["mlm", "sap"])}
    direct_param_grads(True)
    try:
        model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).cuda().train()
        opt = AdamW(build_param_groups(model, 0.01), lr=lr, betas=(0.9, 0.98), max_grad_norm=5.0, runtime=model.rt)
        if graphed:
            step = GraphedTrainStep(model, opt, warmup=1)
            losses = [float(step(batches[t], t)) for t in seq]
            assert step.launches(batches["mlm"], "mlm") and step.launches(batches["sap"], "sap")
        else:
            losses = []
            for t in seq:
                loss = model(batches[t], t).mean()
                loss.backward()
                opt.step()
                losses.append(float(loss.detach()))
        grads = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    finally:
        direct_param_grads(False)
    return losses, grads


def test_graph_replay_at_lr0_equals_eager_in_deterministic_mode():
    seq = ["mlm", "sap", "mlm", "sap", "mlm", "sap"]
    torch.use_deterministic_algorithms(True)
    try:
        e, _ = _train(False, 0.0, seq)
        g, _ = _train(True, 0.0, seq)
    finally:
        torch.use_deterministic_algorithms(False)
    print("CE lr=0 eager  ", e)
    print("CE lr=0 graphed", g)
    assert e == g


def test_deterministic_mode_gives_bit_identical_training_steps():
    seq = ["mlm", "sap", "mlm", "sap"]
    torch.use_deterministic_algorithms(True)
    try:
        l1, g1 = _train(False, 1e-4, seq)
        l2, g2 = _train(False, 1e-4, seq)
    finally:
        torch.use_deterministic_algorithms(False)
    assert l1 == l2
    assert set(g1) == set(g2) and all(torch.equal(g1[n], g2[n]) for n in g1)


@pytest.mark.parametrize("task", ["mrc", "og", "sem"])
def test_unrunnable_tasks_raise(task):
    cfg, scfg = _case()
    model = GlocalTextPathCMTPreTraining(cfg).cuda()
    with pytest.raises(ValueError):
        model(synth.batch_to(synth.make_batch(scfg, seed=1, task="sap"), "cuda"), task)
