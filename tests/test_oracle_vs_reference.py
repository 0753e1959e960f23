"""Pins the oracle to the real reference: the unmodified reference modules (imported through oracle/ref_shim.py) were
run on the same weights and batches as the restatement, and what they returned is stored in
tests/golden/reference_pins.pt (tests/golden/make_golden.py regenerates it)."""
import os

import pytest
import torch

from bevbert_b200 import synth
from bevbert_b200.model.pretrain_cmt import GlocalTextPathCMTPreTraining
from helpers import small_config, small_synth
from oracle import bevbert_ref as R
from oracle import ref_shim

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins.pt")


def pins():
    return torch.load(PINS, weights_only=False)


def check_rows(x, pin, rtol=0.0, atol=0.0):
    """x against a pinned sample of rows and the float64 sums of the whole tensor."""
    x2 = x.reshape(-1, x.shape[-1])
    assert torch.allclose(x2[pin["idx"]], pin["rows"], rtol=rtol, atol=atol), float((x2[pin["idx"]] - pin["rows"]).abs().max())
    tol = max(rtol, 1e-12) * pin["abs_sum"] + atol * x2.numel()
    assert abs(float(x2.double().sum()) - pin["sum"]) <= tol and abs(float(x2.double().abs().sum()) - pin["abs_sum"]) <= tol


def _ref_model(cfg, sd):
    ref = ref_shim.build_reference_model(cfg, sd).train()
    for m in ref.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
        if isinstance(m, torch.nn.MultiheadAttention):
            m.dropout = 0.0
    return ref


@pytest.mark.parametrize("task", ["mlm", "sap", "masksem"])
def test_restatement_equals_reference(task):
    cfg, scfg = small_config(), small_synth(ragged_txt=True)
    sd = {k: v.detach().clone() for k, v in synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=5).state_dict().items()}
    b = synth.make_batch(scfg, seed=21, task=task)
    want = pins()["restatement"][task]
    got = R.forward(sd, synth.clone_batch(b), task, R.OracleConfig(cfg))
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-6), float((got - want).abs().max())


@pytest.mark.parametrize("case", ["longest_trajectory", "empty_bev"])
def test_restatement_equals_reference_on_edge_cases(case):
    """SURVEY section 4 property cases, pinned on the unmodified reference: 21 panoramas per trajectory (TRAIN_MAX_STEP + 1,
    dataset.py:185-187) and depth maps that are all zero (every point dropped, all BEV cells empty)."""
    cfg = small_config()
    scfg = small_synth(pano_min=21, pano_max=21) if case == "longest_trajectory" else small_synth(depth_zero_frac=1.0)
    sd = {k: v.detach().clone() for k, v in synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=5).state_dict().items()}
    pin = pins()["edge"]
    for task in ("sap", "mlm"):
        b = synth.make_batch(scfg, seed=23, task=task)
        want = pin[case + "/" + task]
        got = R.forward(sd, synth.clone_batch(b), task, R.OracleConfig(cfg))
        assert torch.isfinite(want).all()
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-6), (task, float((got - want).abs().max()))


def test_bev_projection_matches_reference_bit_for_bit():
    """lift + project_bev of the reference (torch bmm / matmul + scatter_mean stub) vs the fixed-order oracle:
    cell indices, pooled features, semantic maps and masks."""
    mismatched = 0
    total = 0
    for seed, pin in zip((1, 2, 3), pins()["bev"]):
        b = synth.make_batch(synth.SynthConfig(batch_size=4), seed=seed)
        bs = 4
        ob_ = dict(b)
        R.lift_splat(ob_, 21, 0.5)
        # the reference leaves the order of the 4-term dot products to bmm/matmul; count index flips instead of failing
        ref_idx = pin["cell_idx"].to(ob_["bev_cell_idx"].dtype)
        mismatched += int((ref_idx != ob_["bev_cell_idx"]).sum())
        total += ref_idx.numel()
        if torch.equal(ref_idx, ob_["bev_cell_idx"]):
            check_rows(ob_["bev_fts"], pin["bev"])
            check_rows(ob_["bev_sems"], pin["sems"])
            assert torch.equal(ob_["bev_sem_masks"], pin["sem_masks"])
            assert torch.equal(ob_["bev_ob_masks"], pin["ob_masks"])
    assert mismatched <= total * 1e-5, "cell-index disagreement with the reference: %d of %d" % (mismatched, total)
