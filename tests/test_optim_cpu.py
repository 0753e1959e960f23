"""oracle/adamw_ref.py (the checker of the CUDA optimizer kernel) is pinned to the UNMODIFIED reference optimizer
(pretrain_src/optim/adamw.py) + torch's clip_grad_norm_ on CPU -- their results on the steps below are stored in
tests/golden/reference_pins.pt; the kernel itself is tested in tests/test_optim_gpu.py against that restatement."""
import importlib.util
import os

import pytest
import torch

from oracle import adamw_ref, ref_shim


def _ref_adamw():
    path = os.path.join(ref_shim.REF_ROOT, "pretrain_src", "optim", "adamw.py")
    spec = importlib.util.spec_from_file_location("_ref_adamw", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.AdamW


def _params(seed=1):
    g = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=g)) for s in ((7, 5), (11,), (3, 3), (130, 9))]


def test_oracle_adamw_matches_reference_optimizer():
    pin = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins.pt"),
                     weights_only=False)["adamw"]
    b = _params()
    wds = [0.01, 0.0, 0.01, 0.01]
    mine = adamw_ref.AdamWRef([p.data for p in b], lr=3e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=wds)
    g = torch.Generator().manual_seed(2)
    for step in range(9):
        grads = [torch.randn(p.shape, generator=g) * (10.0 if step == 4 else 1.0) for p in b]
        skip = step % 4                                   # one parameter without a gradient per step
        mg = [None if i == skip else grads[i].clone() for i in range(len(b))]
        n_ref = pin["clip_norms"][step]
        n_mine = adamw_ref.clip_grad_norm_([x for x in mg if x is not None], 5.0)
        assert abs(float(n_ref) - float(n_mine)) <= 1e-5 * float(n_ref)
        mine.step(mg)
    for pa, pb in zip(pin["params"], b):
        assert torch.allclose(pa.detach(), pb.detach(), rtol=1e-6, atol=1e-7)


def test_param_groups_follow_reference_no_decay_rule():
    from bevbert_b200.optim import build_param_groups
    m = torch.nn.Module()
    m.dense = torch.nn.Linear(4, 4)
    m.LayerNorm = torch.nn.LayerNorm(4)
    groups = build_param_groups(m, 0.01)
    assert [tuple(p.shape) for p in groups[0]["params"]] == [(4, 4)] and groups[0]["weight_decay"] == 0.01
    assert len(groups[1]["params"]) == 3 and groups[1]["weight_decay"] == 0.0
