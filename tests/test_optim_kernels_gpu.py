"""bb_mt_sumsq, bb_adamw_step and bb_mt_cast_bf16 (csrc/optim.cu) element by element on launch tables built directly
with K.MtTable over one arena per field, with sentinel-filled guard gaps between tensors: sizes around the 4096-element
chunk, zero-size entries first / in the middle / last, about 600 tensors (the binary search over chunk0), every pointer
aligned (vector path) or one field offset by one element (scalar path).  m, v and p against fp64 with the bounds of
tests/rowops_cases.py; p16 and g bit for bit.  Also: AdamW.step() returns the pre-clip total norm."""
import math

import pytest
import torch

import rowops_cases as R
from oracle import adamw_ref

pytestmark = pytest.mark.gpu
BF, F32 = R.BF, R.F32
B1, B2, EPS = 0.9, 0.98, 1e-6


@pytest.fixture(scope="module")
def K():
    from bevbert_b200 import kernels as K
    assert torch.cuda.is_available()
    prev = K.set_precision(False)
    yield K
    K.set_precision(prev)
    print("\nerr / bound, optimizer:")
    for k in sorted(R.RATIOS):
        print("  %-28s %.3f" % (k, R.RATIOS[k]))


def _table(K, T, steps, decays, with_p16=True):
    return K.MtTable(T.rows(steps, decays, with_p16), "cuda")


def _sumsq(K, T, tab):
    out = torch.full((1,), float("nan"), device="cuda")
    K.mt_sumsq(tab, out)
    torch.cuda.synchronize()
    ref, d = R.sumsq_ref(T.views["g"], T.chunks)
    R.check("sumsq", out.cpu(), torch.tensor([ref], dtype=torch.float64), torch.tensor([d], dtype=torch.float64))
    return out


def _check_step(T, before, coef, clipped, steps, decays, with_p16=True):
    for i, n in enumerate(T.sizes):
        if n == 0:
            continue
        ref = R.adam_ref(before["p"][i], before["g"][i], before["m"][i], before["v"][i], B1, B2, EPS, coef, clipped,
                         steps[i], decays[i])
        R.check("adamw.m[%d]" % i, T.views["m"][i], ref["m"], ref["d_m"])
        R.check("adamw.v[%d]" % i, T.views["v"][i], ref["v"], ref["d_v"])
        R.check("adamw.p[%d]" % i, T.views["p"][i], ref["p"], ref["d_p"])
        R.check_exact("adamw.g[%d] unchanged" % i, T.views["g"][i], before["g"][i])
        if with_p16:
            R.check_exact("adamw.p16[%d]" % i, T.views["p16"][i], T.views["p"][i].to(BF))
    T.check_gaps("pgmv")
    T._gaps("p16")


OFFSETS = [{}, {"p": 1}, {"g": 1}, {"m": 1}, {"v": 1}, {"p16": 1}]
CLIP = [("active", 1.0, 1.0), ("inactive", 1e6, 1.0), ("max_norm0", 0.0, 1.0), ("no_sumsq", 1.0, 1.0),
        ("active", 0.5, 2.0 ** -8), ("inactive", 1e6, 2.0 ** -8)]


@pytest.mark.parametrize("kind", ["edges", "many"])
@pytest.mark.parametrize("off", OFFSETS, ids=lambda o: "aligned" if not o else "offset_" + next(iter(o)))
def test_sumsq_adamw_cast(K, kind, off):
    if kind == "many" and off not in ({}, {"g": 1}):
        pytest.skip("the deep table runs aligned and with one offset field")
    T = R.OptTable(R.opt_sizes(kind), "cuda", offset=off, seed=len(off))
    t = [0] * len(T.sizes)
    for k, (clip, max_norm, gsc) in enumerate(CLIP):
        # several consecutive steps, step sizes as optim.AdamW._fill computes them (per-tensor counters)
        lr = 1e-3
        steps, decays = [], []
        for i in range(len(T.sizes)):
            t[i] += 1
            steps.append(lr * math.sqrt(1.0 - B2 ** t[i]) / (1.0 - B1 ** t[i]))
            decays.append(lr * 50.0 if i % 2 else 0.0)          # lr * wd = 0.05: decay before / after differ
        tab = _table(K, T, steps, decays)
        s = _sumsq(K, T, tab)
        before = T.snapshot()
        use = None if clip == "no_sumsq" else s
        K.adamw_step(tab, B1, B2, EPS, use, max_norm, gsc)
        torch.cuda.synchronize()
        coef, clipped = R.clip_coef(None if use is None else s.cpu()[0], max_norm, gsc)
        if clip == "active":
            assert clipped
        _check_step(T, before, coef, clipped, steps, decays)
        # the shadow refresh: scribble p16, re-cast
        for v in T.views["p16"]:
            v.fill_(-1.0)
        K.mt_cast_bf16(tab)
        torch.cuda.synchronize()
        for i, v in enumerate(T.views["p16"]):
            R.check_exact("mt_cast_bf16[%d]" % i, v, T.views["p"][i].to(BF))
        T._gaps("p16")


def test_adamw_clip_epsilon_at_tiny_norm(K):
    """total norm about 1e-6: the clip's 1e-6 roughly halves the coefficient"""
    T = R.OptTable(R.opt_sizes("edges"), "cuda", scale=6.4e-9)
    steps, decays = [1e-2] * len(T.sizes), [0.05] * len(T.sizes)
    tab = _table(K, T, steps, decays, with_p16=False)
    s = _sumsq(K, T, tab)
    coef, clipped = R.clip_coef(s.cpu()[0], 1e-6, 1.0)
    assert clipped and 0.3 < coef < 0.7
    before = T.snapshot()
    K.adamw_step(tab, B1, B2, EPS, s, 1e-6, 1.0)
    torch.cuda.synchronize()
    _check_step(T, before, coef, clipped, steps, decays, with_p16=False)
    R.check_exact("p16 untouched without a shadow", T.arena["p16"], R.sentinel_like(T.arena["p16"]))


def test_sumsq_deterministic_is_bit_identical(K):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        T = R.OptTable(R.opt_sizes("many"), "cuda", seed=5)
        tab = _table(K, T, [0.0] * len(T.sizes), [0.0] * len(T.sizes))
        a = _sumsq(K, T, tab).clone()
        b = _sumsq(K, T, tab)
        R.check_exact("sumsq deterministic rerun", a, b)
    finally:
        torch.use_deterministic_algorithms(prev)


def test_adamw_step_returns_the_pre_clip_total_norm(K):
    from bevbert_b200.optim import AdamW
    g = torch.Generator().manual_seed(2)
    shapes = [(300, 7), (5,), (4097,)]
    ps = [torch.nn.Parameter(torch.randn(s, generator=g).cuda()) for s in shapes]
    opt = AdamW(ps, lr=1e-3, max_grad_norm=1.0)
    grads = [torch.randn(s, generator=g) for s in shapes]
    for p, gr in zip(ps, grads):
        p.grad = gr.clone().cuda()
    n_ref = float(adamw_ref.clip_grad_norm_([x.clone() for x in grads], 1.0))
    n = opt.step()
    assert n is not None and n.dim() == 0
    assert abs(float(n) - n_ref) <= 1e-5 * n_ref, (float(n), n_ref)
    assert float(n) == float(opt.total_grad_norm())
    assert AdamW([torch.nn.Parameter(torch.zeros(3, device="cuda"))], lr=1e-3).step() is None     # no gradients
