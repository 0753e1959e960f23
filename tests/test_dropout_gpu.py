"""Training-mode dropout on the GPU: every kernel's keep decisions against the documented mask functions
(tests/drop_masks.py), bit for bit, and whole sub-layers with dropout on against fp64 autograd through the oracle.

Kernel level: each case reads the keep pattern out of the kernel's output exactly (a dropped element is exactly 0, or
exactly the residual for a residual-add epilogue), or, for the softmax gradients, decides for every element whether
the kernel's value is nearer the kept or the dropped fp64 value.  It asserts torch.equal between that pattern and the
documented function, and checks the values against fp64 with a tolerance far below the size of a flipped decision.
Seeds have their high 32 bits set, p = 0.1 (threshold 0x1999_9999: nonzero low 16 bits).
"""
import math
import types

import numpy as np
import pytest
import torch

import drop_masks as DM
from helpers import rel_l2

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
SEED = 0xC0FFEE5EED5A1701          # >= 2^63, like the seeds DropState draws
SALT = 0x2545F4914F6CDD1D
P = 0.1
DEV = "cuda"


@pytest.fixture(scope="module")
def K():
    import bevbert_b200.kernels as K
    from bevbert_b200 import _lib
    assert torch.cuda.is_available()
    _lib.load().bb_set_drop_salt_ptr(None)       # a graph test in the same process may have registered a dropout salt
    return K


def _drop(K, seed=SEED):
    th, sc = K.drop_params(P)
    return seed, th, sc


def _rand(*shape, scale=1.0, seed=0, dtype=BF):
    g = torch.Generator().manual_seed(seed * 7919 + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def _round8(n):
    return (n + 7) // 8 * 8


def _check_inferred_keep(got, keep_val, drop_val, keep_ref, what):
    """`got`: a kernel output element by element; keep_val / drop_val: fp64 values of the element with its decision
    kept / dropped (everything else as the documented mask has it).  Where the two differ by more than 2 % of their
    size (a flip is visible above bf16 noise), the decision nearer to `got` must be the documented one; and every
    element must be within a quarter of a flip (or 2 % of its size) of the documented value."""
    got, keep_val, drop_val = got.double(), keep_val.double(), drop_val.double()
    keep_ref = keep_ref.to(got.device)
    flip = (keep_val - drop_val).abs()
    size = keep_val.abs() + drop_val.abs()
    inform = flip > 0.02 * size + 1e-9 * float(size.max())
    assert float(inform.double().mean()) > 0.8, (what, float(inform.double().mean()))
    inferred = (got - keep_val).abs() < (got - drop_val).abs()
    bad = inform & (inferred != keep_ref)
    assert torch.equal(inferred[inform], keep_ref[inform]), "%s: %d of %d decisions differ from the documented mask" % (
        what, int(bad.sum()), int(inform.sum()))
    ref = torch.where(keep_ref, keep_val, drop_val)
    err = (got - ref).abs()
    assert bool((err[inform] <= 0.25 * flip[inform]).all()), (what, float((err / flip.clamp_min(1e-30))[inform].max()))
    assert bool((err <= 0.02 * size + 1e-7 * float(size.max())).all()), (what, float((err - 0.02 * size).max()))


# ----------------------------------------------------------------------------------------- casts
@pytest.mark.parametrize("n,nseeds", [(1000003, 1), (4099, 16), (7, 16)])
def test_cast_and_dropout_act_masks(K, n, nseeds):
    """bb_cast_f32_bf16 / bb_dropout_bf16: the 8-wide body and the scalar tail (n % 8 = 3 or 7); the short sizes run
    several seeds so that the few tail decisions add up to a few dozen."""
    _, th, sc = _drop(K)
    x = torch.randn(n, generator=torch.Generator().manual_seed(n))
    x[x.abs() < 1e-6] = 1.0
    xb = x.to(BF)
    zero = torch.zeros((), dtype=BF)
    for s in range(nseeds):
        seed = ((SEED + 0x9E3779B97F4A7C15 * s) & 0xFFFFFFFFFFFFFFFF) | (1 << 63)
        keep = DM.keep_elem(seed, torch.arange(n), th)
        y = K.cast_to_act(x.to(DEV), (seed, th, sc)).cpu()
        assert torch.equal(y != 0, keep)
        assert torch.equal(y, torch.where(keep, (x * sc).to(BF), zero))
        z = K.dropout_act(xb.to(DEV), (seed, th, sc)).cpu()
        assert torch.equal(z != 0, keep)
        assert torch.equal(z, torch.where(keep, (xb.float() * sc).to(BF), zero))


# ----------------------------------------------------------------------------------------- GEMM epilogues
def _dgelu(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def _gemm_case(K, variant, bn=0, M=300, N=296, Kd=128, nb=(1, 1), ldd=None, seed=SEED, salt=0):
    """One dropout GEMM launch of `variant` (relu: generic epilogue via ACT_RELU; f32: generic via fp32 output;
    gelu_pre / dgelu / drelu / add: the compile-time variants) -> checks; returns (kernel keep pattern, selection)."""
    nb1, nb2 = nb
    ldd = ldd or N
    _, th, sc = _drop(K)
    arm32 = K.act_dtype() == torch.float32
    dt = K.act_dtype()
    a = _rand(nb2, nb1, M, Kd, scale=0.3, seed=1, dtype=dt)
    b = _rand(nb2, nb1, N, Kd, scale=0.3, seed=2, dtype=dt)
    bias = _rand(N, scale=0.5, seed=3, dtype=torch.float32)
    out_dt = torch.float32 if (variant == "f32" or arm32) else BF
    D = torch.full((nb2, nb1, M, ldd), 7.0, dtype=out_dt, device=DEV)    # sentinel in the padding columns
    aux = torch.full((nb2, nb1, M, ldd), 3.0, dtype=dt, device=DEV)
    aux[..., :N] = _rand(nb2, nb1, M, N, scale=1.5, seed=4, dtype=dt)
    kw = dict(bias=bias)
    if variant == "relu":
        kw["act"] = K.ACT_RELU
    elif variant == "gelu_pre":
        pre = torch.full((nb2, nb1, M, ldd), 7.0, dtype=dt, device=DEV)
        kw.update(act=K.ACT_GELU, aux_out=pre)
    elif variant == "dgelu":
        kw = dict(epi_mul=K.EPI_DGELU, aux_in=aux)
    elif variant == "drelu":
        kw = dict(epi_mul=K.EPI_DRELU, aux_in=aux)
    elif variant == "add":
        kw["add_in"] = aux
    K.gemm(a, b, D, M, N, Kd, lda=Kd, ldb=Kd, ldd=ldd, nb1=nb1, nb2=nb2, a_s=(M * Kd, nb1 * M * Kd),
           b_s=(N * Kd, nb1 * N * Kd), d_s=(M * ldd, nb1 * M * ldd), drop=(seed, th, sc), block_n=bn, **kw)
    acc = a.double() @ b.double().transpose(-1, -2)
    av = aux.double()[..., :N]
    v = acc + bias.double()
    if variant == "relu":
        v = v.clamp_min(0)
    elif variant == "gelu_pre":
        pre_ref = v
        v = 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))
    elif variant == "dgelu":
        v = acc * _dgelu(av)
    elif variant == "drelu":
        v = acc * (av > 0)
    off = torch.arange(D.numel(), dtype=torch.int64).view(D.shape)[..., :N]
    keep = DM.keep_elem(seed, off.reshape(-1), th, salt).view(off.shape).to(DEV)
    add = av if variant == "add" else torch.zeros_like(v)
    ref = torch.where(keep, v * float(np.float32(sc)), torch.zeros_like(v)) + add
    out = D.double()[..., :N]
    # the padding columns of D (and of the pre-activation output) are untouched
    assert bool((D[..., N:] == 7.0).all())
    if variant == "gelu_pre":
        assert bool((pre[..., N:] == 7.0).all())
        tol = 2e-5 if arm32 else 2 ** -8
        assert bool(((pre.double()[..., :N] - pre_ref).abs() <= tol * pre_ref.abs() + 1e-4).all()), "pre-activation"
    # a dropped element is exactly 0 (exactly the residual for EPI_ADD)
    assert torch.equal(out[~keep], add[~keep]), "%s: an element the documented mask drops was kept" % variant
    # the kernel's keep pattern, read where the undropped value is clearly nonzero
    if variant == "add":
        kernel_keep = out != add
        sel = (v * sc).abs() > 2 ** -6 * add.abs() + 1e-3
    else:
        kernel_keep = out != 0
        sel = v.abs() > 1e-3
    assert float(sel.double().mean()) > 0.3
    assert torch.equal(kernel_keep[sel], keep[sel]), "%s: %d decisions differ from the documented mask" % (
        variant, int((kernel_keep != keep)[sel].sum()))
    rtol = 1e-5 if out_dt == torch.float32 else 2 ** -7
    assert bool(((out - ref).abs() <= rtol * ref.abs() + 2e-5).all()), (variant, float((out - ref).abs().max()))
    return kernel_keep, sel


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("variant", ["relu", "f32", "gelu_pre", "dgelu", "drelu", "add"])
def test_gemm_epilogue_dropout_masks(K, variant, bn):
    """Every epilogue that takes dropout, at 64- and 128-wide tiles, on 300 x 296 (interior tiles and ragged M / N
    edges): the mask is drop_keep(seed, element offset in D)."""
    _gemm_case(K, variant, bn)


@pytest.mark.parametrize("variant", ["relu", "add", "gelu_pre"])
def test_gemm_dropout_batched_offsets(K, variant):
    """nb1 = 2, nb2 = 3 batches with ldd > N: the element offset includes the batch offset."""
    _gemm_case(K, variant, M=140, N=136, Kd=64, nb=(2, 3), ldd=152)


@pytest.mark.parametrize("variant", ["relu", "add", "dgelu"])
def test_gemm_dropout_unaligned_ldd(K, variant):
    """ldd % 8 != 0 and odd N: no paired stores anywhere (the scalar edge path for every tile)."""
    _gemm_case(K, variant, M=200, N=197, Kd=64, ldd=203)


def test_gemm_add_epilogue_matches_dropout_act(K):
    """The native executors apply the forward dropout of a residual-add GEMM (ldd = N) in the GEMM epilogue and its
    backward with bb_dropout_bf16 on a tensor of the same shape: both must make the same decisions."""
    M, N = 300, 296
    kernel_keep, sel = _gemm_case(K, "add", M=M, N=N)
    da_keep = (K.dropout_act(torch.ones(M, N, dtype=BF, device=DEV), _drop(K)) != 0).view(1, 1, M, N)
    assert torch.equal(kernel_keep[sel], da_keep[sel])


def test_fp32_arm_gemm_dropout_mask(K):
    prev = K.set_precision(True)
    try:
        _gemm_case(K, "relu", M=150, N=136, Kd=64, nb=(2, 1), ldd=144)
        _gemm_case(K, "add", M=150, N=136, Kd=64)
    finally:
        K.set_precision(prev)


# ----------------------------------------------------------------------------------------- unfused softmax
@pytest.mark.parametrize("nq,nk", [(37, 77), (20, 441), (9, 597)])
def test_softmax_dropout_masks(K, nq, nk):
    """bb_softmax_fwd (keep pattern read from Pd) and bb_softmax_bwd (dS element by element) at ragged nk < ld."""
    B, H = 2, 3
    ld = _round8(nk)
    seed, th, sc = _drop(K)
    s = _rand(B, H, nq, ld, scale=0.5, seed=5, dtype=torch.float32)
    p, pd = K.softmax_fwd(s, None, None, B, H, nq, nk, ld, (seed, th, sc))
    keep = DM.softmax_keep(seed, B, H, nq, nk, ld, th).to(DEV)
    pref = torch.softmax(s.double()[..., :nk], -1)
    pdv = pd.double()
    assert torch.equal(pdv[..., :nk] != 0, keep)
    assert bool((pdv[..., nk:] == 0).all()) and bool((p.double()[..., nk:] == 0).all())
    ref = torch.where(keep, pref * sc, torch.zeros_like(pref))
    assert bool(((pdv[..., :nk] - ref).abs() <= 2 ** -8 * ref + 1e-7).all())
    dp = _rand(B, H, nq, ld, seed=6, dtype=torch.float32)
    ds = K.softmax_bwd(p, dp, B, H, nq, nk, ld, (seed, th, sc), 0.125)
    assert bool((ds.double()[..., nk:] == 0).all())
    _check_softmax_grad(ds.double()[..., :nk], p.double()[..., :nk], dp.double()[..., :nk], keep, sc, "softmax_bwd")


def _check_softmax_grad(ds, P, dP, keep, sc, what, out_scale=0.125):
    """ds = out_scale P o (g - sum_k P g), g = keep o sc dP, checked element by element with the documented mask"""
    g = torch.where(keep, dP * sc, torch.zeros_like(dP))
    dot = (P * g).sum(-1, keepdim=True)
    _check_inferred_keep(ds, out_scale * P * (dP * sc - dot), out_scale * P * (-dot), keep, what)


# ----------------------------------------------------------------------------------------- fused scores
def _heads(t, B, n, H):
    return t.view(B, n, H, 64).permute(0, 2, 1, 3)


@pytest.mark.parametrize("nk", [23, 80, 441])
def test_fused_scores_dropout_masks(K, nk):
    """bb_attn_scores mode 0 (Pd) and mode 1 (dS) against softmax_keep."""
    B, H, nq = 2, 2, 130
    Hd = 64 * H
    ldp = _round8(nk)
    seed, th, sc = _drop(K)
    q = _rand(B * nq, Hd, scale=0.3, seed=7)
    kv = _rand(B * nk, 2 * Hd, scale=0.3, seed=8)
    P, Pd = K.attn_scores_fwd(q, Hd, kv, 2 * Hd, B, H, nq, nk, 64, ldp, None, None, (seed, th, sc))
    keep = DM.softmax_keep(seed, B, H, nq, nk, ldp, th).to(DEV)
    qh, kh = _heads(q.double(), B, nq, H), _heads(kv.double()[:, :Hd], B, nk, H)
    vh = _heads(kv.double()[:, Hd:], B, nk, H)
    pref = torch.softmax(qh @ kh.transpose(-1, -2) / 8.0, -1)
    pdv = Pd.double()
    assert torch.equal(pdv[..., :nk] != 0, keep)
    assert bool((pdv[..., nk:] == 0).all()) and bool((P.double()[..., nk:] == 0).all())
    ref = torch.where(keep, pref * sc, torch.zeros_like(pref))
    assert bool(((pdv[..., :nk] - ref).abs() <= 2 ** -7 * ref + 1e-6).all())
    dctx = _rand(B * nq, Hd, scale=0.5, seed=9)
    dS = K.attn_scores_bwd(dctx, Hd, kv[:, Hd:], 2 * Hd, P, B, H, nq, nk, 64, ldp, (seed, th, sc))
    assert bool((dS.double()[..., nk:] == 0).all())
    dP = _heads(dctx.double(), B, nq, H) @ vh.transpose(-1, -2)
    _check_softmax_grad(dS.double()[..., :nk], P.double()[..., :nk], dP, keep, sc, "attn_scores_bwd")


# ----------------------------------------------------------------------------------------- flash attention
def _onehot_block(B, n, H, j):
    """(B * n, H * 64) bf16 with rows 64 j .. 64 j + 63 = I (per head), all other rows zero"""
    t = torch.zeros(B, n, H, 64)
    r = torch.arange(64 * j, min(64 * j + 64, n))
    t[:, r] = torch.eye(64)[: len(r)][None, :, None, :]
    return t.reshape(B * n, H * 64).to(BF).to(DEV)


def _flash_readout(K, B, H, nq, nk, seed, th, sc, salt=0, backward=True):
    """Reads the keep pattern of bb_flash_fwd (V = one-hot key block) and, with backward, of both backward passes:
    dO = one-hot query block -> dV = Pd^T dO; K = one-hot key block -> dQ = alpha dS; Q = one-hot query block ->
    dK = alpha dS^T.  Checks each against attn_keep."""
    Hd = 64 * H
    drop = (seed, th, sc)
    keep = DM.attn_keep(seed, B, H, nq, nk, th, salt).to(DEV)
    q = _rand(B * nq, Hd, scale=0.5, seed=10)
    k = _rand(B * nk, Hd, scale=0.5, seed=11)
    v = _rand(B * nk, Hd, scale=0.5, seed=12)
    dout = _rand(B, nq, Hd, scale=0.5, seed=13)

    def probs(qq, kk):
        return torch.softmax(_heads(qq.double(), B, nq, H) @ _heads(kk.double(), B, nk, H).transpose(-1, -2) / 8.0, -1)

    def ds_parts(qq, kk, o):
        """fp64 dS with each element's decision kept / dropped (D from the kernel's own O, as the kernels use it)"""
        Pm = probs(qq, kk)
        dP = _heads(dout.double().view(B * nq, Hd), B, nq, H) @ _heads(v.double(), B, nk, H).transpose(-1, -2)
        D = (_heads(dout.double().view(B * nq, Hd), B, nq, H) * _heads(o.double().view(B * nq, Hd), B, nq, H)).sum(-1,
                                                                                                                   keepdim=True)
        return Pm * (dP * sc - D), Pm * (-D)

    nkb, nqb = (nk + 63) // 64, (nq + 63) // 64
    fwd_keep = torch.zeros(B, H, nq, nk, dtype=torch.bool, device=DEV)
    dq_got, dq_kv, dq_dv = (torch.zeros(B, H, nq, nk, dtype=torch.float64, device=DEV) for _ in range(3))
    pref = probs(q, k)
    for j in range(nkb):
        c0, c1 = 64 * j, min(64 * j + 64, nk)
        o, _ = K.flash_fwd(q, k, _onehot_block(B, nk, H, j), B, H, nq, nk, Hd, Hd, Hd, drop=drop)
        oh = _heads(o.double().view(B * nq, Hd), B, nq, H)
        assert bool((oh[..., c1 - c0:] == 0).all())
        fwd_keep[..., c0:c1] = oh[..., : c1 - c0] != 0
        assert torch.equal(fwd_keep[..., c0:c1], keep[..., c0:c1]), "forward: %d decisions of key block %d differ" % (
            int((fwd_keep[..., c0:c1] != keep[..., c0:c1]).sum()), j)
        ref = torch.where(keep[..., c0:c1], pref[..., c0:c1] * sc, torch.zeros_like(pref[..., c0:c1]))
        assert bool(((oh[..., : c1 - c0] - ref).abs() <= 2 ** -7 * ref + 1e-6).all()), "forward values"
        if backward:
            kj = _onehot_block(B, nk, H, j)
            o, lse = K.flash_fwd(q, kj, v, B, H, nq, nk, Hd, Hd, Hd, drop=drop)
            dq, _, _ = K.flash_bwd(q, kj, v, o, lse, dout, B, H, nq, nk, Hd, Hd, Hd, drop=drop)
            kv_, dv_ = ds_parts(q, kj, o)
            dq_got[..., c0:c1] = _heads(dq.double().view(B * nq, Hd), B, nq, H)[..., : c1 - c0] / 0.125
            dq_kv[..., c0:c1], dq_dv[..., c0:c1] = kv_[..., c0:c1], dv_[..., c0:c1]
    assert torch.equal(fwd_keep, keep), "forward: %d decisions differ" % int((fwd_keep != keep).sum())
    if not backward:
        return
    _check_inferred_keep(dq_got, dq_kv, dq_dv, keep, "dQ pass")
    dk_got, dk_kv, dk_dv = (torch.zeros(B, H, nq, nk, dtype=torch.float64, device=DEV) for _ in range(3))
    dv_keep = torch.zeros(B, H, nq, nk, dtype=torch.bool, device=DEV)
    for i in range(nqb):
        r0, r1 = 64 * i, min(64 * i + 64, nq)
        qi = _onehot_block(B, nq, H, i)
        o, lse = K.flash_fwd(qi, k, v, B, H, nq, nk, Hd, Hd, Hd, drop=drop)
        _, dk, _ = K.flash_bwd(qi, k, v, o, lse, dout, B, H, nq, nk, Hd, Hd, Hd, drop=drop)
        kv_, dv_ = ds_parts(qi, k, o)
        dkt = _heads(dk.double().view(B * nk, Hd), B, nk, H).transpose(-1, -2)      # (B, H, 64, nk)
        dk_got[:, :, r0:r1] = dkt[:, :, : r1 - r0] / 0.125
        dk_kv[:, :, r0:r1], dk_dv[:, :, r0:r1] = kv_[:, :, r0:r1], dv_[:, :, r0:r1]
        # dO = one-hot query block: dV[k, c] = Pd[64 i + c, k]
        d1 = _onehot_block(B, nq, H, i).view(B, nq, Hd)
        _, _, dv = K.flash_bwd(qi, k, v, o, lse, d1, B, H, nq, nk, Hd, Hd, Hd, drop=drop)
        dvt = _heads(dv.double().view(B * nk, Hd), B, nk, H).transpose(-1, -2)
        assert bool((dvt[:, :, r1 - r0:] == 0).all())
        dv_keep[:, :, r0:r1] = dvt[:, :, : r1 - r0] != 0
        assert torch.equal(dv_keep[:, :, r0:r1], keep[:, :, r0:r1]), "dK/dV pass (dV): %d decisions of query block %d " \
            "differ" % (int((dv_keep[:, :, r0:r1] != keep[:, :, r0:r1]).sum()), i)
        pi = probs(qi, k)[:, :, r0:r1]
        ref = torch.where(keep[:, :, r0:r1], pi * sc, torch.zeros_like(pi))
        assert bool(((dvt[:, :, : r1 - r0] - ref).abs() <= 2 ** -7 * ref + 1e-6).all()), "dV values"
    assert torch.equal(dv_keep, keep), "dK/dV pass (dV): %d decisions differ" % int((dv_keep != keep).sum())
    _check_inferred_keep(dk_got, dk_kv, dk_dv, keep, "dK/dV pass (dS)")


@pytest.mark.parametrize("nq,nk", [(23, 80), (130, 200), (441, 441), (80, 441)])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_flash_attention_dropout_masks(K, mode, nq, nk):
    """bb_flash_fwd / bb_flash_bwd with the mma.sync kernels (mode 0) and the wgmma kernels (modes 1, 2): the forward,
    the dQ pass and the dK/dV pass each make the decisions of attn_keep."""
    prev = K.set_attn_tc(mode)
    try:
        _flash_readout(K, 2, 2, nq, nk, *_drop(K))
    finally:
        K.set_attn_tc(prev)


# ----------------------------------------------------------------------------------------- graph-replay salt
def test_salt_reaches_every_translation_unit(K):
    """With a salt word registered, one launch from each of the six translation units that hold a copy of the salt
    pointer (gemm_tc, rowops, attn_flash, attn_tc, attn_scores, gemm_f32) makes the decisions of seed ^ salt."""
    from bevbert_b200 import _lib
    lib = _lib.load()
    seed, th, sc = _drop(K)
    word = torch.tensor([SALT], dtype=torch.int64, device=DEV)
    assert lib.bb_set_drop_salt_ptr(word.data_ptr()) == 0
    prev_tc = K.set_attn_tc(0)
    try:
        _gemm_case(K, "relu", M=140, N=136, Kd=64, salt=SALT)                             # gemm_tc
        n = 4099
        z = K.dropout_act(torch.ones(n, dtype=BF, device=DEV), (seed, th, sc))            # rowops
        assert torch.equal((z != 0).cpu(), DM.keep_elem(seed, torch.arange(n), th, SALT))
        _flash_readout(K, 1, 2, 70, 80, seed, th, sc, salt=SALT, backward=False)          # attn_flash
        K.set_attn_tc(2)
        _flash_readout(K, 1, 2, 70, 80, seed, th, sc, salt=SALT, backward=False)          # attn_tc
        B, H, nq, nk = 1, 2, 40, 37
        q = _rand(B * nq, 128, scale=0.3, seed=14)
        kv = _rand(B * nk, 256, scale=0.3, seed=15)
        _, Pd = K.attn_scores_fwd(q, 128, kv, 256, B, H, nq, nk, 64, 40, None, None, (seed, th, sc))   # attn_scores
        assert torch.equal((Pd[..., :nk] != 0).cpu(), DM.softmax_keep(seed, B, H, nq, nk, 40, th, SALT))
        prev = K.set_precision(True)
        try:
            _gemm_case(K, "relu", M=70, N=72, Kd=32, salt=SALT)                            # gemm_f32
        finally:
            K.set_precision(prev)
    finally:
        K.set_attn_tc(prev_tc)
        lib.bb_set_drop_salt_ptr(None)
        torch.cuda.synchronize()
    del word


# ----------------------------------------------------------------------------------------- sub-layers vs fp64 autograd
HD, NH, FD = 768, 12, 3072


def _bfp(*shape, scale, seed):
    """bf16-representable fp32 on the device (the bf16 weight shadows then hold the same values)"""
    return _rand(*shape, scale=scale, seed=seed).float()


def _spec_bert():
    B, n = 2, 70
    kmask = torch.zeros(B, n, device=DEV)
    kmask[1, -7:] = -10000.0
    names = ["L.attention.self.%s.%s" % (m, w) for m in ("query", "key", "value") for w in ("weight", "bias")]
    names += ["L.attention.output.dense.weight", "L.attention.output.dense.bias", "L.attention.output.LayerNorm.weight",
              "L.attention.output.LayerNorm.bias", "L.intermediate.dense.weight", "L.intermediate.dense.bias",
              "L.output.dense.weight", "L.output.dense.bias", "L.output.LayerNorm.weight", "L.output.LayerNorm.bias"]
    shapes = [(HD, HD), (HD,)] * 4 + [(HD,), (HD,), (FD, HD), (FD,), (HD, FD), (HD,), (HD,), (HD,)]

    def ref(R, sd, ins, cfg):
        x, bias = ins
        return R.bert_layer(sd, "L", x, kmask.double()[:, None, None, :] + bias[:, None], cfg)

    return dict(names=names, shapes=shapes, gammas=(8, 14), ins=[("act", (B, n, HD)), ("f32", (B, n, n))],
                consts=lambda ins: [ins[0], kmask, ins[1]], ref=ref, kinds=["attn", "ln", "ln"],
                impl=lambda Bk, rt, p: Bk.BertLayerImpl(rt, NH, 1e-12, p, p), out=(B, n, HD))


def _spec_xattn():
    B, nq, nk = 2, 30, 70
    cmask = torch.zeros(B, nk, device=DEV)
    cmask[0, -5:] = -10000.0
    names = ["L.att.%s.%s" % (m, w) for m in ("query", "key", "value") for w in ("weight", "bias")]
    names += ["L.output.dense.weight", "L.output.dense.bias", "L.output.LayerNorm.weight", "L.output.LayerNorm.bias"]

    def ref(R, sd, ins, cfg):
        x, c = ins
        return R.cross_attention(sd, "L", x, c, cmask.double()[:, None, None, :], cfg)

    return dict(names=names, shapes=[(HD, HD), (HD,)] * 4 + [(HD,), (HD,)], gammas=(8,),
                ins=[("act", (B, nq, HD)), ("act", (B, nk, HD))], consts=lambda ins: [ins[0], ins[1], cmask], ref=ref,
                kinds=["attn", "ln"], impl=lambda Bk, rt, p: Bk.XAttnImpl(rt, NH, 1e-12, p, p), out=(B, nq, HD))


def _spec_pano():
    N, V = 5, 36
    kmask = torch.zeros(N, V, device=DEV)
    kmask[2, -9:] = float("-inf")
    names = ["L.self_attn.in_proj_weight", "L.self_attn.in_proj_bias", "L.self_attn.out_proj.weight",
             "L.self_attn.out_proj.bias", "L.linear1.weight", "L.linear1.bias", "L.linear2.weight", "L.linear2.bias",
             "L.norm1.weight", "L.norm1.bias", "L.norm2.weight", "L.norm2.bias"]
    shapes = [(3 * HD, HD), (3 * HD,), (HD, HD), (HD,), (FD, HD), (FD,), (HD, FD), (HD,), (HD,), (HD,), (HD,), (HD,)]

    def ref(R, sd, ins, cfg):
        return R.pano_layer(sd, "L", ins[0], torch.isinf(kmask), cfg)

    return dict(names=names, shapes=shapes, gammas=(8, 10), ins=[("act", (N, V, HD))],
                consts=lambda ins: [ins[0], kmask], ref=ref, kinds=["attn", "elem", "elem", "elem"],
                impl=lambda Bk, rt, p: Bk.PanoLayerImpl(rt, NH, p, p), out=(N, V, HD))


def _spec_layernorm():
    shape = (2, 37, HD)

    def ref(R, sd, ins, cfg):
        return R._drop(R._ln(sd, "L", ins[0] + ins[1], 1e-12), cfg.drop_p)

    return dict(names=["L.weight", "L.bias"], shapes=[(HD,), (HD,)], gammas=(0,), ins=[("act", shape), ("act", shape)],
                consts=lambda ins: list(ins), ref=ref, kinds=["ln"],
                impl=lambda Bk, rt, p: Bk.LayerNormImpl(rt, 1e-12, p_out=p), out=shape)


def _spec_text():
    B, L, V = 2, 40, 100
    ids = torch.randint(1, V, (B, L), generator=torch.Generator().manual_seed(3)).to(DEV)   # 0 is the padding id
    p = "bert.embeddings."
    names = [p + "word_embeddings.weight", p + "position_embeddings.weight", p + "token_type_embeddings.weight",
             p + "LayerNorm.weight", p + "LayerNorm.bias"]

    def ref(R, sd, ins, cfg):
        return R.text_embeddings(sd, ids, cfg)

    return dict(names=names, shapes=[(V, HD), (512, HD), (2, HD), (HD,), (HD,)], gammas=(3,), ins=[],
                consts=lambda ins: [ids], ref=ref, kinds=["ln"],
                impl=lambda Bk, rt, p: Bk.TextEmbedImpl(rt, 1e-12, p_out=p), out=(B, L, HD))


SPECS = {"bert": _spec_bert, "xattn": _spec_xattn, "pano": _spec_pano, "layernorm": _spec_layernorm, "text": _spec_text}


def _data(spec):
    params = [_bfp(*s, scale=0.5 if len(s) == 2 and s[0] in (100, 512, 2) else 0.03, seed=20 + i)
              for i, s in enumerate(spec["shapes"])]
    for i in spec["gammas"]:
        params[i] = params[i] + 1.0
    ins = [_bfp(*shape, scale=0.5, seed=40 + i) if kind == "act" else _rand(*shape, scale=0.3, seed=40 + i).float()
           for i, (kind, shape) in enumerate(spec["ins"])]
    dy = _bfp(*spec["out"], scale=0.1, seed=60)
    return params, ins, dy


def _run_kernels(K, Bk, spec, data, p, python_composition, seed=5):
    """forward + backward of the block -> (y, input grads, param grads, recorded (seed, thresh, scale) sites)"""
    params0, ins0, dy = data
    params = [torch.nn.Parameter(t.clone()) for t in params0]
    ins = [(t.to(K.act_dtype(), copy=True) if kind == "act" else t.clone()).requires_grad_(True)
           for t, (kind, _) in zip(ins0, spec["ins"])]
    rt = Bk.Runtime()
    impl = spec["impl"](Bk, rt, p)
    native = K.native_sublayers
    if python_composition:
        K.native_sublayers = lambda: False
    try:
        ds = rt.begin(True, seed=seed)
        sites, make = [], ds.make

        def recording_make(prob):
            t = make(prob)
            if t[1]:
                sites.append(t)
            return t
        ds.make = recording_make
        y = Bk.run_block(impl, spec["consts"](ins), params)
        y.backward(dy.to(y.dtype))
        torch.cuda.synchronize()
    finally:
        K.native_sublayers = native
    return y.detach(), [t.grad for t in ins], [t.grad for t in params], sites


def _run_reference(spec, data, sites, flash, p, alter=None):
    """the oracle's layer function in fp64; its dropout calls apply the documented masks of `sites` in call order
    (site `alter` with a different seed)"""
    from oracle import bevbert_ref as R
    params0, ins0, dy = data
    sd = {n: t.double().requires_grad_(True) for n, t in zip(spec["names"], params0)}
    ins = [t.double().requires_grad_(True) for t in ins0]
    cfg = types.SimpleNamespace(num_attention_heads=NH, layer_norm_eps=1e-12, drop_p=p)
    seq = [(s ^ 0x5DEECE66D if i == alter else s, th, sc) for i, (s, th, sc) in enumerate(sites)]
    calls = []

    def documented_drop(x, prob):
        if prob <= 0:
            return x
        i = len(calls)
        calls.append(i)
        assert i < len(seq), "the oracle has more dropout sites than the kernels drew"
        seed, th, sc = seq[i]
        kind = spec["kinds"][i]
        if kind == "attn":
            B, H, nq, nk = x.shape
            keep = DM.attn_keep(seed, B, H, nq, nk, th) if flash else DM.softmax_keep(seed, B, H, nq, nk, _round8(nk), th)
        elif kind == "ln":
            keep = DM.ln_keep(seed, x.numel() // x.shape[-1], x.shape[-1], th).view(x.shape)
        else:
            keep = DM.keep_elem(seed, torch.arange(x.numel()), th).view(x.shape)
        return x * keep.to(x.device, x.dtype) * float(np.float32(sc))

    saved = R._drop
    R._drop = documented_drop
    try:
        y = spec["ref"](R, sd, ins, cfg)
    finally:
        R._drop = saved
    assert len(calls) == len(seq) == len(spec["kinds"] if p > 0 else []), (len(calls), len(seq))
    y.backward(dy.double())
    return y.detach(), [t.grad for t in ins], [sd[n].grad for n in spec["names"]]


def _errors(got, ref):
    """(output, worst input grad, worst parameter grad) relative errors; a parameter gradient is measured against
    max(its norm, 1e-2 x the largest reference gradient norm) (the key bias gradient is mathematically zero)"""
    y, gi, gp = got
    ry, rgi, rgp = ref
    e_in = max([rel_l2(a, b) for a, b in zip(gi, rgi)] or [0.0])
    top = max(float(r.norm()) for r in rgp)
    e_par = max(float((a.double() - b).norm()) / max(float(b.norm()), 1e-2 * top) for a, b in zip(gp, rgp))
    return rel_l2(y, ry), e_in, e_par


# (dropout-off floor, bar) of (output, worst input grad, worst parameter grad); the floors were measured on an H100
# 80GB HBM3 with this test's inputs.  Each bar is about 3x the floor of the same comparison; with dropout on, the
# errors measured there were within 10 % of the floors.  With one site's seed changed (the negative controls) the
# errors measured 4e-2 .. 0.5, at least 20x the bar of some gradient at every site.  TextEmbedImpl has no input grad.
BARS = {
    ("bert", "native"): ((2.84e-3, 1e-2), (4.01e-3, 1.2e-2), (4.87e-3, 1.5e-2)),
    ("bert", "python"): ((2.84e-3, 1e-2), (4.01e-3, 1.2e-2), (4.87e-3, 1.5e-2)),
    ("bert", "fp32"): ((7.53e-7, 3e-6), (9.67e-7, 3e-6), (1.01e-6, 3e-6)),
    ("xattn", "native"): ((1.69e-3, 5e-3), (3.91e-3, 1.2e-2), (4.26e-3, 1.3e-2)),
    ("xattn", "python"): ((1.69e-3, 5e-3), (3.91e-3, 1.2e-2), (4.26e-3, 1.3e-2)),
    ("xattn", "fp32"): ((8.92e-8, 3e-7), (7.57e-7, 3e-6), (6.42e-7, 2e-6)),
    ("pano", "native"): ((3.36e-3, 1e-2), (4.34e-3, 1.3e-2), (5.80e-3, 1.8e-2)),
    ("pano", "python"): ((3.36e-3, 1e-2), (4.34e-3, 1.3e-2), (5.80e-3, 1.8e-2)),
    ("pano", "fp32"): ((1.02e-6, 3e-6), (1.03e-6, 3e-6), (1.46e-6, 5e-6)),
    ("layernorm", "native"): ((1.67e-3, 5e-3), (1.67e-3, 5e-3), (9.9e-8, 3e-7)),
    ("layernorm", "fp32"): ((6.41e-8, 2e-7), (6.43e-8, 2e-7), (9.64e-8, 3e-7)),
    ("text", "native"): ((1.66e-3, 5e-3), None, (1.91e-7, 6e-7)),
    ("text", "fp32"): ((6.6e-8, 2e-7), None, (1.74e-7, 6e-7)),
}


@pytest.mark.parametrize("arm", ["native", "python", "fp32"])
@pytest.mark.parametrize("layer", ["bert", "xattn", "pano", "layernorm", "text"])
def test_sublayer_with_dropout_matches_fp64_autograd(K, layer, arm):
    """BertLayerImpl (graph bias with grad + FFN), XAttnImpl, PanoLayerImpl, LayerNormImpl(p_out), TextEmbedImpl in
    training mode with p_attn = p_hidden = 0.1 against the oracle's layer function in fp64 on the same bf16-valued
    inputs, with the oracle's dropout replaced by the documented mask of each site: native executors, the Python
    composition of the same kernels, and the fp32 verification arm (unfused attention: softmax_keep).
    The bars and the dropout-off floors measured on an H100 are in BARS.  LayerNormImpl and TextEmbedImpl have no
    native executor, so their "python" arm is the "native" one."""
    import bevbert_b200.blocks as Bk
    if layer in ("layernorm", "text") and arm == "python":
        pytest.skip("no native executor: the Python composition is the only bf16 path")
    spec = SPECS[layer]()
    prev = K.set_precision(arm == "fp32")
    try:
        data = _data(spec)
        flash = K.use_flash()
        off = _run_kernels(K, Bk, spec, data, 0.0, arm == "python")
        assert not off[3]
        floor = _errors(off[:3], _run_reference(spec, data, [], flash, 0.0))
        on = _run_kernels(K, Bk, spec, data, P, arm == "python")
        sites = on[3]
        assert len(sites) == len(spec["kinds"])
        err = _errors(on[:3], _run_reference(spec, data, sites, flash, P))
        controls = [_errors(on[:3], _run_reference(spec, data, sites, flash, P, alter=i)) for i in range(len(sites))]
    finally:
        K.set_precision(prev)
    print("%s/%s: dropout off %s | dropout on %s | one site's seed changed %s" % (
        layer, arm, ["%.3g" % e for e in floor], ["%.3g" % e for e in err],
        [["%.3g" % e for e in c] for c in controls]))
    checked = [(i, fb[1]) for i, fb in enumerate(BARS[(layer, arm)]) if fb is not None]
    for i, b in checked:
        what = ("output", "input grads", "param grads")[i]
        assert floor[i] <= b, "%s: dropout-off error %.3g above the bar %.3g" % (what, floor[i], b)
        assert err[i] <= b, "%s: dropout-on error %.3g above the bar %.3g" % (what, err[i], b)
    for s, c in enumerate(controls):
        assert max(c[i] / b for i, b in checked) >= 5.0, "site %d (%s): a wrong mask stays within 5x the bars: %s" % (
            s, spec["kinds"][s], c)
