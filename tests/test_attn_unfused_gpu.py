"""The unfused attention path composed: blocks.attn_core_fwd / attn_core_bwd with the flash cores off (the path of the
fp32 verification arm, of BB_FLASH=0 and of the BB_FUSED_SCORES_MAX experiment), at the model's shapes, per element
against fp64 autograd from the same inputs, in both arms and with the fused-scores kernel off (0) and on (512 keys):
  - 441 x 441 BEV self-attention with a graph bias and its gradient (packed Q|K|V);
  - 80-query x 441-key cross attention with a 0 / -10000 key mask (packed K|V);
  - panorama self-attention (36 views) with -inf padding and one panorama with no valid view, whose rows must give
    ctx = 0 and no gradient (the flash cores' convention).
Bounds: ctx within ulp/2 + e (P |V|); dV within ulp/2 + e (P^T |dctx|); dQ within ulp/2 + 2e alpha (A |K|), dK within
ulp/2 + 2e alpha (A^T |Q|), dbias within 2e sum_h A, with A = P (|g| + |sum P g|) bounding dS (g = dctx V^T).
e = 2^-8 in the bf16 arm (twice the relative rounding of P and dS to bf16, the MMA operands) and (nk + 64) 2^-22 in
the fp32 arm (four times gamma of the longest fp32 reduction behind each output).

Regressions: in the fp32 arm a fused-scores limit of 512 keys must change nothing (the bf16-only kernel must not run on
fp32 data), and a PanoLayerImpl batch with a fully padded panorama must give the other panoramas' outputs and every
weight gradient of the batch without it, with finite rows for the dead one.  The native executor reads BB_FLASH and
BB_FUSED_SCORES_MAX once, so its unfused variant runs in a subprocess with its own environment.
"""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
H, DH = 12, 64
HD = H * DH

SHAPES = {  # name: (B, nq, nk, layout, mask, bias)
    "bev": (2, 441, 441, "self", None, True),
    "cross": (2, 80, 441, "cross", "mix", False),
    "pano": (5, 36, 36, "self", "pano", False),
}
PANO_LENS = (36, 20, 0, 36, 7)          # panorama 2 has no valid view


def _kmask(kind, B, nk, g):
    if kind is None:
        return None
    if kind == "mix":
        km = torch.where(torch.rand(B, nk, generator=g) < 0.3, -10000.0, 0.0)
        km[:, 0] = 0.0
        return km
    valid = torch.arange(nk)[None, :] < torch.tensor(PANO_LENS[:B])[:, None]
    return torch.zeros(B, nk).masked_fill(~valid, float("-inf"))


def _inputs(shape, act, seed=0):
    B, nq, nk, layout, mask, bias = SHAPES[shape]
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=g).to(act).cuda()
    if layout == "self":
        qkv = rnd(B * nq, 3 * HD)
        ops = (qkv, 3 * HD, qkv[:, HD:], 3 * HD, qkv[:, 2 * HD:], 3 * HD)
        grads = torch.empty_like(qkv)
        gops = (grads, 3 * HD, grads[:, HD:], 3 * HD, grads[:, 2 * HD:], 3 * HD)
    else:
        q, kv = rnd(B * nq, HD), rnd(B * nk, 2 * HD)
        ops = (q, HD, kv, 2 * HD, kv[:, HD:], 2 * HD)
        dq, dkv = torch.empty_like(q), torch.empty_like(kv)
        gops = (dq, HD, dkv, 2 * HD, dkv[:, HD:], 2 * HD)
    km = _kmask(mask, B, nk, g)
    bi = (torch.randn(B, nq, nk, generator=g) * 0.5) if bias else None
    dctx = rnd(B * nq, HD)
    return ops, gops, (km.cuda() if km is not None else None), (bi.cuda() if bi is not None else None), dctx


def _heads(t, ld, B, n):
    return torch.as_strided(t, (B, H, n, DH), (n * ld, DH, ld, 1), t.storage_offset())


def run_core(K, shape, act, fused, monkeypatch):
    """attn_core_fwd / _bwd with the flash cores off -> (inputs, ctx, dq, dk, dv, dbias)"""
    from bevbert_b200 import blocks as Bk
    monkeypatch.setattr(K, "FLASH", False)
    monkeypatch.setattr(K, "FUSED_SCORES_MAX_KEYS", fused)
    B, nq, nk = SHAPES[shape][:3]
    ops, gops, km, bi, dctx = _inputs(shape, act)
    q, ldq, k, ldk, v, ldv = ops
    st = {}
    ctx = Bk.attn_core_fwd(st, q, ldq, k, ldk, v, ldv, B, H, nq, nk, DH, km, bi, K.NO_DROP)
    dbias = torch.full((B, nq, nk), 0.25, device="cuda") if bi is not None else None
    dq, lddq, dk, lddk, dv, lddv = gops
    Bk.attn_core_bwd(st, dctx, q, ldq, k, ldk, v, ldv, dq, lddq, dk, lddk, dv, lddv, dbias)
    torch.cuda.synchronize()
    return (ops, km, bi, dctx), ctx, (_heads(dq, lddq, B, nq), _heads(dk, lddk, B, nk), _heads(dv, lddv, B, nk)), dbias


def fp64_ref(ins, B, nq, nk):
    ops, km, bi, dctx = ins
    q, ldq, k, ldk, v, ldv = ops
    qh, kh, vh = (_heads(t, ld, B, n).double().detach().clone().requires_grad_(True)
                  for t, ld, n in ((q, ldq, nq), (k, ldk, nk), (v, ldv, nk)))
    b64 = bi.double().clone().requires_grad_(True) if bi is not None else None
    x = qh @ kh.transpose(-1, -2) * 0.125
    if km is not None:
        x = x + km.double().view(B, 1, 1, nk)
    if b64 is not None:
        x = x + b64.view(B, 1, nq, nk)
    dead = ~torch.isfinite(x).any(-1, keepdim=True)
    P = torch.softmax(torch.where(dead, torch.zeros_like(x), x), -1) * (~dead)
    ctx = P @ vh
    do = _heads(dctx, HD, B, nq).double()
    ctx.backward(do)
    g = do @ vh.detach().transpose(-1, -2)
    Pd = P.detach()
    A = Pd * (g.abs() + (Pd * g).sum(-1, keepdim=True).abs())
    return dict(ctx=ctx.detach(), dq=qh.grad, dk=kh.grad, dv=vh.grad, dbias=b64.grad if b64 is not None else None,
                s_ctx=Pd @ vh.detach().abs(), s_dv=Pd.transpose(-1, -2) @ do.abs(), s_dq=0.125 * A @ kh.detach().abs(),
                s_dk=0.125 * A.transpose(-1, -2) @ qh.detach().abs(), s_db=A.sum(1), dead=dead)


def _check(name, got, ref, scale, e, bf):
    import rowops_cases as R
    bound = e * scale + (R.half_ulp_bf16(ref.abs() + e * scale) if bf else 0.0)
    R.check(name, got, ref, bound)


def check_core(shape, act, res, ref):
    B, nq, nk = SHAPES[shape][:3]
    bf = act == BF
    e = 2.0 ** -8 if bf else (nk + 64) * 2.0 ** -22
    ins, ctx, (dq, dk, dv), dbias = res
    tag = "[%s-%s]" % (shape, "bf16" if bf else "fp32")
    ctxh = _heads(ctx, HD, B, nq)
    _check("unfused.ctx" + tag, ctxh, ref["ctx"], ref["s_ctx"], e, bf)
    _check("unfused.dv" + tag, dv, ref["dv"], ref["s_dv"], e, bf)
    _check("unfused.dq" + tag, dq, ref["dq"], ref["s_dq"], 2 * e, bf)
    _check("unfused.dk" + tag, dk, ref["dk"], ref["s_dk"], 2 * e, bf)
    if dbias is not None:
        import rowops_cases as R
        rdb = ref["dbias"] + 0.25                        # accumulated into a buffer holding 0.25
        R.check("unfused.dbias" + tag, dbias, rdb, 2 * e * ref["s_db"] + 2.0 ** -22 * rdb.abs())
    dead = ref["dead"][..., 0]
    if bool(dead.any()):
        assert bool((ctxh[dead] == 0).all()), "ctx of a row with every key at -inf must be 0"


@pytest.fixture(scope="module")
def K():
    from bevbert_b200 import _lib, kernels as K
    assert torch.cuda.is_available()
    _lib.load().bb_set_drop_salt_ptr(None)
    return K


@pytest.fixture(params=[False, True], ids=["bf16", "fp32"])
def arm(K, request):
    prev = K.set_precision(request.param)
    yield F32 if request.param else BF
    K.set_precision(prev)


@pytest.mark.parametrize("fused", [0, 512])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_attn_core_unfused_matches_fp64(K, arm, shape, fused, monkeypatch):
    B, nq, nk = SHAPES[shape][:3]
    res = run_core(K, shape, arm, fused, monkeypatch)
    check_core(shape, arm, res, fp64_ref(res[0], B, nq, nk))


@pytest.mark.parametrize("shape", list(SHAPES))
def test_fp32_arm_ignores_fused_scores_limit(K, shape, monkeypatch):
    """the fused-scores kernel is bf16 only: in the fp32 arm a limit of 512 keys must leave every result bit-identical
    (in deterministic mode, so that the graph-bias gradient adds in a fixed order)"""
    prev = K.set_precision(True)
    det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        r0 = run_core(K, shape, F32, 0, monkeypatch)
        r1 = run_core(K, shape, F32, 512, monkeypatch)
    finally:
        torch.use_deterministic_algorithms(det)
        K.set_precision(prev)
    flat = lambda r: [r[1]] + list(r[2]) + ([r[3]] if r[3] is not None else [])
    for name, a, b in zip(("ctx", "dq", "dk", "dv", "dbias"), flat(r0), flat(r1)):
        assert torch.equal(a, b), "%s: fused-scores limit 512 changed the fp32 arm (max diff %g)" % (
            name, float((a.double() - b.double()).abs().max()))


# ------------------------------------------------------------------------------------------------ panorama layer
def _pano_params(Hd, Fd, act, seed=1):
    g = torch.Generator().manual_seed(seed)
    shapes = [(3 * Hd, Hd), (3 * Hd,), (Hd, Hd), (Hd,), (Fd, Hd), (Fd,), (Hd, Fd), (Hd,), (Hd,), (Hd,), (Hd,), (Hd,)]
    ps = [torch.nn.Parameter((torch.randn(*s, generator=g) * 0.03).cuda()) for s in shapes]
    for i in (8, 10):
        ps[i].data.add_(1.0)
    return ps


def run_pano(K, x, kmask, dy, params, rt):
    from bevbert_b200 import blocks as Bk
    xi = x.clone().requires_grad_(True)
    for p in params:
        p.grad = None
    rt.begin(True, seed=5)
    y = Bk.run_block(Bk.PanoLayerImpl(rt, H, 0.0, 0.0), [xi, kmask], params)
    y.backward(dy)
    torch.cuda.synchronize()
    return y.detach().clone(), xi.grad.clone(), [p.grad.clone() for p in params]


def pano_dead_vs_without(K, act, Fd=3072, seed=3):
    """(batch with panorama 2 fully padded, same batch without it) -> (run, run, live index)"""
    from bevbert_b200 import blocks as Bk
    g = torch.Generator().manual_seed(seed)
    N, V = len(PANO_LENS), 36
    x = (torch.randn(N, V, HD, generator=g) * 0.5).to(act).cuda()
    dy = (torch.randn(N, V, HD, generator=g) * 0.1).to(act).cuda()
    live = [i for i, n in enumerate(PANO_LENS) if n > 0]
    dy[[i for i in range(N) if i not in live]] = 0
    km = _kmask("pano", N, V, g).cuda()
    params = _pano_params(HD, Fd, act)
    rt = Bk.Runtime()
    a = run_pano(K, x, km, dy, params, rt)
    b = run_pano(K, x[live].contiguous(), km[live].contiguous(), dy[live].contiguous(), params, rt)
    return a, b, live


def test_pano_layer_dead_panorama_fp32_arm(K, monkeypatch):
    """PanoLayerImpl (the Python composition) in the fp32 arm: a panorama with no valid view changes nothing for the
    others -- their outputs and input gradients, and every weight gradient -- and its own rows stay finite"""
    monkeypatch.setattr(K, "FLASH", False)
    prev = K.set_precision(True)
    try:
        (ya, dxa, ga), (yb, dxb, gb), live = pano_dead_vs_without(K, F32)
    finally:
        K.set_precision(prev)
    assert bool(torch.isfinite(ya).all()) and bool(torch.isfinite(dxa).all()), "rows of the dead panorama not finite"
    for name, a, b in [("y", ya[live], yb), ("dx", dxa[live], dxb)] + [("grad %d" % i, a, b) for i, (a, b) in
                                                                           enumerate(zip(ga, gb))]:
        assert bool(torch.isfinite(a).all()), name
        tol = 1e-5 * float(b.abs().max()) + 1e-30
        assert float((a - b).abs().max()) <= tol, "%s: max diff %g, tolerance %g" % (
            name, float((a - b).abs().max()), tol)


@pytest.mark.parametrize("fused", ["0", "512"])
def test_native_unfused_pano_layer_dead_panorama(fused):
    """bb_pano_fwd / _bwd with BB_FLASH=0 (and the fused-scores kernel off / on) in a process of its own: a dead
    panorama gives finite rows, the same results as the Python composition, and the other panoramas' results"""
    env = dict(os.environ, BB_FLASH="0", BB_FUSED_SCORES_MAX=fused)
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] +
                                        ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, "-s", os.path.abspath(__file__), "native_pano"], env=env, capture_output=True,
                       text=True, timeout=1200)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stderr[-6000:]


def _native_pano():
    from bevbert_b200 import kernels as K
    from helpers import rel_l2
    assert not K.FLASH and K.native_sublayers()
    outs = {}
    for native in (True, False):
        K.native_sublayers = (lambda n=native: n)
        outs[native] = pano_dead_vs_without(K, BF)
    (ya, dxa, ga), (yb, dxb, gb), live = outs[True]
    (yp, dxp, gp), _, _ = outs[False]
    assert bool(torch.isfinite(ya).all()) and bool(torch.isfinite(dxa).all()), "rows of the dead panorama not finite"
    assert torch.equal(ya, yp) and torch.equal(dxa, dxp), "native executor differs from the Python composition"
    for a, b in zip(ga, gp):
        assert bool(torch.isfinite(a).all()) and rel_l2(a, b) < 1e-4
    assert rel_l2(ya[live], yb) < 1e-3 and rel_l2(dxa[live], dxb) < 1e-2
    for a, b in zip(ga, gb):
        assert rel_l2(a, b) < 1e-2
    print("native unfused pano layer with a dead panorama: ok (BB_FUSED_SCORES_MAX=%d)" % K.FUSED_SCORES_MAX_KEYS)


if __name__ == "__main__":
    {"native_pano": _native_pano}[sys.argv[1]]()
