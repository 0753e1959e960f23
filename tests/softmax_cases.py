"""Case tables, guarded buffers, fp64 references and a-priori per-element error bounds for the unfused attention path:
bb_softmax_fwd / bb_softmax_bwd (csrc/rowops.cu) in both activation types and the fused-scores kernel bb_attn_scores
(csrc/attn_scores.cu, bf16).  Used by tests/test_softmax_gpu.py, tests/test_attn_scores_gpu.py and, against the torch
restatement in tests/emu_kernels.py, by tests/test_softmax_harness_cpu.py.  Buffers, the checker and the bf16 output
term come from tests/rowops_cases.py; the dropout decisions from drop_masks.softmax_keep.

Contract.  x = s + kmask + bias (s = alpha Q K^T for bb_attn_scores); P = softmax over the nk keys of a row,
Pd = keep(seed, row * ld + key) ? P scale : 0; a row whose keys are all -inf gives P = Pd = 0 (as the flash cores do),
so its dS and its share of dbias are 0.  dS = out_scale P o (g - sum_k P g), g = keep ? dP scale : 0, and
dbias (B, nq, nk) += sum over heads of P o (g - sum P g).  Columns [nk, ld) of P, Pd and dS are written as exact zeros.

Bounds (u = 2^-24, gamma_k = 1.01 k u, E(y) = (2 + 1.173 |y|) 2^-23 the relative error of __expf at argument y <= 0
by the CUDA programming guide's 2 + floor(|1.173 y|) ulp).  Per key, with y = x - max x:
* argument error d_x: bb_softmax_fwd rounds s + kmask and then + bias: 1.01 u ([kmask] |s + kmask| + [bias] |x|).
  bb_attn_scores: the wgmma dot product of 64 exact bf16 products in any order, each addition within one fp32 ulp
  (truncation included): 64 2^-23 alpha sum_i |q_i k_i|; then fmaf(s, alpha, kmask) (one rounding, u |alpha s + km|)
  and + bias (u |x|).
* exponential: rho = 1.01 (d_x + u |y|) + 1.01 E(y) (the subtraction of the row maximum rounds; a common error of the
  maximum cancels in the ratio).
* sum of exponentials: bb_softmax_fwd adds MAXE terms per lane (MAXE = 4 / 16 / 32 for ld <= 128 / 512 / 1024) and
  then 5 shuffle levels, D = MAXE + 5.  bb_attn_scores keeps an online sum per thread over 16 keys of each of the
  nkb = ceil(nk / 64) key blocks, rescaled by __expf(old max - new max) when a block raises the maximum, then 2 quad
  levels: D = 16 nkb + 4, and each term carries the rescale error (nkb + 1)(2^-22 + 2u) + (1.173 2^-23 + u) |y|
  (the rescale arguments of a term telescope to at most |y|).  sigma = sum_k p_k rho_k (+ rescale) + gamma_D.
* P: relative p (rho + sigma + 2.01 u) (1 / sum and the product), plus 2^-125 absolute (__expf flushes results
  below the smallest normal), then the rounding to the output type (half an ulp for bf16).  Keys at -inf and dead
  rows must be exactly 0.  Pd: scale d_P + u P scale (p = 0.5: scale 2, exact).
* dS from the kernel's own P (or any P passed in): g = fl(dP scale) (u |g|; for bb_attn_scores dP = dO V^T carries
  64 2^-23 sum |dO_i V_i| scale).  dot = sum P g: bb_softmax_bwd D = MAXE + 6 (one more for an unfused product),
  bb_attn_scores D = 16 nkb + 3 (fmaf chain over the thread's keys, 2 quad levels):
  d_dot = sum |P| e_g + gamma_D sum |P g|.  d = P (g - dot): E_d = 1.01 |P| (e_g + d_dot + u |g - dot|) + u |d|;
  dS = fl(d out_scale): |out_scale| E_d + u |dS|, then the output rounding.
* dbias = init + sum over the H heads (atomics in any order, or in deterministic mode per-head partials summed in head
  order and added): sum_h E_d,h + gamma_H (|init| + sum_h |d_h|).

Every constant is derived from the kernels' order of operations, none is fitted (C of rowops_cases stays 1 for these
quantities).  The worst err / bound of each quantity measured on an H100 is listed in the module docstrings of
tests/test_softmax_gpu.py and tests/test_attn_scores_gpu.py.

Buffers.  Inputs a kernel must not read hold NaN: score / dP columns [nk, ld), Q / K / V / dO padding columns of the
separate-buffer layout and rows past nq / nk inside its sample stride, the padding columns of an unrelated Pin.
P, Pd, dS and dbias sit between NaN-sentinel guards (rowops_cases.Arena); P, Pd and dS start as the sentinel, so an
element left unwritten fails.  A failure names the first bad (b, h, row, col) or guard offset with got / expected.
"""
import math
from dataclasses import dataclass

import torch

import drop_masks as DM
import rowops_cases as R
from rowops_cases import Arena, check, check_exact, fin, gamma_

U = R.U
BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
SEED = 0xC0FFEE5EED5A1701           # >= 2^63, like the seeds DropState draws
RATIOS = R.RATIOS
E23 = 2.0 ** -23
NAN = float("nan")
SCORE_C = 64                        # wgmma dot-product term: dh additions of at most one ulp each


def drop_params(p):
    if p <= 0:
        return 0, 1.0
    return min(int(p * 4294967296.0), 4294967295), 1.0 / (1.0 - p)


def maxe(ld):
    return 4 if ld <= 128 else (16 if ld <= 512 else 32)


def round8(n):
    return (n + 7) // 8 * 8


def _f32(x):
    return float(torch.tensor(x, dtype=F32))


# ------------------------------------------------------------------------------------------------ masks
MASKS = ("none", "mix", "tail", "dead", "full10k")


def make_kmask(kind, B, nk, g):
    """(B, nk) additive key mask or None.  mix: random 0 / -10000; tail: -inf on the last third of the keys (at least
    one key stays); dead: sample 0 all -inf, the rest mixed; full10k: sample 0 all -10000, the rest with a -inf tail"""
    if kind == "none":
        return None
    km = torch.where(torch.rand(B, nk, generator=g) < 0.3, -10000.0, 0.0)
    km[:, 0] = 0.0                      # every live row keeps one unmasked key
    tail = max(1, nk - nk // 3)
    if kind == "tail":
        km.zero_()
        km[:, tail:] = -math.inf
    elif kind == "dead":
        km[0] = -math.inf
    elif kind == "full10k":
        km.zero_()
        km[:, tail:] = -math.inf
        km[0] = -10000.0
    return km.float()


# ------------------------------------------------------------------------------------------------ fp64 references
def fwd_ref(x, dx, sum_depth, rescale=None):
    """P of fp64 logits x (-inf allowed) with argument errors dx -> (P, bound of P before the output rounding).
    rescale(y, nkb): extra relative error of each term of the online sum (bb_attn_scores), or None."""
    live = torch.isfinite(x)
    m = torch.where(live, x, torch.full_like(x, -math.inf)).amax(-1, keepdim=True)
    dead = ~live.any(-1, keepdim=True)
    y = torch.where(live, x - torch.where(dead, torch.zeros_like(m), m), torch.full_like(x, -math.inf))
    e = torch.exp(y)
    S = e.sum(-1, keepdim=True)
    p = torch.where(dead, torch.zeros_like(e), e / torch.where(dead, torch.ones_like(S), S))
    ya = torch.where(live, y.abs(), torch.zeros_like(y))
    dxl = torch.where(live, dx, torch.zeros_like(dx))
    rho = 1.01 * (dxl + U * ya) + 1.01 * (2 + 1.173 * ya) * E23
    extra = rescale(ya) if rescale is not None else torch.zeros_like(ya)
    sigma = (p * (rho + extra)).sum(-1, keepdim=True) + gamma_(sum_depth)
    d = 1.01 * p * (rho + sigma + 2.01 * U) + 2.0 ** -125
    d = torch.where(live & ~dead, d, torch.zeros_like(d))
    return p, d


def drop_ref(p, d, keep, scale):
    sc = _f32(scale)
    pd = torch.where(keep, p * sc, torch.zeros_like(p))
    dd = torch.where(keep, sc * d + U * pd, torch.zeros_like(d))
    return pd, dd


def bwd_ref(P, g, eg, dot_depth, out_scale, H):
    """dS and its bound from P (fp64 values of the kernel's input) and g (fp64, dropout applied) with error eg.
    -> (dS, E_dS before the output rounding, d, E_d) over (B, H, nq, nk)"""
    Pa = P.abs()
    dot = (P * g).sum(-1, keepdim=True)
    ddot = (Pa * eg).sum(-1, keepdim=True) + gamma_(dot_depth) * (P * g).abs().sum(-1, keepdim=True)
    d = P * (g - dot)
    Ed = 1.01 * Pa * (eg + ddot + U * (g - dot).abs()) + U * d.abs()
    os_ = _f32(out_scale)
    ds = d * os_
    Eds = abs(os_) * Ed + U * ds.abs()
    return ds, Eds, d, Ed


def dbias_ref(init, d, Ed):
    H = d.shape[1]
    ref = init.double() + d.sum(1)
    return ref, Ed.sum(1) + gamma_(H) * (init.double().abs() + d.abs().sum(1))


# ------------------------------------------------------------------------------------------------ bb_softmax_fwd / _bwd
@dataclass(frozen=True)
class SmCase:
    ld: int
    nk: int
    B: int = 3
    H: int = 3
    nq: int = 7                     # B H nq = 63 = 8 * 8 - 1 rows; nq = 9 gives 81 = 8 * 10 + 1
    mask: str = "none"
    bias: bool = False
    p: float = 0.0
    out_scale: float = 0.125
    seed: int = 0

    @property
    def id(self):
        return "ld%d-nk%d-B%dH%dq%d-%s%s-p%g-os%g" % (self.ld, self.nk, self.B, self.H, self.nq, self.mask,
                                                    "-bias" if self.bias else "", self.p, self.out_scale)


LDS = (8, 128, 136, 512, 520, 1024)


def softmax_table():
    T = []
    i = 0
    for ld in LDS:
        for nk in sorted({1, max(1, ld - 7), ld}):
            T.append(SmCase(ld, nk, nq=(7, 9)[i % 2], mask=MASKS[i % len(MASKS)], bias=bool(i % 3 != 1),
                            p=(0.0, 0.1, 0.5)[i % 3], out_scale=(0.125, -1.75)[i % 2], seed=i))
            i += 1
    # the bucket boundaries with every mask and dropout probability
    for ld, nk in ((128, 121), (136, 129), (512, 505), (520, 513)):
        for mask in MASKS:
            for p in (0.0, 0.1, 0.5):
                T.append(SmCase(ld, nk, nq=(7, 9)[i % 2], mask=mask, bias=p != 0.1, p=p, out_scale=0.125, seed=i))
                i += 1
    # several samples and heads with a bias: the row -> (b, h, q) decomposition
    T.append(SmCase(448, 441, B=5, H=3, nq=11, mask="mix", bias=True, p=0.1, seed=i))       # 165 = 8 * 20 + 5
    T.append(SmCase(1024, 1019, B=3, H=5, nq=13, mask="dead", bias=True, p=0.5, seed=i + 1))
    return T


def softmax_inputs(case, device):
    g = torch.Generator().manual_seed(1000 + case.seed)
    B, H, nq, nk, ld = case.B, case.H, case.nq, case.nk, case.ld
    s = (torch.randn(B, H, nq, ld, generator=g) * 3.0).float()
    s[..., nk:] = NAN
    km = make_kmask(case.mask, B, nk, g)
    bias = (torch.randn(B, nq, nk, generator=g) * 0.5).float() if case.bias else None
    dp = torch.randn(B, H, nq, ld, generator=g).float()
    dp[..., nk:] = NAN
    init = (torch.randn(B, nq, nk, generator=g) * 0.1).float()
    return [t.to(device) if t is not None else None for t in (s, km, bias, dp, init)]


def run_softmax(case, act, impl, device):
    """forward, then backward from the forward's own P, of one case into guarded buffers -> (arena, inputs, outputs)"""
    import emu_kernels as E
    s, km, bias, dp, init = softmax_inputs(case, device)
    B, H, nq, nk, ld = case.B, case.H, case.nq, case.nk, case.ld
    th, sc = drop_params(case.p)
    A = Arena(device)
    sA = A.inp("scores", s)
    dpA = A.inp("dP", dp)
    P = A.out("P", (B, H, nq, ld), act)
    Pd = A.out("Pd", (B, H, nq, ld), act)
    dS = A.out("dS", (B, H, nq, ld), act)
    db = A.inp("dbias", init) if case.bias else None
    if impl == "gpu":
        R._call("bb_softmax_fwd", sA.data_ptr(), R._p(km), R._p(bias), B, H, nq, nk, ld, SEED, th, sc, P.data_ptr(),
                Pd.data_ptr())
        R._call("bb_softmax_bwd", P.data_ptr(), dpA.data_ptr(), B, H, nq, nk, ld, SEED, th, sc, case.out_scale,
                dS.data_ptr(), R._p(db))
    else:
        ep, epd = E.softmax_fwd(sA, km, bias, B, H, nq, nk, ld, (SEED, th, sc))
        P.copy_(ep)
        Pd.copy_(epd)
        dS.copy_(E.softmax_bwd(P, dpA, B, H, nq, nk, ld, (SEED, th, sc), case.out_scale, db))
    R._sync(device)
    return A, (s, km, bias, dp, init, P), (P, Pd, dS, db)


def softmax_logits(s, km, bias, nk):
    """fp64 x = s + kmask + bias and its argument error, (B, H, nq, nk)"""
    B = s.shape[0]
    s64 = s[..., :nk].double()
    x = s64.clone()
    dx = torch.zeros_like(x)
    if km is not None:
        x = x + km.double().view(B, 1, 1, nk)
        dx = dx + U * x.abs()
    if bias is not None:
        x = x + bias.double().view(B, 1, -1, nk)
        dx = dx + U * x.abs()
    return x, 1.01 * torch.nan_to_num(dx, nan=0.0, posinf=0.0)


def _keep(case, nk, ld, device, th):
    if not th:
        return torch.ones(case.B, case.H, case.nq, nk, dtype=torch.bool, device=device)
    return DM.softmax_keep(SEED, case.B, case.H, case.nq, nk, ld, th).to(device)


def check_softmax(case, act, A, ins, outs):
    s, km, bias, dp, init, Pb = ins
    P, Pd, dS, db = outs
    nk, ld = case.nk, case.ld
    bf = act == BF
    th, sc = drop_params(case.p)
    tag = "%s-%s" % (case.id, "bf16" if bf else "fp32")
    x, dx = softmax_logits(s, km, bias, nk)
    p, d = fwd_ref(x, dx, maxe(ld) + 5)
    check("softmax_fwd.P[%s]" % tag, P[..., :nk], p, fin(p, d, bf))
    keep = _keep(case, nk, ld, p.device, th)
    pd, dd = drop_ref(p, d, keep, sc)
    check("softmax_fwd.Pd[%s]" % tag, Pd[..., :nk], pd, fin(pd, dd, bf))
    # backward from the P it was given
    g = torch.where(keep, dp[..., :nk].double() * _f32(sc), torch.zeros_like(p))
    eg = U * g.abs()
    ds, Eds, dd_, Ed = bwd_ref(Pb[..., :nk].double(), g, eg, maxe(ld) + 6, case.out_scale, case.H)
    check("softmax_bwd.dS[%s]" % tag, dS[..., :nk], ds, fin(ds, Eds, bf))
    if db is not None:
        rdb, edb = dbias_ref(init, dd_, Ed)
        check("softmax_bwd.dbias[%s]" % tag, db, rdb, edb)
    check_pad_and_dead(tag, (P, Pd, dS), nk, x)
    if not th:
        check_exact("softmax_fwd.Pd = P without dropout[%s]" % tag, Pd, P)
    A.check_guards()


def check_zero(name, t):
    """every element == 0 (either sign: a zero times a negative out_scale is -0); NaN fails"""
    bad = (t.double() != 0).reshape(-1).nonzero()
    if bad.numel():
        f = int(bad[0])
        raise AssertionError("%s: %d bad elements; first at %s: got %r expected 0" % (
            name, bad.numel(), R._where(tuple(t.shape), f), float(t.reshape(-1)[f])))


def check_pad_and_dead(tag, outs, nk, x):
    """padding columns exactly 0; on rows whose keys are all -inf every column exactly 0"""
    dead = ~torch.isfinite(x).any(-1)
    for name, t in zip(("P", "Pd", "dS"), outs):
        if t.shape[-1] > nk:
            check_zero("%s columns [nk, ld)[%s]" % (name, tag), t[..., nk:])
        if bool(dead.any()):
            check_zero("%s of rows with every key at -inf[%s]" % (name, tag), t[dead])


# ------------------------------------------------------------------------------------------------ bb_attn_scores
@dataclass(frozen=True)
class AsCase:
    nq: int
    nk: int
    ldp: int
    B: int = 2
    H: int = 2
    layout: str = "sep"             # sep (own buffers, padded) | self (packed Q|K|V, ld 3 Hd) | cross (Q; packed K|V)
    mask: str = "none"
    bias: bool = False
    p: float = 0.0
    pin: str = "own"                # mode 1 reads the kernel's own P, or an unrelated bf16 P ("other")
    seed: int = 0

    @property
    def id(self):
        return "q%d-k%d-ldp%d-B%dH%d-%s-%s%s-p%g-%s" % (self.nq, self.nk, self.ldp, self.B, self.H, self.layout,
                                                       self.mask, "-bias" if self.bias else "", self.p, self.pin)


AS_NQ = (1, 63, 64, 65, 127, 128, 129, 441)
AS_NK = (1, 8, 63, 64, 65, 128, 441, 512)
PERSIST = (9, 12, 441, 64)          # B, H, nq, nk: 9 * 12 * 4 = 432 tiles >= 3 x 132 SMs


def ldps(nk):
    """round8(nk); round8(nk) + 8; 64 ceil(nk / 64) + 8 (an output block with no product block behind it)"""
    return (round8(nk), round8(nk) + 8, 64 * (-(-nk // 64)) + 8)


def scores_table():
    T = []
    i = 0
    for nq in AS_NQ:
        for nk in AS_NK:
            layout = "cross" if i % 3 == 1 else "sep"
            T.append(AsCase(nq, nk, ldps(nk)[i % 3], layout=layout, mask=MASKS[i % len(MASKS)], bias=i % 4 != 3,
                            p=(0.0, 0.1, 0.5)[i % 3], pin=("own", "other")[(i // 3) % 2], seed=i))
            i += 1
    for nk in (63, 65, 441):
        for j, ldp in enumerate(ldps(nk)):
            T.append(AsCase(129, nk, ldp, mask=MASKS[j + 1], bias=True, p=0.1, seed=i))
            i += 1
    for n in (1, 65, 129, 441):
        T.append(AsCase(n, n, ldps(n)[i % 3], layout="self", mask=MASKS[i % len(MASKS)], bias=True, p=0.1, seed=i))
        i += 1
    for mask in MASKS:
        T.append(AsCase(200, 300, 304, mask=mask, bias=True, p=0.5, pin="other", seed=i))
        i += 1
    B, H, nq, nk = PERSIST
    T.append(AsCase(nq, nk, 72, B=B, H=H, layout="self" if nq == nk else "sep", mask="dead", bias=True, p=0.1,
                    seed=i))
    T.append(AsCase(nq, nk, 64, B=B, H=H, layout="cross", mask="mix", bias=False, p=0.0, pin="other", seed=i + 1))
    return T


class Operands:
    """bf16 Q, K, V, dO in the case's layout: views whose first element is (sample 0, row 0, head 0, dim 0), their row
    strides and sample strides, and the fp64 (B, H, rows, 64) copies"""

    def __init__(self, case, device, g):
        B, H, nq, nk = case.B, case.H, case.nq, case.nk
        Hd = 64 * H
        self.A = A = Arena(device)

        def rnd(*shape, scale):
            return (torch.randn(*shape, generator=g) * scale).to(BF)
        q = rnd(B, nq, Hd, scale=1.0)
        k = rnd(B, nk, Hd, scale=1.0)
        v = rnd(B, nk, Hd, scale=1.0)
        do = rnd(B, nq, Hd, scale=1.0)
        if case.layout == "sep":
            def padded(t, rows_pad, col_pad, name):
                b, n, c = t.shape
                full = torch.full((b, n + rows_pad, c + col_pad), NAN, dtype=BF)
                full[:, :n, :c] = t
                return A.inp(name, full), c + col_pad, (n + rows_pad) * (c + col_pad)
            self.q, self.ldq, self.sq = padded(q, 3, 8, "Q")
            self.k, self.ldk, self.sk = padded(k, 5, 16, "K")
            self.v, self.ldv, self.sv = padded(v, 5, 24, "V")
            self.do, self.ldo, self.so = padded(do, 3, 8, "dO")
        elif case.layout == "self":
            assert nq == nk
            qkv = A.inp("QKV", torch.cat([q, k, v], -1))
            self.q, self.k, self.v = qkv, qkv.view(-1)[Hd:], qkv.view(-1)[2 * Hd:]
            self.ldq = self.ldk = self.ldv = 3 * Hd
            self.sq = self.sk = self.sv = nq * 3 * Hd
            self.do, self.ldo, self.so = A.inp("dO", do), Hd, nq * Hd
        else:
            self.q, self.ldq, self.sq = A.inp("Q", q), Hd, nq * Hd
            kv = A.inp("KV", torch.cat([k, v], -1))
            self.k, self.v = kv, kv.view(-1)[Hd:]
            self.ldk = self.ldv = 2 * Hd
            self.sk = self.sv = nk * 2 * Hd
            self.do, self.ldo, self.so = A.inp("dO", do), Hd, nq * Hd
        heads = lambda t, n: t.double().view(B, n, H, 64).permute(0, 2, 1, 3).to(device)
        self.qh, self.kh, self.vh, self.doh = heads(q, nq), heads(k, nk), heads(v, nk), heads(do, nq)


def scores_inputs(case, device):
    g = torch.Generator().manual_seed(2000 + case.seed)
    ops = Operands(case, device, g)
    B, nq, nk, ldp = case.B, case.nq, case.nk, case.ldp
    km = make_kmask(case.mask, B, nk, g)
    bias = (torch.randn(B, nq, nk, generator=g) * 0.5).float() if case.bias else None
    init = (torch.randn(B, nq, nk, generator=g) * 0.1).float()
    other = torch.rand(B, case.H, nq, ldp, generator=g).double()
    other = (other / other[..., :nk].sum(-1, keepdim=True)).to(BF)   # a bf16 P-like matrix, not the kernel's P
    other[..., nk:] = NAN                                            # columns the kernel reads in pairs but never uses
    return ops, [t.to(device) if t is not None else None for t in (km, bias, init, other)]


def _scores_args(ops, case, mode):
    from bevbert_b200 import _lib
    a = _lib.AttnScoresArgs()
    if mode == 0:
        a.A, a.lda, a.a_s1, a.a_s2 = ops.q.data_ptr(), ops.ldq, 64, ops.sq
        a.Bm, a.ldb, a.b_s1, a.b_s2 = ops.k.data_ptr(), ops.ldk, 64, ops.sk
        a.alpha, a.out_scale = 0.125, 1.0
    else:
        a.A, a.lda, a.a_s1, a.a_s2 = ops.do.data_ptr(), ops.ldo, 64, ops.so
        a.Bm, a.ldb, a.b_s1, a.b_s2 = ops.v.data_ptr(), ops.ldv, 64, ops.sv
        a.alpha, a.out_scale = 1.0, 0.125
    a.B, a.H, a.nq, a.nk, a.ldp, a.mode = case.B, case.H, case.nq, case.nk, case.ldp, mode
    return a


def _strided_heads(t, B, H, n, ld, s2):
    return torch.as_strided(t, (B, H, n, 64), (s2, 64, ld, 1), t.storage_offset())


def run_scores(case, impl, device):
    """mode 0 then mode 1 of bb_attn_scores into guarded buffers -> (arena, inputs, outputs)"""
    import ctypes as C
    import emu_kernels as E
    ops, (km, bias, init, other) = scores_inputs(case, device)
    A = ops.A
    B, H, nq, nk, ldp = case.B, case.H, case.nq, case.nk, case.ldp
    th, sc = drop_params(case.p)
    P = A.out("P", (B, H, nq, ldp), BF)
    Pd = A.out("Pd", (B, H, nq, ldp), BF)
    dS = A.out("dS", (B, H, nq, ldp), BF)
    Pin = P if case.pin == "own" else A.inp("Pin", other)
    db = A.inp("dbias", init) if case.bias else None
    if impl == "gpu":
        from bevbert_b200 import _lib
        lib = _lib.load()
        a = _scores_args(ops, case, 0)
        a.kmask, a.bias = R._p(km), R._p(bias)
        a.seed, a.thresh, a.scale = SEED, th, sc
        a.P, a.Pd = P.data_ptr(), Pd.data_ptr()
        from bevbert_b200 import kernels as K
        _lib.check(lib.bb_attn_scores(C.byref(a), K._stream()), "bb_attn_scores mode 0")
        b = _scores_args(ops, case, 1)
        b.seed, b.thresh, b.scale = SEED, th, sc
        b.Pin, b.dS, b.dbias = Pin.data_ptr(), dS.data_ptr(), R._p(db)
        _lib.check(lib.bb_attn_scores(C.byref(b), K._stream()), "bb_attn_scores mode 1")
    else:
        # the unfused pair it replaces: fp32 scores, then the softmax restatement
        qh = _strided_heads(ops.q, B, H, nq, ops.ldq, ops.sq).float()
        kh = _strided_heads(ops.k, B, H, nk, ops.ldk, ops.sk).float()
        S = torch.full((B, H, nq, ldp), NAN)
        S[..., :nk] = (qh @ kh.transpose(-1, -2)) * 0.125
        ep, epd = E.softmax_fwd(S, km, bias, B, H, nq, nk, ldp, (SEED, th, sc))
        P.copy_(ep)
        Pd.copy_(epd)
        doh = _strided_heads(ops.do, B, H, nq, ops.ldo, ops.so).float()
        vh = _strided_heads(ops.v, B, H, nk, ops.ldv, ops.sv).float()
        dP = torch.full((B, H, nq, ldp), NAN)
        dP[..., :nk] = doh @ vh.transpose(-1, -2)
        dS.copy_(E.softmax_bwd(Pin, dP, B, H, nq, nk, ldp, (SEED, th, sc), 0.125, db))
    R._sync(device)
    return A, (ops, km, bias, init, Pin), (P, Pd, dS, db)


def check_scores(case, A, ins, outs):
    ops, km, bias, init, Pin = ins
    P, Pd, dS, db = outs
    B, nq, nk, ldp = case.B, case.nq, case.nk, case.ldp
    th, sc = drop_params(case.p)
    tag = case.id
    nkb = -(-nk // 64)
    S = ops.qh @ ops.kh.transpose(-1, -2)
    aS = (ops.qh.abs() @ ops.kh.abs().transpose(-1, -2))
    x = 0.125 * S
    dx = 0.125 * SCORE_C * E23 * aS
    if km is not None:
        x = x + km.double().view(B, 1, 1, nk)
        dx = dx + U * x.abs()
    if bias is not None:
        x = x + bias.double().view(B, 1, nq, nk)
        dx = dx + U * x.abs()
    dx = 1.01 * torch.nan_to_num(dx, nan=0.0, posinf=0.0)
    resc = lambda ya: (nkb + 1) * (2 * E23 + 2 * U) + (1.173 * E23 + U) * ya
    p, d = fwd_ref(x, dx, 16 * nkb + 4, resc)
    check("attn_scores.P[%s]" % tag, P[..., :nk], p, fin(p, d, True))
    keep = _keep(case, nk, ldp, p.device, th)
    pd, dd = drop_ref(p, d, keep, sc)
    check("attn_scores.Pd[%s]" % tag, Pd[..., :nk], pd, fin(pd, dd, True))
    if not th:
        check_exact("attn_scores.Pd = P without dropout[%s]" % tag, Pd, P)
    dP = ops.doh @ ops.vh.transpose(-1, -2)
    adP = ops.doh.abs() @ ops.vh.abs().transpose(-1, -2)
    scf = _f32(sc)
    g = torch.where(keep, dP * scf, torch.zeros_like(dP))
    eg = torch.where(keep, SCORE_C * E23 * adP * scf * 1.01 + U * g.abs(), torch.zeros_like(dP))
    ds, Eds, dd_, Ed = bwd_ref(Pin[..., :nk].double(), g, eg, 16 * nkb + 3, 0.125, case.H)
    check("attn_scores.dS[%s]" % tag, dS[..., :nk], ds, fin(ds, Eds, True))
    if db is not None:
        rdb, edb = dbias_ref(init, dd_, Ed)
        check("attn_scores.dbias[%s]" % tag, db, rdb, edb)
    check_pad_and_dead(tag, (P, Pd) + ((dS,) if case.pin == "own" else ()), nk, x)
    if case.pin != "own" and ldp > nk:
        check_zero("dS columns [nk, ldp)[%s]" % tag, dS[..., nk:])
    A.check_guards()


# ------------------------------------------------------------------------------------------------ planted faults
def plant(kind, case, act, A, ins, outs):
    """corrupt one output of a correct run the way a faulty kernel would (the checker must then fail)"""
    s, km, bias, dp, init, Pb = ins
    P, Pd, dS, db = outs
    nk = case.nk
    if kind == "ulp":                  # one bf16 output one ulp away from its value, away from the reference
        x, dx = softmax_logits(s, km, bias, nk)
        p, _ = fwd_ref(x, dx, maxe(case.ld) + 5)
        idx = R._where(tuple(p.shape), int(p.reshape(-1).argmax()))
        bits = R.bits(P)
        bits[idx] += 1 if float(P[idx]) >= float(p[idx]) else -1
    elif kind == "mask":               # Pd of another seed's mask (p = 0.5: the kept values are exact either way)
        th, sc = drop_params(case.p)
        other = DM.softmax_keep(SEED ^ 1, case.B, case.H, case.nq, nk, case.ld, th).to(P.device)
        Pd[..., :nk] = torch.where(other, (P[..., :nk].float() * sc).to(P.dtype), torch.zeros_like(P[..., :nk]))
    elif kind == "pad":                # a padding column left unwritten
        P[0, 0, 0, nk] = R.sentinel_like(P[0, 0, 0, nk:nk + 1])[0]
    elif kind == "dead_nan":           # NaN on a row whose keys are all -inf
        P[0, 0, 0, :] = NAN
    elif kind == "past_end":           # one write past the end of dS
        full, st, n = A.bufs["dS"]
        full[st + n] = 0
    elif kind == "dbias_init":         # dbias written instead of accumulated
        db.sub_(init)
    else:
        raise ValueError(kind)


PLANTS = {"ulp": SmCase(136, 129, mask="mix", bias=True, p=0.1, seed=1),
          "mask": SmCase(136, 129, mask="mix", p=0.5, seed=2),
          "pad": SmCase(136, 129, mask="tail", seed=3),
          "dead_nan": SmCase(128, 121, mask="dead", seed=4),
          "past_end": SmCase(8, 5, mask="none", bias=True, seed=5),
          "dbias_init": SmCase(128, 121, mask="mix", bias=True, seed=6)}
