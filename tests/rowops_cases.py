"""Case tables, guarded buffers, fp64 references and a-priori per-element error bounds for the row kernels
(csrc/rowops.cu) and the multi-tensor optimizer kernels (csrc/optim.cu).  Used by tests/test_rowops_gpu.py,
tests/test_optim_kernels_gpu.py and, against the torch restatement in tests/emu_kernels.py, by
tests/test_rowops_harness_cpu.py.

Every output lives between guard regions of G elements filled with a NaN sentinel bit pattern; the body of an output
that the kernel overwrites is filled with the same sentinel, so an element left unwritten is a NaN and fails its check,
and a write past the end changes a guard.  The checker names the first failing element (row, column) with got /
expected / bound.

Bounds.  u = 2^-24.  sum_k denotes an fp32 summation whose longest chain of additions has k roundings; its error is at
most k u (1 + k u) sum |terms| (written k u' below, the factor 1.01 covers the higher-order term).  A bf16 output of
fp64 value y with fp32 error bound d is bounded by d + ulp/2 of (|y| + d); an fp32 output by d.  Each kernel's order:

* layernorm_fwd: z = x (+ res), one rounding u|z| with res; per lane a sequential sum of its 8 nc values
  (nc = ceil(H/256) chunks), then five shuffle steps: k_s = 8 nc + 4.  d_mu = (k_s u' S + [res] u S) / H + u|mu|,
  S = sum |z|.  var: q = sum fma(d, d, q) over d = fl(z^ - mu^), k_q = 8 nc + 6, plus the exact effect of the mean and
  z errors, A = 2 sum |z - mu| a_i + sum (a_i + d_mu)^2 (a_i = [res] u |z_i|); d_Q = A + k_q u' (Q + A);
  d_V = d_Q / H + u Q/H + u V (the division and the + eps), V = Q/H + eps; rstd = 1 / sqrtf(V) (two correctly
  rounded operations): rho = d_V / 2V (1 + d_V / V) + 2.01 u.  y = fl(fl(fl(z - mu) * rstd) * gamma + beta):
  E_t = (a + d_mu) rstd (1 + rho) + |x^| rho + 2.01 u (|x^| + (a + d_mu) rstd),
  d_y = |gamma| E_t + 2.01 u (|gamma| (|x^| + E_t) + |beta|).
  Constant rows holding a bf16 value are exact: every partial sum k c (k <= 1024) has at most 19 significant bits, so
  y must equal beta (rounded to the activation type).
* layernorm_bwd with the kernel's own fp32 mean / rstd as inputs: E_xh = a rstd + 2.01 u |x^|;
  d_c1 = (k_s + 1) u' sum |g| / H + u |c1|, d_c2 = (sum |g| E_xh + (k_s + 2) u' sum |g x^|) / H + u |c2|,
  E_dz = rstd (u |g| + d_c1 + E_xh |c2| + |x^| d_c2 + E_xh d_c2 + 3.01 u (|g| + |c1| + |x^ c2|)) + u |dz|.
  dgamma / dbeta / dxsum: per lane over the warp's rows (ceil(rows / 8 grid)), eight warps in shared memory, then one
  atomic (or det_reduce term) per block, grid = min(ceil(rows / 8), #SMs), plus the add to the buffer's initial
  value: depth D = ceil(rows / 8 grid) + 9 + grid; d = sum of the per-term errors + D u' sum |terms|.
* colsum: per thread a sequential sum (pairs of pairs in the unrolled part), eight row-threads, then one atomic or
  det_reduce term per row-block (gy = min(ceil(rows / 64), 64)): D = ceil(rows / 8 gy) + 12 + gy.
* segment_wsum: fma over the segment's entries in order: len u' sum |w v|.  Backward: one rounded product and one
  atomic per entry: u sum |w g| + (count + 1) u' (|init| + sum |w g|).
* gelu_bwd: erff within 2 ulp, __expf within 2^-21 relative plus the rounding of its argument
  (-x^2/2, relative 1.5 u x^2): d = |g| (3 u + |x pdf| (2^-21 + 1.5 u x^2 + 4 u)) + u |g gelu'(x)|.
* softmax_xent: __expf terms within e_i = 2^-20 + 4 u |x_i - max|; sum depth D = ceil(V / 256) + 13;
  d_s / s = max e_i + D u'.  loss: d_s / s (1.01) + 2 u |ln s| + u |ln s + max| + u |loss|;
  dlogits: |gs| (p_i (e_i + 1.01 d_s/s + 2.01 u) + u |p_i - onehot_i| + 2^-125) + u |dlogit| (2^-125: __expf
  flushes results below the smallest normal to zero).
* AdamW (one step from the kernel's own previous state; coefficient computed in fp64 from the kernel's own sumsq):
  d_coef = 5.01 u coef when clipping is active, else 0; E_g = |g| d_coef + u |g'|;
  E_m = (1 - b1) E_g + 2.01 u (b1 |m| + (1 - b1) |g'|); E_v = 2 (1 - b2) |g'| E_g + 3.01 u (b2 v + (1 - b2) g'^2);
  E_den = min(E_v / 2 sqrt v', sqrt E_v) + u sqrt v' + u (sqrt v' + eps); q = m' / den: E_q = (E_m + |q| E_den) / den
  + u |q|; p' = p - step q: E_p' = step E_q + u step |q| + u |p'|; p'' = p' - decay p':
  E_p'' = (1 + decay) E_p' + 2.01 u (decay |p'| + |p''|).  sumsq: D = 16 + 9 + chunks, D u' sum g^2.

Bounds are multiplied by the per-quantity constant in C (all 1: the bounds above are derived, not fitted).  The worst
err / bound of every quantity, measured on an H100 80GB HBM3 at 700 W in both precision modes, is listed in the module
docstring of tests/test_rowops_gpu.py: at most 1.0 for bf16 outputs (the half-ulp term), 0.03 to 0.95 elsewhere.
"""
import math
from dataclasses import dataclass

import torch

U = 2.0 ** -24
G = 64                                       # guard elements on each side (128 bytes of bf16, 256 of fp32)
SENT = {torch.float32: (torch.int32, 0x7FA5A5A5), torch.bfloat16: (torch.int16, 0x7FA5)}
BF = torch.bfloat16
F32 = torch.float32
C = {}                                       # per-quantity multiplier of the derived bound (default 1)
RATIOS = {}                                  # quantity -> worst err / bound seen in this process


# ------------------------------------------------------------------------------------------------ buffers
class Arena:
    """Guarded fp32 / bf16 buffers on one device.  `out` fills body and guards with the sentinel; `inp` copies a
    tensor into the body.  `offset` shifts the body by that many elements (misaligned views)."""

    def __init__(self, device):
        self.device = device
        self.bufs = {}

    def _alloc(self, name, shape, dtype, offset=0):
        n = math.prod(shape)
        full = torch.empty(G + offset + n + G, dtype=dtype, device=self.device)
        it, pat = SENT[dtype]
        full.view(it).fill_(pat)
        self.bufs[name] = (full, G + offset, n)
        return full[G + offset:G + offset + n].view(shape)

    def out(self, name, shape, dtype, offset=0):
        return self._alloc(name, tuple(shape), dtype, offset)

    def inp(self, name, t, dtype=None, offset=0):
        v = self._alloc(name, tuple(t.shape), dtype or t.dtype, offset)
        v.copy_(t)
        return v

    def check_guards(self):
        for name, (full, s, n) in self.bufs.items():
            it, pat = SENT[full.dtype]
            b = full.view(it)
            for part, lo in ((b[:s], 0), (b[s + n:], s + n)):
                bad = (part != pat).nonzero()
                if bad.numel():
                    raise AssertionError("%s: guard overwritten, bad elements at %d positions, first at element %d "
                                         "relative to the buffer" % (name, bad.numel(), lo + int(bad[0]) - s))


def sentinel_like(t):
    it, pat = SENT[t.dtype]
    return torch.full(t.shape, pat, dtype=it, device=t.device).view(t.dtype)


# ------------------------------------------------------------------------------------------------ checker
def half_ulp_bf16(a):
    """half the bf16 spacing at |a| (fp64), subnormals included"""
    _, e = torch.frexp(a.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(a), e - 9)


def fin(y, d, bf):
    """bound of an output of fp64 value y, fp32 error d, stored bf16 (bf) or fp32"""
    return d + half_ulp_bf16(y.abs() + d) if bf else d


def _where(shape, flat):
    idx = []
    for s in reversed(shape):
        idx.append(flat % s)
        flat //= s
    return tuple(reversed(idx))


def check(name, got, exp, bound):
    """|got - exp| <= C[name] * bound element by element (NaN fails).  Returns and records the worst ratio."""
    g, e = got.double().reshape(exp.shape), exp.double()
    b = bound.double().expand(e.shape) * C.get(name.split("[")[0], 1.0)
    err = (g - e).abs()
    ok = err <= b
    if not bool(ok.all()):
        bad = (~ok).reshape(-1).nonzero()
        f = int(bad[0])
        w = _where(tuple(e.shape), f)
        raise AssertionError("%s: %d bad elements; first at %s: got %.9g expected %.9g bound %.3g" % (
            name, bad.numel(), w, float(g.reshape(-1)[f]), float(e.reshape(-1)[f]), float(b.reshape(-1)[f])))
    r = float((err / b.clamp_min(1e-300)).max()) if err.numel() else 0.0
    key = name.split("[")[0]
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    return r


def bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float64: torch.int64}[t.dtype])


def check_exact(name, got, exp):
    """bit for bit (dtype and every bit pattern)"""
    assert got.dtype == exp.dtype, (name, got.dtype, exp.dtype)
    g, e = bits(got.contiguous()).reshape(-1), bits(exp.contiguous().to(got.device)).reshape(-1)
    bad = (g != e).nonzero()
    if bad.numel():
        f = int(bad[0])
        raise AssertionError("%s: %d bad elements; first at %s: got %r expected %r" % (
            name, bad.numel(), _where(tuple(exp.shape), f), float(got.reshape(-1)[f]), float(exp.reshape(-1)[f])))


def gamma_(k):
    return k * U * 1.01


# ------------------------------------------------------------------------------------------------ LayerNorm
def ln_inputs(case, device):
    """x (xdt), residual (act) | None, gamma, beta (f32); adversarial rows per case.adv"""
    g = torch.Generator().manual_seed(case.seed)
    rows, H = case.rows, case.H
    x = torch.randn(rows, H, generator=g, dtype=torch.float64)
    if case.adv == "offset":                      # |mean| >> std, as after many residual adds
        x = x + 64.0 if case.xdt == BF else x * 0.5 + 300.0
    elif case.adv == "outlier":
        x[:, H // 3] = 3e3
    elif case.adv == "onehot":
        x.zero_()
        x[:, H - 1] = 1.5
    elif case.adv == "const":
        x = torch.full((rows, H), 0.8125, dtype=torch.float64)
    x = x.to(case.xdt)
    res = (torch.randn(rows, H, generator=g) * 0.5).to(case.act) if case.res else None
    if case.adv == "const" and case.res:
        res.fill_(0.25)
    gam = (torch.rand(H, generator=g) + 0.5).float()
    bet = (torch.randn(H, generator=g) * 0.1).float()
    return [t.to(device) if t is not None else None for t in (x, res, gam, bet)]


def ln_fwd_ref(x, res, gamma, beta, eps):
    z = x.double() + (res.double() if res is not None else 0.0)
    rows, H = z.shape
    nc = -(-H // 256)
    mu = z.mean(1)
    d = z - mu[:, None]
    Q = (d * d).sum(1)
    eps64 = float(torch.tensor(eps, dtype=F32))
    V = Q / H + eps64
    rs = V.rsqrt()
    xh = d * rs[:, None]
    y = xh * gamma.double() + beta.double()
    az = z.abs()
    S = az.sum(1)
    a = U * az if res is not None else torch.zeros_like(az)
    dmu = (gamma_(8 * nc + 4) * S + (U * S if res is not None else 0.0)) / H + U * mu.abs()
    A = 2 * (d.abs() * a).sum(1) + ((a + dmu[:, None]) ** 2).sum(1)
    dQ = A + gamma_(8 * nc + 6) * (Q + A)
    dV = dQ / H + U * Q / H + U * V
    rho = dV / (2 * V) * (1 + dV / V) + 2.01 * U
    ad = a + dmu[:, None]
    Et = ad * rs[:, None] * (1 + rho[:, None]) + xh.abs() * rho[:, None] + 2.01 * U * (xh.abs() + ad * rs[:, None])
    ga, ba = gamma.double().abs(), beta.double().abs()
    dy = ga * Et + 2.01 * U * (ga * (xh.abs() + Et) + ba)
    return dict(y=y, mean=mu, rstd=rs, d_y=dy, d_mean=dmu, d_rstd=rho * rs)


def ln_bwd_ref(dy, x, res, gamma, mean, rstd, grid, init):
    """fp64 backward from the kernel's fp32 mean / rstd; init = initial (dgamma, dbeta, dxsum) buffer values"""
    z = x.double() + (res.double() if res is not None else 0.0)
    rows, H = z.shape
    nc = -(-H // 256)
    d = dy.double()
    rs = rstd.double()[:, None]
    xh = (z - mean.double()[:, None]) * rs
    ga = gamma.double()
    g = d * ga
    c1 = g.mean(1, keepdim=True)
    c2 = (g * xh).mean(1, keepdim=True)
    dz = rs * (g - c1 - xh * c2)
    a = U * z.abs() if res is not None else torch.zeros_like(z)
    Exh = a * rs + 2.01 * U * xh.abs()
    dc1 = gamma_(8 * nc + 5) * g.abs().sum(1, keepdim=True) / H + U * c1.abs()
    dc2 = ((g.abs() * Exh).sum(1, keepdim=True) + gamma_(8 * nc + 6) * (g * xh).abs().sum(1, keepdim=True)) / H + \
        U * c2.abs()
    Edz = rs * (U * g.abs() + dc1 + Exh * c2.abs() + xh.abs() * dc2 + Exh * dc2 +
                3.01 * U * (g.abs() + c1.abs() + (xh * c2).abs())) + U * dz.abs()
    depth = -(-rows // (8 * grid)) + 9 + grid
    i_g, i_b, i_x = (t.double() for t in init)
    out = dict(dz=dz, d_dz=Edz)
    out["dgamma"] = i_g + (d * xh).sum(0)
    out["d_dgamma"] = (d.abs() * Exh).sum(0) + gamma_(depth) * (i_g.abs() + (d * xh).abs().sum(0))
    out["dbeta"] = i_b + d.sum(0)
    out["d_dbeta"] = gamma_(depth) * (i_b.abs() + d.abs().sum(0))
    out["dxsum"] = i_x + dz.sum(0)
    out["d_dxsum"] = Edz.sum(0) + gamma_(depth) * (i_x.abs() + dz.abs().sum(0))
    return out


@dataclass(frozen=True)
class LnCase:
    H: int
    rows: int
    xdt: torch.dtype = BF
    res: bool = True
    eps: float = 1e-12
    adv: str = ""
    act: torch.dtype = BF           # activation type of the precision mode (residual, y, dres)
    seed: int = 0

    @property
    def id(self):
        return "H%d-r%d-x%s%s-e%g%s" % (self.H, self.rows, "f32" if self.xdt == F32 else "bf16",
                                      "-res" if self.res else "", self.eps, "-" + self.adv if self.adv else "")


LN_H = (8, 64, 248, 256, 264, 512, 760, 768, 776, 1016, 1024)
ROWS_SMS = 8 * 132                 # 8 * #SMs on an H100 SXM: one row per warp of a full first grid; +1 wraps


def ln_table(act=BF, big=True):
    T = []
    for i, H in enumerate(LN_H):
        for rows in (1, 7, ROWS_SMS, ROWS_SMS + 1):
            T.append(LnCase(H, rows, BF if rows % 2 else F32, bool(i % 2) or rows == 7, 1e-12 if i % 3 else 1e-5,
                            act=act, seed=i * 10 + rows % 10))
    for H in (264, 768, 1024):
        for adv in ("offset", "outlier", "onehot", "const"):
            for xdt in (BF, F32):
                T.append(LnCase(H, 37, xdt, adv != "onehot", 1e-12 if xdt == BF else 1e-5, adv, act=act, seed=3))
    if big:
        for H in (768, 1024, 264):
            T.append(LnCase(H, 20000, BF, True, 1e-12, act=act, seed=5))
        T.append(LnCase(1016, 20001, F32, False, 1e-5, act=act, seed=6))
    return T


# bf16 product mode: (dy_f32, x_f32, dx_f32) pairings bb_layernorm_bwd accepts; the fp32 mode accepts (1, 1, 1) only
LN_BWD_PAIRS = ((0, 0, 0), (0, 1, 1), (1, 0, 0), (1, 1, 1), (0, 0, 1), (0, 1, 0))


def ln_bwd_table(act=BF):
    T = []
    pairs = LN_BWD_PAIRS if act == BF else ((1, 1, 1),)
    for i, H in enumerate(LN_H):
        for j, rows in enumerate((1, 7, ROWS_SMS, ROWS_SMS + 1, 5000)):
            p = pairs[(i + j) % len(pairs)]
            T.append((LnCase(H, rows, F32 if p[1] else BF, bool((i + j) % 2), act=act, seed=i + 7 * j), p))
    for H in (768, 1024):
        for p in pairs:
            T.append((LnCase(H, 20000, F32 if p[1] else BF, True, act=act, seed=11), p))
    for adv in ("offset", "outlier", "const"):
        T.append((LnCase(1024, 37, F32 if pairs[0][1] else BF, True, adv=adv, act=act, seed=4), pairs[0]))
    return T


# ------------------------------------------------------------------------------------------------ colsum
COLSUM_N = (8, 40, 250, 256, 257, 2304, 3072)
# 1, 7, 64 rows; 200 (4 row-blocks, 6-7 rows per thread: remainders 2 and 3 of the 4-way loop); 2661 and 3585 (42 and
# 57 blocks); 4096 (the first count at the 64-block cap), 4097, 20000 (capped: 39-40 rows per thread, remainder 3)
COLSUM_ROWS = (1, 7, 64, 200, 2661, 3585, 4097, 20000)


def colsum_table():
    T = []
    for i, N in enumerate(COLSUM_N):
        for ld in (N, N + 3, N + 8):
            for j, rows in enumerate(COLSUM_ROWS):
                if rows * ld > 12_000_000 or (rows >= 2661 and (i + j) % 2):
                    continue
                T.append((N, ld, rows))
    T.append((3072, 3072, 20000 // 8))
    return T


def colsum_ref(x, N, init):
    rows = x.shape[0]
    gy = min(-(-rows // 64), 64)
    depth = -(-rows // (8 * gy)) + 12 + gy
    s = x[:, :N].double()
    return init.double() + s.sum(0), gamma_(depth) * (init.double().abs() + s.abs().sum(0))


# ------------------------------------------------------------------------------------------------ segment sums
def seg_inputs(H, device, act, seed=0):
    """segments: empty, length 1, hundreds of entries, repeated sources, negative and zero weights"""
    g = torch.Generator().manual_seed(seed)
    lens = [0, 1, 3, 0, 300, 1, 0, 17, 450, 2, 0]
    nsrc = 40
    off = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32)
    n = int(off[-1])
    idx = torch.randint(0, nsrc, (n,), generator=g, dtype=torch.int32)
    idx[:5] = 7                                          # repeated source: atomic collisions in the backward
    w = torch.randn(n, generator=g)
    w[::7] = 0.0
    w[1::5] = -w[1::5].abs()
    src = torch.randn(nsrc, H, generator=g).to(act)
    return [t.to(device) for t in (src, off, idx, w)]


def seg_fwd_ref(src, off, idx, w, H):
    nseg = off.numel() - 1
    lens = (off[1:] - off[:-1]).long()
    seg = torch.repeat_interleave(torch.arange(nseg, device=src.device), lens)
    t = src.double()[idx.long()] * w.double()[:, None]
    out = torch.zeros(nseg, H, dtype=torch.float64, device=src.device).index_add_(0, seg, t)
    aout = torch.zeros_like(out).index_add_(0, seg, t.abs())
    return out, gamma_(1) * lens.double()[:, None] * aout


def seg_bwd_ref(dout, off, idx, w, init):
    nseg = off.numel() - 1
    lens = (off[1:] - off[:-1]).long()
    seg = torch.repeat_interleave(torch.arange(nseg, device=dout.device), lens)
    t = dout.double()[seg] * w.double()[:, None]
    ref = init.double().index_add(0, idx.long(), t)
    at = torch.zeros_like(ref).index_add_(0, idx.long(), t.abs())
    cnt = torch.bincount(idx.long(), minlength=init.shape[0]).double()[:, None]
    return ref, U * at + gamma_(1) * (cnt + 1) * (init.double().abs() + at)


# ------------------------------------------------------------------------------------------------ activations
def gelu_bwd_ref(g, x):
    x64, g64 = x.double(), g.double()
    pdf = torch.exp(-0.5 * x64 * x64) / math.sqrt(2 * math.pi)
    dg = 0.5 * (1 + torch.erf(x64 / math.sqrt(2))) + x64 * pdf
    y = g64 * dg
    d = g64.abs() * (3 * U + (x64 * pdf).abs() * (2.0 ** -21 + 1.5 * U * x64 * x64 + 4 * U)) + U * y.abs()
    return y, d


def gelu_inputs(n, act, device, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.linspace(-8, 8, n, dtype=torch.float64)
    x[::13] = torch.randn(x[::13].shape, generator=g, dtype=torch.float64) * 1e-39    # subnormal pre-activations
    x[5] = 0.0
    dy = torch.randn(n, generator=g)
    return x.to(act).to(device), dy.to(act).to(device)


# ------------------------------------------------------------------------------------------------ softmax cross entropy
XENT_V = (7, 256, 30522, 250002)


def xent_inputs(rows, V, ld, device, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(rows, ld, generator=g, dtype=torch.float64) * 160 - 80).float()
    x[:, V:] = float("nan")                              # never read
    if rows > 1:
        x[1, :V] = torch.randn(V, generator=g) * 0.1     # an ordinary row
    lab = torch.randint(0, V, (rows,), generator=g)
    lab[0] = V - 1
    if rows > 2:
        lab[2] = -1
    if rows > 3:
        lab[3] = 0
    gs = torch.rand(rows, generator=g) + 0.25
    return x.to(device), lab.to(device), gs.to(device)


def xent_ref(x, lab, V, gs):
    xv = x[:, :V].double()
    mx = xv.max(1, keepdim=True).values
    e = torch.exp(xv - mx)
    s = e.sum(1, keepdim=True)
    ls = torch.log(s)
    valid = (lab >= 0)[:, None]
    lab0 = lab.clamp(min=0)[:, None]
    xl = xv.gather(1, lab0)
    loss = torch.where(valid, ls + mx - xl, torch.zeros_like(ls))
    ei = 2.0 ** -20 + 4 * U * (xv - mx).abs()
    depth = -(-V // 256) + 13
    ds = ei.max(1, keepdim=True).values + gamma_(depth)
    dloss = torch.where(valid, 1.01 * ds + 2 * U * ls.abs() + U * (ls + mx).abs() + U * loss.abs(), torch.zeros_like(ls))
    p = e / s
    oh = torch.zeros_like(p).scatter_(1, lab0, 1.0)
    gsv = (gs.double()[:, None] if gs is not None else torch.ones_like(ls)) * valid
    dl = (p - oh) * gsv
    ddl = gsv.abs() * (p * (ei + 1.01 * ds + 2.01 * U) + U * (p - oh).abs() + 2.0 ** -125) + U * dl.abs()
    return loss[:, 0], dloss[:, 0], dl, ddl


# ------------------------------------------------------------------------------------------------ exact ops
def scatter_sorted_ref(src, src_row, w, dst, H, out):
    """bb_scatter_rows_sorted in fp32 with the kernel's order: per run acc = t_e0, acc = acc + t_e, out = out + acc"""
    out = out.clone().float()
    s = src.float()[src_row]
    t = s * w.float()[:, None] if w is not None else s
    n = dst.numel()
    e = 0
    while e < n:
        d = int(dst[e])
        e1 = e
        while e1 < n and int(dst[e1]) == d:
            e1 += 1
        if d >= 0:
            acc = t[e].clone()
            for k in range(e + 1, e1):
                acc = acc + t[k]
            out[d] = out[d] + acc
        e = e1
    return out


# ------------------------------------------------------------------------------------------------ optimizer
MT_CHUNK = 4096


def adam1_f32(p, g, m, v, b1, b2, eps, coef, step, decay, eps_in_sqrt=False, decay_first=False):
    """fp32 restatement of optim.cu adam1 (no fused multiply-adds): torch fp32 tensors, returns (p, m, v)"""
    f = lambda a: torch.tensor(a, dtype=F32)
    b1, b2, eps, coef, step, decay = (f(t) for t in (b1, b2, eps, coef, step, decay))
    g = g * coef
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    if decay_first:
        p = p - decay * p
    den = torch.sqrt(v + eps) if eps_in_sqrt else torch.sqrt(v) + eps
    p = p - step * (m / den)
    if not decay_first:
        p = p - decay * p
    return p, m, v


def clip_coef(sumsq, max_norm, grad_scale, clip_eps=1e-6):
    """fp64 clip coefficient from the kernel's own fp32 sum of squares (None: no clipping)"""
    if sumsq is None or max_norm <= 0:
        return grad_scale, False
    norm = math.sqrt(float(sumsq)) * grad_scale
    c = min(1.0, float(torch.tensor(max_norm, dtype=F32)) / (norm + clip_eps))
    return grad_scale * c, c < 1.0


def adam_ref(p, g, m, v, b1, b2, eps, coef, clipped, step, decay):
    """fp64 AdamW step and its bounds from fp32 state (p, g, m, v); b1 / b2 / eps / step / decay as the kernel sees
    them (fp32)"""
    f = lambda a: float(torch.tensor(a, dtype=F32))
    b1, b2, eps, step, decay = f(b1), f(b2), f(eps), f(step), f(decay)
    p, g, m, v = (t.double() for t in (p, g, m, v))
    gp = g * coef
    m1 = b1 * m + (1 - b1) * gp
    v1 = b2 * v + (1 - b2) * gp * gp
    sv = v1.sqrt()
    den = sv + eps
    q = m1 / den
    p1 = p - step * q
    p2 = p1 - decay * p1
    Eg = g.abs() * (5.01 * U * abs(coef) if clipped else 0.0) + U * gp.abs()
    Em = (1 - b1) * Eg + 2.01 * U * (b1 * m.abs() + (1 - b1) * gp.abs())
    Ev = 2 * (1 - b2) * gp.abs() * Eg + 3.01 * U * (b2 * v.abs() + (1 - b2) * gp * gp)
    Eden = torch.minimum(Ev / (2 * sv).clamp_min(1e-300), Ev.sqrt()) + U * sv + U * den
    Eq = (Em + q.abs() * Eden) / den + U * q.abs()
    Ep1 = step * Eq + U * step * q.abs() + U * p1.abs()
    Ep2 = (1 + decay) * Ep1 + 2.01 * U * (decay * p1.abs() + p2.abs())
    return dict(p=p2, m=m1, v=v1, d_p=Ep2, d_m=Em, d_v=Ev)


OPT_SIZES = (0, 1, 3, 4, 5, 4095, 4096, 4097, 3 * 4096 + 5)


def opt_sizes(kind):
    """tensor sizes of an optimizer table: 'edges' (every edge size, zero-size entries first, in the middle and last)
    or 'many' (about 600 mixed sizes: the binary search over chunk0 walks a deep table)"""
    if kind == "edges":
        return [0] + list(OPT_SIZES[1:5]) + [0, 0] + list(OPT_SIZES[5:]) + [0]
    g = torch.Generator().manual_seed(9)
    s = torch.randint(1, 9000, (600,), generator=g).tolist()
    for i in range(0, 600, 97):
        s[i] = 0
    s[1::50] = [4096] * len(s[1::50])
    return s


class OptTable:
    """p / g / m / v (fp32) and p16 (bf16) of every tensor in one arena each, with a guard gap of G sentinel elements
    between tensors; `offset` maps a field name to an element offset of every tensor's start (the scalar path)."""

    def __init__(self, sizes, device, offset=None, seed=0, scale=1.0):
        offset = offset or {}
        g = torch.Generator().manual_seed(seed)
        self.sizes = list(sizes)
        self.device = device
        self.arena, self.views, self.starts = {}, {f: [] for f in "pgmv"}, {}
        self.views["p16"] = []
        for f, dt in (("p", F32), ("g", F32), ("m", F32), ("v", F32), ("p16", BF)):
            o = offset.get(f, 0)
            starts, pos = [], G
            for n in self.sizes:
                pos = (pos + 7) // 8 * 8 + o           # 16-byte aligned start (bf16: 8 elements) plus the offset
                starts.append(pos)
                pos += n + G
            full = torch.empty(pos, dtype=dt)
            it, pat = SENT[dt]
            full.view(it).fill_(pat)
            full = full.to(device)
            self.arena[f], self.starts[f] = full, starts
            for s, n in zip(starts, self.sizes):
                self.views[f].append(full[s:s + n])
        for i, n in enumerate(self.sizes):
            self.views["p"][i].copy_((torch.randn(n, generator=g)).to(device))
            self.views["g"][i].copy_((torch.randn(n, generator=g) * scale).to(device))
            self.views["m"][i].copy_((torch.randn(n, generator=g) * 0.01).to(device))
            self.views["v"][i].copy_((torch.rand(n, generator=g) * 1e-4).to(device))

    def rows(self, step_sizes, decays, with_p16=True, with_g=True):
        return [(self.views["p"][i].data_ptr(), self.views["g"][i].data_ptr() if with_g else 0,
                 self.views["m"][i].data_ptr(), self.views["v"][i].data_ptr(),
                 self.views["p16"][i].data_ptr() if with_p16 else 0, n, step_sizes[i], decays[i])
                for i, n in enumerate(self.sizes)]

    def check_gaps(self, fields="pgmv"):
        """every element outside the tensors still holds the sentinel"""
        for f in list(fields):
            self._gaps(f)

    def _gaps(self, f):
        full = self.arena[f]
        it, pat = SENT[full.dtype]
        mask = torch.ones(full.numel(), dtype=torch.bool, device=full.device)
        for s, n in zip(self.starts[f], self.sizes):
            mask[s:s + n] = False
        bad = (full.view(it)[mask] != pat).nonzero()
        if bad.numel():
            pos = int(mask.nonzero()[int(bad[0])])
            raise AssertionError("%s: guard overwritten, bad elements at %d positions, first at arena element %d" % (
                f, bad.numel(), pos))

    def snapshot(self):
        return {f: [t.detach().clone() for t in self.views[f]] for f in self.views}

    @property
    def chunks(self):
        return sum(-(-n // MT_CHUNK) for n in self.sizes)


def sumsq_ref(gs, chunks):
    s = sum(float((t.double() ** 2).sum()) for t in gs)
    return s, gamma_(16 + 9 + chunks) * s


def bf16_rne(t):
    return t.to(BF)


# ------------------------------------------------------------------------------------------------ runners
# impl "gpu": the C ABI on guarded CUDA buffers; impl "emu": tests/emu_kernels.py on CPU into the same kind of buffers.
def _lib():
    from bevbert_b200 import _lib as L
    return L


def _call(name, *args):
    from bevbert_b200 import kernels as K
    L = _lib()
    rc = getattr(L.load(), name)(*args, K._stream())
    L.check(rc, name)


def _p(t):
    return 0 if t is None else t.data_ptr()


def _sync(device):
    if str(device).startswith("cuda"):
        torch.cuda.synchronize()


def num_sms(device):
    return torch.cuda.get_device_properties(device).multi_processor_count if str(device).startswith("cuda") else 132


def run_ln_fwd(case, impl, device):
    import emu_kernels as E
    x, res, gam, bet = ln_inputs(case, device)
    rows, H = case.rows, case.H
    A = Arena(device)
    y, y32 = A.out("y", (rows, H), case.act), A.out("y_f32", (rows, H), F32)
    mean, rstd = A.out("mean", (rows,), F32), A.out("rstd", (rows,), F32)
    if impl == "gpu":
        _call("bb_layernorm_fwd", x.data_ptr(), int(x.dtype == F32), _p(res), gam.data_ptr(), bet.data_ptr(), case.eps,
              rows, H, 0, 0, 1.0, 0, 0, 1.0, y.data_ptr(), y32.data_ptr(), mean.data_ptr(), rstd.data_ptr())
    else:
        out = E.layernorm_fwd(x, res, gam, bet, case.eps, want_f32=True)
        for dst, src in zip((y, y32, mean, rstd), out):
            dst.copy_(src)
    _sync(device)
    return A, (x, res, gam, bet), (y, y32, mean, rstd)


def check_ln_fwd(case, A, ins, outs):
    x, res, gam, bet = ins
    y, y32, mean, rstd = outs
    R = ln_fwd_ref(x, res, gam, bet, case.eps)
    bf = case.act == BF
    check("ln_fwd.y[%s]" % case.id, y, R["y"], fin(R["y"], R["d_y"], bf))
    check("ln_fwd.y_f32[%s]" % case.id, y32, R["y"], R["d_y"])
    check("ln_fwd.mean[%s]" % case.id, mean, R["mean"], R["d_mean"])
    check("ln_fwd.rstd[%s]" % case.id, rstd, R["rstd"], R["d_rstd"])
    if case.adv == "const":
        check_exact("ln_fwd.y const rows", y, bet.to(case.act).expand(case.rows, case.H))
    A.check_guards()


def run_ln_bwd(case, pair, impl, device, det=False):
    """-> (arena, inputs, outputs, grid); mean / rstd are the fp32 roundings of the fp64 forward"""
    import emu_kernels as E
    dyf, xf, dxf = pair
    x, res, gam, _ = ln_inputs(case, device)
    rows, H = case.rows, case.H
    R = ln_fwd_ref(x, res, gam, gam, case.eps)
    mean, rstd = R["mean"].float(), R["rstd"].float()
    g = torch.Generator().manual_seed(case.seed + 100)
    dy = torch.randn(rows, H, generator=g).to(F32 if dyf else case.act).to(device)
    init = [(torch.randn(H, generator=g) * 0.1).to(device) for _ in range(3)]
    A = Arena(device)
    dx = A.out("dx", (rows, H), F32 if dxf else case.act)
    dres = A.out("dres", (rows, H), case.act)
    dg, db, dxs = (A.inp(n, t) for n, t in zip(("dgamma", "dbeta", "dxsum"), init))
    if impl == "gpu":
        _call("bb_layernorm_bwd", dy.data_ptr(), dyf, x.data_ptr(), xf, _p(res), gam.data_ptr(), mean.data_ptr(),
              rstd.data_ptr(), rows, H, 0, 0, 1.0, 0, 0, 1.0, dx.data_ptr(), dxf, dres.data_ptr(), dg.data_ptr(),
              db.data_ptr(), dxs.data_ptr())
    else:
        edx, edres = E.layernorm_bwd(dy, x, res, gam, mean, rstd, want_dres=True, dx_f32=bool(dxf), dgamma=dg,
                                     dbeta=db, dxsum=dxs)
        dx.copy_(edx)
        dres.copy_(edres)
    _sync(device)
    grid = min(-(-rows // 8), num_sms(device))
    return A, (dy, x, res, gam, mean, rstd, init), (dx, dres, dg, db, dxs), grid


def check_ln_bwd(case, pair, A, ins, outs, grid):
    dy, x, res, gam, mean, rstd, init = ins
    dx, dres, dg, db, dxs = outs
    R = ln_bwd_ref(dy, x, res, gam, mean, rstd, grid, init)
    tag = "%s-%s" % (case.id, "".join(map(str, pair)))
    check("ln_bwd.dx[%s]" % tag, dx, R["dz"], fin(R["dz"], R["d_dz"], dx.dtype == BF))
    check("ln_bwd.dres[%s]" % tag, dres, R["dz"], fin(R["dz"], R["d_dz"], dres.dtype == BF))
    check("ln_bwd.dgamma[%s]" % tag, dg, R["dgamma"], R["d_dgamma"])
    check("ln_bwd.dbeta[%s]" % tag, db, R["dbeta"], R["d_dbeta"])
    check("ln_bwd.dxsum[%s]" % tag, dxs, R["dxsum"], R["d_dxsum"])
    if case.adv == "const":
        assert bool(torch.isfinite(dx.float()).all()), "ln_bwd: non-finite dx on constant rows"
    A.check_guards()


def run_colsum(N, ld, rows, act, impl, device, seed=0):
    g = torch.Generator().manual_seed(seed + N + rows)
    x = torch.randn(rows, ld, generator=g).to(act).to(device)
    init = (torch.randn(N, generator=g) * 0.1).to(device)
    A = Arena(device)
    out = A.inp("out", init)
    if impl == "gpu":
        _call("bb_colsum_bf16", x.data_ptr(), rows, N, ld, out.data_ptr())
    else:
        out.add_(x[:, :N].float().sum(0))
    _sync(device)
    return A, x, init, out


def check_colsum(N, ld, rows, A, x, init, out):
    ref, d = colsum_ref(x, N, init)
    check("colsum[N%d-ld%d-r%d]" % (N, ld, rows), out, ref, d)
    A.check_guards()


def run_seg(H, act, impl, device, seed=0):
    import emu_kernels as E
    src, off, idx, w = seg_inputs(H, device, act, seed)
    nseg = off.numel() - 1
    g = torch.Generator().manual_seed(seed + 1)
    A = Arena(device)
    out = A.out("out", (nseg, H), act)
    srcA = A.inp("src", src)
    dout = (torch.randn(nseg, H, generator=g)).to(act).to(device)
    init = (torch.randn(src.shape[0], H, generator=g) * 0.1).to(device)
    dsrc = A.inp("dsrc", init)
    if impl == "gpu":
        _call("bb_segment_wsum", srcA.data_ptr(), off.data_ptr(), idx.data_ptr(), w.data_ptr(), nseg, H, out.data_ptr())
        _call("bb_segment_wsum_bwd", dout.data_ptr(), off.data_ptr(), idx.data_ptr(), w.data_ptr(), nseg, H,
              dsrc.data_ptr())
    else:
        out.copy_(E.segment_wsum(src, off, idx, w, nseg, H))
        E.segment_wsum_bwd(dout, off, idx, w, nseg, H, dsrc)
    _sync(device)
    ref, d = seg_fwd_ref(src, off, idx, w, H)
    check("segment_wsum[H%d]" % H, out, ref, fin(ref, d, act == BF))
    rb, db = seg_bwd_ref(dout, off, idx, w, init)
    check("segment_wsum_bwd[H%d]" % H, dsrc, rb, db)
    A.check_guards()


def run_gelu(n, act, impl, device):
    import emu_kernels as E
    x, dy = gelu_inputs(n, act, device)
    A = Arena(device)
    out = A.out("out", (n,), act)
    rout = A.out("relu", (n,), act)
    if impl == "gpu":
        _call("bb_act_bwd_bf16", dy.data_ptr(), x.data_ptr(), 1, out.data_ptr(), n)
        _call("bb_act_bwd_bf16", dy.data_ptr(), x.data_ptr(), 2, rout.data_ptr(), n)
    else:
        out.copy_(E.gelu_bwd(dy, x))
        rout.copy_(E.relu_bwd(dy, x))
    _sync(device)
    ref, d = gelu_bwd_ref(dy, x)
    check("gelu_bwd[n%d]" % n, out, ref, fin(ref, d, act == BF))
    check_exact("relu_bwd", rout, torch.where(x.float() > 0, dy, torch.zeros_like(dy)))
    A.check_guards()


def run_xent(rows, V, ld, act, use_gs, impl, device, seed=0):
    import emu_kernels as E
    x, lab, gs = xent_inputs(rows, V, ld, device, seed)
    gs = gs if use_gs else None
    A = Arena(device)
    loss = A.out("loss", (rows,), F32)
    dl = A.out("dlogits", (rows, ld), act)
    if impl == "gpu":
        _call("bb_softmax_xent", x.data_ptr(), lab.data_ptr(), rows, V, ld, loss.data_ptr(), _p(gs), dl.data_ptr())
    else:
        prev, E.ACT = E.ACT, F32                  # the restatement has no gscale: scale before the one rounding
        try:
            el, edl = E.softmax_xent(x, lab, V, ld)
        finally:
            E.ACT = prev
        loss.copy_(el)
        dl.copy_(edl * (gs[:, None] if gs is not None else 1.0))
    _sync(device)
    return A, (x, lab, gs), (loss, dl)


def check_xent(V, ld, A, ins, outs):
    x, lab, gs = ins
    loss, dl = outs
    rl, dlo, rdl, ddl = xent_ref(x, lab, V, gs)
    tag = "V%d-ld%d%s" % (V, ld, "-gs" if gs is not None else "")
    check("xent.loss[%s]" % tag, loss, rl, dlo)
    check("xent.dlogits[%s]" % tag, dl[:, :V], rdl, fin(rdl, ddl, dl.dtype == BF))
    if ld > V:
        check_exact("xent.dlogits columns [V, ld)", dl[:, V:], torch.zeros_like(dl[:, V:]))
    inv = lab < 0
    if bool(inv.any()):
        z = torch.zeros(1, dtype=torch.float64, device=loss.device)
        check("xent.loss of label -1", loss[inv], torch.zeros_like(loss[inv], dtype=torch.float64), z)
        check("xent.dlogits of label -1", dl[inv], torch.zeros_like(dl[inv], dtype=torch.float64), z)
    A.check_guards()


def run_exact_rows(H, act, impl, device, seed=0):
    """embed_sum, gather_rows (idx -1), add_rows (every subset of b / table / vec), scale_rows_, add_act"""
    import emu_kernels as E
    g = torch.Generator().manual_seed(seed + H)
    V, L, Bn = 97, 40, 3
    word, pos, typ = (torch.randn(n, H, generator=g).to(device) for n in (V, L, 1))
    ids = torch.randint(0, V, (Bn, L), generator=g)
    ids[0, :3] = V - 1
    ids = ids.to(device)
    A = Arena(device)
    z = A.out("embed", (Bn * L, H), F32)
    src = torch.randn(50, H, generator=g).to(act).to(device)
    gidx = torch.randint(-1, 50, (300,), generator=g)
    gidx[:4] = -1
    gidx = gidx.to(device)
    gat = A.out("gather", (300, H), act)
    rows = 131
    a, b = (torch.randn(rows, H, generator=g).to(act).to(device) for _ in range(2))
    table, vec = torch.randn(5, H, generator=g).to(device), torch.randn(H, generator=g).to(device)
    tidx = torch.randint(0, 5, (rows,), generator=g).to(device)
    subsets = [(bb, tt, vv) for bb in (0, 1) for tt in (0, 1) for vv in (0, 1)]
    outs = [A.out("add_rows%d" % i, (rows, H), act) for i in range(len(subsets))]
    ld = H + 3
    xs = torch.randn(rows, ld, generator=g).to(act).to(device)
    sc = A.inp("scale_rows", xs)
    gsc = torch.rand(rows, generator=g).to(device) * 3
    n = rows * H - 5
    aa = A.out("add_act", (n,), act)
    if impl == "gpu":
        _call("bb_embed_sum", ids.data_ptr(), word.data_ptr(), pos.data_ptr(), typ.data_ptr(), Bn * L, L, H, z.data_ptr())
        _call("bb_gather_rows_bf16", src.data_ptr(), gidx.data_ptr(), 300, H, gat.data_ptr())
        for o, (bb, tt, vv) in zip(outs, subsets):
            _call("bb_add_rows", a.data_ptr(), b.data_ptr() if bb else 0, table.data_ptr() if tt else 0,
                  tidx.data_ptr() if tt else 0, vec.data_ptr() if vv else 0, rows, H, o.data_ptr())
        _call("bb_scale_rows_bf16", sc.data_ptr(), gsc.data_ptr(), rows, ld)
        _call("bb_add_bf16", a.data_ptr(), b.data_ptr(), aa.data_ptr(), n)
    else:
        z.copy_(E.embed_sum(ids, word, pos, typ[0]))
        gat.copy_(E.gather_rows(src, gidx, H))
        for o, (bb, tt, vv) in zip(outs, subsets):
            o.copy_(E.add_rows(a, b if bb else None, table if tt else None, tidx if tt else None, vec if vv else None))
        E.scale_rows_(sc, gsc, rows, ld)
        aa.copy_(E.add_act(a.reshape(-1)[:n], b.reshape(-1)[:n]))
    _sync(device)
    check_exact("embed_sum", z, ((word[ids] + pos[None]) + typ[0]).reshape(-1, H))
    gref = torch.zeros(300, H, dtype=act, device=device)
    keep = gidx >= 0
    gref[keep] = src[gidx[keep]]
    check_exact("gather_rows", gat, gref)
    for o, (bb, tt, vv) in zip(outs, subsets):
        r = a.float()
        if bb:
            r = r + b.float()
        if tt:
            r = r + table[tidx]
        if vv:
            r = r + vec
        check_exact("add_rows b%d table%d vec%d" % (bb, tt, vv), o, r.to(act))
    check_exact("scale_rows_", sc, (xs.float() * gsc[:, None]).to(act))
    check_exact("add_act", aa, (a.reshape(-1)[:n].float() + b.reshape(-1)[:n].float()).to(act))
    A.check_guards()


def scatter_sorted_inputs(H, src_f32, use_w, device, act, seed=0):
    """runs of 1 and of hundreds of entries, leading dst < 0"""
    g = torch.Generator().manual_seed(seed + H)
    lens = [5, 1, 1, 300, 2, 1, 130, 1]
    dst = torch.cat([torch.full((n,), d, dtype=torch.int64) for d, n in zip([-1, 0, 2, 3, 7, 8, 9, 11], lens)])
    n = dst.numel()
    src = torch.randn(60, H, generator=g).to(F32 if src_f32 else act)
    src_row = torch.randint(0, 60, (n,), generator=g)
    w = torch.randn(n, generator=g) if use_w else None
    out0 = torch.randn(12, H, generator=g)
    return [t.to(device) if t is not None else None for t in (src, src_row, w, dst, out0)]


def run_scatter_sorted(H, src_f32, use_w, act, impl, device):
    src, src_row, w, dst, out0 = scatter_sorted_inputs(H, src_f32, use_w, device, act)
    A = Arena(device)
    out = A.inp("out", out0)
    ref = scatter_sorted_ref(src.cpu(), src_row.cpu(), w.cpu() if w is not None else None, dst.cpu(), H, out0.cpu())
    if impl == "gpu":
        _call("bb_scatter_rows_sorted", src.data_ptr(), int(src_f32), src_row.data_ptr(), _p(w), dst.data_ptr(),
              dst.numel(), H, out.data_ptr())
    else:
        out.copy_(scatter_sorted_ref(src, src_row, w, dst, H, out0))
    _sync(device)
    check_exact("scatter_rows_sorted", out.cpu(), ref)
    A.check_guards()


def run_embed_grad(L, H, det, impl, device, seed=0):
    """bb_embed_scatter_grad: padding_idx and V - 1; atomic mode all three tables, deterministic mode dpos / dtype0"""
    import emu_kernels as E
    g = torch.Generator().manual_seed(seed + L)
    V, Bn, pad = 61, 4, 0
    ids = torch.randint(0, V, (Bn, L), generator=g)
    ids[0, 0] = V - 1
    ids[-1, -1] = pad
    ids = ids.to(device)
    dz = torch.randn(Bn * L, H, generator=g).to(device)
    iw, ip, it = (torch.randn(n, H, generator=g).to(device) * 0.1 for n in (V, L, 1))
    A = Arena(device)
    dw, dp, dt = A.inp("dword", iw), A.inp("dpos", ip), A.inp("dtype0", it)
    if impl == "gpu":
        _call("bb_embed_scatter_grad", ids.data_ptr(), dz.data_ptr(), Bn * L, L, H, pad, 0 if det else dw.data_ptr(),
              dp.data_ptr(), dt.data_ptr())
    else:
        rw = torch.zeros_like(dw)
        E.embed_scatter_grad(ids, dz, L, pad, rw, dp, dt[0])
        if not det:
            dw.add_(rw)
    _sync(device)
    flat = ids.reshape(-1)
    d64 = dz.double()
    keep = flat != pad
    rw = iw.double().index_add(0, flat[keep], d64[keep])
    aw = torch.zeros_like(rw).index_add_(0, flat[keep], d64[keep].abs())
    cnt = torch.bincount(flat[keep], minlength=V).double()[:, None]
    if det:
        check_exact("embed_scatter_grad.dword (deterministic: untouched)", dw, iw)
    else:
        check("embed_scatter_grad.dword[L%d]" % L, dw, rw, gamma_(1) * (cnt + 1) * (iw.double().abs() + aw))
    lpos = torch.arange(Bn * L, device=device) % L
    rp = ip.double().index_add(0, lpos, d64)
    ap = torch.zeros_like(rp).index_add_(0, lpos, d64.abs())
    check("embed_scatter_grad.dpos[L%d]" % L, dp, rp, gamma_(Bn + 1) * (ip.double().abs() + ap))
    rt = it.double() + d64.sum(0)
    gy = min(-(-Bn * L // 64), 64)
    depth = max(Bn * L, -(-Bn * L // (8 * gy)) + 12 + gy) + 1
    check("embed_scatter_grad.dtype0[L%d]" % L, dt, rt, gamma_(depth) * (it.double().abs() + d64.abs().sum(0)))
    A.check_guards()
