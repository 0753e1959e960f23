"""Cases of the fused attention contract (include/bevbert_b200.h, bb_flash_args) with an fp64 reference (test
infrastructure, shared by tests/test_attn_gpu.py and tests/test_attn_harness_cpu.py).

Exact-routing family ("exact").  Q and K carry a quadratic code in the first 2 NCODE + 1 head dimensions:
    Q[q] . K[k] = -c * |g(k) - g*(q)|^2          (c alpha = 128; Q's and K's other dimensions have disjoint supports)
so every (sample, head, query) row has a set W of winner keys (code g*(q), |W| in {1, 2, 4, 8}) with logit exactly 0
and every other key at least 128 log2(e) = 184.7 below it in the log2 domain.  ex2 of every loser, and every rescale
factor applied when the first winner arrives, then flush to exactly 0, so P = 1/|W|, O = mean of V over W and
LSE = log2 |W| (plus the fp32 log2-domain offset kmask log2(e) of a sample masked -10000 everywhere, or
bias log2(e) for a per-row graph bias that is a power of two <= -2, where the sum stays exact).  dO and V are sparse
+-1, so dP, D, dS, dQ, dK, dV and dbias are dyadic rationals.  The generator asserts, in fp64, that every value a
kernel rounds to bf16 as an MMA operand (P, Pdrop, alpha dS) is representable, and that every product's sum of
|terms| stays below 2^24 times the granule of its terms, so any summation order is exact.  O, dQ, dK, dV, dbias are
then compared bit for bit and LSE exactly.  Dropout rows use p = 0.5 (scale 2, exact); the keep mask comes from
drop_masks.attn_keep.  This needs ex2.approx.ftz to return exact powers of two at small integer arguments and
log2f(2^k) = k; on an H100 every exact-routing row is bit-exact on both cores, including the mma.sync dK / dV pass on
a sample masked -10000 everywhere (where an FMA of (s alpha + kmask) log2e - lse would leave a 2^-11 residue that the
bf16 rounding of P and dS absorbs).

Error-bounded family ("bound").  Random bf16 inputs, alpha = 0.125, p in {0, 0.1}, compared per element with fp64
from the same bf16 inputs (the backward's D from the O that was passed in):
    O  : |err| <= ulp/2 + C_O 2^-9 sum_k Pdrop_k |v_k|
    dV : |err| <= ulp/2 + C_DV 2^-9 (Pdrop^T |dO|)
    dQ : |err| <= ulp/2 + C_DQ 2^-9 alpha (A |K|),  dK: ulp/2 + C_DK 2^-9 alpha (A^T |Q|),  A = P (|g| + |D|)
    LSE: |err| <= C_LSE (ulp_fp32(row max) + 2^-20)
    dbias: |err| <= C_DB 2^-9 sum_h A
(A bounds |dS| and its rounding: dS = P (g - D) cancels.)  The constants are about twice the worst err / bound
measured on an H100 80GB HBM3 at a 400 W power limit over the table (bf16 rounding of P alone gives up to 2):
    O 1.77 -> 3.5, dV 1.97 -> 4, dQ 1.80 -> 3.6, dK 1.94 -> 4, LSE 4.88 -> 10, dbias 0.019 -> 0.04.
Rows are adversarial: a row maximum that grows in every key block and peaks in the last partial block, a single
unmasked key, |alpha S| up to about 40, -10000 / -inf masks and samples masked entirely with either.

Buffers.  Every pointer has its own buffer (or, for the model's layouts, a packed Q|K|V or K|V buffer) with padding
columns, rows past nq / nk inside the batch stride and gaps between samples.  Input elements a kernel must not read
hold NaN.  o, lse, dsum, dq, dk, dv and dbias sit between guards; guards and every element a kernel must not write
hold a NaN sentinel bit pattern that must survive the launch.  A failure names the first bad (b, h, row, col) or guard
offset with the value it got and the value it expected.
"""
import math
import zlib
from dataclasses import dataclass, replace

import torch

import drop_masks as DM

BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
GUARD = 64
SEED = 0xA77E5EED5A170123          # >= 2^63, like the seeds DropState draws
SENT = {BF: 0x7FA5, F32: 0x7FA5A5A5}
_BITS = {BF: torch.int16, F32: torch.int32}
LOG2E_F32 = torch.tensor(1.4426950408889634, dtype=F32)
NCODE, GCODE = 4, 5                # code vectors in {0..4}^4: 625 distinct codes >= 600 keys
CORES = {"mma": 0, "auto": 1, "tc": 2}
# err / bound constants of the error-bounded family (see the module docstring)
C_O, C_DV, C_DQ, C_DK, C_LSE, C_DB = 3.5, 4.0, 3.6, 4.0, 10.0, 0.04


@dataclass(frozen=True)
class Case:
    family: str              # "exact" | "bound"
    B: int
    H: int
    nq: int
    nk: int
    fwd: str = "auto"        # core of the forward: "mma" (set_attn_tc(0)), "tc" (2), "auto" (1, the default dispatch)
    bwd: str = "auto"        # core of the backward, chosen independently
    mask: str = "none"       # none | mix (0 / -10000) | tail (-inf tail) | full10k / fullinf (sample 0 masked entirely)
    bias: bool = False       # graph bias (B, nq, nk): always the mma.sync core
    dbias: str = ""          # "" | "atomic" | "det" (torch.use_deterministic_algorithms around the backward)
    drop: float = 0.0
    alpha: float = 0.125
    layout: str = "sep"      # sep (own padded buffers) | self (packed Q|K|V, packed dQ|dK|dV) | cross (Q, packed K|V)
    adv: str = ""            # bound family: "ramp" (max grows every block) | "single" (one unmasked key) | "big"

    @property
    def id(self):
        s = "%s-b%dh%d-%dx%d-%s_%s-%s-%s" % (self.family, self.B, self.H, self.nq, self.nk, self.fwd, self.bwd,
                                             self.mask, self.layout)
        if self.bias:
            s += "-bias"
        if self.dbias:
            s += "-dbias_" + self.dbias
        if self.drop:
            s += "-p%g" % self.drop
        if self.alpha != 0.125:
            s += "-a%g" % self.alpha
        if self.adv:
            s += "-" + self.adv
        return s


def _E(*a, **k):
    return Case("exact", *a, **k)


def _Bd(*a, **k):
    return Case("bound", *a, **k)


EXACT_ROWS = [
    # the model's shapes
    _E(2, 12, 441, 441, "tc", "tc", "mix", layout="self"),
    _E(2, 12, 441, 441, "auto", "auto", "none", layout="self", drop=0.5),
    _E(3, 12, 80, 80, "mma", "mma", "mix", layout="self"),
    _E(2, 12, 80, 80, "tc", "mma", "tail", layout="self", drop=0.5),
    _E(2, 12, 441, 80, "mma", "tc", "mix", layout="cross"),
    _E(2, 12, 80, 441, "tc", "tc", "tail", layout="cross", drop=0.5),
    _E(3, 12, 36, 36, "mma", "mma", "full10k", layout="self"),
    _E(3, 12, 36, 36, "tc", "tc", "full10k", layout="self", drop=0.5),
    _E(2, 12, 23, 23, "mma", "mma", "mix", bias=True, dbias="atomic", layout="self"),
    _E(2, 12, 23, 23, "mma", "mma", "none", bias=True, dbias="det", layout="self", drop=0.5),
    _E(3, 12, 1, 80, "auto", "auto", "mix", layout="cross"),
    _E(2, 12, 1, 441, "mma", "tc", "tail", layout="cross", drop=0.5),
    # edges: every listed nq and nk, both cores, mixed cores
    _E(2, 1, 1, 600, "tc", "tc", "mix"),
    _E(2, 1, 15, 7, "mma", "mma", "mix"),
    _E(2, 1, 16, 1, "tc", "tc", "none"),
    _E(3, 12, 17, 23, "tc", "mma", "tail", drop=0.5),
    _E(2, 1, 63, 63, "mma", "tc", "mix", alpha=1.0),
    _E(1, 12, 64, 64, "tc", "tc", "none", alpha=2.0),
    _E(2, 12, 65, 65, "mma", "mma", "tail", drop=0.5),
    _E(2, 1, 127, 127, "tc", "tc", "fullinf"),
    _E(2, 1, 128, 128, "mma", "mma", "fullinf", drop=0.5),
    _E(2, 12, 129, 129, "auto", "auto", "mix"),
    _E(3, 1, 257, 193, "tc", "tc", "mix", drop=0.5),
    _E(2, 1, 257, 512, "mma", "mma", "none", alpha=1.0),
    _E(2, 1, 129, 600, "tc", "tc", "tail"),
    _E(2, 12, 65, 191, "tc", "mma", "full10k"),
    _E(2, 1, 65, 191, "mma", "tc", "full10k", drop=0.5),
    _E(1, 12, 441, 512, "tc", "tc", "mix", drop=0.5),
    _E(2, 1, 127, 36, "tc", "tc", "fullinf", alpha=2.0),
    _E(2, 1, 63, 129, "mma", "tc", "fullinf"),
    _E(2, 1, 17, 36, "mma", "mma", "tail", bias=True, dbias="det"),
    _E(2, 1, 127, 65, "mma", "mma", "mix", bias=True, dbias="atomic", drop=0.5),
    _E(3, 12, 128, 127, "auto", "tc", "none"),
    _E(2, 12, 15, 64, "tc", "tc", "mix", drop=0.5),
]

BOUND_ROWS = [
    _Bd(2, 12, 441, 441, "tc", "tc", "mix", layout="self", drop=0.1, adv="ramp"),
    _Bd(2, 12, 441, 441, "mma", "mma", "none", layout="self", adv="ramp"),
    _Bd(2, 12, 80, 441, "tc", "mma", "tail", layout="cross", drop=0.1),
    _Bd(3, 1, 65, 193, "mma", "tc", "fullinf", adv="ramp"),
    _Bd(2, 1, 129, 600, "tc", "tc", "full10k", adv="ramp", drop=0.1),
    _Bd(2, 12, 17, 7, "mma", "mma", "none", adv="single"),
    _Bd(2, 12, 64, 129, "tc", "tc", "none", adv="single", drop=0.1),
    _Bd(2, 12, 23, 23, "mma", "mma", "mix", bias=True, dbias="atomic", drop=0.1, layout="self"),
    _Bd(3, 12, 36, 36, "auto", "auto", "mix", adv="big", layout="self"),
    _Bd(2, 12, 1, 512, "tc", "tc", "full10k", adv="ramp"),
    _Bd(2, 12, 441, 80, "auto", "auto", "mix", layout="cross", adv="big", drop=0.1),
]

TABLE = EXACT_ROWS + BOUND_ROWS


# ------------------------------------------------------------------------------------------------------- helpers
def bits(t):
    return t.view(_BITS[t.dtype])


def cbits(t):
    """bit patterns with -0 taken as +0 (the sign of a zero output is not part of the contract)"""
    b = bits(t).clone()
    b[t == 0] = 0
    return b


def _sentinel(n, dt, device):
    return torch.full((n,), SENT[dt], dtype=_BITS[dt], device=device).view(dt)


def ulp(x, dt):
    """one unit in the last place of dtype dt (bf16 or fp32) at the magnitude of the fp64 values x"""
    p = 8 if dt == BF else 24
    _, e = torch.frexp(x)
    e = torch.where(x == 0, torch.full_like(e, -125), e).clamp_min(-125)
    return torch.ldexp(torch.ones_like(x), e - p)


def granule(x, dim):
    """largest power of two dividing every element of the fp64 dyadic x along `dim` (1 where all are zero)"""
    m, e = torch.frexp(x)
    n = (m * 2.0 ** 53).to(torch.int64)
    low = torch.log2((n & -n).double().clamp_min(1.0)).round().to(torch.int64)
    lb = torch.where(x == 0, torch.full_like(low, 10 ** 6), e.to(torch.int64) - 53 + low).amin(dim)
    lb = torch.where(lb == 10 ** 6, torch.zeros_like(lb), lb)
    return torch.ldexp(torch.ones(lb.shape, dtype=F64, device=x.device), lb)


def exact_product(a, b, what):
    """a @ b over the last / second-to-last dims is exact in fp32 in any summation order"""
    s = a.abs() @ b.abs()
    gran = granule(a, -1).unsqueeze(-1) * granule(b, -2).unsqueeze(-2)
    assert bool((s < 2.0 ** 24 * gran).all()), "%s: a partial sum may round in fp32" % what
    return a @ b


def bf16_exact(x, what):
    assert bool((x.float().to(BF).double() == x).all()), "%s is not exactly representable in bf16" % what


def drop_params(p):
    return (0, 1.0) if p <= 0 else (min(int(p * 4294967296.0), 4294967295), 1.0 / (1.0 - p))


# ------------------------------------------------------------------------------------------------------ launches
class Slot:
    """logical (B, rows, H, 64) tensor at buffer[start + b*bs + r*ld + h*64 + d]"""

    def __init__(self, buf, start, ld, bs, rows):
        self.buf, self.start, self.ld, self.bs, self.rows = buf, start, ld, bs, rows

    def offsets(self, B, H, device):
        b = torch.arange(B, device=device).view(B, 1, 1, 1) * self.bs
        r = torch.arange(self.rows, device=device).view(1, self.rows, 1, 1) * self.ld
        hd = torch.arange(H * 64, device=device).view(1, 1, H, 64)
        return self.start + b + r + hd                      # (B, rows, H, 64)


class Launch:
    """Buffers, flash arguments and fp64 reference of one case on `device`."""

    def __init__(self, case, device, layout=None):
        c = self.case = case if layout is None else replace(case, layout=layout)
        self.device = device
        B, H, nq, nk = c.B, c.H, c.nq, c.nk
        self.g = torch.Generator().manual_seed(zlib.crc32(replace(c, layout="sep").id.encode()))
        Hd = H * 64
        self.bufs, self.init, self.slots, self.outputs = {}, {}, {}, set()

        # ---- layouts
        def own(name, rows, out, k):
            pad = 8 * (1 + k % 3)
            ld = Hd + pad
            bs = (rows + 1 + k % 2) * ld + 8 * (1 + k % 4)
            n = GUARD + (B - 1) * bs + rows * ld + GUARD + ld
            self._buffer(name, n, out)
            self.slots[name] = Slot(name, GUARD, ld, bs, rows)

        def packed(name, rows, names, out):
            ld = len(names) * Hd
            self._buffer(name, GUARD + B * rows * ld + GUARD, out)
            for i, nm in enumerate(names):
                self.slots[nm] = Slot(name, GUARD + i * Hd, ld, rows * ld, rows)

        def tight(name, rows, out):
            packed(name, rows, [name], out)

        if c.layout == "sep":
            for k, (nm, rows, out) in enumerate([("q", nq, 0), ("k", nk, 0), ("v", nk, 0), ("o", nq, 1), ("dout", nq, 0),
                                                 ("dq", nq, 1), ("dk", nk, 1), ("dv", nk, 1)]):
                own(nm, rows, out, k)
        elif c.layout == "self":
            assert nq == nk
            packed("qkv", nq, ["q", "k", "v"], 0)
            packed("dqkv", nq, ["dq", "dk", "dv"], 1)
            tight("o", nq, 1)
            tight("dout", nq, 0)
        else:
            tight("q", nq, 0)
            packed("kv", nk, ["k", "v"], 0)
            tight("dq", nq, 1)
            packed("dkv", nk, ["dk", "dv"], 1)
            tight("o", nq, 1)
            tight("dout", nq, 0)
        for nm in ("lse", "dsum"):
            self._buffer(nm, 2 * GUARD + B * H * nq, 1, F32)
        self.loff = {nm: s.offsets(B, H, device) for nm, s in self.slots.items()}

        # ---- values (fp64 on the CPU, (B, H, rows, 64) per tensor)
        V = self._values()
        self.val = V
        for nm in ("q", "k", "v", "dout"):
            s = self.slots[nm]
            self.bufs[s.buf][self.loff[nm]] = V[nm].permute(0, 2, 1, 3).to(device=device, dtype=BF)
        # kmask / bias: NaN guards around the addressed elements
        self.kmask = self.bias = self.dbias = None
        if V["kmask"] is not None:
            self._buffer("kmask", 2 * GUARD + B * nk, 0, F32)
            self.bufs["kmask"][GUARD:GUARD + B * nk] = V["kmask"].reshape(-1).to(device=device, dtype=F32)
        if c.bias:
            self._buffer("bias", 2 * GUARD + B * nq * nk, 0, F32)
            self.bufs["bias"][GUARD:GUARD + B * nq * nk] = V["bias"].reshape(-1).to(device=device, dtype=F32)
        if c.dbias:
            self._buffer("dbias", 2 * GUARD + B * nq * nk, 1, F32)
            self.bufs["dbias"][GUARD:GUARD + B * nq * nk] = V["dbias0"].reshape(-1).to(device=device, dtype=F32)
        self.drop = (0, 0, 1.0)
        if c.drop:
            th, sc = drop_params(c.drop)
            self.drop = (SEED, th, sc)
        self.init = {k: v.clone() for k, v in self.bufs.items()}
        self._reference()

    def _buffer(self, name, n, out, dt=BF):
        if out:
            self.bufs[name] = _sentinel(n, dt, self.device)
            self.outputs.add(name)
        else:
            self.bufs[name] = torch.full((n,), float("nan"), dtype=dt, device=self.device)

    # ------------------------------------------------------------------------------------------------ values
    def _mask(self):
        c, g = self.case, self.g
        B, nk = c.B, c.nk
        if c.mask == "none":
            return None
        km = torch.zeros(B, nk, dtype=F64)
        for b in range(B):
            kind = c.mask
            if kind in ("full10k", "fullinf") and b == 0:
                km[b] = -10000.0 if kind == "full10k" else float("-inf")
                continue
            if kind in ("mix", "full10k") and nk > 1:
                sel = torch.rand(nk, generator=g) < 0.3
                sel[int(torch.randint(0, nk, (1,), generator=g))] = False
                km[b, sel] = -10000.0
            if kind in ("tail", "fullinf") and nk > 1:
                km[b, nk - max(1, nk // (4 + b)):] = float("-inf")
        return km

    def _values(self):
        c, g = self.case, self.g
        B, H, nq, nk = c.B, c.H, c.nq, c.nk
        km = self._single_mask() if c.adv == "single" else self._mask()
        V = {"kmask": km}
        if c.family == "exact":
            V.update(self._exact_values(km))
        else:
            V.update(self._bound_values(km))
        if c.dbias:
            V["dbias0"] = torch.randint(-8, 9, (B, nq, nk), generator=g).double() / 4
        return V

    def _exact_values(self, km):
        c, g = self.case, self.g
        B, H, nq, nk = c.B, c.H, c.nq, c.nk
        cc = 128.0 / c.alpha
        nc = 2 * NCODE + 1
        codes = torch.stack(torch.meshgrid(*[torch.arange(GCODE)] * NCODE, indexing="ij"), -1).reshape(-1, NCODE)
        Q = torch.zeros(B, H, nq, 64, dtype=F64)
        K = torch.zeros(B, H, nk, 64, dtype=F64)
        win = torch.zeros(B, H, nq, nk, dtype=torch.bool)
        kfree = torch.ones(B, nk, dtype=torch.bool) if km is None else (km[:, :] == 0)
        for b in range(B):
            allsame = km is not None and bool((km[b] == km[b, 0]).all())
            if km is not None and km[b, 0] == float("-inf") and allsame:
                cand = torch.arange(nk)                     # fully -inf: codes irrelevant
            else:
                cand = torch.arange(nk) if allsame else kfree[b].nonzero()[:, 0]
            for h in range(H):
                # key codes: groups of 1, 2, 4, 8 keys spread over the key range share a code
                perm = torch.randperm(codes.shape[0], generator=g)
                kc = codes[perm[:nk]].clone()                      # distinct codes for every key
                stride = _coprime_stride(len(cand))
                order = cand[(torch.arange(len(cand)) * stride) % len(cand)]
                groups, i, j = [], 0, 0
                while i < len(order):
                    sz = min([1, 2, 4, 8][j % 4], len(order) - i)
                    sz = 1 << (sz.bit_length() - 1)
                    groups.append(order[i:i + sz])
                    kc[order[i:i + sz]] = kc[order[i]].clone()
                    i += sz
                    j += 1
                # queries pick groups so that consecutive queries cover the key range
                qg = torch.tensor([(q * 7 + h * 3 + b) % len(groups) for q in range(nq)])
                tgt = torch.stack([kc[groups[int(x)][0]] for x in qg]).double()         # (nq, NCODE)
                kd = kc.double()
                # Q . K = -cc |g - g*|^2 = sum_i (-cc g_i^2) + (2 cc g*_i) g_i + (-cc g*_i^2) * 1
                K[b, h, :, :NCODE] = kd * kd
                K[b, h, :, NCODE:2 * NCODE] = kd
                K[b, h, :, 2 * NCODE] = 1.0
                Q[b, h, :, :NCODE] = -cc
                Q[b, h, :, NCODE:2 * NCODE] = 2 * cc * tgt
                Q[b, h, :, 2 * NCODE] = -cc * (tgt * tgt).sum(-1)
                for q in range(nq):
                    win[b, h, q, groups[int(qg[q])]] = True
        # the other dimensions: Q on even, K on odd ones (disjoint), small integers
        rest = torch.arange(nc, 64)
        qd, kd_ = rest[rest % 2 == 0], rest[rest % 2 == 1]
        Q[..., qd] = torch.randint(-2, 3, (B, H, nq, len(qd)), generator=g).double()
        K[..., kd_] = torch.randint(-1, 2, (B, H, nk, len(kd_)), generator=g).double()

        def sparse_pm1(*shape, dens):
            return (torch.randint(0, 2, shape, generator=g) * 2 - 1).double() * (torch.rand(*shape, generator=g) < dens)
        Vv = sparse_pm1(B, H, nk, 64, dens=0.3)
        dO = sparse_pm1(B, H, nq, 64, dens=0.15)
        bias = None
        if c.bias:
            # a per-row power of two <= -2 (the row's LSE offset stays exact) plus offsets on entries that lose in every head
            beta = -(2.0 ** torch.randint(1, 4, (B, nq, 1), generator=g).double())
            anyw = win.any(1)
            off = torch.randint(-16, 17, (B, nq, nk), generator=g).double() / 4
            bias = beta + torch.where(anyw, torch.zeros_like(off), off)
        return {"q": Q, "k": K, "v": Vv, "dout": dO, "bias": bias, "win": win}

    def _bound_values(self, km):
        c, g = self.case, self.g
        B, H, nq, nk = c.B, c.H, c.nq, c.nk
        sd = 2.2 if c.adv == "big" else 1.0
        Q = torch.randn(B, H, nq, 64, generator=g) * sd
        K = torch.randn(B, H, nk, 64, generator=g) * sd
        if c.adv == "ramp":
            # logits grow with the key index in every row: a new maximum in every block, peaking at the last key
            Q[..., 0] = 4.0
            K[..., 0] = torch.linspace(-40.0, 80.0, nk)
            Q[..., 1:] *= 0.5
        if c.adv == "big":
            Q[..., 0] = 8.0
            K[..., 0] = (torch.rand(B, H, nk, generator=g) * 2 - 1) * 40.0
        Vv = torch.randn(B, H, nk, 64, generator=g)
        dO = torch.randn(B, H, nq, 64, generator=g) * 0.5
        bias = None
        if c.bias:
            bias = (torch.randn(B, nq, nk, generator=g) * 2.0).to(F32).double()
        out = {nm: t.to(BF).double() for nm, t in (("q", Q), ("k", K), ("v", Vv), ("dout", dO))}
        out["bias"] = bias
        return out

    def _single_mask(self):
        c, g = self.case, self.g
        km = torch.full((c.B, c.nk), float("-inf"), dtype=F64)
        for b in range(c.B):
            km[b, int(torch.randint(0, c.nk, (1,), generator=g))] = 0.0
        return km

    # ------------------------------------------------------------------------------------------------ reference
    def _reference(self):
        c, V = self.case, self.val
        B, H, nq, nk, alpha = c.B, c.H, c.nq, c.nk, c.alpha
        dev = self.device
        Q, K, Vv, dO = (V[n].to(dev) for n in ("q", "k", "v", "dout"))
        km = V["kmask"].to(dev) if V["kmask"] is not None else torch.zeros(B, nk, dtype=F64, device=dev)
        bias = V["bias"].to(dev) if V["bias"] is not None else torch.zeros(B, nq, nk, dtype=F64, device=dev)
        th, sc = self.drop[1], self.drop[2]
        keep = DM.attn_keep(SEED, B, H, nq, nk, th).to(dev) if th else torch.ones(B, H, nq, nk, dtype=torch.bool, device=dev)
        x = alpha * (Q @ K.transpose(-1, -2)) + km.view(B, 1, 1, nk) + bias.view(B, 1, nq, nk)   # natural-log logits
        dead = (x == float("-inf")).all(-1)                                                           # (B,H,nq)
        R = {}
        if c.family == "exact":
            exact_product(Q, K.transpose(-1, -2), "Q K^T")
            win = V["win"].to(dev)
            nw = win.sum(-1, keepdim=True).double()
            assert bool(((nw == 1) | (nw == 2) | (nw == 4) | (nw == 8)).all())
            # winners share the row's offset (mask / bias), the rest sit >= 150 below in the log2 domain
            x2 = x / math.log(2.0)
            wmax = torch.where(win, x2, torch.full_like(x2, float("-inf"))).amax(-1, keepdim=True)
            wmin = torch.where(win, x2, torch.full_like(x2, float("inf"))).amin(-1, keepdim=True)
            live = ~dead.unsqueeze(-1)
            assert bool(((wmax == wmin) | ~live).all()), "winners of a row differ"
            assert bool(((torch.where(win, torch.full_like(x2, -1e9), x2) <= wmax - 150) | ~live).all()), \
                "a loser is too close"
            P = torch.where(win & live, 1.0 / nw, torch.zeros_like(x))
            # LSE: the fp32 log2-domain offset of the winners (kmask log2 e or bias log2 e, one rounding) + log2 |W|
            off = (km.view(B, 1, 1, nk) + bias.view(B, 1, nq, nk)).expand(B, H, nq, nk)
            woff = torch.where(win, off, torch.full_like(off, float("inf"))).amin(-1)   # common offset of the row
            m32 = (woff.float() * LOG2E_F32.to(dev)).double()
            lse = m32 + (torch.frexp(nw[..., 0])[1] - 1).double()                       # log2 |W|, exactly
            assert bool(((lse.float().double() == lse) | dead).all()), "LSE is not exact in fp32"
            R["lse"] = torch.where(dead, torch.full_like(lse, float("inf")), lse)
        else:
            P = torch.softmax(x, -1).nan_to_num(0.0)
            mx = x.amax(-1)
            R["lse"] = torch.where(dead, torch.full_like(mx, float("inf")),
                                   (mx + torch.log(torch.exp(x - mx.unsqueeze(-1)).sum(-1))) / math.log(2.0))
            self.lse_mag = torch.where(dead, torch.zeros_like(mx), mx / math.log(2.0)).abs()
        Pd = torch.where(keep, P * sc, torch.zeros_like(P))
        if c.family == "exact":
            bf16_exact(P, "P")
            bf16_exact(Pd, "Pdrop")
            O = exact_product(Pd, Vv, "Pdrop V")
        else:
            O = Pd @ Vv
        R["o"] = O
        self.P, self.Pd, self.keep = P, Pd, keep
        self.R = R
        self.dO, self.Q, self.K, self.V = dO, Q, K, Vv
        self.sc = sc
        if c.family == "exact":
            self.backward_reference(O.permute(0, 2, 1, 3))

    def backward_reference(self, o_bhrd):
        """the backward's reference from the O passed to it ((B, nq, H, 64) fp64 values)"""
        c, R = self.case, self.R
        B, H, nq, nk, alpha = c.B, c.H, c.nq, c.nk, c.alpha
        O = o_bhrd.permute(0, 2, 1, 3)
        P, keep, sc, dO, Q, K, Vv = self.P, self.keep, self.sc, self.dO, self.Q, self.K, self.V
        exact = c.family == "exact"
        dP = exact_product(dO, Vv.transpose(-1, -2), "dO V^T") if exact else dO @ Vv.transpose(-1, -2)
        gk = torch.where(keep, dP * sc, torch.zeros_like(dP))
        D = (dO * O).sum(-1, keepdim=True)
        dS = P * (gk - D)
        if exact:
            exact_product(dO.unsqueeze(-2), O.unsqueeze(-1), "rowsum(dO o O)")
            bf16_exact(alpha * dS, "alpha dS")
            R["dq"] = exact_product(alpha * dS, K, "alpha dS K")
            R["dk"] = exact_product((alpha * dS).transpose(-1, -2), Q, "alpha dS^T Q")
            R["dv"] = exact_product(self.Pd.transpose(-1, -2), dO, "Pdrop^T dO")
        else:
            R["dq"] = alpha * dS @ K
            R["dk"] = alpha * dS.transpose(-1, -2) @ Q
            R["dv"] = self.Pd.transpose(-1, -2) @ dO
            A = P * (gk.abs() + D.abs())
            self.mag = {"o": self.Pd @ Vv.abs(), "dv": self.Pd.transpose(-1, -2) @ dO.abs(),
                        "dq": alpha * A @ K.abs(), "dk": alpha * A.transpose(-1, -2) @ Q.abs(), "dbias": A.sum(1)}
        if c.dbias:
            d0 = self.val["dbias0"].to(self.device)
            if exact:
                s = dS.abs().sum(1) + d0.abs()
                gran = torch.minimum(granule(dS.reshape(-1), 0), granule(d0.reshape(-1), 0))
                assert bool((s < 2.0 ** 24 * gran).all()), "dbias sum may round in fp32"
            R["dbias"] = d0 + dS.sum(1)

    # ---------------------------------------------------------------------------------------------------- launch
    def args(self, lib_struct):
        """bb_flash_args with every field of the case (the caller passes _lib.FlashArgs)"""
        c, s = self.case, self.slots
        a = lib_struct()

        def ptr(nm):
            sl = s[nm]
            return self.bufs[sl.buf].data_ptr() + 2 * sl.start

        def fptr(nm):
            return self.bufs[nm].data_ptr() + 4 * GUARD if nm in self.bufs else 0
        a.q, a.k, a.v, a.o = ptr("q"), ptr("k"), ptr("v"), ptr("o")
        a.q_bs, a.k_bs, a.v_bs, a.o_bs = s["q"].bs, s["k"].bs, s["v"].bs, s["o"].bs
        a.ldq, a.ldk, a.ldv, a.ldo = s["q"].ld, s["k"].ld, s["v"].ld, s["o"].ld
        a.B, a.H, a.nq, a.nk, a.dh = c.B, c.H, c.nq, c.nk, 64
        a.alpha = c.alpha
        a.kmask, a.bias, a.lse = fptr("kmask"), fptr("bias"), fptr("lse")
        a.seed, a.thresh, a.scale = self.drop
        a.dout, a.do_bs, a.lddo, a.dsum = ptr("dout"), s["dout"].bs, s["dout"].ld, fptr("dsum")
        a.dq, a.dk, a.dv = ptr("dq"), ptr("dk"), ptr("dv")
        a.dq_bs, a.dk_bs, a.dv_bs = s["dq"].bs, s["dk"].bs, s["dv"].bs
        a.lddq, a.lddk, a.lddv = s["dq"].ld, s["dk"].ld, s["dv"].ld
        a.dbias = fptr("dbias")
        return a

    def strided(self, nm):
        """(B, rows, H, 64) tensor aliasing a logical tensor's elements"""
        sl = self.slots[nm]
        buf = self.bufs[sl.buf]
        return torch.as_strided(buf, (self.case.B, sl.rows, self.case.H, 64), (sl.bs, sl.ld, 64, 1), sl.start)

    def view(self, nm):
        """(B, rows, H, 64) view of a logical tensor"""
        return self.bufs[self.slots[nm].buf][self.loff[nm]]

    def fview(self, nm, shape):
        n = 1
        for x in shape:
            n *= x
        return self.bufs[nm][GUARD:GUARD + n].view(shape)

    def reset(self):
        for k, v in self.init.items():
            self.bufs[k].copy_(v)

    # ---------------------------------------------------------------------------------------------------- checks
    def untouched(self, names=None):
        for k in (self.bufs if names is None else names):
            a, b = bits(self.bufs[k]), bits(self.init[k])
            if not torch.equal(a, b):
                self._fail_buf(k, a != b, "changed by a launch that must not write it")

    def _expected_buffer(self, buf, items):
        """initial bits of `buf` with `items` [(name, ref (B, rows, H, 64) fp64)] stored"""
        exp = self.init[buf].clone()
        for nm, ref in items:
            exp[self.loff[nm]] = ref.to(F32).to(exp.dtype)
        return exp

    def check_fwd(self, record=None):
        c = self.case
        B, H, nq = c.B, c.H, c.nq
        self.untouched([k for k in self.bufs if k not in self.outputs])
        o_ref = self.R["o"].permute(0, 2, 1, 3)
        lse = self.fview("lse", (B, H, nq))
        if c.family == "exact":
            self._cmp_exact("o", [("o", o_ref)])
            exp = self.init["lse"].clone()
            exp[GUARD:GUARD + B * H * nq] = self.R["lse"].reshape(-1).float()
            if not torch.equal(cbits(self.bufs["lse"]), cbits(exp)):
                self._fail_buf("lse", cbits(self.bufs["lse"]) != cbits(exp), "not exact", exp)
        else:
            self._cmp_bound("o", "o", o_ref, self.mag_o(), C_O, record)
            self._outside_ok("lse", GUARD, B * H * nq)
            ref = self.R["lse"]
            inf = torch.isinf(ref)
            got = lse.double()
            tol = ulp(self.lse_mag, F32) + 2.0 ** -20
            err = torch.where(inf, torch.zeros_like(ref), (got - ref).abs())
            bad = ~(err <= C_LSE * tol) | (inf & (got != ref))
            if record is not None:
                record["lse"] = max(record.get("lse", 0.0), float((err / tol).max()))
            if bool(bad.any()):
                self._fail_flat("lse", bad, got, ref, "outside the LSE bound")

    def mag_o(self):
        if not hasattr(self, "mag"):
            self.mag = {"o": self.Pd @ self.V.abs()}
        return self.mag["o"].permute(0, 2, 1, 3)

    def check_bwd(self, record=None):
        c = self.case
        B, H, nq, nk = c.B, c.H, c.nq, c.nk
        self.untouched([k for k in self.bufs if k not in self.outputs])
        self._outside_ok("dsum", GUARD, B * H * nq)
        refs = {nm: self.R[nm].permute(0, 2, 1, 3) for nm in ("dq", "dk", "dv")}
        if c.family == "exact":
            groups = {}
            for nm in ("dq", "dk", "dv"):
                groups.setdefault(self.slots[nm].buf, []).append((nm, refs[nm]))
            for buf, items in groups.items():
                self._cmp_exact(buf, items)
        else:
            for nm, cc in (("dq", C_DQ), ("dk", C_DK), ("dv", C_DV)):
                self._cmp_bound(self.slots[nm].buf, nm, refs[nm], self.mag[nm].permute(0, 2, 1, 3), cc, record)
        if c.dbias:
            n = B * nq * nk
            ref = self.R["dbias"].reshape(-1)
            got = self.bufs["dbias"][GUARD:GUARD + n].double()
            self._outside_ok("dbias", GUARD, n)
            if c.family == "exact":
                bad = cbits(self.bufs["dbias"][GUARD:GUARD + n]) != cbits(ref.float())
                what = "not bit-exact"
            else:
                unit = 2.0 ** -9 * self.mag["dbias"].reshape(-1)
                excess = ((got - ref).abs() - ulp(ref, F32)).clamp_min(0)
                if record is not None:
                    record["dbias"] = max(record.get("dbias", 0.0), float((excess / (unit + 1e-300)).max()))
                bad = ~(excess <= C_DB * unit)
                what = "outside the dbias bound"
            if bool(bad.any()):
                self._fail_flat("dbias", bad, got, ref, what, shape=(B, nq, nk), names=("b", "q", "k"))

    def _outside_ok(self, buf, start, n):
        b, i = bits(self.bufs[buf]), bits(self.init[buf])
        bad = b != i
        bad[start:start + n] = False
        if bool(bad.any()):
            self._fail_buf(buf, bad, "written outside its elements")

    def _cmp_exact(self, buf, items):
        exp = self._expected_buffer(buf, items)
        got = self.bufs[buf]
        if not torch.equal(cbits(got), cbits(exp)):
            self._fail_buf(buf, cbits(got) != cbits(exp), "not bit-exact", exp)

    def _cmp_bound(self, buf, nm, ref, mag, cc, record):
        exp = self._expected_buffer(buf, [])
        got = self.bufs[buf]
        pos = self.loff[nm]
        outside = torch.ones(got.numel(), dtype=torch.bool, device=got.device)
        for other, sl in self.slots.items():
            if sl.buf == buf:
                outside[self.loff[other].reshape(-1)] = False
        bad = torch.zeros_like(outside)
        bad[outside] = bits(got)[outside] != bits(exp)[outside]
        if bool(bad.any()):
            self._fail_buf(buf, bad, "written outside its elements")
        g = got[pos].double()
        half = ulp(ref, BF) / 2
        unit = 2.0 ** -9 * mag
        err = (g - ref).abs()
        if record is not None:
            r = ((err - half).clamp_min(0) / (unit + 1e-300))
            r = torch.where((err - half) <= 0, torch.zeros_like(r), r)
            record[nm] = max(record.get(nm, 0.0), float(r.max()))
        badl = ~(err <= half + cc * unit)
        if bool(badl.any()):
            idx = badl.nonzero()[0].tolist()
            raise AssertionError("%s: %s outside ulp/2 + %g 2^-9 bound: %d bad elements; first at (b=%d, row=%d, h=%d, "
                                 "col=%d): got %r, expected %r (bound %g)" % (
                                     self.case.id, nm, cc, int(badl.sum()), idx[0], idx[1], idx[2], idx[3],
                                     float(g[tuple(idx)]), float(ref[tuple(idx)]),
                                     float((half + cc * unit)[tuple(idx)])))

    def _fail_flat(self, buf, bad, got, ref, what, shape=None, names=("b", "h", "q")):
        c = self.case
        shape = shape or (c.B, c.H, c.nq)
        i = int(bad.reshape(-1).nonzero()[0, 0])
        idx = []
        for s in reversed(shape):
            idx.append(i % s)
            i //= s
        idx = idx[::-1]
        g, r = got.reshape(shape)[tuple(idx)], ref.reshape(shape)[tuple(idx)]
        raise AssertionError("%s: %s %s: %d bad elements; first at (%s): got %r, expected %r" % (
            c.id, buf, what, int(bad.sum()), ", ".join("%s=%d" % (n, v) for n, v in zip(names, idx)), float(g),
            float(r)))

    def _fail_buf(self, buf, bad, what, exp=None):
        c = self.case
        p = int(bad.nonzero()[0, 0])
        t = self.bufs[buf]
        mask = 0xFFFF if t.dtype == BF else 0xFFFFFFFF
        got = "0x%x (%r)" % (int(bits(t)[p]) & mask, float(t[p]))
        where = None
        for nm, sl in self.slots.items():
            if sl.buf != buf:
                continue
            hit = (self.loff[nm] == p).nonzero()
            if hit.numel():
                b, r, h, d = hit[0].tolist()
                where = "%s (b=%d, h=%d, row=%d, col=%d)" % (nm, b, h, r, d)
        if where is None and buf in ("lse", "dsum", "dbias", "kmask", "bias") and GUARD <= p:
            where = "element %d" % (p - GUARD)
        if where is None:
            where = "unaddressed element / guard at offset %d from the buffer's first element" % p
        if exp is not None:
            e = "0x%x (%r)" % (int(bits(exp)[p]) & mask, float(exp[p]))
        elif buf in self.outputs:
            e = "sentinel 0x%x" % SENT[t.dtype]
        else:
            e = "its input value"
        raise AssertionError("%s: %s %s: %d bad elements; first at %s: got %s, expected %s" % (
            c.id, buf, what, int(bad.sum()), where, got, e))


def _coprime_stride(n):
    if n <= 2:
        return 1
    s = max(1, int(n * 0.618))
    while math.gcd(s, n) != 1:
        s += 1
    return s


# ----------------------------------------------------------------------------------------------------- runners
def run_case(L, fwd, bwd, record=None):
    """forward, check, backward from the forward's own O / LSE, check"""
    fwd(L)
    L.check_fwd(record)
    if L.case.family == "bound":
        L.backward_reference(L.view("o").double())
    bwd(L)
    L.check_bwd(record)
