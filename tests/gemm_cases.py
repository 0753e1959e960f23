"""Integer-operand cases of the GEMM contract (include/bevbert_b200.h, bb_gemm_args) with an exact fp64 reference
(test infrastructure, shared by tests/test_gemm_gpu.py and tests/test_gemm_harness_cpu.py).

Every operand element is -1, 0 or 1, so every product and every partial sum is an integer far below 2^24: the fp32
accumulator equals the exact result whatever the MMA order, the split or the order of the atomics.  Bias is a multiple
of 1/4, alpha is 1 or 1/8, aux_in / add_in are multiples of 1/4 and dropout has p = 0.5 (scale 2.0).  Everything the
epilogue does apart from GELU / gelu' is then exact in fp32, and each output is one round-to-nearest-even of an exact
value.  The reference restates the contract in fp64 from the same integers, in the documented order
    alpha*acc + bias -> aux_out -> act -> epi_mul -> dropout -> + add_in -> store or accumulate,
and the outputs are compared bit for bit.  For bf16 outputs the operand density keeps |acc| well below 256, so an
accumulator that is off by one cannot hide in the output rounding; the reference asserts the bound it relies on.

GELU / gelu' (erff, __expf) are compared with fp64 GELU of the exact fp32 pre-activation: within one output ulp plus
2^-22 |x| absolute (x: the value GELU or the gelu' factor is applied to; 1 + erff(x / sqrt 2) cancels for negative x,
so fp32 GELU has only absolute accuracy there, about 2 fp32 ulps of erff times |x| / 2).  For bf16 outputs, at least
99 % of the elements where 2^-22 |x| is below 2^-9 of a bf16 ulp (at least 80 % of them) must be bit-exact.  Over all
elements the bit-exact share is lower (98.6 % measured on an H100 at pre-activations of standard deviation 1.5): for
x below about -2 the absolute error of fp32 GELU is a visible fraction of the bf16 ulp of a result that small.

Buffers: operand elements the kernel must not read (columns k >= K inside lda, rows past M / N inside a batch stride,
batch gaps) hold NaN, so one stray read turns outputs into NaN.  D, aux_out, aux_in and add_in live in larger buffers
with GUARD elements before and after; guards and unaddressed elements (padding columns, batch gaps) hold a NaN
sentinel bit pattern that must survive the launch.  A misaligned pointer is a view that starts 1..7 elements into its
buffer.
"""
import math
import zlib
from dataclasses import dataclass, replace

import torch

import drop_masks as DM

BF = torch.bfloat16
F32 = torch.float32
GUARD = 64
SEED = 0xC0FFEE5EED5A1701          # >= 2^63, like the seeds DropState draws
DROP_P = 0.5
SENTINEL = {BF: 0x7FA5, F32: 0x7FA5A5A5}       # NaN bit patterns of the guards / unaddressed elements
_BITS = {BF: torch.int16, F32: torch.int32}
MAJORS = {"NT": (0, 0), "NN": (0, 1), "TN": (1, 0), "TT": (1, 1)}   # (a_mn, b_mn): T = stored MN-major

# epilogue features of each variant label; the first five are compile-time variants of gemm_tc.cu, the rest reach
# EPI_GENERIC (the fp32-output GELU through out="f32")
VARIANTS = {
    "plain": {},
    "gelu_pre": dict(act=1, aux_out=True),
    "dgelu": dict(epi_mul=1),
    "drelu": dict(epi_mul=2),
    "add": dict(add_in=True),
    "relu": dict(act=2),
    "gelu": dict(act=1),
    "auxout": dict(aux_out=True),
    "gelu_f32": dict(act=1, aux_out=True),
    "dgelu_add": dict(epi_mul=1, add_in=True),
    "drelu_add": dict(epi_mul=2, add_in=True),
    "relu_add": dict(act=2, add_in=True),
}


@dataclass(frozen=True)
class Case:
    variant: str
    M: int
    N: int
    K: int
    maj: str = "NT"
    out: str = "bf16"          # D dtype in the bf16 arm ("f32": fp32 output); the fp32 arm always stores fp32
    alpha: float = 1.0
    bias: bool = False
    drop: bool = False
    accumulate: bool = False
    split_k: int = 1
    block_n: int = 128
    nb: tuple = (1, 1)
    ldd: str = "n"             # "n": ldd = N; "pad": ldd > N, ldd % 8 == 0; "odd": ldd % 8 != 0
    attn: int = 0              # > 0: batch b1 is a column offset of `attn` elements within a row (attention output)
    lda_pad: bool = False      # lda / ldb well past the inner extent
    mis: str = ""              # "D" / "aux_in" / "add_in" / "aux_out": that pointer 1..7 elements off 16-byte alignment
    std: float = 0.0           # target standard deviation of acc (0: by variant)

    @property
    def feats(self):
        f = dict(act=0, aux_out=False, epi_mul=0, add_in=False)
        f.update(VARIANTS[self.variant])
        return f

    @property
    def id(self):
        lay = "ldd_" + self.ldd
        if self.nb != (1, 1):
            lay += "-b%dx%d" % self.nb
        if self.attn:
            lay += "-attn%d" % self.attn
        if self.lda_pad:
            lay += "-ldpad"
        if self.mis:
            lay += "-mis_" + self.mis
        extra = "%s-a%g%s%s" % (self.out, self.alpha, "-bias" if self.bias else "", "-drop" if self.drop else "")
        if self.accumulate:
            extra += "-acc"
        if self.split_k > 1:
            extra += "-split%d" % self.split_k
        return "%s-%dx%dx%d-%s-bn%d-%s-%s" % (self.variant, self.M, self.N, self.K, lay, self.block_n, self.maj, extra)


def _r8(n):
    return (n + 7) // 8 * 8


# ------------------------------------------------------------------------------------------------------- the table
M_RES = [1, 9, 17, 33, 63, 64, 65, 100, 127, 0]
KS = [8, 16, 40, 64, 72, 136, 1000]
LDDS = ["n", "pad", "n", "odd"]


def _plain_rows():
    rows, i = [], 0
    for bn in (64, 128):
        for n in [bn + r for r in range(8)] + [5]:     # every N % 8 residue past a full tile, and N < 8
            rows.append(Case("plain", M=128 * (1 + i % 2) + M_RES[i % 10], N=n, K=KS[i % 7], maj=list(MAJORS)[i % 4],
                             out="f32" if i % 3 == 0 else "bf16", alpha=0.125 if i % 4 in (1, 2) else 1.0,
                             bias=i % 2 == 0, block_n=bn, ldd=LDDS[i % 4], lda_pad=i % 5 == 0))
            i += 1
    for j, (m, n, k, maj) in enumerate([(300, 296, 136, "NT"), (77, 45, 40, "TT"), (1000, 200, 72, "NN")]):
        rows.append(Case("plain", m, n, k, maj=maj, bias=True, alpha=0.125 if j == 1 else 1.0, block_n=0,
                         out="f32" if j == 2 else "bf16"))
    return rows


def _fused_rows():
    rows, i = [], 0
    for v in ("gelu_pre", "dgelu", "drelu", "add"):
        for drop in (False, True):
            for bn in (64, 128):
                for maj in ("NT", "NN"):
                    rows.append(Case(v, M=128 * (1 + i % 3) + M_RES[(3 * i) % 10], N=bn * (1 + i % 2) + (i * 3) % 8,
                                     K=KS[i % 7], maj=maj, alpha=0.125 if i % 2 else 1.0, bias=v != "add" or i % 2 == 0,
                                     drop=drop, block_n=bn, ldd=LDDS[(i // 2) % 4], lda_pad=i % 3 == 0))
                    i += 1
    # the model's widths at a ragged row count, and block_n = 0
    rows.append(Case("gelu_pre", 333, 3072, 768, bias=True, alpha=0.125, block_n=0))
    rows.append(Case("dgelu", 333, 768, 3072, maj="NN", block_n=0, drop=True))
    return rows


def _generic_rows():
    rows, i = [], 0
    specs = [("relu", {}), ("gelu", dict(bias=True)), ("auxout", dict(bias=True, alpha=0.125)),
             ("gelu_f32", dict(out="f32", bias=True, drop=True)), ("dgelu_add", {}), ("drelu_add", dict(drop=True)),
             ("relu_add", dict(bias=True))]
    for v, kw in specs:
        for bn in (64, 128):
            rows.append(Case(v, M=128 + M_RES[(2 * i + 1) % 10], N=bn + 1 + (2 * i) % 7, K=KS[(i + 2) % 7],
                             maj="NN" if i % 2 else "NT", block_n=bn, ldd=LDDS[i % 4], **kw))
            i += 1
    return rows


def _layout_rows():
    rows = []
    # each pointer misaligned alone (the scalar path of every chunk), the others aligned
    for j, (v, mis, kw) in enumerate([("plain", "D", dict(bias=True)), ("plain", "D", dict(out="f32", alpha=0.125)),
                                      ("gelu_pre", "D", dict(bias=True, alpha=0.125)), ("dgelu", "D", {}),
                                      ("add", "D", dict(drop=True)), ("dgelu", "aux_in", dict(drop=True)),
                                      ("drelu", "aux_in", {}), ("add", "add_in", {}),
                                      ("dgelu_add", "add_in", {}), ("gelu_pre", "aux_out", dict(alpha=0.125)),
                                      ("auxout", "aux_out", dict(bias=True))]):
        rows.append(Case(v, M=128 + M_RES[j % 10], N=136 + j % 8, K=KS[j % 7], maj="NN" if j % 2 else "NT",
                         block_n=64 if j % 2 else 128, mis=mis, **kw))
    # batched 2 x 3 with gaps between batches
    for j, (v, maj, kw) in enumerate([("plain", "NT", dict(bias=True)), ("plain", "TT", dict(out="f32")),
                                      ("plain", "TN", dict(alpha=0.125)), ("gelu_pre", "NT", dict(bias=True)),
                                      ("dgelu", "NN", {}), ("add", "NN", dict(drop=True)),
                                      ("relu_add", "NT", dict(drop=True))]):
        rows.append(Case(v, M=100 + 37 * j, N=72 + 9 * j, K=KS[j % 7], maj=maj, nb=(2, 3), block_n=64 if j % 2 else 128,
                         ldd=["n", "pad", "odd"][j % 3], lda_pad=j % 2 == 1, **kw))
    # attention output: heads interleave within a row (ctx), tight, padded and ragged
    for j, (n, ds1, v) in enumerate([(64, 64, "plain"), (61, 64, "plain"), (60, 60, "plain"), (61, 64, "add"),
                                     (57, 57, "plain")]):
        rows.append(Case(v, M=77 + 50 * j, N=n, K=64, nb=(3, 2), attn=ds1, block_n=64, drop=v == "add",
                         out="f32" if j == 4 else "bf16"))
    return rows


def _split_rows():
    """accumulate / split-K rows (EPI_ATOMIC; EPI_SPLIT_DET under the deterministic flag)"""
    rows = []
    for j, maj in enumerate(MAJORS):
        rows.append(Case("plain", 200 + j, 136 + j, 64 * (j + 1) + 8, maj=maj, out="f32", accumulate=True,
                         bias=j % 2 == 0, block_n=64 if j % 2 else 128, ldd="odd" if j == 3 else "n"))
    for j, (m, n, k, split, maj) in enumerate([(256, 256, 1000, 3, "NT"), (200, 136, 1000, 5, "NN"),
                                               (130, 70, 136, 5, "TN"), (300, 190, 72, 3, "TT"),
                                               (129, 257, 520, 2, "TT"), (65, 200, 1000, 2, "NT"),
                                               (333, 129, 640, 5, "TN"), (128, 128, 40, 2, "NN")]):
        rows.append(Case("plain", m, n, k, maj=maj, out="f32", split_k=split, accumulate=j % 2 == 0,
                         bias=j % 3 != 1, block_n=64 if j % 2 else 128, ldd=["n", "odd", "pad"][j % 3],
                         alpha=0.125 if j == 5 else 1.0, lda_pad=j == 6))
    rows.append(Case("plain", 100, 200, 520, out="f32", split_k=3, nb=(2, 3), bias=True, block_n=64))
    return rows


FULL_ROWS = [
    Case("gelu_pre", 14112, 3072, 768, alpha=0.125, bias=True, block_n=0),
    Case("dgelu", 14112, 3072, 768, maj="NN", block_n=0),
    Case("add", 14112, 768, 2304, maj="NN", bias=True, block_n=0),
    Case("plain", 768, 3072, 14112, maj="TT", out="f32", accumulate=True, split_k=8, block_n=0),
]

PINGPONG_TILES = ["1", "2", "3", "sms-1", "sms", "sms+1", "2*sms+1", "3*sms"]


def pingpong_case(variant, tiles_expr, sms):
    """128-wide tiles, one tile column: `tiles_expr` (in terms of the SM count) tiles in all; the last tile row is
    ragged except for a single tile.  K = 136: three k-blocks per tile, so the stage ring wraps."""
    t = eval(tiles_expr, {"sms": sms})
    m = 128 * t - (0 if t == 1 else 37)
    kw = dict(bias=True, alpha=0.125) if variant != "dgelu" else {}
    return Case(variant, m, 128, 136, maj="NN" if variant == "dgelu" else "NT", block_n=128, **kw)


SPLIT_ROWS = _split_rows()
TABLE = _plain_rows() + _fused_rows() + _generic_rows() + _layout_rows() + SPLIT_ROWS


def fp32_arm_rows(rows):
    """the rows that apply to the fp32 verification arm (gemm_f32.cu): no tile width, no alignment paths, one row
    per remaining configuration"""
    seen, out = set(), []
    for c in rows:
        if c.mis:
            continue
        c = replace(c, block_n=0, out="f32")
        if c.id not in seen:
            seen.add(c.id)
            out.append(c)
    return out


# ------------------------------------------------------------------------------------------------------- buffers
def _sentinel(n, dt, device):
    return torch.full((n,), SENTINEL[dt], dtype=_BITS[dt], device=device).view(dt)


def bits(t):
    return t.view(_BITS[t.dtype])


class Launch:
    """Buffers, launch arguments and exact reference of one case.  `arm32`: fp32 operands / aux (verification arm)."""

    def __init__(self, case, device, arm32=False):
        c = self.case = case
        self.device, self.arm32 = device, arm32
        f = c.feats
        adt = F32 if arm32 else BF
        odt = F32 if (arm32 or c.out == "f32") else BF
        self.adt, self.odt = adt, odt
        # the values depend on the logical problem only, so a misaligned launch of it sees the same numbers
        g = torch.Generator().manual_seed(zlib.crc32(replace(c, mis="").id.encode()))
        nb1, nb2 = c.nb
        M, N, Kd = c.M, c.N, c.K
        a_mn, b_mn = MAJORS[c.maj]
        gelu_family = f["act"] == 1 or f["epi_mul"] == 1
        std = c.std or ((12.0 if c.alpha < 1 else 1.5) if f["act"] == 1 else 6.0)
        dens = min(1.0, std / math.sqrt(Kd))

        def operand(rows, mn, pad):
            inner = (rows if mn else Kd)
            outer = (Kd if mn else rows)
            ld = _r8(inner) + (40 if pad else 0)
            s1 = outer * ld + (16 if nb1 > 1 else 0)
            s2 = nb1 * s1 + (24 if nb2 > 1 else 0)
            n = (nb2 - 1) * s2 + (nb1 - 1) * s1 + outer * ld + 16
            buf = torch.full((n,), float("nan"), dtype=adt)
            vals = (torch.randint(0, 2, (nb2, nb1, rows, Kd), generator=g) * 2 - 1) * \
                (torch.rand(nb2, nb1, rows, Kd, generator=g) < dens)
            strides = (s2, s1, 1, ld) if mn else (s2, s1, ld, 1)
            torch.as_strided(buf, vals.shape, strides).copy_(vals)
            return buf.to(device), vals.to(device=device, dtype=torch.float64), ld, (s1 if nb1 > 1 else 0,
                                                                                   s2 if nb2 > 1 else 0)

        self.a, A64, self.lda, self.a_s = operand(M, a_mn, c.lda_pad)
        self.b, B64, self.ldb, self.b_s = operand(N, b_mn, c.lda_pad)
        self.a_mn, self.b_mn = a_mn, b_mn

        # output layout, shared by D, aux_out, aux_in and add_in
        if c.attn:
            ldd = nb1 * c.attn
            d_s1, d_s2 = c.attn, M * ldd
        else:
            ldd = {"n": N, "pad": _r8(N) + 16, "odd": N + 3 if (N + 3) % 8 else N + 5}[c.ldd]
            d_s1 = M * ldd + (16 if ldd % 8 == 0 else 5) if nb1 > 1 else 0
            d_s2 = nb1 * max(d_s1, M * ldd) + 8 if nb2 > 1 else 0
        self.ldd, self.d_s = ldd, (d_s1, d_s2)
        b1 = torch.arange(nb1, dtype=torch.int64, device=device).view(1, nb1, 1, 1)
        b2 = torch.arange(nb2, dtype=torch.int64, device=device).view(nb2, 1, 1, 1)
        m = torch.arange(M, dtype=torch.int64, device=device).view(1, 1, M, 1)
        n = torch.arange(N, dtype=torch.int64, device=device).view(1, 1, 1, N)
        self.loff = b1 * d_s1 + b2 * d_s2 + m * ldd + n          # element offset in D of logical (b2, b1, m, n)
        extent = int(self.loff.max()) + 1
        self.buflen = 2 * GUARD + 8 + extent
        assert torch.unique(self.loff).numel() == self.loff.numel(), "output layout overlaps itself"

        mis = {"D": 3, "aux_in": 5, "add_in": 1, "aux_out": 7}
        self.start = {k: GUARD + (mis[k] if c.mis == k else 0) for k in mis}
        self.bufs, self.views = {}, {}

        def outbuf(name, dt, vals=None):
            buf = _sentinel(self.buflen, dt, device)
            if vals is not None:
                buf[self.start[name] + self.loff] = vals.to(F32).to(dt)
            self.bufs[name] = buf
            self.views[name] = buf[self.start[name]:]
            return vals

        def quarters(lo, hi):
            v = torch.randint(int(4 * lo), int(4 * hi) + 1, (nb2, nb1, M, N), generator=g).double() / 4
            return v.to(device)

        D0 = None
        if c.accumulate or c.split_k > 1:
            D0 = torch.randint(-16, 17, (nb2, nb1, M, N), generator=g).double().to(device)
        outbuf("D", odt, D0)
        aux_in = outbuf("aux_in", adt, quarters(-3, 3)) if f["epi_mul"] else None
        add_in = outbuf("add_in", adt, quarters(-8, 8)) if f["add_in"] else None
        if f["aux_out"]:
            outbuf("aux_out", adt)
        self.bias = None
        if c.bias:
            bias = torch.full((_r8(N) + 8,), float("nan"))
            bias[:N] = torch.randint(-8, 9, (N,), generator=g).double() / 4
            self.bias = bias.to(device)
        self.drop = (0, 0, 1.0)
        if c.drop:
            th, sc = drop_params(DROP_P)
            assert sc == 2.0
            self.drop = (SEED, th, sc)
        self.init = {k: v.clone() for k, v in self.bufs.items()}

        # ---- reference, fp64, in the header's order
        acc = A64 @ B64.transpose(-1, -2)
        amax = float(acc.abs().max())
        bf16_out = odt == BF or (f["aux_out"] and adt == BF)
        assert amax < (256 if bf16_out else 2 ** 24), "operand density too high for an exact bf16 comparison (%g)" % amax
        v = acc * c.alpha
        if self.bias is not None:
            v = v + self.bias[:N].double()
        pre = v
        self.ref = {}
        if f["aux_out"]:
            self.ref["aux_out"] = pre
        if f["act"] == 1:
            v = gelu64(v)
        elif f["act"] == 2:
            v = v.clamp_min(0)
        mag = pre.abs()
        if f["epi_mul"] == 1:
            v = v * dgelu64(aux_in)
        elif f["epi_mul"] == 2:
            v = torch.where(aux_in > 0, v, torch.zeros_like(v))
        if c.drop:
            keep = DM.keep_elem(SEED, self.loff.reshape(-1), self.drop[1]).view(self.loff.shape).to(device)
            v = torch.where(keep, v * 2.0, torch.zeros_like(v))
            mag = torch.where(keep, mag * 2.0, torch.zeros_like(mag))      # a dropped element is exact
        if add_in is not None:
            v = v + add_in
        if D0 is not None:
            v = D0 + v
        self.ref["D"] = v
        self.tol_mag = mag if gelu_family else None     # the D comparison is a tolerance one
        for k, r in self.ref.items():
            if k == "D" and gelu_family:
                continue
            assert bool((r.float().double() == r).all()), "%s reference is not exact in fp32" % k

    # ---------------------------------------------------------------------------------------------------- launch
    def kwargs(self, **over):
        c, f = self.case, self.case.feats
        kw = dict(a=self.a, b=self.b, out=self.views["D"], M=c.M, N=c.N, K=c.K, lda=self.lda, ldb=self.ldb,
                  ldd=self.ldd, a_mn=bool(self.a_mn), b_mn=bool(self.b_mn), nb1=c.nb[0], nb2=c.nb[1], a_s=self.a_s,
                  b_s=self.b_s, d_s=self.d_s, alpha=c.alpha, bias=self.bias, act=f["act"],
                  aux_out=self.views.get("aux_out"), aux_in=self.views.get("aux_in"), epi_mul=f["epi_mul"],
                  add_in=self.views.get("add_in"), accumulate=c.accumulate, split_k=c.split_k, drop=self.drop,
                  block_n=0 if self.arm32 else c.block_n)
        kw.update(over)
        return kw

    def run(self, gemm, **over):
        kw = self.kwargs(**over)
        gemm(kw.pop("a"), kw.pop("b"), kw.pop("out"), kw.pop("M"), kw.pop("N"), kw.pop("K"), kw.pop("lda"),
             kw.pop("ldb"), kw.pop("ldd"), **kw)

    def reset(self):
        for k, v in self.init.items():
            self.bufs[k].copy_(v)

    # ---------------------------------------------------------------------------------------------------- checks
    def logical(self, name):
        """the addressed elements of an output-like buffer as a (nb2, nb1, M, N) tensor"""
        return self.bufs[name][self.start[name] + self.loff]

    def untouched(self, names=None):
        """every buffer (or `names`) bit for bit as before the launch"""
        for k in (self.bufs if names is None else names):
            if not torch.equal(bits(self.bufs[k]), bits(self.init[k])):
                self._fail(k, bits(self.bufs[k]) != bits(self.init[k]), "changed by a launch that must not write it")

    def check(self):
        """outputs against the reference, guards and unaddressed elements against the sentinel, inputs unchanged"""
        self.untouched([k for k in ("aux_in", "add_in") if k in self.bufs])
        for name, ref in self.ref.items():
            buf = self.bufs[name]
            dt = buf.dtype
            pos = (self.start[name] + self.loff).reshape(-1)
            if name == "D" and self.tol_mag is not None:
                outside = torch.ones(self.buflen, dtype=torch.bool, device=buf.device)
                outside[pos] = False
                bad = torch.zeros_like(outside)
                bad[outside] = bits(buf)[outside] != bits(self.init[name])[outside]
                got = buf[pos].double()
                r = ref.reshape(-1)
                tol = ulp(r, dt) + 2.0 ** -22 * self.tol_mag.reshape(-1)
                bad[pos] = ~((got - r).abs() <= tol)           # NaN fails
                if bool(bad.any()):
                    self._fail(name, bad, "outside one output ulp + 2^-22 |x|", ref)
                if dt == BF:
                    # where fp32 GELU / gelu' is accurate to far below a bf16 ulp (not where 1 + erff cancels), the
                    # output is the bf16 rounding of the exact value, bar a rare near-tie
                    well = 2.0 ** -22 * self.tol_mag.reshape(-1) <= 2.0 ** -9 * ulp(r, BF)
                    exact = bits(buf[pos]) == bits(r.float().to(BF))
                    fw, fe = float(well.double().mean()), float(exact[well].double().mean())
                    assert fw >= 0.8 and fe >= 0.99, "%s %s: %.4f of the elements well conditioned, %.4f of those " \
                        "bit-exact (%.4f of all)" % (self.case.id, name, fw, fe, float(exact.double().mean()))
            else:
                exp = self.init[name].clone()
                exp[pos] = ref.reshape(-1).to(F32).to(dt)
                if not torch.equal(bits(buf), bits(exp)):
                    self._fail(name, bits(buf) != bits(exp), "not bit-exact", ref)

    def _fail(self, name, bad, what, ref=None):
        buf = self.bufs[name]
        p = int(bad.nonzero()[0, 0])
        nbad = int(bad.sum())
        inv = torch.full((self.buflen,), -1, dtype=torch.int64, device=buf.device)
        inv[(self.start[name] + self.loff).reshape(-1)] = torch.arange(self.loff.numel(), device=buf.device)
        li = int(inv[p])
        got = "0x%x (%r)" % (int(bits(buf)[p]) & (0xFFFF if buf.dtype == BF else 0xFFFFFFFF), float(buf[p]))
        if li < 0:
            where = "unaddressed element / guard at offset %d from the pointer" % (p - self.start[name])
            exp = "sentinel 0x%x" % SENTINEL[buf.dtype] if name not in ("aux_in", "add_in") else "its input value"
        else:
            nb2, nb1, M, N = self.loff.shape
            b2, r = divmod(li, nb1 * M * N)
            b1, r = divmod(r, M * N)
            row, col = divmod(r, N)
            where = "(b1=%d, b2=%d, row=%d, col=%d)" % (b1, b2, row, col)
            if ref is not None:
                e = ref.reshape(-1)[li]
                eb = bits(e.float().to(buf.dtype).reshape(1))[0]
                exp = "0x%x (%r)" % (int(eb) & (0xFFFF if buf.dtype == BF else 0xFFFFFFFF), float(e))
            else:
                exp = "unchanged"
        raise AssertionError("%s: %s %s: %d bad elements; first at %s: got %s, expected %s" % (
            self.case.id, name, what, nbad, where, got, exp))


def drop_params(p):
    return min(int(p * 4294967296.0), 4294967295), 1.0 / (1.0 - p)


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def dgelu64(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def ulp(x, dt):
    """one unit in the last place of dtype dt (bf16 or fp32) at the magnitude of the fp64 values x"""
    p = 8 if dt == BF else 24
    _, e = torch.frexp(x)
    e = torch.where(x == 0, torch.full_like(e, -125), e).clamp_min(-125)
    return torch.ldexp(torch.ones_like(x), e - p)
