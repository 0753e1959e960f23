"""Cases, references and checkers for the VLN-CE view-embedding sum (bb_add_rows3 through kernels.add_rows(..., c=...),
blocks.AddRows3Impl) and the BEV known-answer points at 11 x 11 / 1 m.  Shared by tests/test_ce_add_rows3_gpu.py and
its CPU rehearsal tests/test_ce_pretrain_cpu.py.

Forward: out = fl_T(((a + b) + c) + table[idx] + vec) with fp32 additions in that order, T the activation type.  Every
operand element is a bf16 (or fp32) value, so fp32 arithmetic is exactly specified: the result must be BIT-IDENTICAL to
the same-order fp32 sum rounded to T (`same_order`), and within `bound` of the exact fp64 sum
(5 fp32 roundings of partial sums no larger than S = |a|+|b|+|c|+|t|+|v|, plus the final rounding to T).
Memory layout: row operands live inside NaN-filled buffers with padded row strides (columns [H, ld) and the rows past
the end hold NaN: a kernel that reads them produces NaN); the output sits between guard rows / columns holding a
sentinel that must survive bit for bit."""
import torch

F64, F32 = torch.float64, torch.float32
SENTINEL = -7.0e3

# (rows, H, lda, ldb, ldc, ldo, table, vec): ragged row counts, padded strides, every optional term on and off
CASES = [
    (1, 8, 8, 8, 8, 8, True, True),
    (7, 768, 768, 768, 768, 768, True, True),        # the model's shape class (H = 768)
    (33, 768, 776, 768, 784, 792, True, True),       # padded strides on every operand
    (257, 64, 72, 64, 64, 80, True, False),
    (255, 128, 128, 136, 128, 128, False, True),
    (1023, 16, 24, 16, 32, 16, False, False),
    (4099, 768, 768, 768, 768, 768, True, True),     # 1538 blocks of 256 threads: several waves
]


def _u(dt):
    return 2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -24


def make_case(case, act, seed, device="cpu"):
    """-> dict of operands (views into NaN-padded buffers), fp32 table / vec, int64 idx, the guarded output buffer."""
    rows, H, lda, ldb, ldc, ldo, use_t, use_v = case
    g = torch.Generator().manual_seed(seed)

    ops = {}
    for name, ld in (("a", lda), ("b", ldb), ("c", ldc)):
        buf = torch.full((rows + 2, ld), float("nan"), dtype=act)
        buf[:rows, :H] = (torch.randn(rows, H, generator=g) * 4).to(act)
        buf = buf.to(device)
        ops[name] = buf[:rows, :H]
        ops[name + "_buf"] = buf
    nt = 3                                               # table row nt is never indexed and holds NaN
    table = torch.cat([torch.randn(nt, H, generator=g) * 2, torch.full((1, H), float("nan"))], 0)
    ops["table"] = table.to(device) if use_t else None
    ops["idx"] = torch.randint(0, nt, (rows,), generator=g).to(device) if use_t else None
    ops["vec"] = torch.randn(H, generator=g).to(device) if use_v else None
    obuf = torch.full((rows + 2, ldo), SENTINEL, dtype=act).to(device)
    ops["out_buf"] = obuf
    ops["out"] = obuf[1:rows + 1, :H]
    return ops


def _terms(ops):
    t = [ops["a"], ops["b"], ops["c"]]
    if ops["table"] is not None:
        t.append(ops["table"][ops["idx"]])
    if ops["vec"] is not None:
        t.append(ops["vec"][None].expand_as(ops["a"]))
    return [x.cpu() for x in t]


def emu_add_rows(base):
    """CPU stand-in for kernels.add_rows with the third row operand (the same-order fp32 sum); `base` is the
    emulation of the two-operand form, which it keeps serving"""
    def add_rows(a, b=None, table=None, idx=None, vec=None, c=None, out=None):
        if c is None:
            return base(a, b, table, idx, vec)
        s = a.to(F32) + b.to(F32) + c.to(F32)
        if table is not None:
            s = s + table[idx]
        if vec is not None:
            s = s + vec[None]
        r = base(s)
        return r if out is None else out.copy_(r)
    return add_rows


def same_order(ops, act):
    """the fp32 left-to-right sum rounded to the activation type: what the kernel must produce bit for bit"""
    t = _terms(ops)
    s = t[0].to(F32)
    for x in t[1:]:
        s = s + x.to(F32)
    return s.to(act)


def check_forward(ops, act, name=""):
    """exactness against the same-order fp32 sum, the fp64 bound, and untouched guards; -> worst error / bound"""
    t = _terms(ops)
    out = ops["out"].cpu()
    exact = sum(x.to(F64) for x in t)
    S = sum(x.to(F64).abs() for x in t)
    bound = _u(act) * exact.abs() + 5 * 2.0 ** -24 * S * (1 + _u(act)) + 1e-30
    err = (out.to(F64) - exact).abs()
    assert torch.isfinite(out).all(), "%s: non-finite output (padding read?)" % name
    assert (err <= bound).all(), "%s: worst err/bound %.3g" % (name, float((err / bound).max()))
    assert torch.equal(out, same_order(ops, act)), "%s: not the same-order fp32 sum" % name
    ob = ops["out_buf"].cpu()
    rows, H = out.shape
    assert (ob[0] == SENTINEL).all() and (ob[rows + 1:] == SENTINEL).all(), "%s: guard row written" % name
    assert (ob[1:rows + 1, H:] == SENTINEL).all(), "%s: padding column written" % name
    return float((err / bound).max())


def check_backward(g, grads, ops, name=""):
    """AddRows3Impl backward: da = db = dc = g exactly; dtable = scatter-add of g by idx and dvec = column sum of g
    within the fp32 accumulation bound of the fp64 sums (n_terms * 2^-24 * sum|g|)."""
    gin, (dt, dv) = grads
    g64 = g.cpu().to(F64)
    for k, x in zip("abc", gin[:3]):
        assert x is not None and torch.equal(x.cpu(), g.cpu()), "%s: d%s is not the output gradient" % (name, k)
    rows = g.shape[0]
    if ops["table"] is not None:
        idx = ops["idx"].cpu()
        want = torch.zeros(ops["table"].shape, dtype=F64).index_add_(0, idx, g64)
        absum = torch.zeros(ops["table"].shape, dtype=F64).index_add_(0, idx, g64.abs())
        assert ((dt.cpu().to(F64) - want).abs() <= rows * 2.0 ** -24 * absum + 1e-30).all(), "%s: dtable" % name
    else:
        assert dt is None
    if ops["vec"] is not None:
        want, absum = g64.sum(0), g64.abs().sum(0)
        assert ((dv.cpu().to(F64)[1] - want).abs() <= rows * 2.0 ** -24 * absum + 1e-30).all(), "%s: dvec" % name
    else:
        assert dv is None


# ------------------------------------------------------------------------------------------ BEV at 11 x 11, 1 m
D_CE, RES_CE = 11, 1.0
# (x, y, z) ego-frame point -> expected flat cell (-1 = dropped); cell = 11 * round_half_even(z + 5) + round(x + 5)
LIFT_KATS = [
    ((0.0, 0.0, 0.0), 60),                                # the origin is the centre cell
    ((0.5, 0.0, 0.0), 61), ((-0.5, 0.0, 0.0), 59),        # x = +-0.5: 5.5 -> 6, 4.5 -> 4 (half to even)
    ((1.5, 0.0, 0.0), 61), ((-1.5, 0.0, 0.0), 59),        # x = +-1.5: 6.5 -> 6, 3.5 -> 4
    ((0.0, 0.0, 0.5), 71), ((0.0, 0.0, -0.5), 49),        # z = +-0.5: rows 6 / 4
    ((0.0, 0.0, 1.5), 71), ((0.0, 0.0, -1.5), 49),        # z = +-1.5: rows 6 / 4
    ((0.49, 0.0, 0.0), 60), ((0.51, 0.0, 0.0), 61),
    ((5.0, 0.0, 5.0), 120), ((-5.0, 0.0, -5.0), 0),       # the last and the first cell
    ((5.5, 0.0, 0.0), 65), ((5.51, 0.0, 0.0), -1),        # 10.5 -> 10 stays on the map, 10.51 -> 11 leaves it
    ((-5.5, 0.0, 0.0), 55), ((-5.51, 0.0, 0.0), -1),      # -0.5 -> 0 stays, -0.51 -> -1 leaves
    ((0.0, 0.5, 0.0), 60), ((0.0, 0.50001, 0.0), -1),     # height clip: y > 0.5 is dropped, y = 0.5 kept
]


def lift_kat_points():
    """(1, n, 3) fp32 points, (1, n) no-depth mask (all False), (n,) expected cells"""
    pts = torch.tensor([p for p, _ in LIFT_KATS], dtype=F32)[None]
    return pts, torch.zeros(1, pts.shape[1], dtype=torch.bool), torch.tensor([c for _, c in LIFT_KATS])
