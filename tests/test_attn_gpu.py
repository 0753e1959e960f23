"""The fused attention cores element by element against fp64 (tests/attn_cases.py explains the two families, the
buffers and the bounds).

- The table through bb_flash_fwd / bb_flash_bwd with FlashArgs built directly (alpha, batch strides and every ld are
  the case's): both cores forced (set_attn_tc 0 / 2) and the default dispatch, forward on one core and backward on
  the other, the graph-bias case, dbias in the atomic and the deterministic mode.  Exact-routing rows bit for bit;
  error-bounded rows within their per-element bounds.
- The model's packed layouts give bit-identical results to the separate-buffer launch.
- The exact-routing rows through the paths that materialise P: bb_softmax_fwd / _bwd at ld on each side of the
  128 / 512 template boundaries and up to 1024, and bb_attn_scores modes 0 and 1; columns [nk, ldp) must be zero.
- Which kernels a call reaches (torch.profiler kernel names).
- Host-side argument checks: the library's message, no launch, buffers untouched.
"""
import contextlib
import ctypes as C
import re

import pytest
import torch

import attn_cases as A
import drop_masks as DM

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def K():
    import bevbert_b200.kernels as K
    from bevbert_b200 import _lib
    assert torch.cuda.is_available()
    _lib.load().bb_set_drop_salt_ptr(None)       # a graph test in the same process may have registered a dropout salt
    prec = K.set_precision(False)
    mode = K.set_attn_tc(1)
    K.set_attn_tc(mode)
    det = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    fill = torch.utils.deterministic.fill_uninitialized_memory
    try:
        yield K
    finally:
        K.set_precision(prec)
        K.set_attn_tc(mode)
        torch.use_deterministic_algorithms(det[0], warn_only=det[1])
        torch.utils.deterministic.fill_uninitialized_memory = fill


@contextlib.contextmanager
def deterministic(on=True):
    """torch's deterministic flag for the launches inside only"""
    prev = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    fill = torch.utils.deterministic.fill_uninitialized_memory
    torch.use_deterministic_algorithms(on)
    torch.utils.deterministic.fill_uninitialized_memory = False
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
        torch.utils.deterministic.fill_uninitialized_memory = fill


@contextlib.contextmanager
def core(K, name):
    prev = K.set_attn_tc(A.CORES[name])
    try:
        yield
    finally:
        K.set_attn_tc(prev)


def _lib():
    from bevbert_b200 import _lib as L
    return L


def flash(K, L, which, **over):
    """one bb_flash_fwd / _bwd call on the case's core; returns (rc, message)"""
    lib = _lib()
    a = L.args(lib.FlashArgs)
    for k, v in over.items():
        setattr(a, k, v)
    fn = lib.load().bb_flash_fwd if which == "fwd" else lib.load().bb_flash_bwd
    with core(K, L.case.fwd if which == "fwd" else L.case.bwd):
        with deterministic(L.case.dbias == "det" and which == "bwd"):
            rc = fn(C.byref(a), K._stream())
    msg = lib.load().bb_last_error()
    return rc, (msg.decode() if msg else "")


def runners(K):
    def fwd(L):
        rc, msg = flash(K, L, "fwd")
        assert rc == 0, msg
        torch.cuda.synchronize()

    def bwd(L):
        rc, msg = flash(K, L, "bwd")
        assert rc == 0, msg
        torch.cuda.synchronize()
    return fwd, bwd


RATIOS = {}


# ---------------------------------------------------------------------------------------------------------- table
@pytest.mark.parametrize("case", A.EXACT_ROWS, ids=lambda c: c.id)
def test_attn_exact(K, case):
    A.run_case(A.Launch(case, DEV), *runners(K))


@pytest.mark.parametrize("case", A.BOUND_ROWS, ids=lambda c: c.id)
def test_attn_bounded(K, case):
    rec = {}
    try:
        A.run_case(A.Launch(case, DEV), *runners(K), record=rec)
    finally:
        print("\nRATIO %s %s" % (case.id, " ".join("%s=%.4g" % kv for kv in sorted(rec.items()))))
        for k, v in rec.items():
            RATIOS[k] = max(RATIOS.get(k, 0.0), v)


@pytest.mark.parametrize("layout", ["self", "cross"])
@pytest.mark.parametrize("cores", ["mma", "tc"])
def test_attn_packed_layouts_bit_identical(K, layout, cores):
    """random bf16 inputs: the model's packed layouts (Q|K|V in one buffer with dQ|dK|dV written into one buffer; Q with
    a packed K|V) give the same bits as the separate-buffer launch of the same problem"""
    nk = 80 if layout == "self" else 441
    case = A.Case("bound", 2, 12, 80, nk, cores, cores, "mix", drop=0.1)
    out = []
    for lay in ("sep", layout):
        L = A.Launch(case, DEV, layout=lay)
        A.run_case(L, *runners(K))
        out.append({nm: A.bits(L.view(nm)).clone() for nm in ("o", "dq", "dk", "dv")} |
                   {"lse": A.bits(L.fview("lse", (2, 12, 80))).clone()})
    for nm in out[0]:
        assert torch.equal(out[0][nm], out[1][nm]), (case.id, layout, nm)


# --------------------------------------------------------------------------------- paths that materialise P
def _routing(B, H, nq, nk, seed, masked=0):
    """winner sets (|W| in 1, 2, 4, 8) among the keys not masked; losers >= 110 below (natural log)"""
    g = torch.Generator().manual_seed(seed)
    kmask = torch.zeros(B, nk, dtype=torch.float64)
    for b in range(B):
        if masked and nk > 8:
            kmask[b, torch.randperm(nk, generator=g)[:masked]] = -10000.0
    win = torch.zeros(B, H, nq, nk, dtype=torch.bool)
    for b in range(B):
        free = (kmask[b] == 0).nonzero()[:, 0]
        for h in range(H):
            for q in range(nq):
                n = min([1, 2, 4, 8][(q + h) % 4], len(free))
                n = 1 << (n.bit_length() - 1)
                win[b, h, q, free[torch.randperm(len(free), generator=g)[:n]]] = True
    s = torch.where(win, torch.zeros(B, H, nq, nk, dtype=torch.float64),
                    -110.0 - torch.randint(0, 400, (B, H, nq, nk), generator=g).double() / 4)
    P = win.double() / win.sum(-1, keepdim=True)
    return s, kmask, P


def _guarded(n, dt):
    return A._sentinel(n + 2 * A.GUARD, dt, DEV)


def _check_rows(name, buf, ref, nk, ld, dt):
    """buf (guards + nb x ld) holds ref in columns < nk, zeros in [nk, ld), guards untouched"""
    nb = ref.shape[0]
    exp = A._sentinel(buf.numel(), dt, DEV)
    body = torch.zeros(nb, ld, dtype=torch.float64, device=DEV)
    body[:, :nk] = ref
    exp[A.GUARD:A.GUARD + nb * ld] = body.reshape(-1).to(torch.float32).to(dt)
    bad = A.cbits(buf) != A.cbits(exp)
    if bool(bad.any()):
        p = int(bad.nonzero()[0, 0]) - A.GUARD
        where = "row %d col %d" % divmod(p, ld) if 0 <= p < nb * ld else "guard offset %d" % p
        raise AssertionError("%s: %d bad elements; first at %s: got %r, expected %r" % (
            name, int(bad.sum()), where, float(buf[p + A.GUARD]), float(exp[p + A.GUARD])))


@pytest.mark.parametrize("nk,ld,drop,dbias", [(1, 8, False, False), (100, 128, True, True), (129, 136, False, True),
                                              (500, 512, True, False), (513, 520, False, False),
                                              (1000, 1024, True, True)])
def test_softmax_exact_routing(K, nk, ld, drop, dbias):
    """bb_softmax_fwd / bb_softmax_bwd on fp32 scores with exact winners: P, Pd and dS bit for bit"""
    lib = _lib().load()
    B, H, nq = 2, 3, 5
    s, kmask, P = _routing(B, H, nq, nk, seed=nk * 7 + ld, masked=nk // 10)
    scores = torch.full((B, H, nq, ld), float("nan"), dtype=torch.float32)
    scores[..., :nk] = s.float()
    scores, km = scores.to(DEV), kmask.float().to(DEV)
    th, sc = A.drop_params(0.5 if drop else 0.0)
    keep = DM.softmax_keep(A.SEED, B, H, nq, nk, ld, th).to(DEV).double() if th else torch.ones_like(P).to(DEV)
    P = P.to(DEV)
    n = B * H * nq * ld
    probs, pd = _guarded(n, A.BF), _guarded(n, A.BF)
    n0 = lib.bb_launch_count()
    _lib().check(lib.bb_softmax_fwd(scores.data_ptr(), km.data_ptr(), 0, B, H, nq, nk, ld, A.SEED, th, sc,
                                    probs.data_ptr() + 2 * A.GUARD, pd.data_ptr() + 2 * A.GUARD, K._stream()),
                 "bb_softmax_fwd")
    torch.cuda.synchronize()
    assert lib.bb_launch_count() == n0 + 1
    _check_rows("P", probs, P.reshape(-1, nk), nk, ld, A.BF)
    Pd = P * keep * sc
    _check_rows("Pd", pd, Pd.reshape(-1, nk), nk, ld, A.BF)
    # backward with respect to the dropped probabilities
    g = torch.Generator().manual_seed(ld)
    dp = torch.randint(-2, 3, (B, H, nq, nk), generator=g).double().to(DEV)
    dpb = torch.full((B, H, nq, ld), float("nan"), dtype=torch.float32, device=DEV)
    dpb[..., :nk] = dp.float()
    gk = dp * keep * sc
    d = P * (gk - (P * gk).sum(-1, keepdim=True))
    ref = d * 0.125
    A.bf16_exact(ref, "dS")
    ds = _guarded(n, A.BF)
    db = None
    if dbias:
        db = _guarded(B * nq * nk, torch.float32)
        db[A.GUARD:A.GUARD + B * nq * nk] = 0.25
    _lib().check(lib.bb_softmax_bwd(probs.data_ptr() + 2 * A.GUARD, dpb.data_ptr(), B, H, nq, nk, ld, A.SEED, th, sc,
                                    0.125, ds.data_ptr() + 2 * A.GUARD, 0 if db is None else db.data_ptr() + 4 * A.GUARD,
                                    K._stream()), "bb_softmax_bwd")
    torch.cuda.synchronize()
    _check_rows("dS", ds, ref.reshape(-1, nk), nk, ld, A.BF)
    if dbias:
        _check_rows("dbias", db, (0.25 + d.sum(1)).reshape(-1, nk), nk, nk, torch.float32)


@pytest.mark.parametrize("case", [A.Case("exact", 2, 12, 80, 80, mask="mix"),
                                  A.Case("exact", 3, 1, 129, 512, mask="full10k", drop=0.5),
                                  A.Case("exact", 2, 12, 23, 23, mask="mix", bias=True, drop=0.5),
                                  A.Case("exact", 2, 1, 65, 7, mask="none", alpha=1.0)], ids=lambda c: c.id)
def test_attn_scores_exact_routing(K, case):
    """bb_attn_scores mode 0 (P, Pd) and mode 1 (dS, dbias) on the exact-routing Q / K / V / dO: bit for bit, with
    columns [nk, ldp) zero"""
    lib = _lib().load()
    L = A.Launch(case, DEV)
    B, H, nq, nk = case.B, case.H, case.nq, case.nk
    ldp = (nk + 7) // 8 * 8 + 8
    n = B * H * nq * ldp
    th, sc = L.drop[1], L.drop[2]
    keep = DM.softmax_keep(A.SEED, B, H, nq, nk, ldp, th).to(DEV) if th else torch.ones(B, H, nq, nk, dtype=torch.bool,
                                                                                          device=DEV)
    P = L.P

    def ptr(nm):
        sl = L.slots[nm]
        return L.bufs[sl.buf].data_ptr() + 2 * sl.start

    def operand(a, nm, which):
        sl = L.slots[nm]
        setattr(a, which, ptr(nm))
        if which == "A":
            a.lda, a.a_s1, a.a_s2 = sl.ld, 64, sl.bs
        else:
            a.ldb, a.b_s1, a.b_s2 = sl.ld, 64, sl.bs

    a = _lib().AttnScoresArgs()
    operand(a, "q", "A")
    operand(a, "k", "Bm")
    a.B, a.H, a.nq, a.nk, a.ldp, a.mode = B, H, nq, nk, ldp, 0
    a.alpha, a.out_scale = case.alpha, 1.0
    a.kmask = L.bufs["kmask"].data_ptr() + 4 * A.GUARD if "kmask" in L.bufs else 0
    a.bias = L.bufs["bias"].data_ptr() + 4 * A.GUARD if "bias" in L.bufs else 0
    a.seed, a.thresh, a.scale = L.drop
    Pb, Pdb = _guarded(n, A.BF), _guarded(n, A.BF)
    a.P, a.Pd = Pb.data_ptr() + 2 * A.GUARD, Pdb.data_ptr() + 2 * A.GUARD
    _lib().check(lib.bb_attn_scores(C.byref(a), K._stream()), "bb_attn_scores")
    torch.cuda.synchronize()
    _check_rows("P", Pb, P.reshape(-1, nk), nk, ldp, A.BF)
    Pd = torch.where(keep, P * sc, torch.zeros_like(P))
    _check_rows("Pd", Pdb, Pd.reshape(-1, nk), nk, ldp, A.BF)
    # mode 1: dS = P o (g - sum_k P g) * out_scale, g = dropout-mask(dO V^T); dbias += unscaled
    b = _lib().AttnScoresArgs()
    operand(b, "dout", "A")
    operand(b, "v", "Bm")
    b.B, b.H, b.nq, b.nk, b.ldp, b.mode = B, H, nq, nk, ldp, 1
    b.alpha, b.out_scale = 1.0, case.alpha
    b.seed, b.thresh, b.scale = L.drop
    dS = _guarded(n, A.BF)
    db = _guarded(B * nq * nk, torch.float32)
    db[A.GUARD:A.GUARD + B * nq * nk] = -0.5
    b.Pin, b.dS, b.dbias = a.P, dS.data_ptr() + 2 * A.GUARD, db.data_ptr() + 4 * A.GUARD
    _lib().check(lib.bb_attn_scores(C.byref(b), K._stream()), "bb_attn_scores")
    torch.cuda.synchronize()
    gk = torch.where(keep, (L.dO @ L.V.transpose(-1, -2)) * sc, torch.zeros_like(P))
    d = P * (gk - (P * gk).sum(-1, keepdim=True))
    A.bf16_exact(d * case.alpha, "dS")
    _check_rows("dS", dS, (d * case.alpha).reshape(-1, nk), nk, ldp, A.BF)
    _check_rows("dbias", db, (-0.5 + d.sum(1)).reshape(-1, nk), nk, nk, torch.float32)


# ------------------------------------------------------------------------------------------------------ dispatch
DISPATCH = {
    # name: (case, forward kernels, backward kernels)
    "auto_80": (A.Case("exact", 2, 12, 80, 80), ["attn_tc_fwd_kernel"], ["attn_tc_bwd_kernel<0>", "attn_tc_bwd_kernel<1>"]),
    "auto_36": (A.Case("exact", 2, 12, 36, 36), ["flash_fwd_kernel"], ["flash_bwd_dq_kernel", "flash_bwd_dkv_kernel"]),
    "tc_36": (A.Case("exact", 2, 12, 36, 36, "tc", "tc"), ["attn_tc_fwd_kernel"],
              ["attn_tc_bwd_kernel<0>", "attn_tc_bwd_kernel<1>"]),
    "mma_441": (A.Case("exact", 1, 12, 441, 441, "mma", "mma"), ["flash_fwd_kernel"],
                ["flash_bwd_dq_kernel", "flash_bwd_dkv_kernel"]),
    "tc_fwd_mma_bwd": (A.Case("exact", 2, 1, 80, 129, "tc", "mma"), ["attn_tc_fwd_kernel"],
                       ["flash_bwd_dq_kernel", "flash_bwd_dkv_kernel"]),
    "bias_tc": (A.Case("exact", 2, 12, 80, 80, "tc", "tc", bias=True), ["flash_fwd_kernel"],
                ["flash_bwd_dq_kernel", "flash_bwd_dkv_kernel"]),
    "dbias_tc": (A.Case("exact", 2, 12, 80, 80, "tc", "tc", bias=True, dbias="atomic"), ["flash_fwd_kernel"],
                 ["flash_bwd_dq_kernel", "flash_bwd_dkv_kernel"]),
}
ALL_ATTN = ["attn_tc_fwd_kernel", "attn_tc_bwd_kernel", "flash_fwd_kernel", "flash_bwd_dq_kernel", "flash_bwd_dkv_kernel"]


@pytest.fixture(scope="module")
def dispatch_trace(K):
    """kernel names of every DISPATCH step, from one profiler session: each step runs inside its own record_function
    range and synchronises before the range closes, so its kernels start inside it"""
    launches = {name: A.Launch(case, DEV) for name, (case, _, _) in DISPATCH.items()}
    fwd, bwd = runners(K)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for name, L in launches.items():
            for which, step in (("fwd", fwd), ("bwd", bwd)):
                with torch.profiler.record_function("dispatch/%s/%s" % (name, which)):
                    step(L)
    ev = prof.events()
    ranges = [(e.name, e.time_range.start, e.time_range.end) for e in ev if e.name.startswith("dispatch/")]
    kernels = [(e.name, e.time_range.start) for e in ev if e.device_type == torch.autograd.DeviceType.CUDA]
    return {tag: [n for n, t in kernels if t0 <= t <= t1] for tag, t0, t1 in ranges}


@pytest.mark.parametrize("name", list(DISPATCH))
def test_attn_dispatch_reaches_the_intended_kernels(dispatch_trace, name):
    _, kf, kb = DISPATCH[name]
    for which, want in (("fwd", kf), ("bwd", kb)):
        names = dispatch_trace["dispatch/%s/%s" % (name, which)]
        ran = sorted({k for k in ALL_ATTN for n in names if k in n} |
                     {m for n in names for m in re.findall(r"attn_tc_bwd_kernel<\d>", n)})
        for k in want:
            assert any(k in n for n in names), (name, which, k, ran)
        others = [k for k in ALL_ATTN if k not in "".join(want) and any(k in n for n in names)]
        assert not others, (name, which, want, others)


# ---------------------------------------------------------------------------------------------- invalid arguments
INVALID = {
    # name: (fwd / bwd, fields, message)
    "dh_32": ("fwd", dict(dh=32), "head dim must be 64"),
    "nq_zero": ("fwd", dict(nq=0), "sizes must be positive"),
    "nk_negative": ("bwd", dict(nk=-1), "sizes must be positive"),
    "B_zero": ("fwd", dict(B=0), "sizes must be positive"),
    "ldq_not_multiple_of_8": ("fwd", dict(ldq="+4"), "row strides must be multiples of 8 elements"),
    "ldo_not_multiple_of_8": ("bwd", dict(ldo="+2"), "row strides must be multiples of 8 elements"),
    "lddq_not_multiple_of_8": ("bwd", dict(lddq="+4"), "bb_flash_bwd: row strides must be multiples of 8"),
    "B_too_large": ("fwd", dict(B=65536), "B, H must be <= 65535"),
    "H_too_large": ("bwd", dict(H=65536), "B, H must be <= 65535"),
    "null_o": ("fwd", dict(o=0), "null o / lse"),
    "null_lse": ("bwd", dict(lse=0), "null o / lse"),
    "null_dq": ("bwd", dict(dq=0), "null gradient pointer"),
    "null_dsum": ("bwd", dict(dsum=0), "null gradient pointer"),
    "null_dout": ("bwd", dict(dout=0), "null gradient pointer"),
}
for _f in ("q", "k", "v", "o"):
    INVALID["misaligned_" + _f] = ("fwd", {_f: "+2"}, "q / k / v / o must be 16-byte aligned")
    INVALID[_f + "_bs_not_multiple_of_8"] = ("fwd", {_f + "_bs": "+4"}, "batch strides must be multiples of 8 elements")
for _f in ("dout", "dq", "dk", "dv"):
    INVALID["misaligned_" + _f] = ("bwd", {_f: "+8"}, "dout / dq / dk / dv must be 16-byte aligned")
for _f in ("do", "dq", "dk", "dv"):
    INVALID[_f + "_bs_not_multiple_of_8"] = ("bwd", {_f + "_bs": "+2"}, "batch strides must be multiples of 8 elements")
INVALID["bwd_misaligned_q"] = ("bwd", dict(q="+8"), "q / k / v / o must be 16-byte aligned")


@pytest.mark.parametrize("tc", ["mma", "tc"])
@pytest.mark.parametrize("name", list(INVALID))
def test_flash_invalid_arguments(K, name, tc):
    """Host-side checks of bb_flash_fwd / _bwd: an error with the library's message, no launch, buffers untouched"""
    which, fields, msg = INVALID[name]
    L = A.Launch(A.Case("exact", 2, 12, 80, 80, tc, tc, "mix"), DEV)
    a0 = L.args(_lib().FlashArgs)
    over = {k: (getattr(a0, k) + int(v[1:]) if isinstance(v, str) else v) for k, v in fields.items()}
    n0 = K.launch_count()
    rc, got = flash(K, L, which, **over)
    torch.cuda.synchronize()
    assert rc != 0 and msg in got, (name, rc, got)
    assert K.launch_count() == n0, "a rejected call launched a kernel"
    L.untouched()


def test_flash_kernels_wrapper_rejects_misaligned_views(K):
    """kernels.flash_fwd on a view that starts 2 elements into its buffer raises instead of launching"""
    q = torch.zeros(2 * 80 * 768 + 8, dtype=torch.bfloat16, device=DEV)
    n0 = K.launch_count()
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        K.flash_fwd(q[2:], q[8:], q[8:], 2, 12, 80, 80, 768, 768, 768)
    torch.cuda.synchronize()
    assert K.launch_count() == n0
