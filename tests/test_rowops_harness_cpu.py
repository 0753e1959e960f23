"""The row-kernel and optimizer harness of tests/test_rowops_gpu.py and tests/test_optim_kernels_gpu.py, rehearsed on
the CPU: the fp64 references and their bounds against the torch restatement in tests/emu_kernels.py (bf16 rounding on
through set_act_dtype) and against an fp32 restatement of the AdamW update.  Also: the case tables reach every feature,
the checker catches planted errors, and the host-side argument checks of the row kernels run before any CUDA call.
No GPU needed."""
import json
import os
import subprocess
import sys

import pytest
import torch

import emu_kernels as E
import rowops_cases as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF, F32 = R.BF, R.F32


@pytest.fixture(params=[BF, F32], ids=["bf16", "fp32"])
def act(request):
    E.set_act_dtype(request.param)
    yield request.param
    E.set_act_dtype(F32)


@pytest.mark.parametrize("i", range(0, len(R.ln_table(big=False)), 3))
def test_harness_ln_fwd(act, i):
    case = R.ln_table(act, big=False)[i]
    A, ins, outs = R.run_ln_fwd(case, "emu", "cpu")
    R.check_ln_fwd(case, A, ins, outs)


@pytest.mark.parametrize("i", range(0, 40, 3))
def test_harness_ln_bwd(act, i):
    small = [c for c in R.ln_bwd_table(act) if c[0].rows <= 1100]
    case, pair = small[i % len(small)]
    A, ins, outs, grid = R.run_ln_bwd(case, pair, "emu", "cpu")
    R.check_ln_bwd(case, pair, A, ins, outs, grid)


@pytest.mark.parametrize("N,ld,rows", [t for t in R.colsum_table() if t[2] <= 4097][::5])
def test_harness_colsum(act, N, ld, rows):
    R.check_colsum(N, ld, rows, *R.run_colsum(N, ld, rows, act, "emu", "cpu"))


@pytest.mark.parametrize("H", [8, 264, 768])
def test_harness_segment_wsum(act, H):
    R.run_seg(H, act, "emu", "cpu")


def test_harness_gelu_relu(act):
    R.run_gelu(4099, act, "emu", "cpu")


@pytest.mark.parametrize("V,ld,gs", [(7, 16, True), (256, 256, False), (30522, 30528, True)])
def test_harness_xent(act, V, ld, gs):
    A, ins, outs = R.run_xent(5, V, ld, act, gs, "emu", "cpu")
    R.check_xent(V, ld, A, ins, outs)


@pytest.mark.parametrize("H", [8, 264, 768])
def test_harness_exact_rows(act, H):
    R.run_exact_rows(H, act, "emu", "cpu")


@pytest.mark.parametrize("src_f32,w", [(False, True), (True, False), (True, True)])
def test_harness_scatter_sorted(src_f32, w):
    E.set_act_dtype(BF)
    try:
        R.run_scatter_sorted(16, src_f32, w, BF, "emu", "cpu")
    finally:
        E.set_act_dtype(F32)


@pytest.mark.parametrize("L,det", [(1, False), (40, True), (80, False)])
def test_harness_embed_grad(L, det):
    R.run_embed_grad(L, 264, det, "emu", "cpu")


# ------------------------------------------------------------------------------------------- AdamW restatement
def _adam_emu(T, b1, b2, eps, coef, steps, decays, **kw):
    for i in range(len(T.sizes)):
        p, m, v = R.adam1_f32(T.views["p"][i].clone(), T.views["g"][i], T.views["m"][i].clone(),
                              T.views["v"][i].clone(), b1, b2, eps, coef, steps[i], decays[i], **kw)
        T.views["p"][i].copy_(p)
        T.views["m"][i].copy_(m)
        T.views["v"][i].copy_(v)
        T.views["p16"][i].copy_(p.to(BF))


def _adam_check(T, before, b1, b2, eps, coef, clipped, steps, decays):
    for i, n in enumerate(T.sizes):
        if n == 0:
            continue
        ref = R.adam_ref(before["p"][i], before["g"][i], before["m"][i], before["v"][i], b1, b2, eps, coef, clipped,
                         steps[i], decays[i])
        R.check("adamw.m[%d]" % i, T.views["m"][i], ref["m"], ref["d_m"])
        R.check("adamw.v[%d]" % i, T.views["v"][i], ref["v"], ref["d_v"])
        R.check("adamw.p[%d]" % i, T.views["p"][i], ref["p"], ref["d_p"])
        R.check_exact("adamw.p16[%d]" % i, T.views["p16"][i], T.views["p"][i].to(BF))
        R.check_exact("adamw.g[%d] unchanged" % i, T.views["g"][i], before["g"][i])
    T.check_gaps("pgmv")
    T._gaps("p16")


def _tiny_norm_case():
    T = R.OptTable(R.opt_sizes("edges"), "cpu", scale=6.4e-9)
    s, _ = R.sumsq_ref(T.views["g"], T.chunks)
    return T, s


def test_harness_adamw_restatement():
    for kind, gsc, max_norm in (("edges", 1.0, 1.0), ("many", 2.0 ** -8, 0.5), ("edges", 1.0, 0.0)):
        T = R.OptTable(R.opt_sizes(kind), "cpu", seed=3)
        s, _ = R.sumsq_ref(T.views["g"], T.chunks)
        coef, clipped = R.clip_coef(torch.tensor(s, dtype=F32), max_norm, gsc)
        steps = [1e-3 * (1 + i % 3) for i in range(len(T.sizes))]
        decays = [0.05 if i % 2 else 0.0 for i in range(len(T.sizes))]
        before = T.snapshot()
        _adam_emu(T, 0.9, 0.98, 1e-6, coef, steps, decays)
        _adam_check(T, before, 0.9, 0.98, 1e-6, coef, clipped, steps, decays)


# ------------------------------------------------------------------------------------------- table coverage
def test_table_reaches_every_feature():
    lt = R.ln_table()
    assert {c.H for c in lt} == set(R.LN_H)
    assert {c.H for c, _ in R.ln_bwd_table()} == set(R.LN_H)
    assert any(c.H <= 768 for c in lt) and any(768 < c.H <= 1024 for c in lt)          # both backward templates
    assert {1, 7, R.ROWS_SMS, R.ROWS_SMS + 1} <= {c.rows for c in lt} and max(c.rows for c in lt) >= 20000
    assert {c.xdt for c in lt} == {BF, F32} and {c.res for c in lt} == {False, True} and {c.eps for c in lt} == {1e-12, 1e-5}
    assert {c.adv for c in lt} == {"", "offset", "outlier", "onehot", "const"}
    bt = R.ln_bwd_table()
    assert {p for _, p in bt} == set(R.LN_BWD_PAIRS) and len(R.LN_BWD_PAIRS) == 6
    # the prefetch loop: some warp takes a second row (rows > 8 * #SMs)
    assert any(c.rows > 8 * 132 and c.H <= 768 for c, _ in bt) and any(c.rows > 8 * 132 and c.H > 768 for c, _ in bt)
    ct = R.colsum_table()
    assert {N for N, _, _ in ct} == set(R.COLSUM_N)
    assert any(ld % 8 for _, ld, _ in ct) and any(N % 8 for N, _, _ in ct)               # the scalar path
    assert any(rows > 64 * 64 for _, _, rows in ct)                                      # the 64-slice cap
    rem = set()
    for N, ld, rows in ct:
        if ld % 8 == 0:
            gy = min(-(-rows // 64), 64)
            for r0 in range(8 * gy):
                rem.add(len(range(r0, rows, 8 * gy)) % 4)
    assert {1, 2, 3} <= rem
    es, ms = R.opt_sizes("edges"), R.opt_sizes("many")
    assert set(R.OPT_SIZES) <= set(es) and es[0] == 0 and es[-1] == 0 and 0 in es[1:-1]
    assert len(ms) >= 600 and 0 in ms and 4096 in ms
    assert set(R.XENT_V) == {7, 256, 30522, 250002}


# ------------------------------------------------------------------------------------------- planted errors
def _bf16_ln_case():
    E.set_act_dtype(BF)
    return R.LnCase(264, 40, BF, True, 1e-12, seed=1)


def _ln_fwd_planted(how):
    case = _bf16_ln_case()
    try:
        A, ins, outs = R.run_ln_fwd(case, "emu", "cpu")
    finally:
        E.set_act_dtype(F32)
    y, y32, mean, rstd = outs
    if how == "truncate":
        ref = R.ln_fwd_ref(*ins, case.eps)["y"]
        r32 = ref.float()
        t = (R.bits(r32) & ~0xFFFF).view(F32)                     # toward zero
        up = (r32 - t).abs() / (R.half_ulp_bf16(ref) * 2)           # position within the bf16 interval
        k = int(up.reshape(-1).argmax())
        assert float(up.reshape(-1)[k]) > 0.8
        y.view(-1)[k] = t.reshape(-1)[k].to(BF)
    elif how == "swap_stats":
        mean[[3, 4]] = mean[[4, 3]].clone()
        rstd[[3, 4]] = rstd[[4, 3]].clone()
    elif how == "unwritten":
        y[5, 8:16] = R.sentinel_like(y[5, 8:16])
    R.check_ln_fwd(case, A, ins, outs)


@pytest.mark.parametrize("how", ["truncate", "swap_stats", "unwritten"])
def test_checker_catches_planted_ln_fwd(how):
    with pytest.raises(AssertionError, match="bad elements"):
        _ln_fwd_planted(how)


def test_checker_catches_dropped_dgamma_partial():
    case = _bf16_ln_case()
    try:
        A, ins, outs, grid = R.run_ln_bwd(case, (0, 0, 0), "emu", "cpu")
    finally:
        E.set_act_dtype(F32)
    dy, x, res, gam, mean, rstd, init = ins
    z = x.double() + res.double()
    xh = (z[:8] - mean[:8, None].double()) * rstd[:8, None].double()
    outs[2].sub_((dy[:8].double() * xh).sum(0).float())              # block 0's eight rows never added
    with pytest.raises(AssertionError, match="bad elements"):
        R.check_ln_bwd(case, (0, 0, 0), A, ins, outs, grid)


def test_checker_catches_nonzero_dlogits_padding():
    E.set_act_dtype(BF)
    try:
        A, ins, outs = R.run_xent(4, 7, 16, BF, True, "emu", "cpu")
    finally:
        E.set_act_dtype(F32)
    outs[1][2, 9] = 1e-3
    with pytest.raises(AssertionError, match="bad elements"):
        R.check_xent(7, 16, A, ins, outs)


@pytest.mark.parametrize("how", ["no_clip_eps", "eps_in_sqrt", "decay_first", "tail", "past_end"])
def test_checker_catches_planted_adamw(how):
    T, s = _tiny_norm_case()                      # total norm about 1e-6: the clip's epsilon halves the coefficient
    max_norm = 1e-6
    coef, clipped = R.clip_coef(torch.tensor(s, dtype=F32), max_norm, 1.0)
    assert 0.3 < coef < 0.7 and clipped
    steps = [1e-2] * len(T.sizes)
    decays = [0.05] * len(T.sizes)
    before = T.snapshot()
    kw = {}
    c = coef
    if how == "no_clip_eps":
        c = R.clip_coef(torch.tensor(s, dtype=F32), max_norm, 1.0, clip_eps=0.0)[0]
    elif how == "eps_in_sqrt":
        kw["eps_in_sqrt"] = True
    elif how == "decay_first":
        kw["decay_first"] = True
    _adam_emu(T, 0.9, 0.98, 1e-6, c, steps, decays, **kw)
    i = T.sizes.index(4097)
    if how == "tail":
        T.views["p"][i][-1] = before["p"][i][-1]
    elif how == "past_end":
        T.arena["p"][T.starts["p"][i] + 4097] = 0.0
    with pytest.raises(AssertionError, match="bad elements"):
        _adam_check(T, before, 0.9, 0.98, 1e-6, coef, clipped, steps, decays)


# ------------------------------------------------------------------------------------ host-side argument checks
_REJECT = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import __graft_entry__  # noqa: F401
from bevbert_b200 import _lib
lib = _lib.load()
A = 0x100000000          # never dereferenced: the calls must be rejected before any CUDA call
out = []
for fn, args in json.loads(sys.argv[2]):
    n0 = lib.bb_launch_count()
    rc = getattr(lib, fn)(*args)
    msg = lib.bb_last_error()
    out.append([fn, rc, lib.bb_launch_count() - n0, msg.decode() if msg else ""])
print(json.dumps(out))
"""

A0 = 0x100000000


def _ln_fwd(x=A0, res=A0, gamma=A0, beta=A0, y=A0, y32=A0, H=768):
    return ["bb_layernorm_fwd", [x, 0, res, gamma, beta, 1e-12, 16, H, 0, 0, 1.0, 0, 0, 1.0, y, y32, A0, A0, None]]


def _ln_bwd(dy=A0, x=A0, res=A0, gamma=A0, dx=A0, dres=A0, H=768):
    return ["bb_layernorm_bwd", [dy, 0, x, 0, res, gamma, A0, A0, 16, H, 0, 0, 1.0, 0, 0, 1.0, dx, 0, dres, A0, A0, A0,
                                 None]]


def _add_rows(a=A0, b=A0, table=A0, vec=A0, out=A0):
    return ["bb_add_rows", [a, b, table, A0, vec, 16, 768, out, None]]


MIS = 2       # one bf16 element
REJECTED = [(_ln_fwd(**{k: A0 + MIS}), "bb_layernorm_fwd: x / residual / gamma / beta / y / y_f32 must be 16-byte aligned")
            for k in ("x", "res", "y")] + \
    [(_ln_fwd(**{k: A0 + 4}), "must be 16-byte aligned") for k in ("gamma", "beta", "y32")] + \
    [(_ln_bwd(**{k: A0 + MIS}), "bb_layernorm_bwd: dy / x / residual / gamma / dx / dres must be 16-byte aligned")
     for k in ("dy", "x", "res", "dx", "dres")] + \
    [(_ln_bwd(gamma=A0 + 8), "must be 16-byte aligned")] + \
    [(_add_rows(**{k: A0 + (MIS if k in "ab" or k == "out" else 4)}), "bb_add_rows: a / b / table / vec / out must be")
     for k in ("a", "b", "table", "vec", "out")] + \
    [(["bb_gather_rows_bf16", [A0 + MIS, A0, 4, 768, A0, None]], "bb_gather_rows_bf16: in / out must be 16-byte aligned"),
     (["bb_gather_rows_bf16", [A0, A0, 4, 768, A0 + 8, None]], "bb_gather_rows_bf16: in / out must be 16-byte aligned"),
     (["bb_segment_wsum", [A0 + MIS, A0, A0, A0, 4, 768, A0, None]], "bb_segment_wsum: src / out must be"),
     (["bb_segment_wsum", [A0, A0, A0, A0, 4, 768, A0 + MIS, None]], "bb_segment_wsum: src / out must be"),
     (["bb_segment_wsum_bwd", [A0 + MIS, A0, A0, A0, 4, 768, A0, None]], "bb_segment_wsum_bwd: dout must be"),
     (["bb_embed_sum", [A0, A0 + 4, A0, A0, 8, 4, 768, A0, None]], "bb_embed_sum: word / pos / type0 / out must be"),
     (["bb_embed_sum", [A0, A0, A0 + 8, A0, 8, 4, 768, A0, None]], "bb_embed_sum: word / pos / type0 / out must be"),
     (["bb_embed_sum", [A0, A0, A0, A0 + 4, 8, 4, 768, A0, None]], "bb_embed_sum: word / pos / type0 / out must be"),
     (["bb_embed_sum", [A0, A0, A0, A0, 8, 4, 768, A0 + 12, None]], "bb_embed_sum: word / pos / type0 / out must be"),
     (["bb_colsum_bf16", [A0 + MIS, 16, 768, 768, A0, None]], "bb_colsum_bf16: x must be 16-byte aligned when ld"),
     # the shape limits
     (_ln_fwd(H=772), "bb_layernorm_fwd: H must be a multiple of 8 and <= 1024"),
     (_ln_fwd(H=1032), "bb_layernorm_fwd: H must be a multiple of 8 and <= 1024"),
     (_ln_bwd(H=1032), "bb_layernorm_bwd: H must be a multiple of 8 and <= 1024"),
     (_ln_bwd(H=36), "bb_layernorm_bwd: H must be a multiple of 8 and <= 1024"),
     (["bb_add_rows", [A0, A0, A0, A0, A0, 16, 20, A0, None]], "bb_add_rows: H must be a multiple of 8"),
     (["bb_softmax_fwd", [A0, 0, 0, 1, 1, 8, 1030, 1032, 0, 0, 1.0, A0, 0, None]], "need nk <= ld <= 1024"),
     (["bb_softmax_bwd", [A0, A0, 1, 1, 8, 8, 1032, 0, 0, 1.0, 1.0, A0, 0, None]], "need nk <= ld <= 1024")]


def test_misaligned_row_arguments_are_rejected_before_any_cuda_call():
    """Each misaligned pointer of an entry point whose kernel issues 16-byte accesses, H % 8 != 0, H > 1024 and
    ld > 1024: the call returns its message and launches nothing.  Fake pointers, never dereferenced, in a process that
    sees no GPU."""
    lib = os.path.join(ROOT, "vln-bevbert_b200", "libbevbert_b200.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    spec = json.dumps([c for c, _ in REJECTED])
    r = subprocess.run([sys.executable, "-c", _REJECT, ROOT, spec], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(res) == len(REJECTED)
    for (fn, rc, launched, msg), (call, want) in zip(res, REJECTED):
        assert rc != 0 and launched == 0, (call, rc, launched, msg)
        assert want in msg, (call, msg)
