"""The row kernels of csrc/rowops.cu element by element against fp64 references with a-priori bounds
(tests/rowops_cases.py), through the C ABI on guarded buffers: every case in the bf16 product mode and again in the
fp32 verification mode (K.set_precision(True)), whose bounds have no half-ulp bf16 term.  The fp32 mode's rejections
(bf16 pairings of bb_layernorm_bwd, a bf16 source of bb_scatter_rows_sorted) are asserted.  LayerNorm backward, colsum
and the embedding gradients also run in the deterministic mode, twice, bit-identical.

Worst err / bound per quantity (printed at the end of the module with -s), measured on an H100 80GB HBM3 at 700 W,
bf16 mode / fp32 mode.  Every constant of rowops_cases.C is 1: the bounds are derived from each kernel's order of
operations, not fitted.  A bf16 output's bound is its half ulp plus a small fp32 term, so a ratio near 1 is expected
there; a single element rounded toward zero instead of to nearest lands above 1.
  ln_fwd.y 1.000 / 0.222, y_f32 0.246 / 0.222, mean 0.166 / 0.197, rstd 0.264 / 0.264
  ln_bwd.dx 1.000 / 0.413, dres 1.000 / 0.413, dgamma 0.252 / 0.325, dbeta 0.216 / 0.216, dxsum 0.107 / 0.124
  colsum 0.071 / 0.253; segment_wsum 1.000 / 0.954, backward 0.215 / 0.234; gelu_bwd 1.000 / 0.692
  embed_scatter_grad dword 0.544 / 0.501, dpos 0.496 / 0.496, dtype0 0.124 / 0.124
  softmax_xent loss 0.135 / 0.135, dlogits 0.999 / 0.315
The optimizer (tests/test_optim_kernels_gpu.py): adamw m 0.629, v 0.556, p 0.598; sumsq 0.033.
"""
import pytest
import torch

import rowops_cases as R

pytestmark = pytest.mark.gpu
BF, F32 = R.BF, R.F32


@pytest.fixture(scope="module", params=[False, True], ids=["bf16", "fp32"])
def act(request):
    from bevbert_b200 import kernels as K
    assert torch.cuda.is_available()
    prev = K.set_precision(request.param)
    yield F32 if request.param else BF
    K.set_precision(prev)
    print("\nerr / bound, %s mode:" % ("fp32" if request.param else "bf16"))
    for k in sorted(R.RATIOS):
        print("  %-28s %.3f" % (k, R.RATIOS[k]))
    R.RATIOS.clear()


@pytest.fixture
def det():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def _rejects(fn, *args):
    """the entry point returns an error (and launches nothing) -> its message"""
    from bevbert_b200 import _lib, kernels as K
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    rc = getattr(lib, fn)(*args, K._stream())
    assert rc != 0 and lib.bb_launch_count() == n0
    return lib.bb_last_error().decode()


LN = [R.ln_table(BF), R.ln_table(F32)]


@pytest.mark.parametrize("i", range(len(R.ln_table())))
def test_layernorm_fwd(act, i):
    case = LN[act == F32][i]
    A, ins, outs = R.run_ln_fwd(case, "gpu", "cuda")
    R.check_ln_fwd(case, A, ins, outs)


LNB = [R.ln_bwd_table(BF), R.ln_bwd_table(F32)]


@pytest.mark.parametrize("i", range(len(R.ln_bwd_table(BF))))
def test_layernorm_bwd(act, i):
    table = LNB[act == F32]
    if i >= len(table):
        pytest.skip("the fp32 mode has one dtype pairing")
    case, pair = table[i]
    A, ins, outs, grid = R.run_ln_bwd(case, pair, "gpu", "cuda")
    R.check_ln_bwd(case, pair, A, ins, outs, grid)


@pytest.mark.parametrize("i", range(0, len(R.ln_bwd_table(BF)), 4))
def test_layernorm_bwd_deterministic(act, det, i):
    table = LNB[act == F32]
    case, pair = table[i % len(table)]
    A, ins, outs, grid = R.run_ln_bwd(case, pair, "gpu", "cuda")
    R.check_ln_bwd(case, pair, A, ins, outs, grid)
    _, _, outs2, _ = R.run_ln_bwd(case, pair, "gpu", "cuda")
    for a, b in zip(outs, outs2):
        R.check_exact("ln_bwd deterministic rerun", a, b)


def test_layernorm_bwd_fp32_mode_rejects_bf16_pairings(act):
    if act != F32:
        pytest.skip("bf16 mode accepts the six pairings")
    for dyf, xf, dxf in R.LN_BWD_PAIRS[:3] + R.LN_BWD_PAIRS[4:]:
        x = torch.zeros(8, 64, device="cuda")
        msg = _rejects("bb_layernorm_bwd", x.data_ptr(), dyf, x.data_ptr(), xf, None, x.data_ptr(), x.data_ptr(),
                       x.data_ptr(), 8, 64, 0, 0, 1.0, 0, 0, 1.0, x.data_ptr(), dxf, None, None, None, None)
        assert "the fp32 verification mode needs fp32 dy / x / dx" in msg


@pytest.mark.parametrize("N,ld,rows", R.colsum_table())
@pytest.mark.parametrize("mode", ["atomic", "det"])
def test_colsum(act, N, ld, rows, mode):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(mode == "det")
    try:
        r = R.run_colsum(N, ld, rows, act, "gpu", "cuda")
        R.check_colsum(N, ld, rows, *r)
        if mode == "det":
            r2 = R.run_colsum(N, ld, rows, act, "gpu", "cuda")
            R.check_exact("colsum deterministic rerun", r[3], r2[3])
    finally:
        torch.use_deterministic_algorithms(prev)


@pytest.mark.parametrize("H", [8, 264, 768])
def test_segment_wsum(act, H):
    R.run_seg(H, act, "gpu", "cuda")


def test_segment_wsum_bwd_rejected_in_deterministic_mode(act, det):
    x = torch.zeros(8, 64, device="cuda")
    from bevbert_b200 import kernels as K
    K._stream()
    assert "in deterministic mode use bb_scatter_rows_sorted" in _rejects(
        "bb_segment_wsum_bwd", x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), 2, 64, x.data_ptr())


@pytest.mark.parametrize("n", [4099, 1 << 20])
def test_gelu_relu_bwd(act, n):
    R.run_gelu(n, act, "gpu", "cuda")


XENT = [(5, 7, 7), (5, 7, 16), (9, 256, 256), (9, 256, 264), (37, 30522, 30528), (4, 250002, 250008)]


@pytest.mark.parametrize("rows,V,ld", XENT)
@pytest.mark.parametrize("gs", [False, True])
def test_softmax_xent(act, rows, V, ld, gs):
    A, ins, outs = R.run_xent(rows, V, ld, act, gs, "gpu", "cuda")
    R.check_xent(V, ld, A, ins, outs)


@pytest.mark.parametrize("H", [8, 264, 768])
def test_exact_rows(act, H):
    R.run_exact_rows(H, act, "gpu", "cuda")


@pytest.mark.parametrize("src_f32,w", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("H", [8, 768])
def test_scatter_rows_sorted(act, H, src_f32, w):
    if act == F32 and not src_f32:
        x = torch.zeros(8, H, device="cuda")
        i = torch.zeros(2, dtype=torch.int64, device="cuda")
        assert "the fp32 verification mode needs fp32 src" in _rejects(
            "bb_scatter_rows_sorted", x.data_ptr(), 0, i.data_ptr(), None, i.data_ptr(), 2, H, x.data_ptr())
        return
    R.run_scatter_sorted(H, src_f32, w, act, "gpu", "cuda")


@pytest.mark.parametrize("L", [1, 40, 80])
@pytest.mark.parametrize("mode", ["atomic", "det"])
def test_embed_scatter_grad(act, L, mode):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(mode == "det")
    try:
        R.run_embed_grad(L, 264, mode == "det", "gpu", "cuda")
    finally:
        torch.use_deterministic_algorithms(prev)
