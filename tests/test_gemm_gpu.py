"""bb_gemm_bf16 on integer-valued operands, bit for bit against an fp64 restatement of the header's contract
(tests/gemm_cases.py explains why the accumulator and the epilogue are then exact).

The table covers every epilogue variant the dispatch picks (plain, GELU + pre-activation, gelu', relu', residual
add, the generic one through each feature combination the others do not take), both tile widths and the automatic
choice, all four operand majors, every N % 8 residue, row counts that end in either 64-row half and in different
iterations of the staged epilogue loop, strided / odd / batched / attention-output layouts, each pointer misaligned
on its own, ping-pong schedules at tile counts around the SM count, fp32 atomic accumulation and split-K in both the
atomic and the deterministic mode, the model's full-size shapes, and the host-side argument checks.  The same table
runs through the fp32 verification arm (gemm_f32.cu), which the model-parity tests rest on.
"""
import contextlib
import re
from dataclasses import replace

import pytest
import torch

import gemm_cases as G

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def K():
    import bevbert_b200.kernels as K
    from bevbert_b200 import _lib
    assert torch.cuda.is_available()
    _lib.load().bb_set_drop_salt_ptr(None)       # a graph test in the same process may have registered a dropout salt
    prec = K.set_precision(False)
    det = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    fill = torch.utils.deterministic.fill_uninitialized_memory
    try:
        yield K
    finally:
        K.set_precision(prec)
        torch.use_deterministic_algorithms(det[0], warn_only=det[1])
        torch.utils.deterministic.fill_uninitialized_memory = fill


@contextlib.contextmanager
def fp32_arm(K):
    prev = K.set_precision(True)
    try:
        yield
    finally:
        K.set_precision(prev)


@contextlib.contextmanager
def deterministic():
    """torch's deterministic flag for the launches inside only (references are computed outside it)"""
    prev = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    fill = torch.utils.deterministic.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
        torch.utils.deterministic.fill_uninitialized_memory = fill


def _run_case(K, case, arm32=False):
    L = G.Launch(case, DEV, arm32)
    L.run(K.gemm)
    torch.cuda.synchronize()
    L.check()
    return L


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------- table
@pytest.mark.parametrize("case", G.TABLE, ids=lambda c: c.id)
def test_gemm_exact(K, case):
    _run_case(K, case)


@pytest.mark.parametrize("case", G.fp32_arm_rows(G.TABLE), ids=lambda c: c.id)
def test_gemm_exact_fp32_arm(K, case):
    with fp32_arm(K):
        _run_case(K, case, arm32=True)


@pytest.mark.parametrize("tiles", G.PINGPONG_TILES)
@pytest.mark.parametrize("variant", ["plain", "gelu_pre", "dgelu"])
def test_gemm_pingpong_tile_counts(K, variant, tiles):
    """Total tile counts around the card's SM count: one tile, fewer tiles than consumer warpgroups, a partial last
    wave, and three tiles per CTA (each consumer warpgroup reuses its staging buffer)."""
    _run_case(K, G.pingpong_case(variant, tiles, _sms()))


@pytest.mark.parametrize("tiles", ["1", "sms+1", "3*sms"])
def test_gemm_pingpong_tile_counts_fp32_arm(K, tiles):
    with fp32_arm(K):
        _run_case(K, G.pingpong_case("gelu_pre", tiles, _sms()), arm32=True)


@pytest.mark.parametrize("case", G.FULL_ROWS, ids=lambda c: c.id)
def test_gemm_full_size(K, case):
    """The model's FFN and QKV shapes: many tiles per CTA and the real K."""
    _run_case(K, case)


@pytest.mark.parametrize("case", G.FULL_ROWS, ids=lambda c: c.id)
def test_gemm_full_size_fp32_arm(K, case):
    with fp32_arm(K):
        _run_case(K, G.fp32_arm_rows([case])[0], arm32=True)


# ------------------------------------------------------------------------------------------ vector and scalar paths
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("variant,mis", [("gelu_pre", "D"), ("gelu_pre", "aux_out"), ("dgelu", "D"),
                                         ("dgelu", "aux_in")])
def test_gemm_vector_and_scalar_paths_agree(K, variant, mis, bn):
    """The same logical problem with every pointer aligned (16-byte vectors) and with one pointer misaligned (the
    scalar path of every chunk): same arithmetic, so bit-identical outputs, GELU / gelu' included."""
    case = G.Case(variant, 300, 2 * bn + 40, 136, maj="NN" if variant == "dgelu" else "NT", bias=variant != "dgelu",
                  alpha=0.125, drop=True, block_n=bn)
    ref = _run_case(K, case)
    other = _run_case(K, replace(case, mis=mis))
    for name in ref.ref:
        assert torch.equal(G.bits(ref.logical(name)), G.bits(other.logical(name))), (case.id, mis, name)


# ------------------------------------------------------------------------------------------------------- split-K
@pytest.mark.parametrize("case", G.SPLIT_ROWS, ids=lambda c: c.id)
def test_gemm_split_k_deterministic(K, case):
    """The accumulate / split-K rows under torch.use_deterministic_algorithms (EPI_SPLIT_DET: partial tiles summed in
    split order by the last split): exactly the reference, so bit-equal to the atomic results as well."""
    L = G.Launch(case, DEV)
    with deterministic():
        L.run(K.gemm)
        torch.cuda.synchronize()
    L.check()


def test_gemm_split_det_counters_reset(K):
    """Two launches in a row, then another shape, each exact: every launch leaves the arrival counters at zero."""
    a = G.Launch(G.Case("plain", 300, 200, 1000, maj="TT", out="f32", split_k=4, bias=True, block_n=64), DEV)
    b = G.Launch(G.Case("plain", 129, 136, 520, out="f32", split_k=3, accumulate=True), DEV)
    with deterministic():
        a.run(K.gemm)
        torch.cuda.synchronize()
    a.check()
    a.reset()
    with deterministic():
        a.run(K.gemm)
        b.run(K.gemm)
        torch.cuda.synchronize()
    a.check()
    b.check()


def test_gemm_split_det_workspace_too_small(K):
    """A split-K weight gradient whose partial tiles exceed the 32 MB workspace raises with the size it needs and
    launches nothing."""
    case = G.Case("plain", 768, 3072, 14112, maj="TT", out="f32", split_k=8, block_n=128)
    L = G.Launch(case, DEV)
    kb = (case.K + 63) // 64
    split = -(-kb // -(-kb // case.split_k))
    need = 65536 + split * (768 // 128) * (3072 // 128) * 128 * 128 * 4
    assert need > K.DET_WS_BYTES
    n0 = K.launch_count()
    with deterministic():
        with pytest.raises(RuntimeError, match="at least %d bytes" % need):
            L.run(K.gemm)
    torch.cuda.synchronize()
    assert K.launch_count() == n0
    L.untouched()


# ---------------------------------------------------------------------------------------------- invalid arguments
def _invalid_rows():
    nt = G.Case("plain", 200, 136, 64)
    f32 = G.Case("plain", 200, 136, 64, out="f32")
    return {
        "accumulate_bf16_out": (nt, dict(accumulate=True), "accumulate / split_k need fp32 output"),
        "split_act": (f32, dict(split_k=2, act=1), "cannot be combined with a non-linear epilogue"),
        "split_aux_out": (replace(f32, variant="auxout"), dict(split_k=2),
                          "cannot be combined with a non-linear epilogue"),
        "split_epi_mul": (replace(f32, variant="drelu"), dict(split_k=2),
                          "cannot be combined with a non-linear epilogue"),
        "split_add_in": (replace(f32, variant="add"), dict(split_k=2), "cannot be combined with a non-linear epilogue"),
        "split_dropout": (replace(f32, drop=True), dict(split_k=2), "cannot be combined with a non-linear epilogue"),
        "epi_mul_no_aux_in": (nt, dict(epi_mul=1), "epi_mul needs aux_in"),
        "block_n_8": (nt, dict(block_n=8), "invalid block_n"),
        "block_n_272": (nt, dict(block_n=272), "invalid block_n"),
        "block_n_96_b_mn": (replace(nt, maj="NN"), dict(block_n=96), "invalid block_n"),
        "a_base_unaligned": (nt, "a_base", "base not 16-byte aligned"),
        "lda_not_multiple_of_8": (replace(nt, lda_pad=True), dict(lda=68), "leading dimension must be a multiple of 8"),
        "batch_stride_not_multiple_of_8": (replace(nt, nb=(2, 1)), "a_s", "batch strides must be multiples of 8"),
        "M_zero": (nt, dict(M=0), "M, N, K must be positive"),
        "N_negative": (nt, dict(N=-1), "M, N, K must be positive"),
        "K_zero": (nt, dict(K=0), "M, N, K must be positive"),
    }


INVALID = _invalid_rows()


def _check_invalid(K, name, arm32=False):
    case, over, msg = INVALID[name]
    L = G.Launch(case, DEV, arm32)
    if over == "a_base":
        over = dict(a=L.a[3:])
    elif over == "a_s":
        over = dict(a_s=(L.a_s[0] - 4, 0))
    n0 = K.launch_count()
    with pytest.raises(RuntimeError, match=re.escape(msg)):
        L.run(K.gemm, **over)
    torch.cuda.synchronize()
    assert K.launch_count() == n0, "a rejected call launched a kernel"
    L.untouched()


@pytest.mark.parametrize("name", list(INVALID))
def test_gemm_invalid_arguments(K, name):
    """Host-side checks of bb_gemm_bf16: a RuntimeError with the library's message, no launch, buffers untouched."""
    _check_invalid(K, name)


@pytest.mark.parametrize("name", ["M_zero", "N_negative", "K_zero"])
def test_gemm_invalid_arguments_fp32_arm(K, name):
    with fp32_arm(K):
        _check_invalid(K, name, arm32=True)
