"""The integer-operand GEMM harness of tests/test_gemm_gpu.py, rehearsed on the CPU against the torch emulation of the
GEMM (tests/emu_kernels.py): buffers, guards and the fp64 reference for every dropout-free row of the table at small
size, in both storage types.  This also pins the emulator, which the host-logic CPU tests trust, to the header's
contract.  No GPU needed."""
from dataclasses import replace

import pytest
import torch

import emu_kernels
import gemm_cases as G

SMALL = [c for c in G.TABLE + [G.pingpong_case(v, "3", 132) for v in ("plain", "gelu_pre", "dgelu")]
         if not c.drop and c.M * c.N * c.K * c.nb[0] * c.nb[1] <= 4e7]


@pytest.mark.parametrize("case", SMALL, ids=lambda c: c.id)
def test_harness_bf16_storage(case):
    L = G.Launch(case, "cpu")
    L.run(emu_kernels.gemm)
    L.check()


@pytest.mark.parametrize("case", G.fp32_arm_rows(SMALL), ids=lambda c: c.id)
def test_harness_fp32_storage(case):
    L = G.Launch(case, "cpu", arm32=True)
    L.run(emu_kernels.gemm)
    L.check()


def test_table_reaches_every_feature():
    """every epilogue variant at both tile widths, every N % 8 residue at both widths, every major for the plain and
    split rows, each pointer misaligned alone"""
    for v in G.VARIANTS:
        assert {c.block_n for c in G.TABLE if c.variant == v} >= {64, 128}, v
    for bn in (64, 128):
        assert {c.N % 8 for c in G.TABLE if c.variant == "plain" and c.block_n == bn} == set(range(8))
        assert any(c.N < 8 for c in G.TABLE if c.block_n == bn)
    assert {c.M % 128 for c in G.TABLE} >= {1, 9, 17, 33, 63, 64, 65, 100, 127, 0}
    assert {c.K for c in G.TABLE} >= {8, 16, 40, 64, 72, 136, 1000}
    assert {c.maj for c in G.TABLE if c.variant == "plain" and c.split_k == 1} == set(G.MAJORS)
    assert {c.maj for c in G.SPLIT_ROWS if c.split_k > 1} == set(G.MAJORS)
    assert {c.mis for c in G.TABLE} == {"", "D", "aux_in", "add_in", "aux_out"}
    assert {c.ldd for c in G.TABLE} == {"n", "pad", "odd"}
    for v in ("gelu_pre", "dgelu", "drelu", "add"):
        assert {c.drop for c in G.TABLE if c.variant == v} == {False, True}
    assert len({c.id for c in G.TABLE}) == len(G.TABLE)


def _corrupt(how):
    """the emulated GEMM with one placement error"""
    def gemm(a, b, out, M, N, K, lda, ldb, ldd, **kw):
        emu_kernels.gemm(a, b, out, M, N, K, lda, ldb, ldd, **kw)
        if how == "swap_cols":
            row = out[ldd * 5: ldd * 5 + N]
            row[[2, 3]] = row[[3, 2]].clone()
        elif how == "pad_write":
            out[N] = 0
        elif how == "guard_write":
            out[-1] = 0
        elif how == "off_by_one":
            out[ldd * 7 + 1] += 1
    return gemm


@pytest.mark.parametrize("how", ["swap_cols", "pad_write", "guard_write", "off_by_one"])
def test_harness_catches_placement_errors(how):
    case = G.Case("plain", 70, 45, 40, ldd="pad", bias=True, alpha=0.125)
    L = G.Launch(case, "cpu")
    L.run(_corrupt(how))
    with pytest.raises(AssertionError, match=r"bad element"):
        L.check()


def test_harness_catches_gelu_error():
    """a GELU output three bf16 ulps off in a single element fails the tolerance check"""
    case = G.Case("gelu_pre", 70, 45, 40, alpha=0.125)
    L = G.Launch(case, "cpu")
    L.run(emu_kernels.gemm)
    L.check()
    d = L.views["D"]
    i = int((d[:case.N].float().abs() > 0.5).nonzero()[0, 0])
    d.view(torch.int16)[i] += 3
    with pytest.raises(AssertionError, match=r"outside one output ulp"):
        L.check()


def test_misaligned_launch_sees_the_same_problem():
    a = G.Launch(G.Case("dgelu", 70, 45, 40), "cpu")
    b = G.Launch(replace(a.case, mis="aux_in"), "cpu")
    assert torch.equal(a.logical("aux_in"), b.logical("aux_in")) and torch.equal(G.bits(a.a), G.bits(b.a))
    assert b.views["aux_in"].data_ptr() % 16 != 0 and b.views["D"].data_ptr() % 16 == 0
