"""Runs the GEMM self-test cases that exercise the ping-pong tile schedule and the compile-time epilogue variants
(vln-bevbert_b200/csrc/selftest_gemm.cu): an odd number of tiles per CTA, a single tile, one tile more than the grid,
and the full-size gelu' dX and residual-add dX probes, each compared element by element with an fp32 reference."""
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
BIN = os.path.join(os.path.dirname(HERE), "vln-bevbert_b200", "csrc", "build", "selftest_gemm")

CASES = ["pp_odd_tiles", "pp_one_tile", "pp_grid_plus_1", "perf_dgelu", "perf_qkv_dx"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_gemm_selftest_pingpong_case_passes(case):
    if not os.path.exists(BIN):
        pytest.skip("selftest_gemm not built (run `make -C vln-bevbert_b200/csrc`)")
    out = subprocess.run([BIN, case], capture_output=True, text=True, timeout=300)
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("CASE")]
    assert len(lines) == 1, out.stdout[-2000:] + out.stderr[-2000:]
    assert " PASS " in lines[0] and out.returncode == 0, lines[0] + out.stderr[-2000:]
