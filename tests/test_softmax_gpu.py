"""bb_softmax_fwd / bb_softmax_bwd element by element against fp64 references with a-priori bounds
(tests/softmax_cases.py), through the C ABI on guarded buffers: every case in the bf16 product mode and again in the
fp32 verification mode (K.set_precision(True)), whose bounds have no half-ulp bf16 term.  The table crosses the MAXE
buckets (ld = 128 | 136, 512 | 520, 1024), nk in {1, ld - 7, ld}, row counts 8k +- 1, several heads with a graph bias,
0 / -10000 / -inf key masks including a sample masked -inf everywhere (P = Pd = dS = 0) or -10000 everywhere
(uniform), dropout p in {0, 0.1, 0.5} and a negative out_scale.  The graph-bias gradient accumulates into a non-zero
buffer with atomics and, in deterministic mode, twice, bit-identical.

Worst err / bound per quantity (printed at the end of the module with -s), measured on an H100 80GB HBM3 at 700 W,
bf16 mode / fp32 mode.  The bounds are derived, not fitted; a bf16 output's bound is its half ulp plus a small fp32
term, so a ratio near 1 is expected there.
  softmax_fwd.P 0.999 / 0.702, Pd 0.999 / 0.702; softmax_bwd.dS 1.000 / 0.557, dbias 0.958 / 0.916
"""
import pytest
import torch

import rowops_cases as R
import softmax_cases as S

pytestmark = pytest.mark.gpu
BF, F32 = S.BF, S.F32


@pytest.fixture(scope="module", params=[False, True], ids=["bf16", "fp32"])
def act(request):
    from bevbert_b200 import _lib, kernels as K
    assert torch.cuda.is_available()
    _lib.load().bb_set_drop_salt_ptr(None)      # a graph test in the same process may have registered a dropout salt
    prev = K.set_precision(request.param)
    yield F32 if request.param else BF
    K.set_precision(prev)
    print("\nerr / bound, %s mode:" % ("fp32" if request.param else "bf16"))
    for k in sorted(R.RATIOS):
        print("  %-28s %.3f" % (k, R.RATIOS[k]))
    R.RATIOS.clear()


TABLE = S.softmax_table()


@pytest.mark.parametrize("i", range(len(TABLE)), ids=[c.id for c in TABLE])
def test_softmax(act, i):
    case = TABLE[i]
    A, ins, outs = S.run_softmax(case, act, "gpu", "cuda")
    S.check_softmax(case, act, A, ins, outs)


@pytest.mark.parametrize("i", [i for i, c in enumerate(TABLE) if c.bias][::3])
def test_softmax_dbias_deterministic(act, i):
    """deterministic mode: per-head partials summed in head order; two runs bit-identical, both within the bound"""
    case = TABLE[i]
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        A, ins, outs = S.run_softmax(case, act, "gpu", "cuda")
        S.check_softmax(case, act, A, ins, outs)
        _, _, outs2 = S.run_softmax(case, act, "gpu", "cuda")
    finally:
        torch.use_deterministic_algorithms(prev)
    for name, a, b in zip(("P", "Pd", "dS", "dbias"), outs, outs2):
        R.check_exact("deterministic rerun " + name, a, b)
