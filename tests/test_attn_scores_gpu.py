"""bb_attn_scores (the fused-scores kernel of the BB_FUSED_SCORES_MAX experiment) element by element against fp64 from
the same bf16 Q, K, V and dO (tests/softmax_cases.py): mode 0 (P, Pd) and mode 1 (dS, dbias into a non-zero buffer)
from the kernel's own P and from an unrelated bf16 P.  The table covers the tile tails (nq around 64 and 128, nk around
64), ldp = round8(nk), round8(nk) + 8 and 64 ceil(nk / 64) + 8 (an output block with no product block), the separate,
packed Q|K|V and packed K|V layouts, 0 / -10000 / -inf masks with a dead sample, dropout, and a grid of 432 tiles
(over three waves of the persistent loop, so the two-stage shared-memory ring flips phase).

Argument checks: misaligned P / Pd / Pin / dS, a call in the fp32 verification mode, and empty sizes, each without a
launch.

Worst err / bound per quantity (printed at the end of the module with -s), measured on an H100 80GB HBM3 at 700 W.
The score term uses the derived constant 64 (dh additions of at most one fp32 ulp each); nothing is fitted.
  attn_scores.P 0.984, Pd 0.984, dS 0.994, dbias 0.382
"""
import ctypes as C

import pytest
import torch

import rowops_cases as R
import softmax_cases as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from bevbert_b200 import _lib, kernels as K
    assert torch.cuda.is_available()
    _lib.load().bb_set_drop_salt_ptr(None)
    prev = K.set_precision(False)
    yield K
    K.set_precision(prev)
    print("\nerr / bound, bb_attn_scores:")
    for k in sorted(R.RATIOS):
        print("  %-28s %.3f" % (k, R.RATIOS[k]))
    R.RATIOS.clear()


TABLE = S.scores_table()


@pytest.mark.parametrize("i", range(len(TABLE)), ids=[c.id for c in TABLE])
def test_attn_scores(K, i):
    case = TABLE[i]
    A, ins, outs = S.run_scores(case, "gpu", "cuda")
    S.check_scores(case, A, ins, outs)


# ------------------------------------------------------------------------------------------------ argument checks
def _case_args(K, mode, **over):
    case = S.AsCase(65, 80, 88)
    ops, _ = S.scores_inputs(case, "cuda")
    buf = torch.zeros(2 * 2 * 65 * 88 + 8, dtype=torch.bfloat16, device="cuda")
    a = S._scores_args(ops, case, mode)
    if mode == 0:
        a.P, a.Pd = buf.data_ptr(), buf.data_ptr()
    else:
        a.Pin, a.dS = buf.data_ptr(), buf.data_ptr()
    for k, v in over.items():
        setattr(a, k, v)
    return a, (ops, buf)


def _rc(K, a):
    """-> (status, launches, message) of one bb_attn_scores call"""
    from bevbert_b200 import _lib
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    rc = lib.bb_attn_scores(C.byref(a), K._stream())
    return rc, lib.bb_launch_count() - n0, lib.bb_last_error().decode()


@pytest.mark.parametrize("field,mode", [("P", 0), ("Pd", 0), ("Pin", 1), ("dS", 1)])
def test_attn_scores_rejects_misaligned_outputs(K, field, mode):
    """P / Pd / Pin / dS are stored and read as bf16 pairs: an odd bf16 offset is refused before any launch"""
    a, keep = _case_args(K, mode)
    setattr(a, field, getattr(a, field) + 2)
    rc, n, msg = _rc(K, a)
    assert rc != 0 and n == 0 and "4-byte aligned" in msg, (rc, n, msg)


def test_attn_scores_rejects_fp32_mode(K):
    a, keep = _case_args(K, 0)
    prev = K.set_precision(True)
    try:
        rc, n, msg = _rc(K, a)
    finally:
        K.set_precision(prev)
    assert rc != 0 and n == 0 and "fp32 verification mode" in msg, (rc, n, msg)
    with pytest.raises(TypeError):
        q = torch.zeros(65, 128, device="cuda")
        K.attn_scores_fwd(q, 128, q, 128, 1, 2, 65, 65, 64, 72, None, None, K.NO_DROP)


@pytest.mark.parametrize("field", ["B", "H", "nq"])
@pytest.mark.parametrize("mode", [0, 1])
def test_attn_scores_empty_sizes_launch_nothing(K, field, mode):
    for v in (0, -1):
        a, keep = _case_args(K, mode, **{field: v})
        rc, n, msg = _rc(K, a)
        assert rc == 0 and n == 0, (field, v, rc, n, msg)
