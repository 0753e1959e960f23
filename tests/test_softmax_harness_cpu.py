"""The unfused-attention harness of tests/test_softmax_gpu.py and tests/test_attn_scores_gpu.py, rehearsed on the CPU:
the fp64 references and their bounds (tests/softmax_cases.py) against the torch restatement in tests/emu_kernels.py
(bf16 rounding on through set_act_dtype), the case tables reach every feature the issue of each kernel needs, and the
checkers reject each kind of fault a kernel could have.  No GPU needed."""
import pytest
import torch

import emu_kernels as E
import softmax_cases as S

BF, F32 = S.BF, S.F32


@pytest.fixture(params=[BF, F32], ids=["bf16", "fp32"])
def act(request):
    E.set_act_dtype(request.param)
    yield request.param
    E.set_act_dtype(F32)


SM = S.softmax_table()


@pytest.mark.parametrize("i", range(0, len(SM), 2))
def test_harness_softmax(act, i):
    case = SM[i]
    A, ins, outs = S.run_softmax(case, act, "emu", "cpu")
    S.check_softmax(case, act, A, ins, outs)


AS = [c for c in S.scores_table() if c.B * c.H * c.nq * c.ldp <= 2_000_000]


@pytest.mark.parametrize("i", range(0, len(AS), 3))
def test_harness_attn_scores(i):
    E.set_act_dtype(BF)
    try:
        case = AS[i]
        A, ins, outs = S.run_scores(case, "emu", "cpu")
        S.check_scores(case, A, ins, outs)
    finally:
        E.set_act_dtype(F32)


def test_tables_reach_every_feature():
    sm = S.softmax_table()
    for ld in S.LDS:
        assert {c.nk for c in sm if c.ld == ld} >= {1, max(1, ld - 7), ld}, ld
    rows = {c.B * c.H * c.nq % 8 for c in sm}
    assert {1, 7} <= rows
    assert all({m for m in S.MASKS} <= {c.mask for c in sm if c.ld == ld} for ld in (128, 136, 512, 520))
    assert {0.0, 0.1, 0.5} <= {c.p for c in sm} and any(c.out_scale not in (0.125,) for c in sm)
    assert any(c.H > 1 and c.bias and c.B > 1 for c in sm)
    sc = S.scores_table()
    assert set(S.AS_NQ) <= {c.nq for c in sc} and set(S.AS_NK) <= {c.nk for c in sc}
    for nk in (63, 65, 441):
        assert set(S.ldps(nk)) <= {c.ldp for c in sc if c.nk == nk}
    assert any(c.ldp > 64 * -(-c.nk // 64) for c in sc)             # an output block with no product block
    tiles = [c.B * c.H * -(-c.nq // 128) for c in sc]
    assert min(tiles) < 132 and max(tiles) >= 3 * 132
    assert {"sep", "self", "cross"} == {c.layout for c in sc}
    assert set(S.MASKS) <= {c.mask for c in sc} and {0.0, 0.1, 0.5} <= {c.p for c in sc}
    assert {"own", "other"} == {c.pin for c in sc} and any(c.bias for c in sc)


@pytest.mark.parametrize("kind", sorted(S.PLANTS))
def test_checker_rejects_planted_fault(kind):
    """one-ulp bf16 error, wrong dropout mask, unwritten padding column, NaN on a dead row, write past the end,
    dbias without its initial value: each must fail the check of an otherwise correct run"""
    E.set_act_dtype(BF)
    try:
        case = S.PLANTS[kind]
        A, ins, outs = S.run_softmax(case, BF, "emu", "cpu")
        S.check_softmax(case, BF, A, ins, outs)                  # the correct run passes
        A, ins, outs = S.run_softmax(case, BF, "emu", "cpu")
        S.plant(kind, case, BF, A, ins, outs)
        with pytest.raises(AssertionError):
            S.check_softmax(case, BF, A, ins, outs)
    finally:
        E.set_act_dtype(F32)


def test_dead_rows_are_zero_in_the_restatement():
    """a row with every key at -inf gives P = Pd = dS = 0 and adds nothing to dbias (the flash cores' convention)"""
    B, H, nq, nk, ld = 2, 2, 3, 5, 8
    s = torch.randn(B, H, nq, ld)
    km = torch.zeros(B, nk)
    km[1] = float("-inf")
    p, _ = E.softmax_fwd(s, km, None, B, H, nq, nk, ld)
    assert torch.equal(p[1], torch.zeros_like(p[1])) and bool(torch.isfinite(p).all())
    db = torch.zeros(B, nq, nk)
    ds = E.softmax_bwd(p, torch.randn(B, H, nq, ld), B, H, nq, nk, ld, (0, 0, 1.0), 0.125, db)
    assert torch.equal(ds[1], torch.zeros_like(ds[1])) and torch.equal(db[1], torch.zeros_like(db[1]))
