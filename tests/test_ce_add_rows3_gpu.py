"""bb_add_rows3 (the VLN-CE view-embedding sum) element by element against fp64, on the bf16 product path and the fp32
verification arm: ragged row counts, padded row strides, NaN in every byte it must not read, guard rows and padding
columns of the output that must stay untouched, argument checks, and the AddRows3Impl backward; bit-identical repeats
under torch.use_deterministic_algorithms(True).  The checkers live in tests/ce_cases.py and are rehearsed against
planted faults on CPU by tests/test_ce_pretrain_cpu.py."""
import pytest
import torch

import ce_cases as C
from bevbert_b200 import blocks as Bk
from bevbert_b200 import kernels as K
from bevbert_b200 import _lib

pytestmark = pytest.mark.gpu


def _arm(fp32):
    return torch.float32 if fp32 else torch.bfloat16


@pytest.mark.parametrize("fp32", [False, True])
@pytest.mark.parametrize("case", C.CASES)
def test_forward_against_fp64(case, fp32):
    prev = K.set_precision(fp32)
    try:
        act = _arm(fp32)
        ops = C.make_case(case, act, seed=case[0], device="cuda")
        K.add_rows(ops["a"], ops["b"], ops["table"], ops["idx"], ops["vec"], c=ops["c"], out=ops["out"])
        torch.cuda.synchronize()
        r = C.check_forward(ops, act, str(case))
        print("add_rows3 %s %s worst err/bound %.3f" % (case, act, r))
    finally:
        K.set_precision(prev)


@pytest.mark.parametrize("fp32", [False, True])
@pytest.mark.parametrize("case", [C.CASES[1], C.CASES[2], C.CASES[3], C.CASES[6]])
def test_backward_and_deterministic_mode(case, fp32):
    prev = K.set_precision(fp32)
    try:
        act = _arm(fp32)
        ops = C.make_case(case, act, seed=7, device="cuda")
        H = ops["a"].shape[1]
        vsrc = torch.stack([torch.randn(H, device="cuda"), ops["vec"]]) if ops["vec"] is not None else None
        g = (torch.randn(ops["a"].shape, device="cuda") * 3).to(act)

        def step():
            impl, st = Bk.AddRows3Impl(vec_row=1), {}
            out = impl.fwd(st, [ops["a"], ops["b"], ops["c"], ops["idx"]], [ops["table"], vsrc])
            gin, gp = impl.bwd(st, [g], [ops["table"], vsrc])
            torch.cuda.synchronize()
            return out, gin, gp

        out, gin, gp = step()
        ops["out"] = out
        ops["out_buf"] = torch.full((out.shape[0] + 2, H), C.SENTINEL, dtype=act, device="cuda")
        ops["out_buf"][1:-1] = out
        C.check_forward(ops, act, "impl")
        C.check_backward(g, (gin, gp), ops, "impl")
        torch.use_deterministic_algorithms(True)
        try:
            r1, r2 = step(), step()
        finally:
            torch.use_deterministic_algorithms(False)
        assert torch.equal(r1[0], r2[0])
        for x, y in zip(r1[2], r2[2]):
            assert (x is None and y is None) or torch.equal(x, y)
        C.check_backward(g, (r1[1], r1[2]), ops, "deterministic")
    finally:
        K.set_precision(prev)


def test_argument_checks_leave_output_untouched():
    ops = C.make_case(C.CASES[2], torch.bfloat16, seed=3, device="cuda")
    lib = _lib.load()
    a, b, c, o = ops["a"], ops["b"], ops["c"], ops["out"]
    rows, H = a.shape
    base = dict(a=a.data_ptr(), lda=a.stride(0), b=b.data_ptr(), ldb=b.stride(0), c=c.data_ptr(), ldc=c.stride(0),
                t=ops["table"].data_ptr(), i=ops["idx"].data_ptr(), v=ops["vec"].data_ptr(), rows=rows, H=H,
                o=o.data_ptr(), ldo=o.stride(0))
    bad = [dict(H=20), dict(c=0), dict(i=0), dict(lda=H - 8), dict(ldo=H + 4), dict(a=a.data_ptr() + 2),
           dict(o=o.data_ptr() + 8), dict(v=ops["vec"].data_ptr() + 4)]
    before = ops["out_buf"].clone()
    for d in bad:
        k = dict(base, **d)
        rc = lib.bb_add_rows3(k["a"], k["lda"], k["b"], k["ldb"], k["c"], k["ldc"], k["t"], k["i"], k["v"], k["rows"],
                              k["H"], k["o"], k["ldo"], None)
        assert rc != 0, d
        assert b"bb_add_rows3" in lib.bb_last_error()
    assert lib.bb_add_rows3(base["a"], base["lda"], base["b"], base["ldb"], base["c"], base["ldc"], 0, 0, 0, 0, H,
                            base["o"], base["ldo"], None) == 0          # rows = 0: nothing to do
    torch.cuda.synchronize()
    assert torch.equal(ops["out_buf"].view(torch.int16), before.view(torch.int16))
