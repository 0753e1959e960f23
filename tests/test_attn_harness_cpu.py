"""The attention harness of tests/test_attn_gpu.py, rehearsed on the CPU against the fp32 torch restatement of the
kernels' arithmetic (tests/emu_kernels.py flash_core_*): buffers, guards, sentinels and the fp64 reference of every
dropout-free exact-routing row, bit for bit.  Also: the table reaches every feature, the checker catches planted
errors, and the host-side alignment checks of bb_flash_fwd / bb_flash_bwd run before any CUDA call.  No GPU needed."""
import json
import os
import subprocess
import sys

import pytest
import torch

import attn_cases as A
import emu_kernels as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = [c for c in A.EXACT_ROWS if not c.drop]


def _kw(L):
    kw = {}
    if "kmask" in L.bufs:
        kw["kmask"] = L.fview("kmask", (L.case.B, L.case.nk))
    if "bias" in L.bufs:
        kw["bias"] = L.fview("bias", (L.case.B, L.case.nq, L.case.nk))
    return kw


def emu_fwd(L):
    c = L.case
    E.flash_core_fwd(L.strided("q"), L.strided("k"), L.strided("v"), L.strided("o"), L.fview("lse", (c.B, c.H, c.nq)),
                     c.alpha, **_kw(L))


def emu_bwd(L):
    c = L.case
    db = L.fview("dbias", (c.B, c.nq, c.nk)) if "dbias" in L.bufs else None
    E.flash_core_bwd(L.strided("q"), L.strided("k"), L.strided("v"), L.strided("o"), L.fview("lse", (c.B, c.H, c.nq)),
                     L.strided("dout"), L.strided("dq"), L.strided("dk"), L.strided("dv"), c.alpha, dbias=db, **_kw(L))
    L.fview("dsum", (c.B, c.H, c.nq)).zero_()


@pytest.mark.parametrize("case", ROWS, ids=lambda c: c.id)
def test_harness_exact_rows(case):
    A.run_case(A.Launch(case, "cpu"), emu_fwd, emu_bwd)


@pytest.mark.parametrize("layout", ["sep", "self"])
def test_harness_layouts_see_the_same_problem(layout):
    """a packed launch of a case holds the same values as its separate-buffer launch"""
    case = A.Case("exact", 2, 12, 80, 80, "mma", "mma", "mix")
    a, b = A.Launch(case, "cpu"), A.Launch(case, "cpu", layout=layout)
    for nm in ("q", "k", "v", "dout"):
        assert torch.equal(A.bits(a.view(nm)), A.bits(b.view(nm)))
    assert torch.equal(a.R["dq"], b.R["dq"])


def test_table_reaches_every_feature():
    T = A.TABLE
    assert {c.nq for c in T} >= {1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 257, 441}
    assert {c.nk for c in T} >= {1, 7, 23, 36, 63, 64, 65, 127, 128, 129, 191, 193, 441, 512, 600}
    model = {(441, 441), (80, 80), (441, 80), (80, 441), (36, 36), (1, 80)}
    assert model <= {(c.nq, c.nk) for c in A.EXACT_ROWS}
    assert any(c.nq == 23 and c.nk == 23 and c.bias and c.H == 12 for c in A.EXACT_ROWS)
    assert {c.H for c in T} == {1, 12} and max(c.B for c in T) == 3
    for fam in (A.EXACT_ROWS, A.BOUND_ROWS):
        assert {c.fwd for c in fam} >= {"mma", "tc", "auto"} and {c.bwd for c in fam} >= {"mma", "tc", "auto"}
        assert {(c.fwd, c.bwd) for c in fam} >= {("mma", "tc"), ("tc", "mma")}
        assert {c.mask for c in fam} == {"none", "mix", "tail", "full10k", "fullinf"}
        assert {c.layout for c in fam} == {"sep", "self", "cross"}
        assert {c.drop > 0 for c in fam} == {False, True}
    assert {c.dbias for c in A.EXACT_ROWS} == {"", "atomic", "det"}
    assert {c.alpha for c in A.EXACT_ROWS} >= {0.125, 1.0, 2.0}
    assert {c.adv for c in A.BOUND_ROWS} == {"", "ramp", "single", "big"}
    assert all(c.fwd == "mma" and c.bwd == "mma" for c in T if c.bias)
    # the stage ring wraps: key blocks >= 4 and >= 7 on both cores
    for core in ("mma", "tc"):
        assert any(-(-c.nk // 64) >= 7 and c.fwd == core for c in A.EXACT_ROWS)
        assert any(-(-c.nq // 64) >= 4 and c.bwd == core for c in A.EXACT_ROWS)
    assert len({c.id for c in T}) == len(T)


@pytest.mark.parametrize("case", [A.Case("exact", 2, 1, 257, 512, "mma", "mma", "none", alpha=1.0),
                                  A.Case("exact", 2, 1, 129, 600, "tc", "tc", "tail"),
                                  A.Case("exact", 3, 12, 128, 127, "auto", "tc", "none")], ids=lambda c: c.id)
def test_winners_reach_every_key_block(case):
    """every key block of every (sample, head) with unmasked keys holds some query's winners, and some rows meet their first winner
    after a block of losers (the online-softmax rescale flushes the losers' running maximum)"""
    L = A.Launch(case, "cpu")
    win = L.val["win"]
    nblk = -(-case.nk // 64)
    blk = win.reshape(case.B, case.H, case.nq, -1)
    pad = nblk * 64 - case.nk
    w = torch.nn.functional.pad(blk, (0, pad)).reshape(case.B, case.H, case.nq, nblk, 64).any(-1)
    km = L.val["kmask"] if L.val["kmask"] is not None else torch.zeros(case.B, case.nk, dtype=torch.float64)
    live = torch.nn.functional.pad(km > float("-inf"), (0, pad)).reshape(case.B, 1, nblk, 64).any(-1)
    assert bool((w.any(2) | ~live).all()), "a key block with unmasked keys but without winners"
    first = w.float().argmax(-1)
    assert bool((first > 0).any())


# ------------------------------------------------------------------------------------------- planted errors
def _planted(how):
    def fwd(L):
        c = L.case
        if how == "key_block":
            km = torch.zeros(c.B, c.nk) if "kmask" not in L.bufs else L.fview("kmask", (c.B, c.nk)).clone()
            km[:, 64:128] = float("-inf")                       # one key block left out of the softmax
            E.flash_core_fwd(L.strided("q"), L.strided("k"), L.strided("v"), L.strided("o"),
                             L.fview("lse", (c.B, c.H, c.nq)), c.alpha, kmask=km)
            return
        emu_fwd(L)
        o = L.strided("o")
        if how == "swap_rows":
            o[0, [3, 4]] = o[0, [4, 3]].clone()
        elif how == "pad_write":
            sl = L.slots["o"]
            L.bufs["o"][sl.start + c.H * 64] = 0              # first padding column of row 0
        elif how == "guard_write":
            L.bufs["lse"][-1] = 0
        elif how == "lse_ulp":
            lse = L.fview("lse", (c.B, c.H, c.nq))
            lse.view(torch.int32)[1, 0, 5] += 1

    def bwd(L):
        emu_bwd(L)
        if how == "dk_row":
            dk = L.strided("dk")
            dk[1, 7] = dk[1, 8].clone() if not torch.equal(dk[1, 7], dk[1, 8]) else dk[1, 7] + 1
    return fwd, bwd


@pytest.mark.parametrize("how", ["swap_rows", "pad_write", "guard_write", "key_block", "lse_ulp", "dk_row"])
def test_checker_catches_planted_errors(how):
    case = A.Case("exact", 2, 12, 80, 191, "mma", "mma", "none")
    L = A.Launch(case, "cpu")
    fwd, bwd = _planted(how)
    with pytest.raises(AssertionError, match=r"bad elements"):
        A.run_case(L, fwd, bwd)


def test_checker_catches_bound_violation():
    """error-bounded family: one O element moved by 32 bf16 ulps (about 25 %) fails its bound"""
    case = A.Case("bound", 2, 1, 65, 193, "mma", "mma", "none")
    L = A.Launch(case, "cpu")
    emu_fwd(L)
    L.check_fwd()
    o = L.strided("o")
    o.view(torch.int16)[1, 3, 0, 5] += 32
    with pytest.raises(AssertionError, match=r"outside ulp/2"):
        L.check_fwd()


# ------------------------------------------------------------------------------------ host-side argument checks
_MISALIGNED = r"""
import ctypes as C, json, sys
sys.path.insert(0, sys.argv[1])
import __graft_entry__  # noqa: F401
from bevbert_b200 import _lib
lib = _lib.load()
BASE = 0x100000000          # never dereferenced: the calls must be rejected before any CUDA call


def args():
    a = _lib.FlashArgs()
    for n in ("q", "k", "v", "o", "lse", "dout", "dsum", "dq", "dk", "dv"):
        setattr(a, n, BASE)
    a.q_bs = a.k_bs = a.v_bs = a.o_bs = a.do_bs = a.dq_bs = a.dk_bs = a.dv_bs = 80 * 768
    a.ldq = a.ldk = a.ldv = a.ldo = a.lddo = a.lddq = a.lddk = a.lddv = 768
    a.B, a.H, a.nq, a.nk, a.dh, a.alpha = 2, 12, 80, 80, 64, 0.125
    return a


out = []
for fn, field, val in json.loads(sys.argv[2]):
    a = args()
    setattr(a, field, getattr(a, field) + val)
    n0 = lib.bb_launch_count()
    rc = getattr(lib, fn)(C.byref(a), None)
    msg = lib.bb_last_error()
    out.append([fn, field, rc, lib.bb_launch_count() - n0, msg.decode() if msg else ""])
print(json.dumps(out))
"""

MISALIGNED = [("bb_flash_fwd", f, 2, "q / k / v / o must be 16-byte aligned") for f in ("q", "k", "v", "o")] + \
    [("bb_flash_fwd", f, 4, "batch strides must be multiples of 8 elements") for f in ("q_bs", "k_bs", "v_bs", "o_bs")] + \
    [("bb_flash_bwd", f, 8, "dout / dq / dk / dv must be 16-byte aligned") for f in ("dout", "dq", "dk", "dv")] + \
    [("bb_flash_bwd", f, 2, "batch strides must be multiples of 8 elements") for f in ("do_bs", "dq_bs", "dk_bs", "dv_bs")] + \
    [("bb_flash_bwd", "q", 4, "q / k / v / o must be 16-byte aligned")]


def test_misaligned_flash_arguments_are_rejected_before_any_cuda_call():
    """Each misaligned pointer and each batch stride that is not a multiple of 8 elements: bb_flash_fwd / _bwd return
    the alignment message and launch nothing.  Fake pointers, never dereferenced; the calls run in a process that sees
    no GPU, so a library that let one through could not launch it anywhere."""
    lib = os.path.join(ROOT, "vln-bevbert_b200", "libbevbert_b200.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    spec = json.dumps([[fn, f, v] for fn, f, v, _ in MISALIGNED])
    r = subprocess.run([sys.executable, "-c", _MISALIGNED, ROOT, spec], env=env, capture_output=True, text=True,
                       timeout=120)
    assert r.returncode == 0, r.stderr
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for (fn, field, rc, launched, msg), (_, _, _, want) in zip(res, MISALIGNED):
        assert rc != 0 and launched == 0, (fn, field, rc, launched, msg)
        assert want in msg, (fn, field, msg)
