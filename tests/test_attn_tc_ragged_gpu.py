"""csrc/attn_tc.cu at ragged query counts (1, 63, 65, 80, 441): the forward and the dQ pass stage each key block's mask
in shared memory, and the dK/dV pass stages -lse, D (written by the dQ pass) and the dropout row hash of each query
block.  Forward and both backward passes against fp32 torch autograd, with a key mask and with dropout off and on
(keep mask from drop_masks.attn_keep)."""
import pytest
import torch

import drop_masks as DM
from helpers import rel_l2

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _rnd(*shape, scale, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(BF).cuda()


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("nq,nk,cross", [(1, 80, True), (63, 441, True), (65, 80, True), (80, 80, False),
                                         (441, 441, False), (441, 80, True)])
def test_attn_tc_ragged_queries_match_fp32_autograd(nq, nk, cross, dropout):
    import bevbert_b200.kernels as K
    from bevbert_b200 import _lib
    _lib.load().bb_set_drop_salt_ptr(None)       # a graph test in the same process may have registered a dropout salt
    B, H, Hd, seed = 2, 12, 768, 31
    if not cross:
        qkv = _rnd(B * nq, 3 * Hd, scale=0.8, seed=1)
        q, k, v, ldq, ldk, ldv = qkv, qkv[:, Hd:], qkv[:, 2 * Hd:], 3 * Hd, 3 * Hd, 3 * Hd
    else:
        q = _rnd(B * nq, Hd, scale=0.8, seed=1)
        kv = _rnd(B * nk, 2 * Hd, scale=0.8, seed=2)
        k, v, ldq, ldk, ldv = kv, kv[:, Hd:], Hd, 2 * Hd, 2 * Hd
    kmask = torch.zeros(B, nk)
    kmask[1, nk // 2:] = -10000.0
    kmask[0, -3:] = float("-inf")
    kmask = kmask.cuda()
    dout = _rnd(B, nq, Hd, scale=0.5, seed=3)
    th, sc = K.drop_params(0.1 if dropout else 0.0)
    drop = (seed, th, sc) if dropout else K.NO_DROP
    prev = K.set_attn_tc(2)
    try:
        o, lse = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, None, drop)
        dq, dk, dv = K.flash_bwd(q, k, v, o, lse, dout, B, H, nq, nk, ldq, ldk, ldv, kmask, None, drop)
    finally:
        K.set_attn_tc(prev)

    def heads(t, n, ld):
        return torch.as_strided(t, (B, H, n, 64), (n * ld, 64, ld, 1), t.storage_offset()).float().clone().requires_grad_(True)
    qh, kh, vh = heads(q, nq, ldq), heads(k, nk, ldk), heads(v, nk, ldv)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * 0.125 + kmask.view(B, 1, 1, nk), -1)
    if dropout:
        p = p * DM.attn_keep(seed, B, H, nq, nk, th).cuda() * sc
    ro = (p @ vh).permute(0, 2, 1, 3).reshape(B, nq, Hd)
    ro.backward(dout.float())

    def unheads(t, n):
        return t.permute(0, 2, 1, 3).reshape(B, n, Hd)
    assert rel_l2(o.view(B, nq, Hd), ro.detach()) < 6e-3
    assert rel_l2(dq.view(B, nq, Hd), unheads(qh.grad, nq)) < 1.2e-2
    assert rel_l2(dk.view(B, nk, Hd), unheads(kh.grad, nk)) < 1.2e-2
    assert rel_l2(dv.view(B, nk, Hd), unheads(vh.grad, nk)) < 1.2e-2
