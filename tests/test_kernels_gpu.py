"""Per-kernel parity on the GPU, through the C ABI (bevbert_b200.kernels -> ctypes -> libbevbert_b200.so).

Each kernel is compared with its torch restatement (tests/emu_kernels.py, fp32 on CPU) on the same
bf16-rounded inputs.  Tolerances: integer / index work bit-exact; fp32 outputs 1e-4 relative;
bf16 outputs 1e-2 relative (one bf16 rounding = 2^-9)."""
import math

import pytest
import torch

import emu_kernels as E
from helpers import rel_l2

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


@pytest.fixture(scope="module")
def K():
    import bevbert_b200.kernels as K
    assert torch.cuda.is_available()
    return K


def rnd(*shape, scale=1.0, dtype=BF, seed=0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dtype)


def dev(t):
    return t.cuda() if t is not None else None


def f32(t):
    return t.float().cpu() if t is not None else None


# ----------------------------------------------------------------------------------------- BEV
def test_lift_index_bit_exact(K):
    from bevbert_b200 import synth
    from oracle import bevbert_ref as R
    for D, res in ((21, 0.5), (11, 1.0)):
        b = synth.make_batch(synth.SynthConfig(batch_size=3, bev_dim=D, bev_res=res), seed=5)
        idx, pc = K.bev_lift_index(dev(b["depths"]).reshape(3, 12, 14, 14), dev(b["T_c2w"]), dev(b["S_w2c"]).reshape(3, 3),
                                   dev(b["T_w2c"]).reshape(3, 4, 4), D, res, want_pc=True)
        rpc, nod = R.lift_points(b["depths"], b["T_c2w"], b["S_w2c"], b["T_w2c"])
        ridx = R.cell_index(rpc, nod, D, res)
        assert torch.equal(pc.cpu(), rpc), "ego-frame point cloud must match the oracle bit for bit"
        assert torch.equal(idx.cpu().long(), ridx), "cell indices must be bit-exact"
        assert (ridx >= 0).float().mean() > 0.3


def test_lift_index_known_answers(K):
    """Hand-built cases (SURVEY.md 8c): centre cell, round-half-even at +-0.25 m, y clip, zero depth, outside."""
    D, res = 21, 0.5

    def cell_of(x, y, z):
        # one pixel image whose un-projection is (x*?..): use T_c2w translation to place the point, depth tiny
        T = torch.eye(4)
        T[0, 3], T[1, 3], T[2, 3] = x, y, z
        depths = torch.full((1, 1, 1, 1), 1e-30)          # non-zero depth, negligible offset
        idx, _ = K.bev_lift_index(dev(depths), dev(T[None, None]), dev(torch.zeros(1, 3)), dev(torch.eye(4)[None]), D,
                                  res, fx=1.0, fy=1.0, cx=0.5, cy=0.5)
        return int(idx.cpu()[0, 0])
    centre = (D * D - 1) // 2
    assert cell_of(0, 0, 0) == centre
    assert cell_of(0.25, 0, 0) == centre          # 0.25/0.5+10 = 10.5 -> rounds to even 10
    assert cell_of(0.75, 0, 0) == centre + 2      # 11.5 -> 12
    assert cell_of(-0.25, 0, 0) == centre         # 9.5 -> 10 (even)
    assert cell_of(0, 0.5, 0) == centre           # y == clip is kept
    assert cell_of(0, 0.5001, 0) == -1            # above the clip
    assert cell_of(5.3, 0, 0) == -1               # 20.6 -> 21 >= D: outside
    assert cell_of(0, 0, -5.3) == -1
    z = torch.zeros(1, 1, 1, 1)
    idx, _ = K.bev_lift_index(dev(z), dev(torch.eye(4)[None, None]), dev(torch.zeros(1, 3)), dev(torch.eye(4)[None]), D,
                              res)
    assert int(idx.cpu()[0, 0]) == -1             # depth 0 dropped


def test_scatter_mean_deterministic_and_exact(K):
    B, P, C, ncell = 3, 2352, 768, 441
    g = torch.Generator().manual_seed(1)
    feats = torch.randn(B, P, C, generator=g)
    idx = torch.randint(-1, ncell, (B, P), generator=g, dtype=torch.int32)
    idx[0, :50] = 7                      # heavily shared cell
    idx[1] = -1                          # sample with no valid point
    idx[2, idx[2] == 5] = 6              # guaranteed empty cell
    o32, o16, ob, cnt = K.bev_scatter_mean(dev(feats), dev(idx), ncell)
    r32, _, rob, rcnt = E.bev_scatter_mean(feats, idx, ncell)
    assert torch.equal(o32.cpu(), r32), "sequential-order sum + divide must be bit-exact"
    assert torch.equal(ob.cpu(), rob) and torch.equal(cnt.cpu(), rcnt)
    assert torch.equal(o16.cpu(), r32.to(BF))
    assert not ob.cpu()[1].any() and float(o32[1].abs().max()) == 0.0
    o32b, _, _, _ = K.bev_scatter_mean(dev(feats), dev(idx), ncell)
    assert torch.equal(o32, o32b), "run-to-run deterministic"
    # 16-bit wire format: bf16 point features pool exactly like their fp32 images (same fp32 sums, same order)
    w32, w16, wob, wcnt = K.bev_scatter_mean(dev(feats.to(BF)), dev(idx), ncell)
    x32, _, xob, _ = E.bev_scatter_mean(feats.to(BF).float(), idx, ncell)
    assert torch.equal(w32.cpu(), x32) and torch.equal(wob.cpu(), xob) and torch.equal(wcnt.cpu(), rcnt)
    sems = torch.nn.functional.one_hot(torch.randint(0, 40, (B, P), generator=g), 40).double()
    s, sm = K.bev_scatter_sem(dev(sems), dev(idx), ncell)
    rs, rsm = E.bev_scatter_sem(sems, idx, ncell)
    assert torch.equal(s.cpu(), rs) and torch.equal(sm.cpu(), rsm)


# ----------------------------------------------------------------------------------------- casts / dropout
def test_cast_and_dropout(K):
    x = torch.randn(1000003)
    y = K.cast_to_act(dev(x))
    assert torch.equal(y.cpu(), x.to(BF))
    assert torch.equal(K.cast_to_f32(y).cpu(), x.to(BF).float())
    p = 0.1
    th, sc = K.drop_params(p)
    d1 = K.cast_to_act(dev(x), (1234, th, sc)).cpu().float()
    d2 = K.cast_to_act(dev(x), (1234, th, sc)).cpu().float()
    d3 = K.cast_to_act(dev(x), (1235, th, sc)).cpu().float()
    assert torch.equal(d1, d2) and not torch.equal(d1, d3)
    keep = d1 != 0
    assert abs(float(keep.float().mean()) - (1 - p)) < 3e-3
    assert torch.equal(d1[keep], (x * sc).to(BF).float()[keep])
    # the bf16->bf16 dropout regenerates the same mask
    d4 = K.dropout_act(y, (1234, th, sc)).cpu().float()
    nz = (y.cpu().float() != 0) & (x != 0)
    assert torch.equal((d4 != 0)[nz], keep[nz])


# ----------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("x_f32,res", [(False, True), (False, False), (True, False)])
def test_layernorm_fwd_bwd(K, x_f32, res):
    rows, H = 1037, 768
    x = rnd(rows, H, dtype=torch.float32 if x_f32 else BF)
    r = rnd(rows, H, seed=1) if res else None
    gam, bet = torch.rand(H) + 0.5, torch.randn(H) * 0.1
    dy = rnd(rows, H, seed=2)
    y, y32, mean, rstd = K.layernorm_fwd(dev(x), dev(r), dev(gam), dev(bet), 1e-12, want_f32=True)
    ry, _, rm, rr = E.layernorm_fwd(f32(x), f32(r), gam, bet, 1e-12)
    assert rel_l2(y32, ry) < 1e-5 and rel_l2(y, ry) < 5e-3
    assert rel_l2(mean, rm) < 1e-5 and rel_l2(rstd, rr) < 1e-5
    dg, db = torch.zeros(H).cuda(), torch.zeros(H).cuda()
    dxs = torch.zeros(H).cuda()
    dx, dres = K.layernorm_bwd(dev(dy), dev(x), dev(r), dev(gam), mean, rstd, want_dres=res, dx_f32=x_f32, dgamma=dg,
                               dbeta=db, dxsum=dxs)
    rdg, rdb = torch.zeros(H), torch.zeros(H)
    rdx, rdres = E.layernorm_bwd(f32(dy), f32(x), f32(r), gam, rm, rr, want_dres=res, dgamma=rdg, dbeta=rdb)
    assert rel_l2(dx, rdx) < (1e-4 if x_f32 else 6e-3)
    if res:
        assert rel_l2(dres, rdres) < 6e-3
    assert rel_l2(dg, rdg) < 1e-4 and rel_l2(db, rdb) < 1e-4
    assert float((dxs.cpu() - rdx.sum(0)).norm()) < 1e-3 * float(rdx.abs().sum(0).norm())   # bias grad of the dense before LN


def _ln_keep_mask(seed, rows, H, thresh):
    """torch restatement of the LayerNorm-site dropout decisions (csrc/rowops.cu ln_keep8: one hash per 8-element vector,
    four mixes, 16-bit halves), for checking that forward and backward apply the documented function."""
    M = 0xFFFFFFFF
    vec = torch.arange(rows * H // 8, dtype=torch.int64)
    x = (vec & M) ^ (((vec >> 32) * 0x9E3779B1) & M) ^ (seed & M) ^ (((seed >> 32) * 0x85EBCA6B) & M)
    x = x ^ (x >> 16)
    x = (x * 0x7FEB352D) & M
    x = x ^ (x >> 15)
    x = (x * 0x846CA68B) & M
    h = x ^ (x >> 16)
    t16 = thresh >> 16
    keep = torch.zeros(rows * H // 8, 8, dtype=torch.bool)
    for k in range(4):
        y = (h + (k + 1) * 0x9E3779B1) & M
        y = y ^ (y >> 15)
        y = (y * 0x2C1B3C6D) & M
        y = y ^ (y >> 16)
        keep[:, 2 * k] = (y & 0xFFFF) >= t16
        keep[:, 2 * k + 1] = (y >> 16) >= t16
    return keep.reshape(rows, H)


def test_layernorm_dropout_replay(K):
    from bevbert_b200 import _lib
    _lib.load().bb_set_drop_salt_ptr(None)       # a graph test in the same process may have registered a dropout salt
    rows, H = 512, 768
    x, r = rnd(rows, H), rnd(rows, H, seed=1)
    gam, bet = torch.ones(H), torch.zeros(H)
    th, sc = K.drop_params(0.1)
    di, do = (77, th, sc), (78, th, sc)
    y, _, mean, rstd = K.layernorm_fwd(dev(x), dev(r), dev(gam), dev(bet), 1e-12, drop_in=di, drop_out=do)
    out_keep = (y.cpu().float() != 0)
    assert abs(float(out_keep.float().mean()) - 0.9) < 5e-3
    assert torch.equal(out_keep | (y.cpu().float() == 0), _ln_keep_mask(78, rows, H, th) | (y.cpu().float() == 0))
    assert (out_keep & ~_ln_keep_mask(78, rows, H, th)).sum() == 0          # nothing the documented mask drops survives
    # backward with dy = 1 : dx must vanish exactly where the input mask dropped x
    dy = torch.ones(rows, H).to(BF)
    dx, dres = K.layernorm_bwd(dev(dy), dev(x), dev(r), dev(gam), mean, rstd, drop_in=di, drop_out=do, want_dres=True)
    dropped = ~_ln_keep_mask(77, rows, H, th)
    assert abs(float(dropped.float().mean()) - 0.1) < 5e-3
    # the forward used the same input mask: recompute LN(drop(x) + r) on the host from the documented mask
    z = x.float() * (~dropped).float() * sc + r.float()
    yref = ((z - z.mean(1, keepdim=True)) / torch.sqrt(z.var(1, unbiased=False, keepdim=True) + 1e-12)) * sc
    live = _ln_keep_mask(78, rows, H, th)
    assert rel_l2(y.cpu().float()[live], yref[live]) < 1e-2
    assert float(dx.cpu().float()[dropped].abs().max()) == 0.0
    kept = ~dropped
    assert torch.allclose(dx.cpu().float()[kept], (dres.cpu().float() * sc)[kept], rtol=2e-2, atol=1e-3)


# ----------------------------------------------------------------------------------------- reductions / softmax
def test_colsum(K):
    x = rnd(3001, 2304)
    assert rel_l2(K.colsum(dev(x), 2304), E.colsum(f32(x), 2304)) < 1e-5
    x = rnd(77, 40)
    assert rel_l2(K.colsum(dev(x), 40), E.colsum(f32(x), 40)) < 1e-5


@pytest.mark.parametrize("nq,nk,neg", [(441, 441, -10000.0), (20, 80, -10000.0), (36, 36, float("-inf")), (80, 491, -10000.0)])
def test_softmax_fwd_bwd(K, nq, nk, neg):
    B, H = 3, 12
    ld = (nk + 7) // 8 * 8
    s = torch.randn(B, H, nq, ld) * 2
    kmask = torch.zeros(B, nk)
    kmask[1, nk // 2:] = neg
    bias = torch.randn(B, nq, nk) * 0.5
    p, pd = K.softmax_fwd(dev(s), dev(kmask), dev(bias), B, H, nq, nk, ld)
    rp, _ = E.softmax_fwd(s, kmask, bias, B, H, nq, nk, ld)
    assert rel_l2(p, rp) < 4e-3
    assert float(p.cpu().float()[..., nk:].abs().max() if ld > nk else 0.0) == 0.0
    dp = torch.randn(B, H, nq, ld)
    dbias = torch.zeros(B, nq, nk).cuda()
    ds = K.softmax_bwd(p, dev(dp), B, H, nq, nk, ld, (0, 0, 1.0), 0.125, dbias)
    rdb = torch.zeros(B, nq, nk)
    rds = E.softmax_bwd(f32(p), dp, B, H, nq, nk, ld, (0, 0, 1.0), 0.125, rdb)
    assert rel_l2(ds, rds) < 6e-3 and rel_l2(dbias, rdb) < 1e-4
    # dropout variant: probabilities kept are scaled, the mask replays in backward
    th, sc = K.drop_params(0.1)
    p2, pd2 = K.softmax_fwd(dev(s), dev(kmask), dev(bias), B, H, nq, nk, ld, (9, th, sc))
    assert torch.equal(p2, p)
    kept = pd2.cpu().float() != 0
    big = rp > 1e-3
    assert abs(float(kept[big].float().mean()) - 0.9) < 2e-2


# ----------------------------------------------------------------------------------------- row utilities
def test_embed_and_rows(K):
    V, L, H, B = 500, 80, 768, 4
    word, pos, typ = torch.randn(V, H), torch.randn(512, H), torch.randn(2, H)
    ids = torch.randint(0, V, (B, L))
    ids[0, -5:] = 0
    z = K.embed_sum(dev(ids), dev(word), dev(pos), dev(typ[0].contiguous()))
    assert torch.equal(z.cpu(), E.embed_sum(ids, word, pos, typ[0]))
    dz = torch.randn(B * L, H)
    dw, dp_, dt = torch.zeros(V, H).cuda(), torch.zeros(512, H).cuda(), torch.zeros(2, H).cuda()
    K.embed_scatter_grad(dev(ids), dev(dz), L, 0, dw, dp_, dt[0])
    rw, rp, rt = torch.zeros(V, H), torch.zeros(512, H), torch.zeros(2, H)
    E.embed_scatter_grad(ids, dz, L, 0, rw, rp, rt[0])
    assert rel_l2(dw, rw) < 1e-5 and rel_l2(dp_, rp) < 1e-5 and rel_l2(dt, rt) < 1e-5
    assert float(dw[0].abs().max()) == 0.0
    src = rnd(300, H)
    idx = torch.randint(-1, 300, (1000,))
    assert torch.equal(K.gather_rows(dev(src), dev(idx), H).cpu().float(), E.gather_rows(f32(src), idx, H))
    out = torch.zeros(300, H).cuda()
    g = rnd(1000, H, seed=3)
    K.scatter_add_rows(dev(g), dev(idx), H, out)
    assert rel_l2(out, E.scatter_add_rows(f32(g), idx, H, torch.zeros(300, H))) < 1e-5
    a, b = rnd(640, H), rnd(640, H, seed=4)
    table, vec = torch.randn(3, H), torch.randn(H)
    ti = torch.randint(0, 3, (640,))
    assert rel_l2(K.add_rows(dev(a), dev(b), dev(table), dev(ti), dev(vec)), E.add_rows(f32(a), f32(b), table, ti, vec)) < 4e-3
    assert rel_l2(K.add_act(dev(a), dev(b)), f32(a) + f32(b)) < 4e-3
    seg_off = torch.tensor([0, 0, 36, 38, 38, 39], dtype=torch.int32)
    sidx = torch.randint(0, 300, (39,), dtype=torch.int32)
    w = torch.rand(39)
    o = K.segment_wsum(dev(src), dev(seg_off), dev(sidx), dev(w), 5, H)
    assert rel_l2(o, E.segment_wsum(f32(src), seg_off, sidx, w, 5, H)) < 4e-3
    d32 = torch.zeros(300, H).cuda()
    K.segment_wsum_bwd(o, dev(seg_off), dev(sidx), dev(w), 5, H, d32)
    assert rel_l2(d32, E.segment_wsum_bwd(f32(o), seg_off, sidx, w, 5, H, torch.zeros(300, H))) < 1e-5
    pre = rnd(1000, H, scale=2.0, seed=5)
    assert rel_l2(K.gelu_bwd(dev(g), dev(pre)), E.gelu_bwd(f32(g), f32(pre))) < 5e-3
    assert rel_l2(K.relu_bwd(dev(g), dev(pre)), E.relu_bwd(f32(g), f32(pre))) < 1e-6
    gs = torch.rand(1000)
    x2 = dev(g.clone())
    K.scale_rows_(x2, dev(gs), 1000, H)
    assert rel_l2(x2, f32(g) * gs[:, None]) < 4e-3


def test_softmax_xent(K):
    rows, V = 37, 30522
    ld = (V + 7) // 8 * 8
    logits = torch.randn(rows, ld) * 3
    labels = torch.randint(0, V, (rows,))
    labels[3] = -1
    loss, dl = K.softmax_xent(dev(logits), dev(labels), V, ld)
    rl, rdl = E.softmax_xent(logits, labels, V, ld)
    assert torch.allclose(loss.cpu(), rl, rtol=1e-5, atol=1e-5)
    assert rel_l2(dl, rdl) < 5e-3
    ref = torch.nn.functional.cross_entropy(logits[:, :V], labels.clamp(min=0), reduction="none")
    assert torch.allclose(loss.cpu()[labels >= 0], ref[labels >= 0], rtol=1e-5, atol=1e-5)


# ----------------------------------------------------------------------------------------- GEMM / attention through blocks
def test_linear_helpers(K):
    import bevbert_b200.blocks as Bk
    M, Kd, N = 1000, 768, 3072
    x, w, b = rnd(M, Kd), rnd(N, Kd, scale=0.05, seed=1), torch.randn(N) * 0.1
    y, pre = Bk.lin_fwd(dev(x), dev(w), dev(b), act=K.ACT_GELU, want_pre=True)
    rpre = f32(x) @ f32(w).T + b
    assert rel_l2(pre, rpre) < 4e-3
    assert rel_l2(y, torch.nn.functional.gelu(rpre)) < 4e-3
    dy = rnd(M, N, seed=2)
    dy2, w2 = rnd(M, Kd, seed=6), rnd(Kd, N, scale=0.05, seed=7)      # FFN output dense backward shape
    dh = Bk.lin_bwd_dx(dev(dy2), dev(w2), epi_mul=K.EPI_DGELU, aux_in=pre, add_in=dev(dy))
    assert rel_l2(dh, E.gelu_bwd(f32(dy2) @ f32(w2), f32(pre)) + f32(dy)) < 6e-3
    dxe = Bk.lin_bwd_dx(dev(dy), dev(w))
    assert rel_l2(dxe, f32(dy) @ f32(w)) < 4e-3
    dw = Bk.lin_bwd_dw(dev(dy), dev(x))
    assert rel_l2(dw, f32(dy).T @ f32(x)) < 1e-4
    # tiny / padded shapes used by the heads and position features
    x8, w8 = rnd(50, 16), rnd(768, 16, seed=3)
    y8, _ = Bk.lin_fwd(dev(x8), dev(w8), None)
    assert rel_l2(y8, f32(x8) @ f32(w8).T) < 4e-3
    h, w1 = rnd(64, 768), rnd(8, 768, seed=4)
    o, _ = Bk.lin_fwd(dev(h), dev(w1), None, out_f32=True)
    assert rel_l2(o, f32(h) @ f32(w1).T) < 1e-4


@pytest.mark.parametrize("B,nq,nk,cross", [(3, 441, 441, False), (3, 441, 80, True), (2, 20, 80, True), (5, 36, 36, False),
                                           (2, 80, 461, True)])
def test_attention_core(K, B, nq, nk, cross):
    import bevbert_b200.blocks as Bk
    H, dh = 12, 64
    Hd = H * dh
    if cross:
        q = rnd(B * nq, Hd)
        kv = rnd(B * nk, 2 * Hd, seed=1)
        qd, kvd = dev(q), dev(kv)
        views = (qd, Hd, kvd, 2 * Hd, kvd[:, Hd:], 2 * Hd)
        qf, kf, vf = f32(q), f32(kv)[:, :Hd], f32(kv)[:, Hd:]
    else:
        qkv = rnd(B * nq, 3 * Hd)
        qd = dev(qkv)
        views = (qd, 3 * Hd, qd[:, Hd:], 3 * Hd, qd[:, 2 * Hd:], 3 * Hd)
        qf, kf, vf = f32(qkv)[:, :Hd], f32(qkv)[:, Hd:2 * Hd], f32(qkv)[:, 2 * Hd:]
    kmask = torch.zeros(B, nk)
    kmask[0, nk - nk // 3:] = -10000.0
    bias = torch.randn(B, nq, nk) * 0.3 if not cross else None
    st = {}
    ctx = Bk.attn_core_fwd(st, *views, B, H, nq, nk, dh, dev(kmask), dev(bias), (0, 0, 1.0))

    def heads(t, n):
        return t.reshape(B, n, H, dh).permute(0, 2, 1, 3)
    qh, kh, vh = heads(qf, nq).requires_grad_(True), heads(kf, nk).requires_grad_(True), heads(vf, nk).requires_grad_(True)
    s = qh @ kh.transpose(-1, -2) / math.sqrt(dh) + kmask[:, None, None, :]
    if bias is not None:
        s = s + bias[:, None]
    ref = (torch.softmax(s, -1) @ vh).permute(0, 2, 1, 3).reshape(B * nq, Hd)
    assert rel_l2(ctx, ref) < 8e-3
    dctx = rnd(B * nq, Hd, seed=5)
    ref.backward(f32(dctx))
    if cross:
        dq, dkv = torch.zeros_like(qd), torch.zeros_like(kvd)
        Bk.attn_core_bwd(st, dev(dctx), *views, dq, Hd, dkv, 2 * Hd, dkv[:, Hd:], 2 * Hd)
        gq, gk, gv = f32(dq), f32(dkv)[:, :Hd], f32(dkv)[:, Hd:]
    else:
        dqkv = torch.zeros_like(qd)
        dbias = torch.zeros(B, nq, nk).cuda()
        Bk.attn_core_bwd(st, dev(dctx), *views, dqkv, 3 * Hd, dqkv[:, Hd:], 3 * Hd, dqkv[:, 2 * Hd:], 3 * Hd, dbias)
        gq, gk, gv = f32(dqkv)[:, :Hd], f32(dqkv)[:, Hd:2 * Hd], f32(dqkv)[:, 2 * Hd:]

    def unheads(t, n):
        return t.permute(0, 2, 1, 3).reshape(B * n, Hd)
    assert rel_l2(gq, unheads(qh.grad, nq)) < 1.5e-2
    assert rel_l2(gk, unheads(kh.grad, nk)) < 1.5e-2
    assert rel_l2(gv, unheads(vh.grad, nk)) < 1.5e-2


def test_launch_counter(K):
    K.reset_launch_count()
    K.cast_to_act(torch.zeros(64, device="cuda"))
    assert K.launch_count() == 1


@pytest.mark.parametrize("cross", [False, True])
def test_native_sublayer_executor_equals_python_composition(K, monkeypatch, cross):
    """csrc/layers.cu (one C call per sub-layer) enqueues the same kernels as the Python composition in blocks.py."""
    import bevbert_b200.blocks as Bk
    from bevbert_b200.config import make_config
    torch.manual_seed(0)
    B, nq, nk, Hd, H = 3, 50, 36, 768, 12
    rt = Bk.Runtime()
    x = (torch.randn(B, nq, Hd) * 0.5).to(BF).cuda()
    c = (torch.randn(B, nk, Hd) * 0.5).to(BF).cuda()
    kmask = torch.zeros(B, nk if cross else nq).cuda()
    kmask[1, -7:] = -10000.0
    bias = None if cross else (torch.randn(B, nq, nq) * 0.3).cuda().requires_grad_(True)
    n_par = 10 if cross else 16
    shapes = [(Hd, Hd), (Hd,)] * 4 + [(Hd,), (Hd,)]
    if not cross:
        shapes += [(4 * Hd, Hd), (4 * Hd,), (Hd, 4 * Hd), (Hd,), (Hd,), (Hd,)]
    params = [torch.nn.Parameter((torch.randn(*s_) * 0.03).cuda()) for s_ in shapes]
    assert len(params) == n_par
    dy = (torch.randn(B, nq, Hd) * 0.1).to(BF).cuda()
    outs = {}
    for native in (True, False):
        monkeypatch.setattr(K, "native_sublayers", lambda native=native: native)
        xi = x.clone().requires_grad_(True)
        ci = c.clone().requires_grad_(True)
        for p_ in params:
            p_.grad = None
        if bias is not None:
            bias.grad = None
        rt.begin(True, seed=5)
        if cross:
            y = Bk.run_block(Bk.XAttnImpl(rt, H, 1e-12), [xi, ci, kmask], params)
        else:
            y = Bk.run_block(Bk.BertLayerImpl(rt, H, 1e-12), [xi, kmask, bias], params)
        y.backward(dy)
        outs[native] = (y.detach().clone(), xi.grad.clone(), ci.grad.clone() if cross else bias.grad.clone(),
                        [p_.grad.clone() for p_ in params])
    yn, dxn, d2n, gn = outs[True]
    yp, dxp, d2p, gp = outs[False]
    assert torch.equal(yn, yp) and torch.equal(dxn, dxp)
    assert rel_l2(d2n, d2p) < 1e-5
    for a, b in zip(gn, gp):
        assert rel_l2(a, b) < 1e-4     # split-K / reduction atomics: order-dependent last bits only


@pytest.mark.parametrize("nq,nk", [(441, 441), (50, 36), (20, 80), (130, 500)])
def test_fused_scores_match_unfused_path_and_replay_dropout(K, nq, nk):
    """bb_attn_scores (softmax / softmax-backward on the wgmma accumulators) vs GEMM -> fp32 scores -> softmax kernels:
    same probabilities, identical dropout mask (same counters), same dS and dbias."""
    B, H, dh = 2, 12, 64
    Hd = H * dh
    ldp = (nk + 7) // 8 * 8
    q = rnd(B * nq, Hd, scale=0.6).cuda()
    kv = rnd(B * nk, 2 * Hd, scale=0.6, seed=1).cuda()
    kmask = torch.zeros(B, nk)
    kmask[1, nk // 2:] = -10000.0
    bias = (torch.randn(B, nq, nk) * 0.3)
    th, sc = K.drop_params(0.1)
    drop = (4242, th, sc)
    P, Pd = K.attn_scores_fwd(q, Hd, kv, 2 * Hd, B, H, nq, nk, dh, ldp, dev(kmask), dev(bias), drop)
    S = torch.empty(B, H, nq, ldp, dtype=torch.float32, device="cuda")
    K.gemm(q, kv, S, nq, nk, dh, lda=Hd, ldb=2 * Hd, ldd=ldp, nb1=H, nb2=B, a_s=(dh, nq * Hd), b_s=(dh, nk * 2 * Hd),
           d_s=(nq * ldp, H * nq * ldp), alpha=0.125)
    P2, Pd2 = K.softmax_fwd(S, dev(kmask), dev(bias), B, H, nq, nk, ldp, drop)
    assert rel_l2(P, P2) < 4e-3
    assert float(P.float()[..., nk:].abs().max() if ldp > nk else 0.0) == 0.0
    big = P2.float() > 1e-3
    assert torch.equal((Pd.float() != 0)[big], (Pd2.float() != 0)[big]), "dropout masks must coincide"
    dctx = rnd(B * nq, Hd, seed=2).cuda()
    v = kv[:, Hd:]
    db1 = torch.zeros(B, nq, nk, device="cuda")
    dS = K.attn_scores_bwd(dctx, Hd, v, 2 * Hd, P2, B, H, nq, nk, dh, ldp, drop, db1)
    dP = torch.empty(B, H, nq, ldp, dtype=torch.float32, device="cuda")
    K.gemm(dctx, v, dP, nq, nk, dh, lda=Hd, ldb=2 * Hd, ldd=ldp, nb1=H, nb2=B, a_s=(dh, nq * Hd), b_s=(dh, nk * 2 * Hd),
           d_s=(nq * ldp, H * nq * ldp))
    db2 = torch.zeros(B, nq, nk, device="cuda")
    dS2 = K.softmax_bwd(P2, dP, B, H, nq, nk, ldp, drop, 0.125, db2)
    assert rel_l2(dS, dS2) < 6e-3 and rel_l2(db1, db2) < 1e-4


def _flash_ref(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, bias, keep=None, scale=1.0):
    """fp32 torch attention on the same strided views; -> (o (B,nq,H*64), leaf tensors (qh, kh, vh, bias))."""
    def heads(t, n, ld):
        return torch.as_strided(t, (B, H, n, 64), (n * ld, 64, ld, 1), t.storage_offset()).float().clone().requires_grad_(True)
    qh, kh, vh = heads(q, nq, ldq), heads(k, nk, ldk), heads(v, nk, ldv)
    bl = bias.clone().requires_grad_(True) if bias is not None else None
    s = qh @ kh.transpose(-1, -2) * 0.125
    if kmask is not None:
        s = s + kmask.view(B, 1, 1, nk)
    if bl is not None:
        s = s + bl.view(B, 1, nq, nk)
    p = torch.softmax(s, -1)
    pd = p if keep is None else p * keep * scale
    o = (pd @ vh).permute(0, 2, 1, 3).reshape(B, nq, H * 64)
    return o, p, (qh, kh, vh, bl)


@pytest.mark.parametrize("nq,nk,cross", [(441, 441, False), (80, 80, False), (36, 36, False), (23, 23, False),
                                         (23, 80, True), (441, 80, True), (80, 441, True), (130, 200, True), (64, 128, True)])
def test_flash_attention_matches_fp32_reference(K, nq, nk, cross):
    """bb_flash_fwd / bb_flash_bwd (csrc/attn_flash.cu) vs fp32 torch attention + autograd on the same packed
    Q|K|V views: key masks (-10000 and -inf), additive bias and its gradient, ragged tile tails."""
    B, H, Hd = 2, 12, 768
    if not cross:
        qkv = rnd(B * nq, 3 * Hd, scale=0.8).cuda()
        q, k, v, ldq, ldk, ldv = qkv, qkv[:, Hd:], qkv[:, 2 * Hd:], 3 * Hd, 3 * Hd, 3 * Hd
    else:
        q = rnd(B * nq, Hd, scale=0.8).cuda()
        kv = rnd(B * nk, 2 * Hd, scale=0.8, seed=1).cuda()
        k, v, ldq, ldk, ldv = kv, kv[:, Hd:], Hd, 2 * Hd, 2 * Hd
    kmask = torch.zeros(B, nk)
    kmask[1, nk // 2:] = -10000.0
    kmask[0, -3:] = float("-inf")
    kmask = kmask.cuda()
    bias = (torch.randn(B, nq, nk) * 0.3).cuda()
    dout = rnd(B, nq, Hd, scale=0.5, seed=2).cuda()
    o, lse = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, bias)
    ro, _, (qh, kh, vh, bl) = _flash_ref(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, bias)
    assert rel_l2(o, ro) < 6e-3
    ro.backward(dout.float())
    dbias = torch.zeros(B, nq, nk, device="cuda")
    dq, dk, dv = K.flash_bwd(q, k, v, o, lse, dout, B, H, nq, nk, ldq, ldk, ldv, kmask, bias, dbias=dbias)

    def unheads(t, n):
        return t.permute(0, 2, 1, 3).reshape(B, n, Hd)
    assert rel_l2(dq, unheads(qh.grad, nq)) < 1.2e-2
    assert rel_l2(dk, unheads(kh.grad, nk)) < 1.2e-2
    assert rel_l2(dv, unheads(vh.grad, nk)) < 1.2e-2
    assert rel_l2(dbias, bl.grad) < 1.2e-2
    assert torch.isfinite(o.float()).all() and torch.isfinite(dq.float()).all() and torch.isfinite(dk.float()).all()
    # without mask / bias, written into packed views (the executors' layout)
    o2, lse2 = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv)
    ro2, _, (qh, kh, vh, _) = _flash_ref(q, k, v, B, H, nq, nk, ldq, ldk, ldv, None, None)
    assert rel_l2(o2, ro2) < 6e-3
    ro2.backward(dout.float())
    dpack = torch.zeros(B * nk, 2 * Hd, dtype=BF, device="cuda")
    dqo = torch.zeros(B * nq, Hd, dtype=BF, device="cuda")
    K.flash_bwd(q, k, v, o2, lse2, dout, B, H, nq, nk, ldq, ldk, ldv, out=(dqo, Hd, dpack, 2 * Hd, dpack[:, Hd:], 2 * Hd))
    assert rel_l2(dqo.view(B, nq, Hd), unheads(qh.grad, nq)) < 1.2e-2
    assert rel_l2(dpack[:, :Hd].reshape(B, nk, Hd), unheads(kh.grad, nk)) < 1.2e-2
    assert rel_l2(dpack[:, Hd:].reshape(B, nk, Hd), unheads(vh.grad, nk)) < 1.2e-2


def test_flash_attention_dropout_is_replayed_in_backward(K):
    """With V = identity per head, O is the dropped probability matrix itself: the kept fraction matches p, kept
    entries are P / (1-p), and backward with the same seed equals autograd through that exact mask."""
    B, H, Hd, nq, nk = 2, 12, 768, 100, 64
    q = rnd(B * nq, Hd, scale=0.8).cuda()
    kv = rnd(B * nk, 2 * Hd, scale=0.8, seed=1).cuda()
    eye = torch.eye(64).repeat(B, 1, H).view(B * nk, Hd)            # V_h = I for every head
    kv[:, Hd:] = eye.to(BF).cuda()
    k, v = kv, kv[:, Hd:]
    th, sc = K.drop_params(0.1)
    drop = (977, th, sc)
    o, lse = K.flash_fwd(q, k, v, B, H, nq, nk, Hd, 2 * Hd, 2 * Hd, drop=drop)
    o_nodrop, _ = K.flash_fwd(q, k, v, B, H, nq, nk, Hd, 2 * Hd, 2 * Hd)
    pd = o.float().view(B, nq, H, 64).permute(0, 2, 1, 3)           # (B,H,nq,nk)
    p = o_nodrop.float().view(B, nq, H, 64).permute(0, 2, 1, 3)
    big = p > 1e-3
    keep = (pd != 0)
    frac = 1.0 - keep[big].float().mean().item()
    assert abs(frac - 0.1) < 0.01, frac
    assert rel_l2(pd[big & keep], p[big & keep] * sc) < 1e-2
    o_b, _ = K.flash_fwd(q, k, v, B, H, nq, nk, Hd, 2 * Hd, 2 * Hd, drop=(978, th, sc))
    assert not torch.equal(o, o_b) and torch.equal(o, K.flash_fwd(q, k, v, B, H, nq, nk, Hd, 2 * Hd, 2 * Hd, drop=drop)[0])
    # backward through the same mask (entries with p <= 1e-3 that were dropped are indistinguishable: treat as kept,
    # their contribution is below the tolerance)
    mask = (keep | ~big).float()
    dout = rnd(B, nq, Hd, scale=0.5, seed=2).cuda()
    ro, _, (qh, kh, vh, _) = _flash_ref(q, k, v, B, H, nq, nk, Hd, 2 * Hd, 2 * Hd, None, None, keep=mask, scale=sc)
    ro.backward(dout.float())
    dq, dk, dv = K.flash_bwd(q, k, v, o, lse, dout, B, H, nq, nk, Hd, 2 * Hd, 2 * Hd, drop=drop)

    def unheads(t, n):
        return t.permute(0, 2, 1, 3).reshape(B, n, Hd)
    assert rel_l2(dq, unheads(qh.grad, nq)) < 2e-2
    assert rel_l2(dk, unheads(kh.grad, nk)) < 2e-2
    assert rel_l2(dv, unheads(vh.grad, nk)) < 2e-2


def test_native_pano_layer_equals_python_composition(K, monkeypatch):
    import bevbert_b200.blocks as Bk
    torch.manual_seed(1)
    N, V, Hd, H, Fd = 7, 36, 768, 12, 3072
    rt = Bk.Runtime()
    x = (torch.randn(N, V, Hd) * 0.5).to(BF).cuda()
    kmask = torch.zeros(N, V).cuda()
    kmask[2, -9:] = float("-inf")
    shapes = [(3 * Hd, Hd), (3 * Hd,), (Hd, Hd), (Hd,), (Fd, Hd), (Fd,), (Hd, Fd), (Hd,), (Hd,), (Hd,), (Hd,), (Hd,)]
    params = [torch.nn.Parameter((torch.randn(*s_) * 0.03).cuda()) for s_ in shapes]
    for i in (8, 10):
        params[i].data.add_(1.0)
    dy = (torch.randn(N, V, Hd) * 0.1).to(BF).cuda()
    outs = {}
    for native in (True, False):
        monkeypatch.setattr(K, "native_sublayers", lambda native=native: native)
        xi = x.clone().requires_grad_(True)
        for p_ in params:
            p_.grad = None
        rt.begin(True, seed=11)
        y = Bk.run_block(Bk.PanoLayerImpl(rt, H, 0.1, 0.1), [xi, kmask], params)
        y.backward(dy)
        outs[native] = (y.detach().clone(), xi.grad.clone(), [p_.grad.clone() for p_ in params])
    assert torch.equal(outs[True][0], outs[False][0]) and torch.equal(outs[True][1], outs[False][1])
    for a, b in zip(outs[True][2], outs[False][2]):
        assert rel_l2(a, b) < 1e-4


@pytest.mark.parametrize("nq,nk,cross,mode", [(441, 441, False, 1), (441, 80, True, 1), (80, 441, True, 1), (80, 80, False, 1),
                                              (130, 200, True, 1), (64, 128, True, 1), (100, 512, True, 1),
                                              (512, 441, True, 1), (300, 600, True, 1), (36, 36, False, 2), (23, 80, True, 2),
                                              (5, 7, True, 2)])
def test_tcgen05_attention_forward_matches_fp32_and_mma_sync_paths(K, nq, nk, cross, mode):
    """csrc/attn_tc.cu (wgmma + TMA, S in registers) vs fp32 torch attention and vs the mma.sync kernel (same LSE, same
    dropout decisions): key masks (-10000 / -inf, a fully masked sample), ragged tails, 1..3 super-blocks."""
    B, H, Hd = 3, 12, 768
    if not cross:
        qkv = rnd(B * nq, 3 * Hd, scale=0.8).cuda()
        q, k, v, ldq, ldk, ldv = qkv, qkv[:, Hd:], qkv[:, 2 * Hd:], 3 * Hd, 3 * Hd, 3 * Hd
    else:
        q = rnd(B * nq, Hd, scale=0.8).cuda()
        kv = rnd(B * nk, 2 * Hd, scale=0.8, seed=1).cuda()
        k, v, ldq, ldk, ldv = kv, kv[:, Hd:], Hd, 2 * Hd, 2 * Hd
    kmask = torch.zeros(B, nk)
    kmask[1, nk // 2:] = -10000.0
    kmask[0, -3:] = float("-inf")
    kmask[2, :] = float("-inf")                      # every key masked: zero output rows, lse = +inf
    kmask = kmask.cuda()
    prev = K.set_attn_tc(mode)
    try:
        o, lse = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, None)
        o2, _ = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv)
        th, sc = K.drop_params(0.1)
        od, lsed = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, None, (4242, th, sc))
        K.set_attn_tc(0)
        o_ref, lse_ref = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, None)
        od_ref, _ = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, None, (4242, th, sc))
    finally:
        K.set_attn_tc(prev)
    ro, _, _ = _flash_ref(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, None)     # sample 2 of the reference is NaN
    assert rel_l2(o[:2], ro[:2]) < 6e-3
    assert float(o[2].float().abs().max()) == 0.0 and torch.isinf(lse[2]).all()
    ro2, _, _ = _flash_ref(q, k, v, B, H, nq, nk, ldq, ldk, ldv, None, None)
    assert rel_l2(o2, ro2) < 6e-3
    assert torch.isfinite(o.float()).all()
    fin = torch.isfinite(lse_ref)
    assert torch.equal(fin, torch.isfinite(lse)) and (lse[fin] - lse_ref[fin]).abs().max() < 2e-3
    assert rel_l2(o[:2], o_ref[:2]) < 4e-3 and float(o_ref[2].float().abs().max()) == 0.0
    # identical dropout decisions: the dropped outputs agree as closely as the undropped ones
    assert rel_l2(od[:2], od_ref[:2]) < 6e-3 and (lsed[fin] - lse_ref[fin]).abs().max() < 2e-3


def test_project_bev_reference_entry_point_bit_exact(K):
    """PointCloud.project_bev(pc, mask, feat[, sem]) -- the entry point the agents call (map_nav_src/r2r/agent.py:170) --
    against the oracle's cell_index + scatter_mean: indices, features, semantics and masks bit for bit, including
    boundary points (exact .5 cell edges -> round half to even), y == clip, points outside, and a ragged list input."""
    from bevbert_b200.model.bev_utils import PointCloud
    from oracle import bevbert_ref as R
    import math
    D, res = 21, 0.5
    pcl = PointCloud(math.radians(90), 1, 14, 14, D, res)
    g = torch.Generator().manual_seed(5)
    B, N, C = 3, 1500, 768
    pc = (torch.rand(B, N, 3, generator=g) - 0.5) * 14.0
    pc[0, :6] = torch.tensor([[0.0, 0.0, 0.0], [0.25, 0.5, 0.75], [-0.25, 0.5000001, 1.25], [5.25, 0.0, -5.25],
                              [5.26, 0.0, 0.0], [-5.25, 0.2, 5.24]])
    nod = torch.rand(B, N, generator=g) < 0.05
    feat = torch.randn(B, N, C, generator=g)
    sem = torch.nn.functional.one_hot(torch.randint(0, 40, (B, N), generator=g), 40).double()
    bev, ob, s, sm = pcl.project_bev(pc.cuda(), nod.cuda(), feat.cuda(), sem.cuda())
    idx = R.cell_index(pc, nod, D, res, 0.5)
    for i in range(B):
        rb = R.scatter_mean(feat[i], idx[i], D * D).reshape(D, D, C)
        assert torch.equal(bev[i].cpu(), rb)
        assert torch.equal(ob[i].cpu(), ~((rb.max(-1)[0] == 0) & (rb.min(-1)[0] == 0)))
        rs = R.scatter_mean(sem[i], idx[i], D * D).reshape(D, D, 40)
        rs[rs > 0] = 1
        assert torch.equal(s[i].cpu(), rs) and torch.equal(sm[i].cpu(), rs.sum(2) > 0)
    # agent-side variant: no semantics, ragged per-sample clouds
    lens = [1500, 700, 1]
    bev2, ob2 = pcl.project_bev([pc[i, :n].cuda() for i, n in enumerate(lens)], [nod[i, :n].cuda() for i, n in enumerate(lens)],
                                [feat[i, :n].cuda() for i, n in enumerate(lens)])
    for i, n in enumerate(lens):
        rb = R.scatter_mean(feat[i, :n], idx[i, :n], D * D).reshape(D, D, C)
        assert torch.equal(bev2[i].cpu(), rb)


@pytest.mark.parametrize("nq,nk,cross,mode", [(441, 441, False, 1), (441, 80, True, 1), (80, 441, True, 1), (80, 80, False, 1),
                                              (130, 200, True, 1), (100, 512, True, 1), (512, 441, True, 1),
                                              (36, 36, False, 2), (23, 80, True, 2), (5, 7, True, 2)])
def test_tcgen05_attention_backward_matches_fp32_autograd(K, nq, nk, cross, mode):
    """csrc/attn_tc.cu backward (two wgmma passes: dQ per query tile, dK/dV per key tile) vs fp32 torch autograd with
    key masks (-10000 / -inf) and ragged tails, outputs written into packed views; plus dropout replay against the
    mma.sync backward on the same forward state."""
    B, H, Hd = 2, 12, 768
    if not cross:
        qkv = rnd(B * nq, 3 * Hd, scale=0.8).cuda()
        q, k, v, ldq, ldk, ldv = qkv, qkv[:, Hd:], qkv[:, 2 * Hd:], 3 * Hd, 3 * Hd, 3 * Hd
    else:
        q = rnd(B * nq, Hd, scale=0.8).cuda()
        kv = rnd(B * nk, 2 * Hd, scale=0.8, seed=1).cuda()
        k, v, ldq, ldk, ldv = kv, kv[:, Hd:], Hd, 2 * Hd, 2 * Hd
    kmask = torch.zeros(B, nk)
    kmask[1, nk // 2:] = -10000.0
    kmask[0, -3:] = float("-inf")
    kmask = kmask.cuda()
    dout = rnd(B, nq, Hd, scale=0.5, seed=2).cuda()
    th, sc = K.drop_params(0.1)
    prev = K.set_attn_tc(mode)
    try:
        o, lse = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, None)
        dpack = torch.zeros(B * nk, 2 * Hd, dtype=BF, device="cuda")
        dqo = torch.zeros(B * nq, Hd, dtype=BF, device="cuda")
        K.flash_bwd(q, k, v, o, lse, dout, B, H, nq, nk, ldq, ldk, ldv, kmask, None,
                    out=(dqo, Hd, dpack, 2 * Hd, dpack[:, Hd:], 2 * Hd))
        od, lsed = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, None, (77, th, sc))
        dq_d, dk_d, dv_d = K.flash_bwd(q, k, v, od, lsed, dout, B, H, nq, nk, ldq, ldk, ldv, kmask, None, (77, th, sc))
        K.set_attn_tc(0)
        dq_r, dk_r, dv_r = K.flash_bwd(q, k, v, od, lsed, dout, B, H, nq, nk, ldq, ldk, ldv, kmask, None, (77, th, sc))
    finally:
        K.set_attn_tc(prev)
    ro, _, (qh, kh, vh, _) = _flash_ref(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, None)
    ro.backward(dout.float())

    def unheads(t, n):
        return t.permute(0, 2, 1, 3).reshape(B, n, Hd)
    assert rel_l2(dqo.view(B, nq, Hd), unheads(qh.grad, nq)) < 1.2e-2
    assert rel_l2(dpack[:, :Hd].reshape(B, nk, Hd), unheads(kh.grad, nk)) < 1.2e-2
    assert rel_l2(dpack[:, Hd:].reshape(B, nk, Hd), unheads(vh.grad, nk)) < 1.2e-2
    assert torch.isfinite(dqo.float()).all() and torch.isfinite(dpack.float()).all()
    # same dropout mask in both backward implementations
    assert rel_l2(dq_d, dq_r) < 1.2e-2 and rel_l2(dk_d, dk_r) < 1.2e-2 and rel_l2(dv_d, dv_r) < 1.2e-2
