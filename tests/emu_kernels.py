"""TEST INFRASTRUCTURE ONLY -- torch restatement of every function in bevbert_b200.kernels.

`install()` monkey-patches the kernel wrappers so that the host-side logic (blocks.py forward/backward
composition, index builders, model glue, state-dict surface) can run on CPU in fp32 and be compared with
the oracle.  It is never imported by the product; the product raises without the CUDA library.
Semantics follow the C ABI contracts in include/bevbert_b200.h (strides, majorness, epilogue order).
"""
import math

import torch

F32 = torch.float32
ACT = F32      # storage dtype of activations; set_act_dtype(torch.bfloat16) makes every emulated kernel round its
               # outputs where the CUDA kernels store bf16 (precision studies / tolerance derivations on CPU)


ROUND = None   # study mode (ACT = float64 container): the set of sites whose outputs are rounded to bf16; None = n/a


def set_act_dtype(dt, round_sites=None):
    """dt = torch.bfloat16: every activation is stored (rounded) as bf16, like the CUDA kernels.
    dt = torch.float64 + round_sites: activations live in an exact container and only the named sites round to
    bf16 (scripts/precision_study.py): gemm_in gemm_out gemm_dx ln_y ln_dx ln_dres flash_p flash_ds flash_o
    flash_dqkv other."""
    global ACT, ROUND
    ACT = dt
    ROUND = set(round_sites) if round_sites is not None else None


def _a(t, site="other"):
    if ROUND is not None and ACT == torch.float64:
        return t.to(torch.bfloat16).to(ACT) if site in ROUND else t.to(F32).to(ACT)
    return t.to(ACT)


def _strided(base, shape, strides):
    return torch.as_strided(base, shape, strides, base.storage_offset())


def gemm(a, b, out, M, N, K, lda, ldb, ldd, a_mn=False, b_mn=False, nb1=1, nb2=1, a_s=(0, 0), b_s=(0, 0),
         d_s=(0, 0), alpha=1.0, bias=None, act=0, aux_out=None, aux_in=None, epi_mul=0, add_in=None,
         accumulate=False, split_k=1, drop=(0, 0, 1.0), block_n=0):
    assert drop[1] == 0, "emulation runs with dropout disabled"
    A = _strided(a, (nb2, nb1, M, K), (a_s[1], a_s[0], 1, lda) if a_mn else (a_s[1], a_s[0], lda, 1))
    Bm = _strided(b, (nb2, nb1, N, K), (b_s[1], b_s[0], 1, ldb) if b_mn else (b_s[1], b_s[0], ldb, 1))
    if ROUND is not None and "gemm_in" in ROUND:
        A, Bm = A.to(torch.bfloat16), Bm.to(torch.bfloat16)
    v = torch.matmul(A.to(F32), Bm.to(F32).transpose(-1, -2)) * alpha
    if bias is not None:
        v = v + bias[:N].to(F32)
    dshape, dstr = (nb2, nb1, M, N), (d_s[1], d_s[0], ldd, 1)
    osite = "gemm_dx" if add_in is not None else "gemm_out"
    if aux_out is not None:
        _strided(aux_out, dshape, dstr).copy_(_a(v, osite) if aux_out.dtype == ACT else v)
    if act == 1:
        v = v * 0.5 * (1.0 + torch.erf(v / math.sqrt(2.0)))
    elif act == 2:
        v = torch.relu(v)
    if epi_mul:
        x = _strided(aux_in, dshape, dstr).to(F32)
        if epi_mul == 1:
            v = v * (0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi))
        else:
            v = torch.where(x > 0, v, torch.zeros_like(v))
    if add_in is not None:
        v = v + _strided(add_in, dshape, dstr).to(F32)
    D = _strided(out, dshape, dstr)
    if accumulate or split_k > 1:
        D.add_(v)
    else:
        D.copy_(_a(v, osite) if out.dtype == ACT and out.dtype != F32 else v)
    return out


def act_dtype():
    return ACT


def native_sublayers():
    """The emulation has no C++ executors: blocks.py falls back to its Python composition of the same kernels."""
    return False


FUSED_SCORES_MAX_KEYS = 512


def attn_scores_fwd(q, ldq, k, ldk, B, H, nq, nk, dh, ldp, kmask, bias, drop):
    S = torch.zeros(B, H, nq, ldp, dtype=F32)
    gemm(q, k, S, nq, nk, dh, lda=ldq, ldb=ldk, ldd=ldp, nb1=H, nb2=B, a_s=(dh, nq * ldq), b_s=(dh, nk * ldk),
         d_s=(nq * ldp, H * nq * ldp), alpha=1.0 / math.sqrt(dh))
    return softmax_fwd(S, kmask, bias, B, H, nq, nk, ldp, drop)


def attn_scores_bwd(dctx, ldd, v, ldv, P, B, H, nq, nk, dh, ldp, drop, dbias=None):
    dP = torch.zeros(B, H, nq, ldp, dtype=F32)
    gemm(dctx, v, dP, nq, nk, dh, lda=ldd, ldb=ldv, ldd=ldp, nb1=H, nb2=B, a_s=(dh, nq * ldd), b_s=(dh, nk * ldv),
         d_s=(nq * ldp, H * nq * ldp))
    return softmax_bwd(P, dP, B, H, nq, nk, ldp, drop, 1.0 / math.sqrt(dh), dbias)


FLASH = True


def _heads(t, B, n, H, ld):
    return _strided(t, (B, H, n, 64), (n * ld, 64, ld, 1))


def _flash_probs(q, k, B, H, nq, nk, ldq, ldk, kmask, bias):
    s = torch.matmul(_heads(q, B, nq, H, ldq).to(F32), _heads(k, B, nk, H, ldk).to(F32).transpose(-1, -2)) * 0.125
    if kmask is not None:
        s = s + kmask.view(B, 1, 1, nk)
    if bias is not None:
        s = s + bias.view(B, 1, nq, nk)
    return torch.nan_to_num(torch.softmax(s, -1), nan=0.0)          # rows with every key at -inf give zeros


_LOG2E = torch.tensor(1.4426950408889634, dtype=F32)


def _flash_logits2(qh, kh, alpha, kmask, bias):
    """log2-domain logits in the kernels' fp32 order: fma(S, alpha log2e, kmask log2e) (+ bias log2e); (B,H,nq,nk)"""
    B, H, nq, nk = qh.shape[0], qh.shape[1], qh.shape[2], kh.shape[2]
    a2 = (torch.tensor(alpha, dtype=F32) * _LOG2E).double()
    s = torch.matmul(qh.to(F32), kh.to(F32).transpose(-1, -2)).double() * a2
    if kmask is not None:
        s = s + (kmask.to(F32) * _LOG2E).double().view(B, 1, 1, nk)
    s = s.to(F32).double()
    if bias is not None:
        s = s + bias.to(F32).double().view(B, 1, nq, nk) * _LOG2E.double()
    return s.to(F32)


def flash_core_fwd(q, k, v, o, lse, alpha, kmask=None, bias=None):
    """bb_flash_fwd restated in fp32 on (B, rows, H, 64) views (any strides): ex2 of the log2-domain logits against the
    row maximum, bf16 probabilities into the P V product, one scale by 1/l, LSE = max + log2 l (+inf for rows whose
    keys are all -inf, which give zeros).  Dropout is not emulated."""
    qh, kh, vh = (t.permute(0, 2, 1, 3) for t in (q, k, v))
    s = _flash_logits2(qh, kh, alpha, kmask, bias)
    m = s.amax(-1, keepdim=True)
    e = torch.exp2(s - torch.where(m == float("-inf"), torch.zeros_like(m), m))
    l = e.sum(-1, keepdim=True)
    oh = torch.matmul(e.to(torch.bfloat16).to(F32), vh.to(F32)) * torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    o.copy_(oh.permute(0, 2, 1, 3).to(o.dtype))
    lse.copy_(torch.where(l > 0, m + torch.log2(l), torch.full_like(l, float("inf")))[..., 0])


def flash_core_bwd(q, k, v, o, lse, dout, dq, dk, dv, alpha, kmask=None, bias=None, dbias=None):
    """bb_flash_bwd restated in fp32 on (B, rows, H, 64) views: P = ex2(logit - lse), D = rowsum(dO o O),
    dS = P (dO V^T - D) (dbias += sum over heads), dQ = bf16(alpha dS) K, dK = bf16(alpha dS)^T Q, dV = bf16(P)^T dO."""
    qh, kh, vh, oh, doh = (t.permute(0, 2, 1, 3).to(F32) for t in (q, k, v, o, dout))
    s = _flash_logits2(qh, kh, alpha, kmask, bias)
    p = torch.exp2(s - lse.unsqueeze(-1))
    d = (doh * oh).sum(-1, keepdim=True)
    ds = p * (torch.matmul(doh, vh.transpose(-1, -2)) - d)
    if dbias is not None:
        dbias.add_(ds.sum(1))
    dsb = (ds * alpha).to(torch.bfloat16).to(F32)
    dq.copy_(torch.matmul(dsb, kh).permute(0, 2, 1, 3).to(dq.dtype))
    dk.copy_(torch.matmul(dsb.transpose(-1, -2), qh).permute(0, 2, 1, 3).to(dk.dtype))
    dv.copy_(torch.matmul(p.to(torch.bfloat16).to(F32).transpose(-1, -2), doh).permute(0, 2, 1, 3).to(dv.dtype))


def flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask=None, bias=None, drop=(0, 0, 1.0)):
    assert drop[1] == 0, "emulation runs with dropout disabled"
    p = _flash_probs(q, k, B, H, nq, nk, ldq, ldk, kmask, bias)
    o = torch.matmul(_a(p, 'flash_p').to(F32), _heads(v, B, nk, H, ldv).to(F32))          # (B,H,nq,64); P feeds the MMA as ACT
    qh, kh = _heads(q, B, nq, H, ldq).to(F32), _heads(k, B, nk, H, ldk).to(F32)
    s = _flash_logits2(qh, kh, 0.125, kmask, bias)                                        # the row log-sum-exp, log2 domain
    m = s.amax(-1, keepdim=True)
    l = torch.exp2(s - torch.where(m == float("-inf"), torch.zeros_like(m), m)).sum(-1, keepdim=True)
    lse = torch.where(l > 0, m + torch.log2(l), torch.full_like(l, float("inf")))[..., 0]
    return _a(o.permute(0, 2, 1, 3).reshape(B, nq, H * 64).contiguous(), 'flash_o'), lse


def flash_bwd(q, k, v, o, lse, dout, B, H, nq, nk, ldq, ldk, ldv, kmask=None, bias=None, drop=(0, 0, 1.0), dbias=None,
              out=None):
    assert drop[1] == 0
    Hd = H * 64
    p = _flash_probs(q, k, B, H, nq, nk, ldq, ldk, kmask, bias)
    do = _heads(dout, B, nq, H, Hd).to(F32)
    dp = torch.matmul(do, _heads(v, B, nk, H, ldv).to(F32).transpose(-1, -2))
    dsum = (do * _heads(o, B, nq, H, Hd).to(F32)).sum(-1, keepdim=True)      # rowsum(dO o O), as the kernel does
    ds = p * (dp - dsum)
    if dbias is not None:
        dbias.add_(ds.sum(1))
    ds = _a(ds, 'flash_ds').to(F32)
    if out is None:
        dq, dk, dv = torch.zeros(B, nq, Hd, dtype=ACT), torch.zeros(B, nk, Hd, dtype=ACT), torch.zeros(B, nk, Hd, dtype=ACT)
        lddq = lddk = lddv = Hd
    else:
        dq, lddq, dk, lddk, dv, lddv = out
    _heads(dv, B, nk, H, lddv).copy_(_a(torch.matmul(_a(p, 'flash_p').to(F32).transpose(-1, -2), do), 'flash_dqkv'))
    _heads(dq, B, nq, H, lddq).copy_(_a(torch.matmul(ds, _heads(k, B, nk, H, ldk).to(F32)) * 0.125, 'flash_dqkv'))
    _heads(dk, B, nk, H, lddk).copy_(_a(torch.matmul(ds.transpose(-1, -2), _heads(q, B, nq, H, ldq).to(F32)) * 0.125, 'flash_dqkv'))
    return dq, dk, dv


def gemm_profile(enable):
    pass


def gemm_profile_records():
    return []


def _no_native(*a, **k):
    raise RuntimeError("native sub-layer executors are not emulated")


attn_desc = ffn_desc = pano_desc = sublayer_ws_bytes = sublayer_fwd = sublayer_bwd = _no_native


def drop_params(p):
    return (0, 1.0) if p <= 0 else (min(int(p * 4294967296.0), 4294967295), 1.0 / (1.0 - p))


_count = [0]


def launch_count():
    return _count[0]


def reset_launch_count():
    _count[0] = 0


def bev_lift_index(depths, T_c2w, S_w2c, T_w2c, map_dim, map_res, depth_scale=10.0, fx=7.0, fy=7.0, cx=7.0, cy=7.0,
                   y_clip=0.5, want_pc=False):
    from oracle import bevbert_ref as R
    pc, nod = R.lift_points(depths, T_c2w, S_w2c, T_w2c, depth_scale, fx, fy, cx, cy)
    idx = R.cell_index(pc, nod, map_dim, map_res, y_clip)
    return idx.to(torch.int32), (pc if want_pc else None)


def bev_cell_index(pc, no_depth, map_dim, map_res, y_clip=0.5):
    from oracle import bevbert_ref as R
    nd = no_depth if no_depth is not None else torch.zeros(pc.shape[:-1], dtype=torch.bool)
    return R.cell_index(pc, nd.bool(), map_dim, map_res, y_clip).to(torch.int32)


def bev_scatter_mean(feats, cell_idx, ncell, want_f32=True, want_bf16=True):
    from oracle import bevbert_ref as R
    feats = feats.float()                      # bf16 wire features pool in fp32, like the kernel
    out = torch.stack([R.scatter_mean(feats[i], cell_idx[i].long(), ncell) for i in range(feats.shape[0])], 0)
    ob = ~((out.max(-1)[0] == 0) & (out.min(-1)[0] == 0))
    cnt = torch.stack([torch.bincount(cell_idx[i][cell_idx[i] >= 0].long(), minlength=ncell) for i in range(feats.shape[0])], 0)
    return (out if want_f32 else None), (_a(out) if want_bf16 else None), ob, cnt.to(torch.int32)


def bev_scatter_sem(sems, cell_idx, ncell, num_classes=40):
    from oracle import bevbert_ref as R
    if sems.dtype == torch.uint8:
        sems = torch.nn.functional.one_hot(sems.long(), num_classes).to(torch.float64)
    out = torch.stack([R.scatter_mean(sems[i], cell_idx[i].long(), ncell) for i in range(sems.shape[0])], 0)
    out[out > 0] = 1
    return out, out.sum(2) > 0


def cast_to_act(src, drop=(0, 0, 1.0), out=None):
    assert drop[1] == 0
    if out is None:
        return _a(src.to(F32).clone())
    out.copy_(src)
    return out


def cast_to_f32(src):
    return src.to(F32).clone()


def dropout_act(src, drop, out=None):
    assert drop[1] == 0
    return src.clone()


def layernorm_fwd(x, residual, gamma, beta, eps, drop_in=(0, 0, 1.0), drop_out=(0, 0, 1.0), want_f32=False):
    assert drop_in[1] == 0 and drop_out[1] == 0
    z = x.to(F32) + (residual.to(F32) if residual is not None else 0)
    mean = z.mean(-1)
    var = ((z - mean[:, None]) ** 2).mean(-1)
    rstd = 1.0 / torch.sqrt(var + eps)
    y = (z - mean[:, None]) * rstd[:, None] * gamma + beta
    return _a(y, 'ln_y'), (y.clone() if want_f32 else None), mean, rstd


def layernorm_bwd(dy, x, residual, gamma, mean, rstd, drop_in=(0, 0, 1.0), drop_out=(0, 0, 1.0), want_dx=True,
                  want_dres=False, dx_f32=False, dgamma=None, dbeta=None, dxsum=None):
    z = x.to(F32) + (residual.to(F32) if residual is not None else 0)
    xh = (z - mean[:, None]) * rstd[:, None]
    d = dy.to(F32)
    g = d * gamma
    c1 = g.mean(-1, keepdim=True)
    c2 = (g * xh).mean(-1, keepdim=True)
    dz = rstd[:, None] * (g - c1 - xh * c2)
    if dgamma is not None:
        dgamma.add_((d * xh).sum(0))
    if dbeta is not None:
        dbeta.add_(d.sum(0))
    if dxsum is not None:
        dxsum.add_(dz.sum(0))
    return ((dz.clone() if dx_f32 else _a(dz, 'ln_dx')) if want_dx else None), (_a(dz, 'ln_dres') if want_dres else None)


def colsum(x, N, out=None):
    s = x.reshape(-1, N).to(F32).sum(0)
    if out is None:
        return s
    out.add_(s)
    return out


def softmax_fwd(scores, kmask, bias, nbatch, H, nq, nk, ld, drop=(0, 0, 1.0)):
    assert drop[1] == 0
    s = scores[..., :nk].clone()
    if kmask is not None:
        s = s + kmask.view(nbatch, 1, 1, nk)
    if bias is not None:
        s = s + bias.view(nbatch, 1, nq, nk)
    p = torch.zeros(nbatch, H, nq, ld, dtype=ACT)
    p[..., :nk] = torch.softmax(s, -1)
    return p, p


def softmax_bwd(probs, dprobs, nbatch, H, nq, nk, ld, drop, out_scale, dbias=None):
    p, g = probs[..., :nk].to(F32), dprobs[..., :nk]
    d = p * (g - (p * g).sum(-1, keepdim=True))
    ds = torch.zeros(nbatch, H, nq, ld, dtype=ACT)
    ds[..., :nk] = d * out_scale
    if dbias is not None:
        dbias.add_(d.sum(1))
    return ds


def embed_sum(ids, word, pos, type0):
    L = ids.shape[1]
    return ((word[ids] + pos[:L][None]) + type0[None, None]).reshape(-1, word.shape[1])


def embed_scatter_grad(ids, dz, L, padding_idx, dword, dpos, dtype0):
    flat = ids.reshape(-1)
    keep = flat != padding_idx
    dword.index_add_(0, flat[keep], dz[keep])
    dpos.index_add_(0, torch.arange(flat.numel()) % L, dz)
    dtype0.add_(dz.sum(0))


def gather_rows(src, idx, H):
    out = torch.zeros(idx.numel(), H, dtype=ACT)
    keep = idx >= 0
    out[keep] = src.reshape(-1, H)[idx[keep]].to(ACT)
    return out


def scatter_add_rows(src, idx, H, out_f32):
    keep = idx >= 0
    out_f32.view(-1, H).index_add_(0, idx[keep], src.reshape(-1, H)[keep].to(F32))
    return out_f32


def _act_bwd(dy, aux, mode):
    x = aux.to(F32)
    if mode == 1:
        return _a(dy.to(F32) * (0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)))
    return torch.where(x > 0, dy, torch.zeros_like(dy))


def gelu_bwd(dy, pre):
    return _act_bwd(dy, pre, 1)


def relu_bwd(dy, post):
    return _act_bwd(dy, post, 2)


def add_rows(a, b=None, table=None, idx=None, vec=None):
    out = a.to(F32).clone()
    if b is not None:
        out = out + b.to(F32)
    if table is not None:
        out = out + table[idx]
    if vec is not None:
        out = out + vec[None]
    return _a(out)


def scale_rows_(x, g, rows, ld):
    x.copy_(x.to(F32) * g[:, None])
    return x


def segment_wsum(src, seg_off, idx, w, nseg, H):
    out = torch.zeros(nseg, H, dtype=F32)
    seg = torch.repeat_interleave(torch.arange(nseg), (seg_off[1:] - seg_off[:-1]).long())
    out.index_add_(0, seg, src[idx.long()].to(F32) * w[:, None])
    return _a(out)


def segment_wsum_bwd(dout, seg_off, idx, w, nseg, H, dsrc_f32):
    seg = torch.repeat_interleave(torch.arange(nseg), (seg_off[1:] - seg_off[:-1]).long())
    dsrc_f32.view(-1, H).index_add_(0, idx.long(), dout[seg].to(F32) * w[:, None])
    return dsrc_f32


def add_act(a, b):
    return _a(a.to(F32) + b.to(F32))


def axpy_f32_from_act(x, y):
    y.add_(x.to(F32))
    return y


def softmax_xent(logits, labels, V, ld, want_grad=True):
    x = logits[:, :V]
    lse = torch.logsumexp(x, -1)
    valid = labels >= 0
    lab = labels.clamp(min=0)
    loss = torch.where(valid, lse - x.gather(1, lab[:, None])[:, 0], torch.zeros_like(lse))
    dl = None
    if want_grad:
        dl = torch.zeros(logits.shape[0], ld, dtype=ACT)
        g = torch.softmax(x, -1)
        g[torch.arange(x.shape[0]), lab] -= 1.0
        dl[:, :V] = g * valid[:, None]
    return loss, dl


def _no_mt(*a, **k):
    raise RuntimeError("multi-tensor optimizer kernels take raw device pointers and are not emulated")


MtTable = mt_cast_bf16 = mt_sumsq = adamw_step = _no_mt


def set_attn_tc(mode):
    return 1


def set_precision(fp32):
    return False


def set_side_stream(stream):
    pass


def side_stream():
    return None


def side_join():
    pass


def use_flash():
    return FLASH


_NAMES = ["set_side_stream", "side_stream", "side_join", "set_precision", "use_flash", "bev_cell_index", "set_attn_tc", "MtTable", "mt_cast_bf16", "mt_sumsq", "adamw_step", "flash_fwd", "flash_bwd", "attn_scores_fwd", "attn_scores_bwd", "gemm_profile", "gemm_profile_records", "native_sublayers", "attn_desc", "ffn_desc", "pano_desc", "sublayer_ws_bytes", "sublayer_fwd", "sublayer_bwd", "gemm", "act_dtype", "drop_params", "launch_count", "reset_launch_count", "bev_lift_index",
          "bev_scatter_mean", "bev_scatter_sem", "cast_to_act", "cast_to_f32", "dropout_act", "layernorm_fwd",
          "layernorm_bwd", "colsum", "softmax_fwd", "softmax_bwd", "embed_sum", "embed_scatter_grad", "gather_rows",
          "scatter_add_rows", "gelu_bwd", "relu_bwd", "add_rows", "scale_rows_", "segment_wsum", "segment_wsum_bwd",
          "add_act", "axpy_f32_from_act", "softmax_xent"]


def install(monkeypatch=None):
    """Patches bevbert_b200.kernels in place (use pytest's monkeypatch to undo automatically)."""
    import bevbert_b200.kernels as K
    g = globals()
    missing = [n for n in dir(K) if callable(getattr(K, n)) and not n.startswith("_") and n not in _NAMES
               and getattr(getattr(K, n), "__module__", "") == K.__name__]
    assert not missing, "kernels without an emulation: %s" % missing
    for n in _NAMES:
        if monkeypatch is not None:
            monkeypatch.setattr(K, n, g[n])
        else:
            setattr(K, n, g[n])
