"""Forward / backward of the encoder blocks, composed from the C-ABI kernels (kernels.py).

Each block is a pair of plain functions (`fwd` records what backward needs in a dict, `bwd` replays the
kernels in reverse): no PyTorch arithmetic inside a block, and one autograd node per block (`run_block`)
instead of one per op.  Activations between kernels are bf16, all reductions / statistics fp32, parameter
gradients fp32.

Reference semantics (pretrain_src/model/vilmodel.py): BertSelfAttention :103-141, BertSelfOutput :150-154,
BertIntermediate/BertOutput :177-193, BertOutAttention :325-352, GraphLXRTXLayer :383-421;
transformer.py:170-182 for the pre-norm panorama layer.
"""
import math

import torch

from . import kernels as K

NO_DROP = (0, 0, 1.0)


# =============================================================================================== utilities
class DropState:
    """Per-forward dropout bookkeeping: every dropout site takes a fresh seed so masks are independent,
    and the same (seed, thresh, scale) triple is replayed in backward."""

    def __init__(self, training: bool = False, base_seed: int = 0):
        self.training = training
        self.base = (base_seed & 0xFFFFFFFF) << 24
        self.n = 0

    def make(self, p):
        if not self.training or p <= 0.0:
            return NO_DROP
        self.n += 1
        th, sc = K.drop_params(p)
        # the kernels hash (element index XOR seed): consecutive site numbers would give masks that are XOR-shifted
        # copies of each other, so every site gets a fully mixed 64-bit seed (splitmix64 finaliser)
        return (_mix64(self.base + self.n), th, sc)


def _mix64(x):
    x = (x + 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
    return x ^ (x >> 31)


class Runtime:
    """State shared by all blocks of one model: bf16 weight shadows + the dropout state of the current forward."""

    def __init__(self):
        self.wc = WeightCache()
        self.ds = DropState()
        self.feat_p = 0.0     # feature dropout requested by the pre-training wrapper (pretrain_cmt.py:102-106)
        self.calls = 0
        self._stream_id = None
        self._training = False    # mode of the previous begin(): a train -> eval switch re-casts the shadows

    def begin(self, training: bool, seed=None, tag=None):
        self.calls += 1
        if seed is None:
            if self._stream_id is None:
                # dropout stream = f(torch.manual_seed, data-parallel rank): ranks draw different masks, and
                # re-seeding torch re-seeds the kernels' counter-based RNG
                import os
                self._stream_id = _mix64(torch.initial_seed() ^ (int(os.environ.get("RANK", "0")) << 48)) & 0xFFFFFF
            seed = (self.calls * 7919 + 17) ^ self._stream_id
        self.ds = DropState(training, seed)
        if training:
            ARENA.new_step(tag)
            SCRATCH.new_step(tag)
            if not self.wc.managed:     # a foreign optimizer may have stepped since the last forward (see WeightCache)
                self.wc.refresh_all()
        elif self._training and not self.wc.managed:
            self.wc.refresh_all()       # first eval forward after training: the last optimizer step is not seen yet
        self._training = training
        return self.ds


class _Shadow:
    __slots__ = ("params", "buf", "ver", "epoch", "plain", "vec", "view")

    def __init__(self, params, buf, plain, vec=False, view=None):
        self.params, self.buf, self.plain, self.vec = params, buf, plain, vec
        self.view = view            # copy source of a re-laid-out shadow: view(param) has buf's shape
        self.ver, self.epoch = None, -1


class WeightCache:
    """bf16 shadows of the fp32 parameters (the GEMM operands).  Several parameters can be stacked row-wise into one
    operand (packed Q|K|V), and tiny matrices are zero-padded to the 8-element granularity TMA needs.

    Freshness.  Optimizers update `p.data` in place, which does NOT bump `p._version` (neither torch's fused AdamW nor
    the reference's `p.data.addcdiv_`, pretrain_src/optim/adamw.py:99,110), so versions alone cannot tell when a
    shadow is out of date.  Every shadow therefore also carries the cache epoch at which it was written:
      * `bevbert_b200.optim.AdamW` (`managed`) writes the bf16 shadow of every parameter it updates inside its own
        update kernel and marks stale only the shadows it could not write (zero-padded tiny operands);
      * with any other optimizer `Runtime.begin(training=True)` advances the epoch at the
        start of every training forward, which re-casts all stacked / plain shadows in ONE multi-tensor launch
        (`refresh_all`, ~1.1 GB of traffic = ~0.2 ms per step on this model), and the first `begin(training=False)`
        after a training forward does the same once, so validation after an optimizer step evaluates the new weights;
      * `p._version` is still compared, which covers `load_state_dict` / `copy_` in eval mode.
    An in-place update that bumps no version (`p.data.add_()`, torch's fused AdamW) made while the model stays in eval
    mode is not seen: call `invalidate()` after it."""

    def __init__(self):
        self._c = {}
        self.epoch = 0
        self.managed = False       # True once an optimizer that maintains the shadows itself is attached
        self._table = None         # cached (key-set signature, device table, chunks) of refresh_all

    # ------------------------------------------------------------------ lookups
    def _fresh(self, ent):
        return ent.epoch == self.epoch and ent.ver == tuple(p._version for p in ent.params)

    def get(self, *params, pad_k: int = 0, pad_n: int = 0):
        key = tuple(p.data_ptr() for p in params) + (pad_k, pad_n, K.act_dtype())
        ent = self._c.get(key)
        if ent is not None and self._fresh(ent):
            return ent.buf
        with torch.no_grad():
            plain = not pad_k and not pad_n
            if ent is None:
                n = sum(p.shape[0] for p in params)
                k = params[0].shape[1]
                shape = (n, k) if plain else (max(n, pad_n), max(k, pad_k))
                buf = (torch.empty if plain else torch.zeros)(shape, dtype=K.act_dtype(), device=params[0].device)
                ent = _Shadow(params, buf, plain)
                self._c[key] = ent
                self._table = None
            self._cast(ent)
        return ent.buf

    def f32(self, p):
        """fp32 copy of a 1-D parameter held in another dtype (CLIP's fp16 biases, clip/model.py:372-393), kept fresh
        like the bf16 shadows (in place, so a CUDA graph that reads it sees `refresh_all(padded=True)`); an fp32
        parameter is returned as it is."""
        if p.dtype == torch.float32:
            return p.detach()
        key = ("f32", p.data_ptr())
        ent = self._c.get(key)
        if ent is not None and self._fresh(ent):
            return ent.buf
        if ent is None:
            ent = self._c[key] = _Shadow((p,), torch.empty(p.shape, dtype=torch.float32, device=p.device), False)
        self._cast(ent)
        return ent.buf

    def conv_nhwc(self, p, dtype):
        """A conv weight (Cout, Cin, R, S) as a (Cout, R, S, Cin) `dtype` copy (the depth encoder's fp16 implicit-GEMM
        operand, fp32 in the verification arm), kept fresh like the other shadows (in place, so a CUDA graph that reads
        it sees `refresh_all(padded=True)`)."""
        key = ("nhwc", p.data_ptr(), dtype)
        ent = self._c.get(key)
        if ent is not None and self._fresh(ent):
            return ent.buf
        if ent is None:
            buf = torch.empty(p.shape[0], p.shape[2], p.shape[3], p.shape[1], dtype=dtype, device=p.device)
            ent = self._c[key] = _Shadow((p,), buf, False, view=lambda t: t.permute(0, 2, 3, 1))
        self._cast(ent)
        return ent.buf

    def _cast(self, ent):
        if ent.plain and ent.params[0].dtype == torch.float32:
            r = 0
            for p in ent.params:
                K.cast_to_act(p.detach(), out=ent.buf[r:r + p.shape[0]])
                r += p.shape[0]
        else:  # tiny padded operands, other source dtypes (fp16) and fp32 copies: plain copies, done once per change
            r = 0
            with torch.no_grad():
                for p in ent.params:
                    dst = ent.buf[r:r + p.shape[0]]
                    if p.dim() == 2:
                        dst = dst[:, :p.shape[1]]
                    dst.copy_(p.detach() if ent.view is None else ent.view(p.detach()))
                    r += p.shape[0]
        ent.ver, ent.epoch = tuple(p._version for p in ent.params), self.epoch

    def vec(self, *params):
        """fp32 concatenation of 1-D parameters (packed Q|K|V bias) WITHOUT a copy per step: on first use the
        parameters' storage is re-homed into one contiguous buffer (`p.data` becomes a view of it), so the packed
        vector is always current whatever updates the parameters.  `module.to()` / `.cuda()` replace `p.data` and
        break the aliasing; that is detected and the parameters are re-homed again."""
        if len(params) == 1:
            return params[0].detach()
        key = ("v",) + tuple(id(p) for p in params)
        ent = self._c.get(key)
        if ent is not None:
            off, ok = 0, True
            for p in params:
                ok = ok and p.data_ptr() == ent.buf.data_ptr() + off * 4 and p.device == ent.buf.device
                off += p.numel()
            if ok:
                return ent.buf
        with torch.no_grad():
            buf = torch.cat([p.detach().reshape(-1) for p in params])
            off = 0
            for p in params:
                p.data = buf[off:off + p.numel()].view(p.shape)
                off += p.numel()
            self._c[key] = _Shadow(params, buf, False, vec=True)
        return buf

    # ------------------------------------------------------------------ invalidation / bulk refresh
    def invalidate(self):
        """Every shadow is out of date (parameters changed behind the cache's back)."""
        self.epoch += 1

    def refresh_all(self, padded=False):
        """Advance the epoch and re-cast every plain / stacked bf16 shadow in ONE multi-tensor launch; padded and
        fp32-vector entries (a handful of tiny tensors) are refreshed lazily by `get` / `vec`.  `padded=True`
        re-casts those padded entries (and the fp32 shadows of the verification arm) now as well, in place, for CUDA
        graphs that read them without calling `get`."""
        self.epoch += 1
        if padded:
            for e in self._c.values():
                if not e.vec and (not e.plain or e.buf.dtype != torch.bfloat16 or e.params[0].dtype != torch.float32):
                    self._cast(e)
        ents = [e for e in self._c.values() if e.plain and not e.vec and e.buf.dtype == torch.bfloat16
                and e.params[0].dtype == torch.float32]
        if not ents or not ents[0].buf.is_cuda:
            return
        if self._table is None:
            rows = []
            for e in ents:
                off = 0
                for p in e.params:
                    rows.append((p.data_ptr(), 0, 0, 0, e.buf.data_ptr() + off * 2, p.numel(), 0.0, 0.0))
                    off += p.numel()
            self._table = K.MtTable(rows, ents[0].buf.device)
        K.mt_cast_bf16(self._table)
        for e in ents:
            e.ver, e.epoch = tuple(p._version for p in e.params), self.epoch

    def shadow_slots(self):
        """{param data_ptr: [(bf16 address of the parameter's slot, entry)]} over the plain / stacked shadows: where an
        optimizer kernel can write the bf16 copy of a parameter it has just updated."""
        out = {}
        for e in self._c.values():
            if not e.plain or e.vec or e.buf.dtype != torch.bfloat16:
                continue
            off = 0
            for p in e.params:
                out.setdefault(p.data_ptr(), []).append((e.buf.data_ptr() + off * 2, e))
                off += p.numel()
        return out

    def entries_with(self, param_ptrs):
        """bf16 shadow entries (plain and padded) that hold at least one of the given parameters."""
        return [e for e in self._c.values() if not e.vec and any(p.data_ptr() in param_ptrs for p in e.params)]


class _ZeroArena:
    """fp32 zeros for the gradient buffers of one training step: one allocation and ONE fill per step instead of one
    per backward block (~130 fills per step otherwise).  The size is learned per tag (the task) from the previous
    step with that tag; requests that do not fit fall back to their own torch.zeros, so it is always correct.
    Slices are handed out once and never reused: gradients stay valid for as long as something references them."""

    def __init__(self):
        self.buf = None
        self.off = 0
        self.need = 0
        self.tag = None
        self.est = {}
        self.step_id = 0        # incremented per step: identifies the current arena (id() of a freed tensor is reused)

    def new_step(self, tag=None):
        if self.need:
            self.est[self.tag] = self.need
        self.buf, self.off, self.need, self.tag = None, 0, 0, tag
        self.step_id += 1

    def take(self, device, n):
        n4 = (n + 3) // 4 * 4                       # keep every slice 16-byte aligned
        self.need += n4
        if self.buf is None:
            est = self.est.get(self.tag, 0)
            if est >= n4:
                self.buf, self.off = torch.zeros(est, dtype=torch.float32, device=device), 0
        if self.buf is not None and self.off + n4 <= self.buf.numel() and self.buf.device == device:
            v = self.buf[self.off:self.off + n4]
            self.off += n4
            return v
        return torch.zeros(n4, dtype=torch.float32, device=device)


ARENA = _ZeroArena()      # parameter gradients only: same carve order and sizes on every data-parallel rank
SCRATCH = _ZeroArena()    # everything else that must start at zero (activation gradients, graph-bias gradient)


def zeros_f32(device, *shape, scratch=False):
    """zero-filled fp32 tensor of `shape` from the step arena: ARENA for accumulate-into PARAMETER gradients (so that
    parallel.FlatGradAllReduce can reduce the arena in place), SCRATCH for data-dependent-size buffers."""
    n = 1
    for d in shape:
        n *= d
    return (SCRATCH if scratch else ARENA).take(device, n)[:n].view(shape)


class ZeroPool:
    """The accumulate-into buffers of one backward block (split-K weight gradients, bias / LayerNorm reductions),
    carved from the step arena."""

    def __init__(self, device, *shapes):
        sizes = []
        for sh in shapes:
            n = 1
            for d in sh:
                n *= d
            sizes.append((n + 3) // 4 * 4)
        self.buf = ARENA.take(device, sum(sizes))
        self.out, off = [], 0
        for sh, n in zip(shapes, sizes):
            m = 1
            for d in sh:
                m *= d
            self.out.append(self.buf[off:off + m].view(sh))
            off += n


def _empty(shape, like, dtype=None):
    return torch.empty(shape, dtype=dtype or K.act_dtype(), device=like.device)


def _round8(n):
    return (n + 7) // 8 * 8


# =============================================================================================== linear pieces
def lin_fwd(x, w16, bias, act=K.ACT_NONE, want_pre=False, drop=NO_DROP, add_in=None, out_f32=False):
    """y = epi(x @ W^T + b): x (M,Kd), w16 (N,Kd) -> (y (M,N), pre-activation | None)."""
    M, Kd = x.shape
    N = w16.shape[0]
    out = _empty((M, N), x, torch.float32 if out_f32 else None)
    pre = _empty((M, N), x) if want_pre else None
    K.gemm(x, w16, out, M, N, Kd, lda=Kd, ldb=Kd, ldd=N, bias=bias, act=act, aux_out=pre, drop=drop, add_in=add_in)
    return out, pre


def lin_bwd_dx(dy, w16, epi_mul=K.EPI_NONE, aux_in=None, add_in=None, drop=NO_DROP):
    """dx = epi(dy @ W): dy (M,N), w16 (N,Kd) read MN-major -> (M,Kd)."""
    M, N = dy.shape
    Kd = w16.shape[1]
    out = _empty((M, Kd), dy)
    K.gemm(dy, w16, out, M, Kd, N, lda=N, ldb=Kd, ldd=Kd, b_mn=True, epi_mul=epi_mul, aux_in=aux_in, add_in=add_in,
           drop=drop)
    return out


_SMS = {}


def _num_sms(device) -> int:
    """Streaming multiprocessors of `device`, for host-side tiling heuristics (132, an H100 SXM, off the GPU)."""
    if device.type != "cuda":
        return 132
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _SMS:
        _SMS[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
    return _SMS[idx]


def lin_bwd_dw(dy, x, out=None):
    """dW = dy^T @ x in fp32: dy (M,N), x (M,Kd), both read MN-major, split over the token dimension.
    `out` (zero-filled fp32 (N,Kd)) is accumulated into when given."""
    M, N = dy.shape
    Kd = x.shape[1]
    if out is None:
        out = zeros_f32(dy.device, N, Kd)
    # few output tiles (weights are small) but a long reduction over tokens: prefer 64-wide tiles when 128-wide
    # ones cannot fill half the SMs, then split the token dimension until about one CTA per SM, keeping >= 8 k-blocks
    # per split
    sms = _num_sms(dy.device)
    m_t = (N + 127) // 128
    bn = 128 if m_t * ((Kd + 127) // 128) >= sms // 2 else 64
    if Kd <= bn:
        bn = 0
    tiles = m_t * ((Kd + max(bn, 1) - 1) // max(bn, 1)) if bn else m_t
    kb = (M + 63) // 64
    split = max(1, min((sms + tiles // 2) // max(tiles, 1), kb // 8 if kb >= 8 else 1))
    K.gemm(dy, x, out, N, Kd, M, lda=N, ldb=Kd, ldd=Kd, a_mn=True, b_mn=True, split_k=split, block_n=bn)
    return out


# =============================================================================================== attention core
def attn_core_fwd(st, q, ldq, k, ldk, v, ldv, B, H, nq, nk, dh, kmask, bias, drop):
    """softmax(Q K^T / sqrt(dh) + kmask + bias) V for every (sample, head).  q/k/v are views whose first
    element is (sample 0, row 0, head 0, dim 0); rows are ld* apart, heads dh apart.  -> ctx (B*nq, H*dh)."""
    ldp = _round8(nk)
    if K.use_flash() and dh == 64:
        ctx, lse = K.flash_fwd(q, k, v, B, H, nq, nk, ldq, ldk, ldv, kmask, bias, drop)
        st.update(lse=lse, fctx=ctx, geo=(B, H, nq, nk, dh, ldp), adrop=drop, amask=(kmask, bias))
        return ctx.view(B * nq, H * dh)
    if K._fused_scores(nk, dh):
        P, Pd = K.attn_scores_fwd(q, ldq, k, ldk, B, H, nq, nk, dh, ldp, kmask, bias, drop)
    else:
        S = _empty((B, H, nq, ldp), q, torch.float32)
        K.gemm(q, k, S, nq, nk, dh, lda=ldq, ldb=ldk, ldd=ldp, nb1=H, nb2=B, a_s=(dh, nq * ldq), b_s=(dh, nk * ldk),
               d_s=(nq * ldp, H * nq * ldp), alpha=1.0 / math.sqrt(dh))
        P, Pd = K.softmax_fwd(S, kmask, bias, B, H, nq, nk, ldp, drop)
        del S
    ctx = _empty((B * nq, H * dh), q)
    K.gemm(Pd, v, ctx, nq, dh, nk, lda=ldp, ldb=ldv, ldd=H * dh, b_mn=True, nb1=H, nb2=B,
           a_s=(nq * ldp, H * nq * ldp), b_s=(dh, nk * ldv), d_s=(dh, nq * H * dh))
    st.update(P=P, Pd=Pd, geo=(B, H, nq, nk, dh, ldp), adrop=drop)
    return ctx


def attn_core_bwd(st, dctx, q, ldq, k, ldk, v, ldv, dq, lddq, dk, lddk, dv, lddv, dbias=None):
    """Writes dQ / dK / dV into the given views (same geometry as q/k/v)."""
    B, H, nq, nk, dh, ldp = st["geo"]
    if "lse" in st:
        kmask, bias = st["amask"]
        K.flash_bwd(q, k, v, st["fctx"], st["lse"], dctx, B, H, nq, nk, ldq, ldk, ldv, kmask, bias, st["adrop"], dbias,
                    out=(dq, lddq, dk, lddk, dv, lddv))
        return
    P, Pd, drop = st["P"], st["Pd"], st["adrop"]
    HD = H * dh
    # dV = Pd^T dctx
    K.gemm(Pd, dctx, dv, nk, dh, nq, lda=ldp, ldb=HD, ldd=lddv, a_mn=True, b_mn=True, nb1=H, nb2=B,
           a_s=(nq * ldp, H * nq * ldp), b_s=(dh, nq * HD), d_s=(dh, nk * lddv))
    if K._fused_scores(nk, dh):
        dS = K.attn_scores_bwd(dctx, HD, v, ldv, P, B, H, nq, nk, dh, ldp, drop, dbias)
    else:
        # dPd = dctx V^T
        dP = _empty((B, H, nq, ldp), dctx, torch.float32)
        K.gemm(dctx, v, dP, nq, nk, dh, lda=HD, ldb=ldv, ldd=ldp, nb1=H, nb2=B, a_s=(dh, nq * HD), b_s=(dh, nk * ldv),
               d_s=(nq * ldp, H * nq * ldp))
        dS = K.softmax_bwd(P, dP, B, H, nq, nk, ldp, drop, 1.0 / math.sqrt(dh), dbias)
        del dP
    # dQ = dS K ; dK = dS^T Q
    K.gemm(dS, k, dq, nq, dh, nk, lda=ldp, ldb=ldk, ldd=lddq, b_mn=True, nb1=H, nb2=B, a_s=(nq * ldp, H * nq * ldp),
           b_s=(dh, nk * ldk), d_s=(dh, nq * lddq))
    K.gemm(dS, q, dk, nk, dh, nq, lda=ldp, ldb=ldq, ldd=lddk, a_mn=True, b_mn=True, nb1=H, nb2=B,
           a_s=(nq * ldp, H * nq * ldp), b_s=(dh, nq * ldq), d_s=(dh, nk * lddk))


# =============================================================================================== sub-layers
def attn_sublayer_fwd(st, wc, x, c, kmask, bias, p, H, eps, ds, p_attn, p_hidden):
    """LN(dropout(dense(attention(x, c))) + x); c is None for self-attention (packed QKV projection).
    p = (Wq,bq,Wk,bk,Wv,bv,Wo,bo,gamma,beta); x (B,nq,Hd), c (B,nk,Hd)."""
    B, nq, Hd = x.shape
    dh = Hd // H
    x2 = x.reshape(B * nq, Hd)
    if c is None:
        nk = nq
        wqkv = wc.get(p[0], p[2], p[4])
        bqkv = wc.vec(p[1], p[3], p[5])
        qkv, _ = lin_fwd(x2, wqkv, bqkv)
        q, k, v = qkv, qkv[:, Hd:], qkv[:, 2 * Hd:]
        ldq = ldk = ldv = 3 * Hd
        st.update(qkv=qkv)
    else:
        nk = c.shape[1]
        c2 = c.reshape(B * nk, Hd)
        q, _ = lin_fwd(x2, wc.get(p[0]), p[1].detach())
        wkv = wc.get(p[2], p[4])
        kv, _ = lin_fwd(c2, wkv, wc.vec(p[3], p[5]))
        k, v = kv, kv[:, Hd:]
        ldq, ldk, ldv = Hd, 2 * Hd, 2 * Hd
        st.update(q=q, kv=kv, c2=c2)
    ctx = attn_core_fwd(st, q, ldq, k, ldk, v, ldv, B, H, nq, nk, dh, kmask, bias, ds.make(p_attn))
    ao, _ = lin_fwd(ctx, wc.get(p[6]), p[7].detach())
    hdrop = ds.make(p_hidden)
    y, _, mean, rstd = K.layernorm_fwd(ao, x2, p[8].detach(), p[9].detach(), eps, drop_in=hdrop)
    st.update(x2=x2, ctx=ctx, ao=ao, mean=mean, rstd=rstd, hdrop=hdrop, cross=c is not None, nk=nk)
    return y.view(B, nq, Hd)


def attn_sublayer_bwd(st, wc, dy, p, H, want_dbias=False):
    """-> (dx (B*nq,Hd), dc (B*nk,Hd) | None, param grads (10), dbias | None)."""
    x2, ctx, ao = st["x2"], st["ctx"], st["ao"]
    B, Hh, nq, nk, dh, ldp = st["geo"]
    Hd = x2.shape[1]
    dev = x2.device
    cross = st["cross"]
    shapes = [(Hd,), (Hd,), (Hd, Hd), (Hd,)]                       # dgamma, dbeta, dWo, dbo
    shapes += [(Hd, Hd), (Hd,), (2 * Hd, Hd), (2 * Hd,)] if cross else [(3 * Hd, Hd), (3 * Hd,)]
    z = ZeroPool(dev, *shapes).out
    if want_dbias:
        z = z + [zeros_f32(dev, B, nq, nk, scratch=True)]      # activation gradient: its size depends on the batch
    dg, db, dWo, dbo = z[0], z[1], z[2], z[3]
    dbias = z[-1] if want_dbias else None
    dao, dres = K.layernorm_bwd(dy.reshape(-1, Hd), ao, x2, p[8].detach(), st["mean"], st["rstd"], drop_in=st["hdrop"],
                                want_dres=True, dgamma=dg, dbeta=db, dxsum=dbo)
    lin_bwd_dw(dao, ctx, dWo)
    dctx = lin_bwd_dx(dao, wc.get(p[6]))
    if not cross:
        qkv = st["qkv"]
        dqkv = _empty(qkv.shape, qkv)
        L = 3 * Hd
        attn_core_bwd(st, dctx, qkv, L, qkv[:, Hd:], L, qkv[:, 2 * Hd:], L, dqkv, L, dqkv[:, Hd:], L,
                      dqkv[:, 2 * Hd:], L, dbias)
        dW, dbq = z[4], z[5]
        lin_bwd_dw(dqkv, x2, dW)
        K.colsum(dqkv, L, out=dbq)
        dx = lin_bwd_dx(dqkv, wc.get(p[0], p[2], p[4]), add_in=dres)
        grads = [dW[:Hd], dbq[:Hd], dW[Hd:2 * Hd], dbq[Hd:2 * Hd], dW[2 * Hd:], dbq[2 * Hd:], dWo, dbo, dg, db]
        return dx, None, grads, dbias
    q, kv, c2 = st["q"], st["kv"], st["c2"]
    dq = _empty(q.shape, q)
    dkv = _empty(kv.shape, kv)
    attn_core_bwd(st, dctx, q, Hd, kv, 2 * Hd, kv[:, Hd:], 2 * Hd, dq, Hd, dkv, 2 * Hd, dkv[:, Hd:], 2 * Hd, dbias)
    dWq, dbq, dWkv, dbkv = z[4], z[5], z[6], z[7]
    lin_bwd_dw(dq, x2, dWq)
    K.colsum(dq, Hd, out=dbq)
    dx = lin_bwd_dx(dq, wc.get(p[0]), add_in=dres)
    lin_bwd_dw(dkv, c2, dWkv)
    K.colsum(dkv, 2 * Hd, out=dbkv)
    dc = lin_bwd_dx(dkv, wc.get(p[2], p[4]))
    grads = [dWq, dbq, dWkv[:Hd], dbkv[:Hd], dWkv[Hd:], dbkv[Hd:], dWo, dbo, dg, db]
    return dx, dc, grads, dbias


def ffn_sublayer_fwd(st, wc, a, p, eps, ds, p_hidden):
    """LN(dropout(W2 gelu(W1 a + b1) + b2) + a); p = (W1,b1,W2,b2,gamma,beta); a (M,Hd)."""
    h, hpre = lin_fwd(a, wc.get(p[0]), p[1].detach(), act=K.ACT_GELU, want_pre=True)
    fo, _ = lin_fwd(h, wc.get(p[2]), p[3].detach())
    hdrop = ds.make(p_hidden)
    y, _, mean, rstd = K.layernorm_fwd(fo, a, p[4].detach(), p[5].detach(), eps, drop_in=hdrop)
    st.update(f_a=a, f_h=h, f_hpre=hpre, f_fo=fo, f_mean=mean, f_rstd=rstd, f_drop=hdrop)
    return y


def ffn_sublayer_bwd(st, wc, dy, p):
    a, h, hpre, fo = st["f_a"], st["f_h"], st["f_hpre"], st["f_fo"]
    Hd = a.shape[1]
    Fd = hpre.shape[1]
    dg, db, dW2, db2, dW1, db1 = ZeroPool(a.device, (Hd,), (Hd,), (Hd, Fd), (Hd,), (Fd, Hd), (Fd,)).out
    dfo, dres = K.layernorm_bwd(dy, fo, a, p[4].detach(), st["f_mean"], st["f_rstd"], drop_in=st["f_drop"],
                                want_dres=True, dgamma=dg, dbeta=db, dxsum=db2)
    lin_bwd_dw(dfo, h, dW2)
    dhpre = lin_bwd_dx(dfo, wc.get(p[2]), epi_mul=K.EPI_DGELU, aux_in=hpre)
    lin_bwd_dw(dhpre, a, dW1)
    K.colsum(dhpre, Fd, out=db1)
    da = lin_bwd_dx(dhpre, wc.get(p[0]), add_in=dres)
    return da, [dW1, db1, dW2, db2, dg, db]


# =============================================================================================== native sub-layers
def _ws(nbytes, dev):
    return torch.empty(nbytes, dtype=torch.uint8, device=dev)


def attn_native_fwd(st, rt, x, c, kmask, bias, p, H, eps, p_attn, p_hidden):
    """Same math as attn_sublayer_fwd, enqueued by one C call (csrc/layers.cu bb_attn_fwd)."""
    wc, ds = rt.wc, rt.ds
    B, nq, Hd = x.shape
    dev = x.device
    x2 = x.reshape(B * nq, Hd)
    if not x2.is_contiguous():
        x2 = x2.contiguous()
    d = K.attn_desc()
    d.B, d.nq, d.Hd, d.heads, d.eps = B, nq, Hd, H, eps
    keep = [x2, kmask, bias]
    d.x = x2.data_ptr()
    if c is None:
        d.nk, d.cross = nq, 0
        wq, bq = wc.get(p[0], p[2], p[4]), wc.vec(p[1], p[3], p[5])
        d.w_qkv, d.b_qkv = wq.data_ptr(), bq.data_ptr()
        keep += [wq, bq]
    else:
        nk = c.shape[1]
        c2 = c.reshape(B * nk, Hd)
        if not c2.is_contiguous():
            c2 = c2.contiguous()
        d.nk, d.cross, d.c = nk, 1, c2.data_ptr()
        wq, bq, wkv, bkv = wc.get(p[0]), p[1].detach(), wc.get(p[2], p[4]), wc.vec(p[3], p[5])
        d.w_qkv, d.b_qkv, d.w_kv, d.b_kv = wq.data_ptr(), bq.data_ptr(), wkv.data_ptr(), bkv.data_ptr()
        keep += [c2, wq, bq, wkv, bkv]
    wo = wc.get(p[6])
    d.w_o, d.b_o, d.gamma, d.beta = wo.data_ptr(), p[7].data_ptr(), p[8].data_ptr(), p[9].data_ptr()
    keep.append(wo)
    d.kmask = kmask.data_ptr() if kmask is not None else None
    d.bias = bias.data_ptr() if bias is not None else None
    d.seed_attn, d.th_attn, d.sc_attn = ds.make(p_attn)
    d.seed_h, d.th_h, d.sc_h = ds.make(p_hidden)
    fb, bb_ = K.sublayer_ws_bytes(d)
    ws = _ws(fb, dev)
    y = torch.empty(B * nq, Hd, dtype=K.act_dtype(), device=dev)
    d.ws, d.y = ws.data_ptr(), y.data_ptr()
    K.sublayer_fwd(d)
    st.update(a_d=d, a_keep=keep, a_ws=ws, a_bwd=bb_, a_geo=(B, nq, d.nk, Hd), a_cross=c is not None)
    return y.view(B, nq, Hd)


def attn_native_bwd(st, dy, want_dbias=False):
    d = st["a_d"]
    B, nq, nk, Hd = st["a_geo"]
    cross = st["a_cross"]
    dev = dy.device
    dy = dy.reshape(-1, Hd)
    if not dy.is_contiguous():
        dy = dy.contiguous()
    shapes = [(Hd,), (Hd,), (Hd, Hd), (Hd,)]
    shapes += [(Hd, Hd), (Hd,), (2 * Hd, Hd), (2 * Hd,)] if cross else [(3 * Hd, Hd), (3 * Hd,)]
    z = ZeroPool(dev, *shapes).out
    if want_dbias:
        z = z + [zeros_f32(dev, B, nq, nk, scratch=True)]      # activation gradient: its size depends on the batch
    gws = _ws(st["a_bwd"], dev)
    st["a_gws"] = (gws, dy)      # side-stream mode: read by kernels that may still be in flight after this call returns
    dx = torch.empty(B * nq, Hd, dtype=K.act_dtype(), device=dev)
    dc = torch.empty(B * nk, Hd, dtype=K.act_dtype(), device=dev) if cross else None
    d.dy, d.gws, d.dx = dy.data_ptr(), gws.data_ptr(), dx.data_ptr()
    d.dc = dc.data_ptr() if cross else None
    d.dgamma, d.dbeta, d.dw_o, d.db_o = z[0].data_ptr(), z[1].data_ptr(), z[2].data_ptr(), z[3].data_ptr()
    d.dw_qkv, d.db_qkv = z[4].data_ptr(), z[5].data_ptr()
    if cross:
        d.dw_kv, d.db_kv = z[6].data_ptr(), z[7].data_ptr()
    d.want_dbias = int(want_dbias)
    d.dbias = z[-1].data_ptr() if want_dbias else None
    K.sublayer_bwd(d)
    dbias = z[-1] if want_dbias else None
    if not cross:
        dW, dbq = z[4], z[5]
        grads = [dW[:Hd], dbq[:Hd], dW[Hd:2 * Hd], dbq[Hd:2 * Hd], dW[2 * Hd:], dbq[2 * Hd:], z[2], z[3], z[0], z[1]]
    else:
        dWkv, dbkv = z[6], z[7]
        grads = [z[4], z[5], dWkv[:Hd], dbkv[:Hd], dWkv[Hd:], dbkv[Hd:], z[2], z[3], z[0], z[1]]
    return dx, dc, grads, dbias


def ffn_native_fwd(st, rt, a, p, eps, p_hidden):
    wc = rt.wc
    M, Hd = a.shape
    dev = a.device
    if not a.is_contiguous():
        a = a.contiguous()
    w1, w2 = wc.get(p[0]), wc.get(p[2])
    d = K.ffn_desc()
    d.M, d.Hd, d.Fd, d.eps = M, Hd, w1.shape[0], eps
    d.a, d.w1, d.w2 = a.data_ptr(), w1.data_ptr(), w2.data_ptr()
    d.b1, d.b2, d.gamma, d.beta = p[1].data_ptr(), p[3].data_ptr(), p[4].data_ptr(), p[5].data_ptr()
    d.seed_h, d.th_h, d.sc_h = rt.ds.make(p_hidden)
    fb, bb_ = K.sublayer_ws_bytes(d)
    ws = _ws(fb, dev)
    y = torch.empty(M, Hd, dtype=K.act_dtype(), device=dev)
    d.ws, d.y = ws.data_ptr(), y.data_ptr()
    K.sublayer_fwd(d)
    st.update(f_d=d, f_keep=[a, w1, w2], f_ws=ws, f_bwd=bb_, f_dims=(M, Hd, w1.shape[0]))
    return y


def ffn_native_bwd(st, dy):
    d = st["f_d"]
    M, Hd, Fd = st["f_dims"]
    dev = dy.device
    if not dy.is_contiguous():
        dy = dy.contiguous()
    dg, db, dW2, db2, dW1, db1 = ZeroPool(dev, (Hd,), (Hd,), (Hd, Fd), (Hd,), (Fd, Hd), (Fd,)).out
    gws = _ws(st["f_bwd"], dev)
    st["f_gws"] = (gws, dy)
    da = torch.empty(M, Hd, dtype=K.act_dtype(), device=dev)
    d.dy, d.gws, d.da = dy.data_ptr(), gws.data_ptr(), da.data_ptr()
    d.dgamma, d.dbeta, d.dw2, d.db2, d.dw1, d.db1 = (dg.data_ptr(), db.data_ptr(), dW2.data_ptr(), db2.data_ptr(),
                                                     dW1.data_ptr(), db1.data_ptr())
    K.sublayer_bwd(d)
    return da, [dW1, db1, dW2, db2, dg, db]


# =============================================================================================== block impls
class BertLayerImpl:
    """BertLayer (vilmodel.py:195-208): self-attention sub-layer + FFN sub-layer, post-LN.
    inputs (x (B,n,Hd), kmask (B,n) f32 | None, bias (B,n,n) f32 | None); 16 params."""

    def __init__(self, rt, heads, eps, p_attn=0.0, p_hidden=0.0):
        self.rt, self.wc, self.H, self.eps, self.pa, self.ph = rt, rt.wc, heads, eps, p_attn, p_hidden

    def fwd(self, st, inputs, p):
        x, kmask, bias = inputs
        ds = self.rt.ds
        st["shape"] = x.shape
        st["bias_grad"] = bias is not None and bias.requires_grad
        st["native"] = K.native_sublayers()
        if st["native"]:
            a = attn_native_fwd(st, self.rt, x, None, kmask, bias, p[:10], self.H, self.eps, self.pa, self.ph)
            y = ffn_native_fwd(st, self.rt, a.reshape(-1, a.shape[-1]), p[10:], self.eps, self.ph)
        else:
            a = attn_sublayer_fwd(st, self.wc, x, None, kmask, bias, p[:10], self.H, self.eps, ds, self.pa, self.ph)
            y = ffn_sublayer_fwd(st, self.wc, a.reshape(-1, a.shape[-1]), p[10:], self.eps, ds, self.ph)
        return y.view(x.shape)

    def bwd(self, st, gouts, p):
        dy = gouts[0].reshape(-1, st["shape"][-1])
        if st["native"]:
            da, g_ffn = ffn_native_bwd(st, dy)
            dx, _, g_att, dbias = attn_native_bwd(st, da, want_dbias=st["bias_grad"])
        else:
            da, g_ffn = ffn_sublayer_bwd(st, self.wc, dy, p[10:])
            dx, _, g_att, dbias = attn_sublayer_bwd(st, self.wc, da, p[:10], self.H, want_dbias=st["bias_grad"])
        return [dx.view(st["shape"]), None, dbias], g_att + g_ffn


class XAttnImpl:
    """BertXAttention (vilmodel.py:354-363): cross-attention + output dense + LN.
    inputs (x (B,nq,Hd), c (B,nk,Hd), cmask (B,nk) f32 | None); 10 params."""

    def __init__(self, rt, heads, eps, p_attn=0.0, p_hidden=0.0):
        self.rt, self.wc, self.H, self.eps, self.pa, self.ph = rt, rt.wc, heads, eps, p_attn, p_hidden

    def fwd(self, st, inputs, p):
        x, c, cmask = inputs
        st["xs"], st["cs"] = x.shape, c.shape
        st["native"] = K.native_sublayers()
        if st["native"]:
            return attn_native_fwd(st, self.rt, x, c, cmask, None, p, self.H, self.eps, self.pa, self.ph)
        return attn_sublayer_fwd(st, self.wc, x, c, cmask, None, p, self.H, self.eps, self.rt.ds, self.pa, self.ph)

    def bwd(self, st, gouts, p):
        dy = gouts[0].reshape(-1, st["xs"][-1])
        if st["native"]:
            dx, dc, grads, _ = attn_native_bwd(st, dy)
        else:
            dx, dc, grads, _ = attn_sublayer_bwd(st, self.wc, dy, p, self.H)
        return [dx.view(st["xs"]), dc.view(st["cs"]), None], grads


class PanoLayerImpl:
    """Pre-norm TransformerEncoderLayer (transformer.py:170-182) with nn.MultiheadAttention's packed in_proj.
    inputs (x (N,V,Hd), kmask (N,V) f32 with -inf on padding, or None); params (in_w,in_b,out_w,out_b,l1w,l1b,l2w,l2b,
    n1w,n1b,n2w,n2b).  `act` is the FFN activation: K.ACT_GELU (the panorama encoder), or K.ACT_QGELU for CLIP's
    ResidualAttentionBlock (clip/model.py:167-188), which runs forward only: the composed launches without the
    pre-activation copy, and no backward."""

    def __init__(self, rt, heads, p_attn=0.0, p_hidden=0.0, act=K.ACT_GELU):
        self.rt, self.wc, self.H, self.pa, self.ph, self.act = rt, rt.wc, heads, p_attn, p_hidden, act

    def _native_fwd(self, st, x, kmask, p):
        wc, ds = self.wc, self.rt.ds
        N, V, Hd = x.shape
        dev = x.device
        x2 = x.reshape(N * V, Hd)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        w_in, w_out, w1, w2 = wc.get(p[0]), wc.get(p[2]), wc.get(p[4]), wc.get(p[6])
        d = K.pano_desc()
        d.N, d.V, d.Hd, d.heads, d.Fd = N, V, Hd, self.H, w1.shape[0]
        d.x, d.kmask = x2.data_ptr(), (kmask.data_ptr() if kmask is not None else None)
        d.w_in, d.w_out, d.w1, d.w2 = w_in.data_ptr(), w_out.data_ptr(), w1.data_ptr(), w2.data_ptr()
        d.b_in, d.b_out, d.b1, d.b2 = p[1].data_ptr(), p[3].data_ptr(), p[5].data_ptr(), p[7].data_ptr()
        d.g1, d.be1, d.g2, d.be2 = p[8].data_ptr(), p[9].data_ptr(), p[10].data_ptr(), p[11].data_ptr()
        d.seed_attn, d.th_attn, d.sc_attn = ds.make(self.pa)
        s1, s2, s3 = ds.make(self.ph), ds.make(self.ph), ds.make(self.ph)
        d.seed1, d.seed2, d.seed3, d.th_h, d.sc_h = s1[0], s2[0], s3[0], s1[1], s1[2]
        fb, bb_ = K.sublayer_ws_bytes(d)
        ws = _ws(fb, dev)
        y = torch.empty(N * V, Hd, dtype=K.act_dtype(), device=dev)
        d.ws, d.y = ws.data_ptr(), y.data_ptr()
        K.sublayer_fwd(d)
        st.update(p_d=d, p_keep=[x2, kmask, w_in, w_out, w1, w2, ws], p_bwd=bb_, shape=x.shape, Fd=w1.shape[0])
        return y.view(x.shape)

    def _native_bwd(self, st, dy):
        d = st["p_d"]
        N, V, Hd = st["shape"]
        Fd = st["Fd"]
        dev = dy.device
        dy = dy.reshape(-1, Hd)
        if not dy.is_contiguous():
            dy = dy.contiguous()
        z = ZeroPool(dev, (3 * Hd, Hd), (3 * Hd,), (Hd, Hd), (Hd,), (Fd, Hd), (Fd,), (Hd, Fd), (Hd,), (Hd,), (Hd,), (Hd,),
                     (Hd,)).out
        gws = _ws(st["p_bwd"], dev)
        st["p_gws"] = (gws, dy)
        dx = torch.empty(N * V, Hd, dtype=K.act_dtype(), device=dev)
        d.dy, d.gws, d.dx = dy.data_ptr(), gws.data_ptr(), dx.data_ptr()
        (d.dw_in, d.db_in, d.dw_out, d.db_out, d.dw1, d.db1, d.dw2, d.db2, d.dg1, d.dbe1, d.dg2, d.dbe2) = \
            [t.data_ptr() for t in z]
        K.sublayer_bwd(d)
        return [dx.view(st["shape"]), None], list(z)

    def fwd(self, st, inputs, p):
        x, kmask = inputs
        st["native"] = self.act == K.ACT_GELU and K.native_sublayers()
        if st["native"]:
            return self._native_fwd(st, x, kmask, p)
        N, V, Hd = x.shape
        dh = Hd // self.H
        x2 = x.reshape(N * V, Hd)
        h1, _, m1, r1 = K.layernorm_fwd(x2, None, p[8].detach(), p[9].detach(), 1e-5)
        qkv, _ = lin_fwd(h1, self.wc.get(p[0]), p[1].detach())
        L = 3 * Hd
        ctx = attn_core_fwd(st, qkv, L, qkv[:, Hd:], L, qkv[:, 2 * Hd:], L, N, self.H, V, V, dh, kmask, None,
                            self.rt.ds.make(self.pa))
        d1 = self.rt.ds.make(self.ph)
        x1, _ = lin_fwd(ctx, self.wc.get(p[2]), p[3].detach(), drop=d1, add_in=x2)
        h2, _, m2, r2 = K.layernorm_fwd(x1, None, p[10].detach(), p[11].detach(), 1e-5)
        d2 = self.rt.ds.make(self.ph)
        gelu = self.act == K.ACT_GELU
        f, fpre = lin_fwd(h2, self.wc.get(p[4]), p[5].detach(), act=self.act, want_pre=gelu, drop=d2)
        d3 = self.rt.ds.make(self.ph)
        y, _ = lin_fwd(f, self.wc.get(p[6]), p[7].detach(), drop=d3, add_in=x1)
        st.update(x2=x2, h1=h1, m1=m1, r1=r1, qkv=qkv, ctx=ctx, x1=x1, h2=h2, m2=m2, r2=r2, f=f, fpre=fpre, d1=d1,
                  d2=d2, d3=d3, shape=x.shape)
        return y.view(x.shape)

    def bwd(self, st, gouts, p):
        if st["native"]:
            return self._native_bwd(st, gouts[0])
        if self.act != K.ACT_GELU:
            raise NotImplementedError("PanoLayerImpl runs backward with GELU only")
        Hd = st["shape"][-1]
        dev = st["x2"].device
        dy = gouts[0].reshape(-1, Hd).contiguous()
        z = lambda n: zeros_f32(dev, n)
        # y = x1 + drop3(f W2^T + b2)
        dy3 = K.dropout_act(dy, st["d3"]) if st["d3"][1] else dy
        dW2 = lin_bwd_dw(dy3, st["f"])
        db2 = K.colsum(dy3, Hd)
        dfpre = lin_bwd_dx(dy3, self.wc.get(p[6]), epi_mul=K.EPI_DGELU, aux_in=st["fpre"], drop=st["d2"])
        dW1 = lin_bwd_dw(dfpre, st["h2"])
        db1 = K.colsum(dfpre, dfpre.shape[1])
        dh2 = lin_bwd_dx(dfpre, self.wc.get(p[4]))
        dg2, dbt2 = z(Hd), z(Hd)
        dx1_ln, _ = K.layernorm_bwd(dh2, st["x1"], None, p[10].detach(), st["m2"], st["r2"], dgamma=dg2, dbeta=dbt2)
        dx1 = K.add_act(dx1_ln, dy)
        # x1 = x + drop1(ctx Wo^T + bo)
        d1g = K.dropout_act(dx1, st["d1"]) if st["d1"][1] else dx1
        dWo = lin_bwd_dw(d1g, st["ctx"])
        dbo = K.colsum(d1g, Hd)
        dctx = lin_bwd_dx(d1g, self.wc.get(p[2]))
        qkv = st["qkv"]
        L = 3 * Hd
        dqkv = _empty(qkv.shape, qkv)
        attn_core_bwd(st, dctx, qkv, L, qkv[:, Hd:], L, qkv[:, 2 * Hd:], L, dqkv, L, dqkv[:, Hd:], L, dqkv[:, 2 * Hd:], L)
        dWin = lin_bwd_dw(dqkv, st["h1"])
        dbin = K.colsum(dqkv, L)
        dh1 = lin_bwd_dx(dqkv, self.wc.get(p[0]))
        dg1, dbt1 = z(Hd), z(Hd)
        dx_ln, _ = K.layernorm_bwd(dh1, st["x2"], None, p[8].detach(), st["m1"], st["r1"], dgamma=dg1, dbeta=dbt1)
        dx = K.add_act(dx_ln, dx1)
        return [dx.view(st["shape"]), None], [dWin, dbin, dWo, dbo, dW1, db1, dW2, db2, dg1, dbt1, dg2, dbt2]


class LinearLNImpl:
    """LN(x W^T + b), eps 1e-12 (vilmodel.py:501,522,541-544,576-583,620-623).  x is fp32 features (cast to the
    activation dtype, with the feature dropout of pretrain_cmt.py:102-106 when `p_in` > 0) or an activation.
    Inner sizes that are not multiples of 8 are zero-padded.  inputs (x (rows,Kd),); params (W,b,gamma,beta)."""

    def __init__(self, rt, eps=1e-12, p_in=0.0):
        self.rt, self.wc, self.eps, self.p_in = rt, rt.wc, eps, p_in

    def fwd(self, st, inputs, p):
        x = inputs[0]
        shape = x.shape
        Kd = shape[-1]
        x2 = x.reshape(-1, Kd)
        Kp = _round8(Kd)
        if Kp != Kd:
            xa = torch.zeros(x2.shape[0], Kp, dtype=K.act_dtype(), device=x.device)
            xa[:, :Kd] = x2
            w = self.wc.get(p[0], pad_k=Kp)
        else:
            if x2.dtype == torch.float32:
                xa = K.cast_to_act(x2, self.rt.ds.make(self.p_in))
            elif self.p_in > 0.0 and self.rt.ds.training and not x.requires_grad:
                xa = K.dropout_act(x2.contiguous(), self.rt.ds.make(self.p_in))   # 16-bit wire features: dropout only
            else:
                xa = x2.contiguous()
            w = self.wc.get(p[0])
        y, _ = lin_fwd(xa, w, p[1].detach())
        o, _, mean, rstd = K.layernorm_fwd(y, None, p[2].detach(), p[3].detach(), self.eps)
        st.update(xa=xa, y=y, mean=mean, rstd=rstd, Kd=Kd, shape=shape, w=w, xgrad=x.requires_grad)
        return o.view(shape[:-1] + (o.shape[-1],))

    def bwd(self, st, gouts, p):
        y = st["y"]
        Hd = y.shape[1]
        dg = zeros_f32(y.device, Hd)
        db = zeros_f32(y.device, Hd)
        dyl, _ = K.layernorm_bwd(gouts[0].reshape(-1, Hd).contiguous(), y, None, p[2].detach(), st["mean"], st["rstd"],
                                 dgamma=dg, dbeta=db)
        dW = lin_bwd_dw(dyl, st["xa"])[:, :st["Kd"]]
        dbias = K.colsum(dyl, Hd)
        dx = None
        if st["xgrad"]:
            dx = lin_bwd_dx(dyl, st["w"])[:, :st["Kd"]].reshape(st["shape"])
        return [dx], [dW, dbias, dg, db]


class LayerNormImpl:
    """y = dropout_out(LN(x + residual)); inputs (x, residual | None); params (gamma, beta)."""

    def __init__(self, rt, eps, p_out=0.0):
        self.rt, self.eps, self.p_out = rt, eps, p_out

    def fwd(self, st, inputs, p):
        x, res = inputs
        Hd = x.shape[-1]
        x2 = x.reshape(-1, Hd)
        r2 = res.reshape(-1, Hd) if res is not None else None
        do = self.rt.ds.make(self.p_out)
        y, _, mean, rstd = K.layernorm_fwd(x2, r2, p[0].detach(), p[1].detach(), self.eps, drop_out=do)
        st.update(x2=x2, r2=r2, mean=mean, rstd=rstd, do=do, shape=x.shape)
        return y.view(x.shape)

    def bwd(self, st, gouts, p):
        Hd = st["shape"][-1]
        dev = st["x2"].device
        dg = zeros_f32(dev, Hd)
        db = zeros_f32(dev, Hd)
        dx, dres = K.layernorm_bwd(gouts[0].reshape(-1, Hd).contiguous(), st["x2"], st["r2"], p[0].detach(), st["mean"],
                                   st["rstd"], drop_out=st["do"], want_dres=st["r2"] is not None, dgamma=dg, dbeta=db)
        return [dx.view(st["shape"]), dres.view(st["shape"]) if dres is not None else None], [dg, db]


class TextEmbedImpl:
    """BertEmbeddings (vilmodel.py:62-77): dropout(LN(word[ids] + pos[arange] + type[0])).
    inputs (txt_ids int64 (B,L),); params (word, pos, type, gamma, beta)."""

    def __init__(self, rt, eps, p_out=0.0):
        self.rt, self.eps, self.p_out = rt, eps, p_out

    def fwd(self, st, inputs, p):
        ids = inputs[0]
        B, L = ids.shape
        z = K.embed_sum(ids, p[0].detach(), p[1].detach(), p[2].detach()[0].contiguous())
        do = self.rt.ds.make(self.p_out)
        y, _, mean, rstd = K.layernorm_fwd(z, None, p[3].detach(), p[4].detach(), self.eps, drop_out=do)
        st.update(ids=ids, z=z, mean=mean, rstd=rstd, do=do, L=L)
        return y.view(B, L, -1)

    def bwd(self, st, gouts, p):
        z = st["z"]
        Hd = z.shape[1]
        dev = z.device
        dg = zeros_f32(dev, Hd)
        db = zeros_f32(dev, Hd)
        dz, _ = K.layernorm_bwd(gouts[0].reshape(-1, Hd).contiguous(), z, None, p[3].detach(), st["mean"], st["rstd"],
                                drop_out=st["do"], dx_f32=True, dgamma=dg, dbeta=db)
        dword = zeros_f32(p[0].device, *p[0].shape)
        dpos = zeros_f32(p[1].device, *p[1].shape)
        dtype_ = zeros_f32(p[2].device, *p[2].shape)
        K.embed_scatter_grad(st["ids"], dz, st["L"], 0, dword, dpos, dtype_[0])
        return [None], [dword, dpos, dtype_, dg, db]


class AddRowsImpl:
    """out = a (+ b) (+ table[idx]) (+ vec_src[vec_row]); a,b activations (rows,Hd); table / vec_src fp32 params.
    inputs (a, b | None, idx | None); params (table | None, vec_src | None)."""

    def __init__(self, vec_row=0):
        self.vec_row = vec_row

    def fwd(self, st, inputs, p):
        a, b, idx = inputs
        table, vsrc = p
        Hd = a.shape[-1]
        a2 = a.reshape(-1, Hd)
        b2 = b.reshape(-1, Hd) if b is not None else None
        i2 = idx.reshape(-1).contiguous() if idx is not None else None
        vec = vsrc.detach()[self.vec_row].contiguous() if vsrc is not None else None
        out = K.add_rows(a2, b2, table.detach() if table is not None else None, i2, vec)
        st.update(idx=i2, shape=a.shape, has_b=b is not None)
        return out.view(a.shape)

    def bwd(self, st, gouts, p):
        table, vsrc = p
        g = gouts[0]
        Hd = st["shape"][-1]
        g2 = g.reshape(-1, Hd).contiguous()
        dt = dv = None
        if table is not None:
            dt = zeros_f32(table.device, *table.shape)
            K.scatter_add_rows(g2, st["idx"], Hd, dt)
        if vsrc is not None:
            dv = zeros_f32(vsrc.device, *vsrc.shape)
            K.colsum(g2, Hd, out=dv[self.vec_row])
        return [g, g if st["has_b"] else None, None], [dt, dv]


class AddRows3Impl(AddRowsImpl):
    """out = ((a + b) + c) (+ table[idx]) (+ vec_src[vec_row]) in one bb_add_rows3 launch; a,b,c activations (rows,Hd).
    inputs (a, b, c, idx | None); params (table | None, vec_src | None).  Backward as AddRowsImpl: the output gradient
    goes to a, b and c unchanged."""

    def fwd(self, st, inputs, p):
        a, b, c, idx = inputs
        table, vsrc = p
        Hd = a.shape[-1]
        i2 = idx.reshape(-1).contiguous() if idx is not None else None
        vec = vsrc.detach()[self.vec_row].contiguous() if vsrc is not None else None
        out = K.add_rows(a.reshape(-1, Hd), b.reshape(-1, Hd), table.detach() if table is not None else None, i2, vec,
                         c=c.reshape(-1, Hd))
        st.update(idx=i2, shape=a.shape, has_b=True)
        return out.view(a.shape)

    def bwd(self, st, gouts, p):
        (g, _, _), dp = super().bwd(st, gouts, p)
        return [g, g, g, None], dp


class SegmentSumImpl:
    """out[s] = sum_e w[e] * src[idx[e]] over CSR segments (gmap node features, vilmodel.py:632-666).
    inputs (src (rows,Hd), seg_off int32, idx int32, w f32); no params."""

    def fwd(self, st, inputs, p):
        src, seg_off, idx, w = inputs
        nseg = seg_off.numel() - 1
        Hd = src.shape[-1]
        out = K.segment_wsum(src.reshape(-1, Hd), seg_off, idx, w, nseg, Hd)
        st.update(seg=(seg_off, idx, w, nseg), sshape=src.shape)
        return out

    def bwd(self, st, gouts, p):
        seg_off, idx, w, nseg = st["seg"]
        Hd = st["sshape"][-1]
        d32 = zeros_f32(gouts[0].device, *st["sshape"], scratch=True)
        K.segment_wsum_bwd(gouts[0].contiguous(), seg_off, idx, w, nseg, Hd, d32)
        return [K.cast_to_act(d32), None, None, None], []


class GatherRowsImpl:
    """out[r] = src[idx[r]] (idx < 0 -> zero row); inputs (src (rows,Hd), idx int64); backward scatter-adds."""

    def fwd(self, st, inputs, p):
        src, idx = inputs
        Hd = src.shape[-1]
        st.update(idx=idx, sshape=src.shape)
        return K.gather_rows(src.reshape(-1, Hd), idx, Hd)

    def bwd(self, st, gouts, p):
        Hd = st["sshape"][-1]
        d32 = zeros_f32(gouts[0].device, *st["sshape"], scratch=True)
        K.scatter_add_rows(gouts[0].contiguous(), st["idx"], Hd, d32.view(-1, Hd))
        return [K.cast_to_act(d32), None], []


class HeadImpl:
    """Linear -> ReLU -> LN(1e-12) -> Linear (pretrain_cmt.py:34-71); output fp32 (rows, n_out).
    inputs (x (rows,Kd) activation,); params (W0,b0,gamma,beta,W3,b3)."""

    def __init__(self, rt):
        self.rt, self.wc = rt, rt.wc

    def fwd(self, st, inputs, p):
        x = inputs[0]
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        h, _ = lin_fwd(x2, self.wc.get(p[0]), p[1].detach(), act=K.ACT_RELU)
        hn, _, mean, rstd = K.layernorm_fwd(h, None, p[2].detach(), p[3].detach(), 1e-12)
        n_out = p[4].shape[0]
        npad = _round8(n_out)
        w3 = self.wc.get(p[4], pad_n=npad) if npad != n_out else self.wc.get(p[4])
        b3 = p[5].detach()
        if npad != n_out:
            b3 = torch.cat([b3, torch.zeros(npad - n_out, dtype=b3.dtype, device=b3.device)])
        out, _ = lin_fwd(hn, w3, b3, out_f32=True)
        st.update(x2=x2, h=h, hn=hn, mean=mean, rstd=rstd, w3=w3, n_out=n_out, npad=npad, xshape=x.shape)
        return out[:, :n_out].reshape(x.shape[:-1] + (n_out,))

    def bwd(self, st, gouts, p):
        n_out, npad = st["n_out"], st["npad"]
        g = gouts[0].reshape(-1, n_out)
        Hd = st["h"].shape[1]
        dev = g.device
        if npad != n_out:
            gp = torch.zeros(g.shape[0], npad, dtype=torch.float32, device=dev)
            gp[:, :n_out] = g
        else:
            gp = g.contiguous()
        g16 = K.cast_to_act(gp)
        dW3 = lin_bwd_dw(g16, st["hn"])[:n_out]
        db3 = K.colsum(g16, npad)[:n_out]
        dhn = lin_bwd_dx(g16, st["w3"])
        dg = zeros_f32(dev, Hd)
        db = zeros_f32(dev, Hd)
        dh, _ = K.layernorm_bwd(dhn, st["h"], None, p[2].detach(), st["mean"], st["rstd"], dgamma=dg, dbeta=db)
        # ReLU': h > 0 -- folded into the dX GEMM epilogue of the first Linear (identity "weights" are avoided
        # by masking dh directly: drelu on an elementwise path = GEMM-free, use the dropout-free multiply kernel)
        dh = K.relu_bwd(dh, st["h"])
        dW0 = lin_bwd_dw(dh, st["x2"])
        db0 = K.colsum(dh, Hd)
        dx = lin_bwd_dx(dh, self.wc.get(p[0])).view(st["xshape"])
        return [dx], [dW0, db0, dg, db, dW3, db3]


class MLMLossImpl:
    """BertOnlyMLMHead (vilmodel.py:258-299) on the masked rows + cross-entropy (pretrain_cmt.py:255-261):
    transform dense -> GELU -> LN -> tied decoder (word embeddings) + bias -> per-row CE.
    inputs (h (m,Hd) activation, labels int64 (m,)); params (Wt,bt,gamma,beta,E,vbias).
    compute_loss=False returns the fp32 logits instead (no backward through them)."""

    def __init__(self, rt, eps, compute_loss=True):
        self.rt, self.wc, self.eps, self.compute_loss = rt, rt.wc, eps, compute_loss

    def fwd(self, st, inputs, p):
        h, labels = inputs
        t, tpre = lin_fwd(h.contiguous(), self.wc.get(p[0]), p[1].detach(), act=K.ACT_GELU, want_pre=True)
        tn, _, mean, rstd = K.layernorm_fwd(t, None, p[2].detach(), p[3].detach(), self.eps)
        V = p[4].shape[0]
        ld = _round8(V)
        m = h.shape[0]
        logits = torch.empty(m, ld, dtype=torch.float32, device=h.device)
        e16 = self.wc.get(p[4])
        K.gemm(tn, e16, logits, m, V, tn.shape[1], lda=tn.shape[1], ldb=tn.shape[1], ldd=ld, bias=p[5].detach())
        if not self.compute_loss:
            return logits[:, :V]
        loss, dlog = K.softmax_xent(logits, labels.contiguous(), V, ld)
        st.update(h=h, t=t, tpre=tpre, tn=tn, mean=mean, rstd=rstd, dlog=dlog, V=V, ld=ld, e16=e16)
        return loss

    def bwd(self, st, gouts, p):
        g = gouts[0].contiguous().to(torch.float32)
        dlog, V, ld, tn = st["dlog"], st["V"], st["ld"], st["tn"]
        m, Hd = tn.shape
        K.scale_rows_(dlog, g, m, ld)
        dE = zeros_f32(g.device, V, Hd)
        kb = (m + 63) // 64
        # a split adds nothing to the occupancy of this many vocabulary tiles; in deterministic mode its partial tiles
        # would need a workspace the size of dE, so the product runs unsplit there
        split = 1 if kb < 8 or torch.are_deterministic_algorithms_enabled() else 2
        K.gemm(dlog, tn, dE, V, Hd, m, lda=ld, ldb=Hd, ldd=Hd, a_mn=True, b_mn=True, split_k=split)
        dvb = zeros_f32(g.device, ld)
        K.colsum(dlog, ld, out=dvb)
        dtn = _empty((m, Hd), tn)
        K.gemm(dlog, st["e16"], dtn, m, Hd, V, lda=ld, ldb=Hd, ldd=Hd, b_mn=True)
        dg = zeros_f32(g.device, Hd)
        db = zeros_f32(g.device, Hd)
        dt, _ = K.layernorm_bwd(dtn, st["t"], None, p[2].detach(), st["mean"], st["rstd"], dgamma=dg, dbeta=db)
        dtpre = K.gelu_bwd(dt, st["tpre"])
        dWt = lin_bwd_dw(dtpre, st["h"].contiguous())
        dbt = K.colsum(dtpre, Hd)
        dh = lin_bwd_dx(dtpre, self.wc.get(p[0]))
        return [dh, None], [dWt, dbt, dg, db, dE, dvb[:V]]


class CastImpl:
    """fp32 -> activation dtype with optional inverted dropout (nn.Dropout on input features,
    pretrain_cmt.py:102-106).  inputs (x f32,); no gradient (inputs are data)."""

    def __init__(self, rt, p=0.0):
        self.rt, self.p = rt, p

    def fwd(self, st, inputs, p):
        return K.cast_to_act(inputs[0], self.rt.ds.make(self.p))

    def bwd(self, st, gouts, p):
        return [None], []


class ToActImpl:
    """fp32 -> activation dtype at an API boundary, differentiable (gradient cast back to fp32)."""

    def fwd(self, st, inputs, p):
        return K.cast_to_act(inputs[0])

    def bwd(self, st, gouts, p):
        return [K.cast_to_f32(gouts[0].contiguous())], []


class ToF32Impl:
    """activation dtype -> fp32 at an API boundary, differentiable."""

    def fwd(self, st, inputs, p):
        return K.cast_to_f32(inputs[0])

    def bwd(self, st, gouts, p):
        return [K.cast_to_act(gouts[0].contiguous().float())], []


def to_act(x):
    return run_block(ToActImpl(), [x], []) if x.dtype == torch.float32 else x


def to_f32(x):
    return run_block(ToF32Impl(), [x], []) if x.dtype != torch.float32 else x


# =============================================================================================== autograd glue
DIRECT_PARAM_GRADS = False   # parallel.direct_param_grads(): blocks assign p.grad themselves
AFTER_BLOCK_BWD = None       # parallel.FlatGradAllReduce: called after every block's backward (overlapped reduction)
DEFER_GRAD_ADDS = False      # a second contribution to a parameter waits in PENDING_ADDS until the reductions are done
PENDING_ADDS = []


SIDE_KEEP = []               # side-stream mode: everything a backward call's side-stream kernels read, kept until the join


def apply_pending_adds():
    for p, g in PENDING_ADDS:
        p.grad.add_(g)
    PENDING_ADDS.clear()


def side_active():
    return K.side_stream() is not None


def join_side():
    """End of backward in side-stream mode (parallel.enable_side_stream): the current stream waits for the weight-gradient
    kernels, the buffers they read are released, second gradient contributions are added."""
    if K.side_stream() is None:
        return
    K.side_join()
    SIDE_KEEP.clear()
    if AFTER_BLOCK_BWD is None:          # with an overlapped reducer, the reducer applies them after its all-reduces
        apply_pending_adds()



class _BlockFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, impl, n_in, *args):
        inputs, params = args[:n_in], args[n_in:]
        st = {}
        with torch.no_grad():
            out = impl.fwd(st, inputs, params)
        ctx.impl, ctx.st, ctx.n_in, ctx.params = impl, st, n_in, params
        return out

    @staticmethod
    def backward(ctx, *gouts):
        with torch.no_grad():
            gin, gpar = ctx.impl.bwd(ctx.st, gouts, ctx.params)
        if side_active():
            SIDE_KEEP.append((ctx.st, gouts))
        ctx.st = None
        gin = list(gin) + [None] * (ctx.n_in - len(gin))
        needs = ctx.needs_input_grad[2:]
        if DIRECT_PARAM_GRADS:
            # hand the parameter gradients over without one AccumulateGrad node per parameter (see parallel.py)
            n_in = ctx.n_in
            for i, (p, g) in enumerate(zip(ctx.params, gpar)):
                if g is not None and needs[n_in + i]:
                    if not g.is_contiguous():          # sliced views of padded operands (tiny K): as AccumulateGrad does
                        g = g.contiguous()
                    if p.grad is None:
                        p.grad = g
                    elif DEFER_GRAD_ADDS or side_active():
                        PENDING_ADDS.append((p, g))
                    else:
                        p.grad.add_(g)
            if AFTER_BLOCK_BWD is not None:
                AFTER_BLOCK_BWD()
            full = [g if n else None for g, n in zip(gin, needs)] + [None] * len(ctx.params)
            return (None, None, *full)
        full = list(gin) + list(gpar)
        full = [g if n else None for g, n in zip(full, needs)]
        return (None, None, *full)


def run_block(impl, inputs, params):
    """Runs `impl` as one autograd node. `inputs` may contain None / non-differentiable tensors."""
    return _BlockFn.apply(impl, len(inputs), *inputs, *params)
