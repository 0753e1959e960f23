// Native sub-layer executors: one C call enqueues the whole kernel sequence of an attention sub-layer
// (projection GEMMs, batched QK^T, masked softmax, PV, output dense, dropout+residual+LayerNorm) or of an FFN
// sub-layer, forward or backward, on the caller's stream.  This is the launch loop of blocks.py moved out of
// Python: same kernels, same order, same math -- the host just stops paying ~40 us of interpreter time per launch.
//
// Reference semantics: BertSelfAttention/BertOutAttention + BertSelfOutput (vilmodel.py:103-154, 325-363),
// BertIntermediate + BertOutput (vilmodel.py:168-193).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/bevbert_b200.h"
#include "common.h"

namespace bb {

static inline int64_t al(int64_t n) { return (n + 255) / 256 * 256; }
// keys-per-row limit of the fused score kernels (BB_FUSED_SCORES_MAX overrides it for experiments; <= 512)
static inline int fused_max_keys() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("BB_FUSED_SCORES_MAX");
    v = e ? atoi(e) : 0;   // default off: with one CTA per SM the softmax arithmetic has too few warps (see DESIGN.md)
    if (v > 512) v = 512;
  }
  return v;
}
bool act_f32();   // gemm_f32.cu: fp32-activation verification mode (bb_set_act_f32)
// fused scores + softmax (attn_scores.cu) instead of the GEMM -> bb_softmax pair: bf16 only, head dim 64
static inline bool fused_scores(int nk, int dh) { return nk <= fused_max_keys() && dh == 64 && !act_f32(); }
static inline int round8(int n) { return (n + 7) / 8 * 8; }
// fused attention core (attn_flash.cu) for head dim 64; BB_FLASH=0 selects the unfused GEMM + softmax sequence
static inline bool flash_on(const bb_attn_desc* d) {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("BB_FLASH");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v && d->Hd / d->heads == 64;
}

struct AttnLayout {
  int ldp;
  int64_t qkv, q, kv, S, P, Pd, lse, ctx, ao, mean, rstd, fwd_bytes;
  int64_t dao, dres, dctx, dqkv, dq, dkv, dP, dS, dsum, bwd_bytes;
};

static AttnLayout attn_layout(const bb_attn_desc* d) {
  AttnLayout L;
  memset(&L, 0, sizeof(L));
  const int64_t Mq = (int64_t)d->B * d->nq, Mk = (int64_t)d->B * d->nk, Hd = d->Hd;
  L.ldp = round8(d->nk);
  const int64_t pn = (int64_t)d->B * d->heads * d->nq * L.ldp;
  int64_t o = 0;
  if (!d->cross) { L.qkv = o; o += al(Mq * 3 * Hd * 2); }
  else { L.q = o; o += al(Mq * Hd * 2); L.kv = o; o += al(Mk * 2 * Hd * 2); }
  const bool flash = flash_on(d);
  const int64_t rows = (int64_t)d->B * d->heads * d->nq;
  if (flash) {
    L.lse = o; o += al(rows * 4);                             // the only attention state saved for backward
  } else {
    L.S = o; if (d->nk > fused_max_keys()) o += al(pn * 4);   // fp32 scores only on the unfused path
    L.P = o; o += al(pn * 2);
    if (d->th_attn) { L.Pd = o; o += al(pn * 2); } else L.Pd = L.P;
  }
  L.ctx = o; o += al(Mq * Hd * 2);
  L.ao = o; o += al(Mq * Hd * 2);
  L.mean = o; o += al(Mq * 4);
  L.rstd = o; o += al(Mq * 4);
  L.fwd_bytes = o;
  o = 0;
  L.dao = o; o += al(Mq * Hd * 2);
  L.dres = o; o += al(Mq * Hd * 2);
  L.dctx = o; o += al(Mq * Hd * 2);
  if (!d->cross) { L.dqkv = o; o += al(Mq * 3 * Hd * 2); }
  else { L.dq = o; o += al(Mq * Hd * 2); L.dkv = o; o += al(Mk * 2 * Hd * 2); }
  if (flash) {
    L.dsum = o; o += al(rows * 4);
  } else {
    L.dP = o; if (d->nk > fused_max_keys()) o += al(pn * 4);
    L.dS = o; o += al(pn * 2);
  }
  L.bwd_bytes = o;
  return L;
}

static inline char* at(void* base, int64_t off) { return reinterpret_cast<char*>(base) + off; }

// Optional side stream for the weight-gradient products (dW = dY^T X, split-K fp32 atomics) and the bias column sums:
// nothing in backward depends on them, they are small (0.4-1.6 waves of tiles on the 2560-row language-encoder
// layers) and so overlap well with the dX chain on the main stream.  side_for() forks: the side stream waits for
// everything enqueued on `main` so far; the caller joins once after backward (bb_side_join) and keeps the buffers those
// kernels read alive until then.  Inside a CUDA-graph capture this becomes a fork / join of the graph.
static cudaStream_t g_side = nullptr;
cudaStream_t side_stream() { return g_side; }
static cudaEvent_t g_fork_ev[32];
static int g_fork_i = 0;
static bool g_side_used = false;
static void* side_for(void* main_stream) {
  if (!g_side) return main_stream;
  cudaEvent_t& ev = g_fork_ev[g_fork_i++ & 31];
  if (!ev) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
  cudaEventRecord(ev, (cudaStream_t)main_stream);
  cudaStreamWaitEvent(g_side, ev, 0);
  g_side_used = true;
  return g_side;
}

// y = epi(x W^T + b)
static int lin_fwd(const void* x, const void* w, void* out, int64_t M, int N, int K, const float* bias, int act,
                   void* pre, uint64_t seed, uint32_t th, float sc, const void* add_in, int out_f32, void* stream) {
  bb_gemm_args g;
  memset(&g, 0, sizeof(g));
  g.A = x; g.B = w; g.D = out; g.M = (int32_t)M; g.N = N; g.K = K; g.nb1 = 1; g.nb2 = 1;
  g.lda = K; g.ldb = K; g.ldd = N; g.alpha = 1.0f; g.bias = bias; g.act = act; g.aux_out = pre; g.out_f32 = out_f32;
  g.drop_seed = seed; g.drop_thresh = th; g.drop_scale = sc; g.add_in = add_in; g.split_k = 1;
  return bb_gemm_bf16(&g, stream);
}
// dx = epi(dy W)
static int lin_bwd_dx(const void* dy, const void* w, void* out, int64_t M, int N, int Kd, int epi_mul, const void* aux_in,
                      const void* add_in, void* stream, uint64_t seed = 0, uint32_t th = 0, float sc = 1.0f) {
  bb_gemm_args g;
  memset(&g, 0, sizeof(g));
  g.A = dy; g.B = w; g.D = out; g.M = (int32_t)M; g.N = Kd; g.K = N; g.nb1 = 1; g.nb2 = 1;
  g.lda = N; g.ldb = Kd; g.ldd = Kd; g.b_mn = 1; g.alpha = 1.0f; g.epi_mul = epi_mul; g.aux_in = aux_in;
  g.add_in = add_in; g.split_k = 1; g.drop_seed = seed; g.drop_thresh = th; g.drop_scale = sc;
  return bb_gemm_bf16(&g, stream);
}
static int num_sms() {     // split-K factor of the weight-gradient products: fill the machine this library runs on
  static int n = 0;
  if (!n) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;   // H100 SXM
  }
  return n;
}
// dW (N, Kd) += dy^T x   (fp32, zeroed by the caller)
static int lin_bwd_dw(const void* dy, const void* x, float* out, int64_t M, int N, int Kd, void* stream) {
  bb_gemm_args g;
  memset(&g, 0, sizeof(g));
  // same tiling rule as blocks.lin_bwd_dw: 128-wide tiles when they fill half the SMs, else 64-wide, then split the
  // token dimension until about one CTA per SM, keeping >= 8 k-blocks per split
  const int m_t = (N + 127) / 128;
  int bn = (m_t * ((Kd + 127) / 128) >= num_sms() / 2) ? 128 : 64;
  if (Kd <= bn) bn = 0;
  const int tiles = bn ? m_t * ((Kd + bn - 1) / bn) : m_t;
  const int64_t kb = (M + 63) / 64;
  int64_t split = (num_sms() + tiles / 2) / (tiles > 0 ? tiles : 1);
  const int64_t cap = kb >= 8 ? kb / 8 : 1;
  if (split > cap) split = cap;
  if (split < 1) split = 1;
  g.A = dy; g.B = x; g.D = out; g.M = N; g.N = Kd; g.K = (int32_t)M; g.nb1 = 1; g.nb2 = 1;
  g.lda = N; g.ldb = Kd; g.ldd = Kd; g.a_mn = 1; g.b_mn = 1; g.out_f32 = 1; g.split_k = (int32_t)split;
  g.accumulate = split > 1 ? 1 : 0; g.alpha = 1.0f; g.block_n = bn; g.drop_scale = 1.0f;
  return bb_gemm_bf16(&g, stream);
}

#define TRY(x)          \
  do {                  \
    int rc_ = (x);      \
    if (rc_) return rc_; \
  } while (0)

// softmax(Q K^T / sqrt(dh) + kmask + bias) V ; q/k/v are element pointers to (sample 0, row 0, head 0, dim 0)
static int attn_core_fwd(const bb_attn_desc* d, const AttnLayout& L, const void* q, int ldq, const void* k, int ldk,
                         const void* v, int ldv, void* stream) {
  const int B = d->B, H = d->heads, nq = d->nq, nk = d->nk, dh = d->Hd / d->heads, ldp = L.ldp;
  if (flash_on(d)) {
    bb_flash_args f;
    memset(&f, 0, sizeof(f));
    f.q = q; f.k = k; f.v = v; f.o = at(d->ws, L.ctx);
    f.q_bs = (int64_t)nq * ldq; f.k_bs = (int64_t)nk * ldk; f.v_bs = (int64_t)nk * ldv; f.o_bs = (int64_t)nq * d->Hd;
    f.ldq = ldq; f.ldk = ldk; f.ldv = ldv; f.ldo = d->Hd;
    f.B = B; f.H = H; f.nq = nq; f.nk = nk; f.dh = dh; f.alpha = 1.0f / sqrtf((float)dh);
    f.kmask = d->kmask; f.bias = d->bias; f.lse = reinterpret_cast<float*>(at(d->ws, L.lse));
    f.seed = d->seed_attn; f.thresh = d->th_attn; f.scale = d->sc_attn;
    return bb_flash_fwd(&f, stream);
  }
  bb_gemm_args g;
  if (fused_scores(nk, dh)) {
    bb_attn_scores_args s;
    memset(&s, 0, sizeof(s));
    s.A = q; s.lda = ldq; s.a_s1 = dh; s.a_s2 = (int64_t)nq * ldq;
    s.Bm = k; s.ldb = ldk; s.b_s1 = dh; s.b_s2 = (int64_t)nk * ldk;
    s.B = B; s.H = H; s.nq = nq; s.nk = nk; s.ldp = ldp; s.mode = 0; s.alpha = 1.0f / sqrtf((float)dh);
    s.kmask = d->kmask; s.bias = d->bias; s.seed = d->seed_attn; s.thresh = d->th_attn; s.scale = d->sc_attn;
    s.P = at(d->ws, L.P); s.Pd = d->th_attn ? at(d->ws, L.Pd) : nullptr;
    TRY(bb_attn_scores(&s, stream));
  } else {
  memset(&g, 0, sizeof(g));
  g.A = q; g.B = k; g.D = at(d->ws, L.S); g.M = nq; g.N = nk; g.K = dh; g.nb1 = H; g.nb2 = B;
  g.lda = ldq; g.a_s1 = dh; g.a_s2 = (int64_t)nq * ldq; g.ldb = ldk; g.b_s1 = dh; g.b_s2 = (int64_t)nk * ldk;
  g.ldd = ldp; g.d_s1 = (int64_t)nq * ldp; g.d_s2 = (int64_t)H * nq * ldp; g.out_f32 = 1; g.split_k = 1;
  g.alpha = 1.0f / sqrtf((float)dh); g.drop_scale = 1.0f;
  TRY(bb_gemm_bf16(&g, stream));
  TRY(bb_softmax_fwd(reinterpret_cast<const float*>(at(d->ws, L.S)), d->kmask, d->bias, B, H, nq, nk, ldp, d->seed_attn,
                     d->th_attn, d->sc_attn, at(d->ws, L.P), d->th_attn ? at(d->ws, L.Pd) : nullptr, stream));
  }
  memset(&g, 0, sizeof(g));
  g.A = at(d->ws, L.Pd); g.B = v; g.D = at(d->ws, L.ctx); g.M = nq; g.N = dh; g.K = nk; g.nb1 = H; g.nb2 = B;
  g.lda = ldp; g.a_s1 = (int64_t)nq * ldp; g.a_s2 = (int64_t)H * nq * ldp; g.ldb = ldv; g.b_s1 = dh;
  g.b_s2 = (int64_t)nk * ldv; g.b_mn = 1; g.ldd = d->Hd; g.d_s1 = dh; g.d_s2 = (int64_t)nq * d->Hd; g.split_k = 1;
  g.alpha = 1.0f; g.drop_scale = 1.0f;
  return bb_gemm_bf16(&g, stream);
}

static int attn_core_bwd(const bb_attn_desc* d, const AttnLayout& L, const void* q, int ldq, const void* k, int ldk,
                         const void* v, int ldv, void* dq, int lddq, void* dk, int lddk, void* dv, int lddv,
                         void* stream) {
  const int B = d->B, H = d->heads, nq = d->nq, nk = d->nk, dh = d->Hd / d->heads, ldp = L.ldp, HD = d->Hd;
  const void* dctx = at(d->gws, L.dctx);
  if (flash_on(d)) {
    bb_flash_args f;
    memset(&f, 0, sizeof(f));
    f.q = q; f.k = k; f.v = v; f.o = at(d->ws, L.ctx);   // the saved context (read-only here)
    f.q_bs = (int64_t)nq * ldq; f.k_bs = (int64_t)nk * ldk; f.v_bs = (int64_t)nk * ldv; f.o_bs = (int64_t)nq * HD;
    f.ldq = ldq; f.ldk = ldk; f.ldv = ldv; f.ldo = HD;
    f.B = B; f.H = H; f.nq = nq; f.nk = nk; f.dh = dh; f.alpha = 1.0f / sqrtf((float)dh);
    f.kmask = d->kmask; f.bias = d->bias; f.lse = reinterpret_cast<float*>(at(d->ws, L.lse));
    f.seed = d->seed_attn; f.thresh = d->th_attn; f.scale = d->sc_attn;
    f.dout = dctx; f.do_bs = (int64_t)nq * HD; f.lddo = HD;
    f.dsum = reinterpret_cast<float*>(at(d->gws, L.dsum));
    f.dq = dq; f.dq_bs = (int64_t)nq * lddq; f.lddq = lddq;
    f.dk = dk; f.dk_bs = (int64_t)nk * lddk; f.lddk = lddk;
    f.dv = dv; f.dv_bs = (int64_t)nk * lddv; f.lddv = lddv;
    f.dbias = d->want_dbias ? d->dbias : nullptr;
    return bb_flash_bwd(&f, stream);
  }
  const int64_t ps1 = (int64_t)nq * ldp, ps2 = (int64_t)H * nq * ldp;
  bb_gemm_args g;
  // dV = Pd^T dctx
  memset(&g, 0, sizeof(g));
  g.A = at(d->ws, L.Pd); g.B = dctx; g.D = dv; g.M = nk; g.N = dh; g.K = nq; g.nb1 = H; g.nb2 = B; g.a_mn = 1; g.b_mn = 1;
  g.lda = ldp; g.a_s1 = ps1; g.a_s2 = ps2; g.ldb = HD; g.b_s1 = dh; g.b_s2 = (int64_t)nq * HD;
  g.ldd = lddv; g.d_s1 = dh; g.d_s2 = (int64_t)nk * lddv; g.split_k = 1; g.alpha = 1.0f; g.drop_scale = 1.0f;
  TRY(bb_gemm_bf16(&g, stream));
  if (fused_scores(nk, dh)) {
    bb_attn_scores_args s;
    memset(&s, 0, sizeof(s));
    s.A = dctx; s.lda = HD; s.a_s1 = dh; s.a_s2 = (int64_t)nq * HD;
    s.Bm = v; s.ldb = ldv; s.b_s1 = dh; s.b_s2 = (int64_t)nk * ldv;
    s.B = B; s.H = H; s.nq = nq; s.nk = nk; s.ldp = ldp; s.mode = 1; s.alpha = 1.0f; s.out_scale = 1.0f / sqrtf((float)dh);
    s.seed = d->seed_attn; s.thresh = d->th_attn; s.scale = d->sc_attn;
    s.Pin = at(d->ws, L.P); s.dS = at(d->gws, L.dS); s.dbias = d->want_dbias ? d->dbias : nullptr;
    TRY(bb_attn_scores(&s, stream));
  } else {
  // dPd = dctx V^T
  memset(&g, 0, sizeof(g));
  g.A = dctx; g.B = v; g.D = at(d->gws, L.dP); g.M = nq; g.N = nk; g.K = dh; g.nb1 = H; g.nb2 = B;
  g.lda = HD; g.a_s1 = dh; g.a_s2 = (int64_t)nq * HD; g.ldb = ldv; g.b_s1 = dh; g.b_s2 = (int64_t)nk * ldv;
  g.ldd = ldp; g.d_s1 = ps1; g.d_s2 = ps2; g.out_f32 = 1; g.split_k = 1; g.alpha = 1.0f; g.drop_scale = 1.0f;
  TRY(bb_gemm_bf16(&g, stream));
  TRY(bb_softmax_bwd(at(d->ws, L.P), reinterpret_cast<const float*>(at(d->gws, L.dP)), B, H, nq, nk, ldp, d->seed_attn,
                     d->th_attn, d->sc_attn, 1.0f / sqrtf((float)dh), at(d->gws, L.dS), d->want_dbias ? d->dbias : nullptr,
                     stream));
  }
  // dQ = dS K
  memset(&g, 0, sizeof(g));
  g.A = at(d->gws, L.dS); g.B = k; g.D = dq; g.M = nq; g.N = dh; g.K = nk; g.nb1 = H; g.nb2 = B; g.b_mn = 1;
  g.lda = ldp; g.a_s1 = ps1; g.a_s2 = ps2; g.ldb = ldk; g.b_s1 = dh; g.b_s2 = (int64_t)nk * ldk;
  g.ldd = lddq; g.d_s1 = dh; g.d_s2 = (int64_t)nq * lddq; g.split_k = 1; g.alpha = 1.0f; g.drop_scale = 1.0f;
  TRY(bb_gemm_bf16(&g, stream));
  // dK = dS^T Q
  memset(&g, 0, sizeof(g));
  g.A = at(d->gws, L.dS); g.B = q; g.D = dk; g.M = nk; g.N = dh; g.K = nq; g.nb1 = H; g.nb2 = B; g.a_mn = 1; g.b_mn = 1;
  g.lda = ldp; g.a_s1 = ps1; g.a_s2 = ps2; g.ldb = ldq; g.b_s1 = dh; g.b_s2 = (int64_t)nq * ldq;
  g.ldd = lddk; g.d_s1 = dh; g.d_s2 = (int64_t)nk * lddk; g.split_k = 1; g.alpha = 1.0f; g.drop_scale = 1.0f;
  return bb_gemm_bf16(&g, stream);
}

}  // namespace bb

using namespace bb;

extern "C" int bb_attn_ws_bytes(const bb_attn_desc* d, int64_t* fwd_bytes, int64_t* bwd_bytes) {
  if (!d) return set_error("bb_attn_ws_bytes: null descriptor");
  if (d->Hd % d->heads != 0 || d->Hd % 8 != 0) return set_error("bb_attn: hidden size must divide into heads, multiple of 8");
  const AttnLayout L = attn_layout(d);
  if (fwd_bytes) *fwd_bytes = L.fwd_bytes;
  if (bwd_bytes) *bwd_bytes = L.bwd_bytes;
  return 0;
}

extern "C" int bb_attn_fwd(const bb_attn_desc* d, void* stream) {
  if (!d || !d->x || !d->ws || !d->y) return set_error("bb_attn_fwd: null argument");
  const AttnLayout L = attn_layout(d);
  const int Hd = d->Hd;
  const int64_t Mq = (int64_t)d->B * d->nq, Mk = (int64_t)d->B * d->nk;
  if (!d->cross) {
    char* qkv = at(d->ws, L.qkv);
    TRY(lin_fwd(d->x, d->w_qkv, qkv, Mq, 3 * Hd, Hd, d->b_qkv, 0, nullptr, 0, 0, 1.0f, nullptr, 0, stream));
    TRY(attn_core_fwd(d, L, qkv, 3 * Hd, qkv + (int64_t)Hd * 2, 3 * Hd, qkv + (int64_t)2 * Hd * 2, 3 * Hd, stream));
  } else {
    if (!d->c) return set_error("bb_attn_fwd: cross attention needs a context");
    char* q = at(d->ws, L.q);
    char* kv = at(d->ws, L.kv);
    TRY(lin_fwd(d->x, d->w_qkv, q, Mq, Hd, Hd, d->b_qkv, 0, nullptr, 0, 0, 1.0f, nullptr, 0, stream));
    TRY(lin_fwd(d->c, d->w_kv, kv, Mk, 2 * Hd, Hd, d->b_kv, 0, nullptr, 0, 0, 1.0f, nullptr, 0, stream));
    TRY(attn_core_fwd(d, L, q, Hd, kv, 2 * Hd, kv + (int64_t)Hd * 2, 2 * Hd, stream));
  }
  TRY(lin_fwd(at(d->ws, L.ctx), d->w_o, at(d->ws, L.ao), Mq, Hd, Hd, d->b_o, 0, nullptr, 0, 0, 1.0f, nullptr, 0, stream));
  return bb_layernorm_fwd(at(d->ws, L.ao), 0, d->x, d->gamma, d->beta, d->eps, Mq, Hd, d->seed_h, d->th_h, d->sc_h, 0, 0,
                          1.0f, d->y, nullptr, reinterpret_cast<float*>(at(d->ws, L.mean)),
                          reinterpret_cast<float*>(at(d->ws, L.rstd)), stream);
}

extern "C" int bb_attn_bwd(const bb_attn_desc* d, void* stream) {
  if (!d || !d->x || !d->ws || !d->gws || !d->dy || !d->dx) return set_error("bb_attn_bwd: null argument");
  const AttnLayout L = attn_layout(d);
  const int Hd = d->Hd;
  const int64_t Mq = (int64_t)d->B * d->nq, Mk = (int64_t)d->B * d->nk;
  char* dao = at(d->gws, L.dao);
  char* dres = at(d->gws, L.dres);
  TRY(bb_layernorm_bwd(d->dy, 0, at(d->ws, L.ao), 0, d->x, d->gamma, reinterpret_cast<const float*>(at(d->ws, L.mean)),
                       reinterpret_cast<const float*>(at(d->ws, L.rstd)), Mq, Hd, d->seed_h, d->th_h, d->sc_h, 0, 0, 1.0f,
                       dao, 0, dres, d->dgamma, d->dbeta, d->db_o, stream));
  TRY(lin_bwd_dw(dao, at(d->ws, L.ctx), d->dw_o, Mq, Hd, Hd, side_for(stream)));
  TRY(lin_bwd_dx(dao, d->w_o, at(d->gws, L.dctx), Mq, Hd, Hd, 0, nullptr, nullptr, stream));
  if (!d->cross) {
    char* qkv = at(d->ws, L.qkv);
    char* dqkv = at(d->gws, L.dqkv);
    const int Lq = 3 * Hd;
    TRY(attn_core_bwd(d, L, qkv, Lq, qkv + (int64_t)Hd * 2, Lq, qkv + (int64_t)2 * Hd * 2, Lq, dqkv, Lq,
                      dqkv + (int64_t)Hd * 2, Lq, dqkv + (int64_t)2 * Hd * 2, Lq, stream));
    TRY(lin_bwd_dw(dqkv, d->x, d->dw_qkv, Mq, 3 * Hd, Hd, side_for(stream)));
    TRY(bb_colsum_bf16(dqkv, Mq, 3 * Hd, 3 * Hd, d->db_qkv, side_for(stream)));
    return lin_bwd_dx(dqkv, d->w_qkv, d->dx, Mq, 3 * Hd, Hd, 0, nullptr, dres, stream);
  }
  if (!d->dc) return set_error("bb_attn_bwd: cross attention needs dc");
  char* q = at(d->ws, L.q);
  char* kv = at(d->ws, L.kv);
  char* dq = at(d->gws, L.dq);
  char* dkv = at(d->gws, L.dkv);
  TRY(attn_core_bwd(d, L, q, Hd, kv, 2 * Hd, kv + (int64_t)Hd * 2, 2 * Hd, dq, Hd, dkv, 2 * Hd, dkv + (int64_t)Hd * 2,
                    2 * Hd, stream));
  TRY(lin_bwd_dw(dq, d->x, d->dw_qkv, Mq, Hd, Hd, side_for(stream)));
  TRY(bb_colsum_bf16(dq, Mq, Hd, Hd, d->db_qkv, side_for(stream)));
  TRY(lin_bwd_dx(dq, d->w_qkv, d->dx, Mq, Hd, Hd, 0, nullptr, dres, stream));
  TRY(lin_bwd_dw(dkv, d->c, d->dw_kv, Mk, 2 * Hd, Hd, side_for(stream)));
  TRY(bb_colsum_bf16(dkv, Mk, 2 * Hd, 2 * Hd, d->db_kv, side_for(stream)));
  return lin_bwd_dx(dkv, d->w_kv, d->dc, Mk, 2 * Hd, Hd, 0, nullptr, nullptr, stream);
}

// ------------------------------------------------------------------------------------------------ FFN sub-layer
namespace bb {
struct FfnLayout {
  int64_t hpre, h, fo, mean, rstd, fwd_bytes, dfo, dres, dhpre, bwd_bytes;
};
static FfnLayout ffn_layout(const bb_ffn_desc* d) {
  FfnLayout L;
  int64_t o = 0;
  L.hpre = o; o += al(d->M * d->Fd * 2);
  L.h = o; o += al(d->M * d->Fd * 2);
  L.fo = o; o += al(d->M * d->Hd * 2);
  L.mean = o; o += al(d->M * 4);
  L.rstd = o; o += al(d->M * 4);
  L.fwd_bytes = o;
  o = 0;
  L.dfo = o; o += al(d->M * d->Hd * 2);
  L.dres = o; o += al(d->M * d->Hd * 2);
  L.dhpre = o; o += al(d->M * d->Fd * 2);
  L.bwd_bytes = o;
  return L;
}
}  // namespace bb

extern "C" int bb_ffn_ws_bytes(const bb_ffn_desc* d, int64_t* fwd_bytes, int64_t* bwd_bytes) {
  if (!d) return set_error("bb_ffn_ws_bytes: null descriptor");
  const FfnLayout L = ffn_layout(d);
  if (fwd_bytes) *fwd_bytes = L.fwd_bytes;
  if (bwd_bytes) *bwd_bytes = L.bwd_bytes;
  return 0;
}

extern "C" int bb_ffn_fwd(const bb_ffn_desc* d, void* stream) {
  if (!d || !d->a || !d->ws || !d->y) return set_error("bb_ffn_fwd: null argument");
  const FfnLayout L = ffn_layout(d);
  TRY(lin_fwd(d->a, d->w1, at(d->ws, L.h), d->M, d->Fd, d->Hd, d->b1, 1, at(d->ws, L.hpre), 0, 0, 1.0f, nullptr, 0, stream));
  TRY(lin_fwd(at(d->ws, L.h), d->w2, at(d->ws, L.fo), d->M, d->Hd, d->Fd, d->b2, 0, nullptr, 0, 0, 1.0f, nullptr, 0, stream));
  return bb_layernorm_fwd(at(d->ws, L.fo), 0, d->a, d->gamma, d->beta, d->eps, d->M, d->Hd, d->seed_h, d->th_h, d->sc_h, 0,
                          0, 1.0f, d->y, nullptr, reinterpret_cast<float*>(at(d->ws, L.mean)),
                          reinterpret_cast<float*>(at(d->ws, L.rstd)), stream);
}

extern "C" int bb_ffn_bwd(const bb_ffn_desc* d, void* stream) {
  if (!d || !d->a || !d->ws || !d->gws || !d->dy || !d->da) return set_error("bb_ffn_bwd: null argument");
  const FfnLayout L = ffn_layout(d);
  char* dfo = at(d->gws, L.dfo);
  char* dres = at(d->gws, L.dres);
  char* dhpre = at(d->gws, L.dhpre);
  TRY(bb_layernorm_bwd(d->dy, 0, at(d->ws, L.fo), 0, d->a, d->gamma, reinterpret_cast<const float*>(at(d->ws, L.mean)),
                       reinterpret_cast<const float*>(at(d->ws, L.rstd)), d->M, d->Hd, d->seed_h, d->th_h, d->sc_h, 0, 0,
                       1.0f, dfo, 0, dres, d->dgamma, d->dbeta, d->db2, stream));
  TRY(lin_bwd_dw(dfo, at(d->ws, L.h), d->dw2, d->M, d->Hd, d->Fd, side_for(stream)));
  TRY(lin_bwd_dx(dfo, d->w2, dhpre, d->M, d->Hd, d->Fd, 1, at(d->ws, L.hpre), nullptr, stream));
  TRY(lin_bwd_dw(dhpre, d->a, d->dw1, d->M, d->Fd, d->Hd, side_for(stream)));
  TRY(bb_colsum_bf16(dhpre, d->M, d->Fd, d->Fd, d->db1, side_for(stream)));
  return lin_bwd_dx(dhpre, d->w1, d->da, d->M, d->Fd, d->Hd, 0, nullptr, dres, stream);
}

// ------------------------------------------------------------------------------------------------ panorama layer
namespace bb {
struct PanoLayout {
  AttnLayout A;   // attention-core regions (P, Pd, ctx / dctx, dP, dS) relative to ws / gws
  int64_t h1, m1, r1, qkv, x1, h2, m2, r2, f, fpre, fwd_bytes;
  int64_t dy3, dfpre, dh2, dx1ln, dx1, d1g, dqkv, dh1, dxln, bwd_bytes;
};
static void pano_attn_desc(const bb_pano_desc* d, bb_attn_desc* a) {
  memset(a, 0, sizeof(*a));
  a->B = d->N; a->nq = d->V; a->nk = d->V; a->Hd = d->Hd; a->heads = d->heads;
  a->kmask = d->kmask; a->seed_attn = d->seed_attn; a->th_attn = d->th_attn; a->sc_attn = d->sc_attn;
  a->ws = d->ws; a->gws = d->gws;
}
static PanoLayout pano_layout(const bb_pano_desc* d) {
  PanoLayout L;
  memset(&L, 0, sizeof(L));
  const int64_t M = (int64_t)d->N * d->V, Hd = d->Hd, Fd = d->Fd;
  const int ldp = round8(d->V);
  const int64_t pn = (int64_t)d->N * d->heads * d->V * ldp;
  const bool fused = d->V <= fused_max_keys() && Hd / d->heads == 64;
  int64_t o = 0;
  L.h1 = o; o += al(M * Hd * 2);
  L.m1 = o; o += al(M * 4);
  L.r1 = o; o += al(M * 4);
  L.qkv = o; o += al(M * 3 * Hd * 2);
  L.A.ldp = ldp;
  bb_attn_desc probe;
  pano_attn_desc(d, &probe);
  const bool flash = flash_on(&probe);
  const int64_t rows = (int64_t)d->N * d->heads * d->V;
  if (flash) {
    L.A.lse = o; o += al(rows * 4);
  } else {
    L.A.S = o; if (!fused) o += al(pn * 4);
    L.A.P = o; o += al(pn * 2);
    if (d->th_attn) { L.A.Pd = o; o += al(pn * 2); } else L.A.Pd = L.A.P;
  }
  L.A.ctx = o; o += al(M * Hd * 2);
  L.x1 = o; o += al(M * Hd * 2);
  L.h2 = o; o += al(M * Hd * 2);
  L.m2 = o; o += al(M * 4);
  L.r2 = o; o += al(M * 4);
  L.f = o; o += al(M * Fd * 2);
  L.fpre = o; o += al(M * Fd * 2);
  L.fwd_bytes = o;
  o = 0;
  L.dy3 = o; o += al(M * Hd * 2);
  L.dfpre = o; o += al(M * Fd * 2);
  L.dh2 = o; o += al(M * Hd * 2);
  L.dx1ln = o; o += al(M * Hd * 2);
  L.dx1 = o; o += al(M * Hd * 2);
  L.d1g = o; o += al(M * Hd * 2);
  L.A.dctx = o; o += al(M * Hd * 2);
  L.dqkv = o; o += al(M * 3 * Hd * 2);
  if (flash) {
    L.A.dsum = o; o += al(rows * 4);
  } else {
    L.A.dP = o; if (!fused) o += al(pn * 4);
    L.A.dS = o; o += al(pn * 2);
  }
  L.dh1 = o; o += al(M * Hd * 2);
  L.dxln = o; o += al(M * Hd * 2);
  L.bwd_bytes = o;
  return L;
}
}  // namespace bb

extern "C" int bb_pano_ws_bytes(const bb_pano_desc* d, int64_t* fwd_bytes, int64_t* bwd_bytes) {
  if (!d) return set_error("bb_pano_ws_bytes: null descriptor");
  const PanoLayout L = pano_layout(d);
  if (fwd_bytes) *fwd_bytes = L.fwd_bytes;
  if (bwd_bytes) *bwd_bytes = L.bwd_bytes;
  return 0;
}

extern "C" int bb_pano_fwd(const bb_pano_desc* d, void* stream) {
  if (!d || !d->x || !d->ws || !d->y) return set_error("bb_pano_fwd: null argument");
  const PanoLayout L = pano_layout(d);
  const int Hd = d->Hd, Fd = d->Fd;
  const int64_t M = (int64_t)d->N * d->V;
  bb_attn_desc a;
  pano_attn_desc(d, &a);
  char* qkv = at(d->ws, L.qkv);
  TRY(bb_layernorm_fwd(d->x, 0, nullptr, d->g1, d->be1, 1e-5f, M, Hd, 0, 0, 1.0f, 0, 0, 1.0f, at(d->ws, L.h1), nullptr,
                       reinterpret_cast<float*>(at(d->ws, L.m1)), reinterpret_cast<float*>(at(d->ws, L.r1)), stream));
  TRY(lin_fwd(at(d->ws, L.h1), d->w_in, qkv, M, 3 * Hd, Hd, d->b_in, 0, nullptr, 0, 0, 1.0f, nullptr, 0, stream));
  TRY(attn_core_fwd(&a, L.A, qkv, 3 * Hd, qkv + (int64_t)Hd * 2, 3 * Hd, qkv + (int64_t)2 * Hd * 2, 3 * Hd, stream));
  TRY(lin_fwd(at(d->ws, L.A.ctx), d->w_out, at(d->ws, L.x1), M, Hd, Hd, d->b_out, 0, nullptr, d->seed1, d->th_h, d->sc_h,
              d->x, 0, stream));
  TRY(bb_layernorm_fwd(at(d->ws, L.x1), 0, nullptr, d->g2, d->be2, 1e-5f, M, Hd, 0, 0, 1.0f, 0, 0, 1.0f, at(d->ws, L.h2),
                       nullptr, reinterpret_cast<float*>(at(d->ws, L.m2)), reinterpret_cast<float*>(at(d->ws, L.r2)),
                       stream));
  TRY(lin_fwd(at(d->ws, L.h2), d->w1, at(d->ws, L.f), M, Fd, Hd, d->b1, 1, at(d->ws, L.fpre), d->seed2, d->th_h, d->sc_h,
              nullptr, 0, stream));
  return lin_fwd(at(d->ws, L.f), d->w2, d->y, M, Hd, Fd, d->b2, 0, nullptr, d->seed3, d->th_h, d->sc_h, at(d->ws, L.x1), 0,
                 stream);
}

extern "C" int bb_pano_bwd(const bb_pano_desc* d, void* stream) {
  if (!d || !d->x || !d->ws || !d->gws || !d->dy || !d->dx) return set_error("bb_pano_bwd: null argument");
  const PanoLayout L = pano_layout(d);
  const int Hd = d->Hd, Fd = d->Fd;
  const int64_t M = (int64_t)d->N * d->V;
  bb_attn_desc a;
  pano_attn_desc(d, &a);
  // y = x1 + drop3(f W2^T + b2)
  const void* dy3 = d->dy;
  if (d->th_h) {
    TRY(bb_dropout_bf16(d->dy, at(d->gws, L.dy3), M * Hd, d->seed3, d->th_h, d->sc_h, stream));
    dy3 = at(d->gws, L.dy3);
  }
  TRY(lin_bwd_dw(dy3, at(d->ws, L.f), d->dw2, M, Hd, Fd, side_for(stream)));
  TRY(bb_colsum_bf16(dy3, M, Hd, Hd, d->db2, side_for(stream)));
  TRY(lin_bwd_dx(dy3, d->w2, at(d->gws, L.dfpre), M, Hd, Fd, 1, at(d->ws, L.fpre), nullptr, stream, d->seed2, d->th_h,
                 d->sc_h));
  TRY(lin_bwd_dw(at(d->gws, L.dfpre), at(d->ws, L.h2), d->dw1, M, Fd, Hd, side_for(stream)));
  TRY(bb_colsum_bf16(at(d->gws, L.dfpre), M, Fd, Fd, d->db1, side_for(stream)));
  TRY(lin_bwd_dx(at(d->gws, L.dfpre), d->w1, at(d->gws, L.dh2), M, Fd, Hd, 0, nullptr, nullptr, stream));
  TRY(bb_layernorm_bwd(at(d->gws, L.dh2), 0, at(d->ws, L.x1), 0, nullptr, d->g2,
                       reinterpret_cast<const float*>(at(d->ws, L.m2)), reinterpret_cast<const float*>(at(d->ws, L.r2)), M,
                       Hd, 0, 0, 1.0f, 0, 0, 1.0f, at(d->gws, L.dx1ln), 0, nullptr, d->dg2, d->dbe2, nullptr, stream));
  TRY(bb_add_bf16(at(d->gws, L.dx1ln), d->dy, at(d->gws, L.dx1), M * Hd, stream));
  // x1 = x + drop1(ctx Wo^T + bo)
  const void* d1g = at(d->gws, L.dx1);
  if (d->th_h) {
    TRY(bb_dropout_bf16(at(d->gws, L.dx1), at(d->gws, L.d1g), M * Hd, d->seed1, d->th_h, d->sc_h, stream));
    d1g = at(d->gws, L.d1g);
  }
  TRY(lin_bwd_dw(d1g, at(d->ws, L.A.ctx), d->dw_out, M, Hd, Hd, side_for(stream)));
  TRY(bb_colsum_bf16(d1g, M, Hd, Hd, d->db_out, side_for(stream)));
  TRY(lin_bwd_dx(d1g, d->w_out, at(d->gws, L.A.dctx), M, Hd, Hd, 0, nullptr, nullptr, stream));
  char* qkv = at(d->ws, L.qkv);
  char* dqkv = at(d->gws, L.dqkv);
  const int Lq = 3 * Hd;
  TRY(attn_core_bwd(&a, L.A, qkv, Lq, qkv + (int64_t)Hd * 2, Lq, qkv + (int64_t)2 * Hd * 2, Lq, dqkv, Lq,
                    dqkv + (int64_t)Hd * 2, Lq, dqkv + (int64_t)2 * Hd * 2, Lq, stream));
  TRY(lin_bwd_dw(dqkv, at(d->ws, L.h1), d->dw_in, M, 3 * Hd, Hd, side_for(stream)));
  TRY(bb_colsum_bf16(dqkv, M, 3 * Hd, 3 * Hd, d->db_in, side_for(stream)));
  TRY(lin_bwd_dx(dqkv, d->w_in, at(d->gws, L.dh1), M, 3 * Hd, Hd, 0, nullptr, nullptr, stream));
  TRY(bb_layernorm_bwd(at(d->gws, L.dh1), 0, d->x, 0, nullptr, d->g1, reinterpret_cast<const float*>(at(d->ws, L.m1)),
                       reinterpret_cast<const float*>(at(d->ws, L.r1)), M, Hd, 0, 0, 1.0f, 0, 0, 1.0f, at(d->gws, L.dxln), 0,
                       nullptr, d->dg1, d->dbe1, nullptr, stream));
  return bb_add_bf16(at(d->gws, L.dxln), at(d->gws, L.dx1), d->dx, M * Hd, stream);
}

extern "C" int bb_set_side_stream(void* side_stream) {
  bb::g_side = (cudaStream_t)side_stream;
  return 0;
}
extern "C" int bb_side_join(void* main_stream) {
  using namespace bb;
  if (!g_side || !g_side_used) return 0;
  static cudaEvent_t ev = nullptr;
  if (!ev) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
  if (cudaEventRecord(ev, g_side) != cudaSuccess || cudaStreamWaitEvent((cudaStream_t)main_stream, ev, 0) != cudaSuccess)
    return set_error("bb_side_join: event record / wait failed");
  g_side_used = false;
  return 0;
}
