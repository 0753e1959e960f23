// Attention core on wgmma tensor cores, fed by TMA, for head dim 64 and >= 64 keys.
//
//   O = dropout(softmax(alpha Q K^T + kmask)) V        per (sample, head), scores / probabilities never leave the SM
//
// Three kernels live here (dispatch at the bottom: launch_fwd / launch_bwd, called from attn_flash.cu):
//   attn_tc_fwd_kernel     forward: a CTA owns 128 queries of one (sample, head); K / V stream through a ring of
//                          shared-memory stages in 64-key blocks;
//   attn_tc_bwd_kernel<M>  backward, dQ pass (M = 0, CTA = 128 queries) and dK / dV pass (M = 1, CTA = 128 keys).
// Every CTA is two consumer warpgroups (warps 0..7, 64 rows each) and one TMA producer warp (warp 8).  Scores are
// wgmma accumulators in registers: thread t of a warpgroup holds rows r0 = 16 (t / 32) + (t % 32) / 4 and r0 + 8 and,
// of every 8-column group, columns 2 (t % 4) and 2 (t % 4) + 1, so a row lives in the four threads of a quad and row
// reductions are two shuffles.  That fragment, converted to bf16, is exactly the register A operand of the next
// wgmma (P V, dS K, P^T dO, dS^T Q), so probabilities and score gradients never touch shared memory; the other
// operand of those products is the K / V / Q / dO tile read MN-major from the same 128B-swizzled TMA tile.
// The forward keeps a running row maximum (online softmax, O rescaled when it grows).
//
// Reference semantics: BertSelfAttention / BertOutAttention (vilmodel.py:103-154, 325-363); same dropout function and
// log2-domain LSE as csrc/attn_flash.cu (mma.sync path, kept for < 64 keys and for the graph-bias case).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/bevbert_b200.h"
#include "attn_tc.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {
namespace fat {

typedef __nv_bfloat16 bf16;
constexpr int BM = 128;          // rows per CTA (two warpgroups of 64)
constexpr int KB = 64;           // keys (forward, MODE 0) or queries (MODE 1) per streamed block
constexpr int NT = 288;          // 8 consumer warps + 1 producer warp
constexpr int NST = 3;           // depth of the streamed-block ring
constexpr int R_BYTES = BM * 128, BLK_BYTES = KB * 128;
constexpr float LOG2E = 1.4426950408889634f;

struct FwdParams {
  bf16* out;
  int64_t o_bs;
  int ldo;
  float* lse;
  const float* kmask;
  int B, H, nq, nk;
  float a2;           // alpha * log2(e)
  uint64_t seed;
  uint32_t thresh;
  float scale;
};

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// same decisions as csrc/attn_flash.cu: one hash per (sample, head, query) row, one mix per PAIR of adjacent keys
__device__ __forceinline__ uint32_t mix_pair(uint32_t rowhash, uint32_t pair) {
  // one multiply-xorshift round on a Weyl step of the (already fully mixed) row hash: 6 integer instructions per
  // PAIR of keys; measured on 20000 x 512 decisions at p = 0.1: drop rate 0.10003, adjacent-key correlation < 1e-4
  uint32_t x = rowhash + pair * 0x9E3779B1u;
  x ^= x >> 15;
  x *= 0x2C1B3C6Du;
  x ^= x >> 16;
  return x;
}
// keep decision of key k (of the pair hash x): the even key of a pair tests the low 16 bits, the odd key the high 16
__device__ __forceinline__ bool keep_key(uint32_t x, int k, uint32_t t16s) {
  return (k & 1) ? x >= t16s : (x << 16) >= t16s;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// accumulator fragment (64 columns) -> bf16 A-operand fragments of the four 16-deep K steps
__device__ __forceinline__ void to_afrag(const float (&s)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int i = 0; i < 4; ++i) a[kk][i] = pack2(s[8 * kk + 2 * i], s[8 * kk + 2 * i + 1]);
}
// S (+)= A B^T over head dim 64, A and B both K-major 64-row tiles in shared memory
__device__ __forceinline__ void qk_product(float (&s)[32], uint32_t a, uint32_t b) {
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_m64n64_ss<0, 0>(s, wgmma_desc(a + k * 32, 16, 1024), wgmma_desc(b + k * 32, 16, 1024), k > 0 ? 1u : 0u);
}
// D += P X with P the register fragment (64 rows x 64) and X a [64][64] tile read MN-major
__device__ __forceinline__ void pv_product(float (&d)[32], const uint32_t (&a)[4][4], uint32_t x) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wgmma_m64n64_rs<1>(d, a[kk], wgmma_desc(x + kk * 2048, 8192, 1024), 1u);
}
__device__ __forceinline__ void store_row_pair(bf16* dst, float v0, float v1) {
  *reinterpret_cast<uint32_t*>(dst) = pack2(v0, v1);
}

// ================================================================================================ forward
__global__ void __launch_bounds__(NT, 1)
attn_tc_fwd_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                   const __grid_constant__ CUtensorMap tv, const FwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + R_BYTES;
  uint8_t* sV = sK + NST * BLK_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + NST * BLK_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;          // [NST]
  uint64_t* kv_free = bars + 1 + NST;    // [NST]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BM, h = blockIdx.y, b = blockIdx.z;
  const int nblk = (p.nk + KB - 1) / KB;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tq);
    tma_prefetch_desc(&tk);
    tma_prefetch_desc(&tv);
    mbar_init(q_full, 1);
    for (int i = 0; i < NST; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_free[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      mbar_expect_tx(q_full, R_BYTES);
      tma_load_4d(sQ, &tq, q_full, 0, q0, h, b);
      for (int j = 0; j < nblk; ++j) {
        const int st = j % NST;
        mbar_wait_relaxed(&kv_free[st], ((j / NST) & 1) ^ 1);
        mbar_expect_tx(&kv_full[st], 2 * BLK_BYTES);
        tma_load_4d(sK + st * BLK_BYTES, &tk, &kv_full[st], 0, j * KB, h, b);
        tma_load_4d(sV + st * BLK_BYTES, &tv, &kv_full[st], 0, j * KB, h, b);
      }
    }
    return;
  }
  // -------------------------------------------------------------------- consumers (softmax + epilogue)
  const int wg = warp >> 2;
  const int r0 = (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t t16s = p.thresh & 0xFFFF0000u;
  int q[2];
  uint32_t rh[2];
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    q[hh] = q0 + wg * 64 + r0 + 8 * hh;
    rh[hh] = p.thresh ? rng_u32(p.seed, (uint64_t)(((int64_t)b * p.H + h) * p.nq + q[hh])) : 0u;
  }
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  const uint32_t aQ = smem_u32(sQ) + wg * 8192;
  mbar_wait(q_full, 0);
  for (int j = 0; j < nblk; ++j) {
    const int st = j % NST;
    float km[16];   // log2-domain key mask of this thread's 16 columns
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = j * KB + 8 * jj + cq + e;
        km[2 * jj + e] = c < p.nk ? (p.kmask ? __ldg(p.kmask + (int64_t)b * p.nk + c) * LOG2E : 0.f) : -INFINITY;
      }
    mbar_wait(&kv_full[st], (j / NST) & 1);
    float s[32];
    fence_regs(s);
    wgmma_fence();
    qk_product(s, aQ, smem_u32(sK + st * BLK_BYTES));
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float& v = s[4 * jj + i];
        v = fmaf(v, p.a2, km[2 * jj + (i & 1)]);
        mx[i >> 1] = fmaxf(mx[i >> 1], v);
      }
    float ms[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float mn = fmaxf(m[hh], quad_max(mx[hh]));
      ms[hh] = mn == -INFINITY ? 0.f : mn;
      const float corr = ex2f(m[hh] - ms[hh]);
      m[hh] = mn;
      l[hh] *= corr;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        o[4 * jj + 2 * hh] *= corr;
        o[4 * jj + 2 * hh + 1] *= corr;
      }
    }
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int c = j * KB + 8 * jj + cq;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float e0 = ex2f(s[4 * jj + 2 * hh] - ms[hh]), e1 = ex2f(s[4 * jj + 2 * hh + 1] - ms[hh]);
        l[hh] += e0 + e1;
        if (p.thresh) {     // kept probabilities are NOT rescaled here: 1/(1-p) is folded into the O epilogue
          const uint32_t x = mix_pair(rh[hh], (uint32_t)c >> 1);
          e0 = keep_key(x, c, t16s) ? e0 : 0.f;
          e1 = keep_key(x, c + 1, t16s) ? e1 : 0.f;
        }
        s[4 * jj + 2 * hh] = e0;
        s[4 * jj + 2 * hh + 1] = e1;
      }
    }
    uint32_t a[4][4];
    to_afrag(s, a);
    fence_regs(o);
    wgmma_fence();
    pv_product(o, a, smem_u32(sV + st * BLK_BYTES));
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    if (lane == 0) mbar_arrive(&kv_free[st]);
  }
  // ---- epilogue: normalise, store bf16 rows and the log2-domain log-sum-exp
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float lt = quad_sum(l[hh]);
    if (q[hh] >= p.nq) continue;
    const float inv = lt > 0.f ? (p.thresh ? p.scale : 1.0f) / lt : 0.f;
    bf16* dst = p.out + (int64_t)b * p.o_bs + (int64_t)q[hh] * p.ldo + h * 64 + cq;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) store_row_pair(dst + 8 * jj, o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
    if ((lane & 3) == 0 && p.lse)
      p.lse[((int64_t)b * p.H + h) * p.nq + q[hh]] = lt > 0.f ? m[hh] + log2f(lt) : INFINITY;
  }
}

// ================================================================================================ backward
// Two passes over the (query x key) grid of a (sample, head), both with P = 2^(a2 S + kmask - lse) recomputed from the
// forward's log-sum-exp and dS = alpha P o (drop(dP) - D):
//   MODE 0 (CTA = 128 queries): D = rowsum(dO o O);  per 64-key block: S = Q K^T, dP = dO V^T -> dS -> dQ += dS K
//   MODE 1 (CTA = 128 keys)   : per 64-query block: S^T = K Q^T, dP^T = V dO^T -> Pdrop^T, dS^T
//                               -> dV += Pdrop^T dO, dK += dS^T Q
// MODE 1 forms the transposed products directly, so its fragments have keys as rows and feed the accumulating
// products as register A operands without any transposition.  No atomics.
struct BwdParams {
  const bf16 *o, *dout;
  bf16 *dq, *dk, *dv;
  int64_t o_bs, do_bs, dq_bs, dk_bs, dv_bs;
  int ldo, lddo, lddq, lddk, lddv;
  const float* lse;
  float* dsum;
  const float* kmask;
  int B, H, nq, nk;
  float a2, alpha;
  uint64_t seed;
  uint32_t thresh;
  float scale;
};

// tr0 / tr1: the CTA's resident 128-row tiles (Q, dO for MODE 0; K, V for MODE 1), box 128 rows;
// ts0 / ts1: the streamed 64-row blocks (K, V for MODE 0; Q, dO for MODE 1), box 64 rows.
template <int MODE>
__global__ void __launch_bounds__(NT, 1)
attn_tc_bwd_kernel(const __grid_constant__ CUtensorMap tr0, const __grid_constant__ CUtensorMap tr1,
                   const __grid_constant__ CUtensorMap ts0, const __grid_constant__ CUtensorMap ts1, const BwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sR0 = smem;
  uint8_t* sR1 = sR0 + R_BYTES;
  uint8_t* sS0 = sR1 + R_BYTES;             // [NST] streamed block 0 (K_j / Q_i)
  uint8_t* sS1 = sS0 + NST * BLK_BYTES;     // [NST] streamed block 1 (V_j / dO_i)
  uint64_t* bars = reinterpret_cast<uint64_t*>(sS1 + NST * BLK_BYTES);
  uint64_t* r_full = bars;
  uint64_t* st_full = bars + 1;          // [NST]
  uint64_t* st_free = bars + 1 + NST;    // [NST]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t0 = blockIdx.x * BM, h = blockIdx.y, b = blockIdx.z;   // first query (MODE 0) / key (MODE 1) of this CTA
  const int nblk = MODE == 0 ? (p.nk + KB - 1) / KB : (p.nq + KB - 1) / KB;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tr0);
    tma_prefetch_desc(&tr1);
    tma_prefetch_desc(&ts0);
    tma_prefetch_desc(&ts1);
    mbar_init(r_full, 1);
    for (int i = 0; i < NST; ++i) {
      mbar_init(&st_full[i], 1);
      mbar_init(&st_free[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(r_full, 2 * R_BYTES);
      tma_load_4d(sR0, &tr0, r_full, 0, t0, h, b);
      tma_load_4d(sR1, &tr1, r_full, 0, t0, h, b);
      for (int j = 0; j < nblk; ++j) {
        const int st = j % NST;
        mbar_wait_relaxed(&st_free[st], ((j / NST) & 1) ^ 1);
        mbar_expect_tx(&st_full[st], 2 * BLK_BYTES);
        tma_load_4d(sS0 + st * BLK_BYTES, &ts0, &st_full[st], 0, j * KB, h, b);
        tma_load_4d(sS1 + st * BLK_BYTES, &ts1, &st_full[st], 0, j * KB, h, b);
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const int r0 = (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t t16s = p.thresh & 0xFFFF0000u;
  const float scale_eff = p.thresh ? p.scale : 1.0f, inv_scale = 1.0f / scale_eff, as_ = p.alpha * scale_eff;
  const int64_t bh = (int64_t)b * p.H + h;
  const uint32_t aR0 = smem_u32(sR0) + wg * 8192, aR1 = smem_u32(sR1) + wg * 8192;
  int row[2];   // this thread's two rows: queries (MODE 0) / keys (MODE 1)
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) row[hh] = t0 + wg * 64 + r0 + 8 * hh;

  // per-row state: MODE 0 -> -lse, D / scale and the dropout row hash of the query; MODE 1 -> key mask of the key
  float rs_a[2], rs_b[2];
  uint32_t rh[2] = {0u, 0u};
  if (MODE == 0) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int qq = row[hh];
      const bool ok = qq < p.nq;
      // D = rowsum(dO o O): each thread of the quad covers 16 of the 64 columns
      float acc = 0.f;
      if (ok) {
        const uint4* po = reinterpret_cast<const uint4*>(p.o + (int64_t)b * p.o_bs + (int64_t)qq * p.ldo + h * 64 + (lane & 3) * 16);
        const uint4* pd = reinterpret_cast<const uint4*>(p.dout + (int64_t)b * p.do_bs + (int64_t)qq * p.lddo + h * 64 + (lane & 3) * 16);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const uint4 a = __ldg(po + i), d = __ldg(pd + i);
          const __nv_bfloat162* ap = reinterpret_cast<const __nv_bfloat162*>(&a);
          const __nv_bfloat162* dp = reinterpret_cast<const __nv_bfloat162*>(&d);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 x = __bfloat1622float2(ap[e]), y = __bfloat1622float2(dp[e]);
            acc = fmaf(x.x, y.x, acc);
            acc = fmaf(x.y, y.y, acc);
          }
        }
      }
      acc = quad_sum(acc);
      if (ok && (lane & 3) == 0) p.dsum[bh * p.nq + qq] = acc;
      rs_a[hh] = ok ? -__ldg(p.lse + bh * p.nq + qq) : -INFINITY;
      rs_b[hh] = acc * inv_scale;
      rh[hh] = p.thresh ? rng_u32(p.seed, (uint64_t)(bh * p.nq + qq)) : 0u;
    }
  } else {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int kk = row[hh];
      rs_a[hh] = kk < p.nk ? (p.kmask ? __ldg(p.kmask + (int64_t)b * p.nk + kk) * LOG2E : 0.f) : -INFINITY;
      rs_b[hh] = 0.f;
    }
  }

  float acc0[32], acc1[32];   // dQ (MODE 0) / dV, dK (MODE 1)
#pragma unroll
  for (int i = 0; i < 32; ++i) acc0[i] = acc1[i] = 0.f;
  mbar_wait(r_full, 0);
  for (int j = 0; j < nblk; ++j) {
    const int st = j % NST;
    mbar_wait(&st_full[st], (j / NST) & 1);
    const uint32_t a0 = smem_u32(sS0 + st * BLK_BYTES), a1 = smem_u32(sS1 + st * BLK_BYTES);
    float s[32], g[32];
    fence_regs(s);
    fence_regs(g);
    wgmma_fence();
    qk_product(s, aR0, a0);   // S = Q K^T (MODE 0) / S^T = K Q^T (MODE 1)
    qk_product(g, aR1, a1);   // dP = dO V^T        / dP^T = V dO^T
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    fence_regs(g);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int c = j * KB + 8 * jj + cq;
      // per-column state: MODE 0 -> key mask; MODE 1 -> -lse, D / scale and the dropout hash of the query
      float ca[2], cb[2] = {0.f, 0.f};
      uint32_t ch[2] = {0u, 0u};
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        if (MODE == 0) {
          ca[e] = c + e < p.nk ? (p.kmask ? __ldg(p.kmask + (int64_t)b * p.nk + c + e) * LOG2E : 0.f) : -INFINITY;
        } else {
          const bool ok = c + e < p.nq;
          ca[e] = ok ? -__ldg(p.lse + bh * p.nq + c + e) : -INFINITY;
          cb[e] = ok ? __ldg(p.dsum + bh * p.nq + c + e) * inv_scale : 0.f;
          ch[e] = p.thresh ? rng_u32(p.seed, (uint64_t)(bh * p.nq + c + e)) : 0u;
        }
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float pe[2], pd[2], ds[2];
        // the dropout hash is keyed by (query, key pair): MODE 0 rows are queries, MODE 1 rows are keys
        const uint32_t x = p.thresh ? (MODE == 0 ? mix_pair(rh[hh], (uint32_t)c >> 1) : 0u) : 0u;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 4 * jj + 2 * hh + e;
          float gv = g[i];
          float dsub;
          if (MODE == 0) {
            pe[e] = ex2f(fmaf(s[i], p.a2, ca[e] + rs_a[hh]));
            dsub = rs_b[hh];
            pd[e] = pe[e];
            if (p.thresh && !keep_key(x, c + e, t16s)) gv = 0.f;
          } else {
            pe[e] = ex2f(fmaf(s[i], p.a2, rs_a[hh] + ca[e]));
            dsub = cb[e];
            pd[e] = pe[e];
            if (p.thresh) {
              const uint32_t xk = mix_pair(ch[e], (uint32_t)row[hh] >> 1);
              if (!keep_key(xk, row[hh], t16s)) {
                gv = 0.f;
                pd[e] = 0.f;
              }
            }
          }
          ds[e] = (pe[e] * as_) * (gv - dsub);
        }
        s[4 * jj + 2 * hh] = pd[0];
        s[4 * jj + 2 * hh + 1] = pd[1];
        g[4 * jj + 2 * hh] = ds[0];
        g[4 * jj + 2 * hh + 1] = ds[1];
      }
    }
    uint32_t fds[4][4];
    to_afrag(g, fds);
    fence_regs(acc0);
    fence_regs(acc1);
    wgmma_fence();
    if (MODE == 0) {
      pv_product(acc0, fds, a0);            // dQ += dS K_j
    } else {
      uint32_t fpd[4][4];
      to_afrag(s, fpd);
      pv_product(acc0, fpd, a1);            // dV += Pdrop^T dO_i
      pv_product(acc1, fds, a0);            // dK += dS^T Q_i
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(acc0);
    fence_regs(acc1);
    if (lane == 0) mbar_arrive(&st_free[st]);
  }

  // ---- accumulators -> bf16 rows (MODE 0: dQ rows = queries; MODE 1: dV / dK rows = keys)
  const int nrows = MODE == 0 ? p.nq : p.nk;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int64_t r = row[hh];
    if (r >= nrows) continue;
    if (MODE == 0) {
      bf16* dst = p.dq + (int64_t)b * p.dq_bs + r * p.lddq + h * 64 + cq;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) store_row_pair(dst + 8 * jj, acc0[4 * jj + 2 * hh], acc0[4 * jj + 2 * hh + 1]);
    } else {
      bf16* dv = p.dv + (int64_t)b * p.dv_bs + r * p.lddv + h * 64 + cq;   // Pdrop is unscaled
      bf16* dk = p.dk + (int64_t)b * p.dk_bs + r * p.lddk + h * 64 + cq;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        store_row_pair(dv + 8 * jj, acc0[4 * jj + 2 * hh] * scale_eff, acc0[4 * jj + 2 * hh + 1] * scale_eff);
        store_row_pair(dk + 8 * jj, acc1[4 * jj + 2 * hh], acc1[4 * jj + 2 * hh + 1]);
      }
    }
  }
}

constexpr size_t FWD_SMEM = 1024 + R_BYTES + 2 * (size_t)NST * BLK_BYTES + (1 + 2 * NST) * 8;
constexpr size_t BWD_SMEM = 1024 + 2 * R_BYTES + 2 * (size_t)NST * BLK_BYTES + (1 + 2 * NST) * 8;

static int g_init = 0;
static int init_once() {
  if (g_init) return 0;
  if (cudaFuncSetAttribute(attn_tc_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FWD_SMEM) != cudaSuccess ||
      cudaFuncSetAttribute(attn_tc_bwd_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM) != cudaSuccess ||
      cudaFuncSetAttribute(attn_tc_bwd_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM) != cudaSuccess)
    return set_error("cudaFuncSetAttribute failed for the attn_tc kernels");
  g_init = 1;
  return 0;
}

// BB_ATTN_TC: 0 = never, 1 (default) = when nk >= 64, 2 = whenever the kernel supports the call (tests)
static int g_tc_mode = -1;
int tc_mode() {
  if (g_tc_mode < 0) {
    const char* e = getenv("BB_ATTN_TC");
    g_tc_mode = e ? atoi(e) : 1;
  }
  return g_tc_mode;
}
int set_tc_mode(int mode) {
  const int prev = tc_mode();
  g_tc_mode = mode;
  return prev;
}

bool fwd_supported(const bb_flash_args* a) {
  const int mode = tc_mode();
  if (mode == 0 || a->dh != 64 || a->bias != nullptr) return false;
  if (mode == 1 && a->nk < 64) return false;
  const uintptr_t al = reinterpret_cast<uintptr_t>(a->q) | reinterpret_cast<uintptr_t>(a->k) |
                       reinterpret_cast<uintptr_t>(a->v) | reinterpret_cast<uintptr_t>(a->o);
  if (al & 15) return false;
  if ((a->ldq | a->ldk | a->ldv | a->ldo) % 8) return false;
  if ((a->q_bs | a->k_bs | a->v_bs | a->o_bs) % 8) return false;
  return true;
}

int launch_fwd(const bb_flash_args* a, void* stream) {
  if (int e = init_once()) return e;
  FwdParams p;
  memset(&p, 0, sizeof(p));
  p.out = (bf16*)a->o; p.o_bs = a->o_bs; p.ldo = a->ldo; p.lse = a->lse; p.kmask = a->kmask;
  p.B = a->B; p.H = a->H; p.nq = a->nq; p.nk = a->nk;
  p.a2 = a->alpha * LOG2E;
  p.seed = a->seed; p.thresh = a->thresh; p.scale = a->scale;
  CUtensorMap tq, tk, tv;
  if (int e = make_tmap_bf16_4d(&tq, a->q, 64, a->nq, a->H, a->B, a->ldq, 64, a->q_bs, BM)) return e;
  if (int e = make_tmap_bf16_4d(&tk, a->k, 64, a->nk, a->H, a->B, a->ldk, 64, a->k_bs, KB)) return e;
  if (int e = make_tmap_bf16_4d(&tv, a->v, 64, a->nk, a->H, a->B, a->ldv, 64, a->v_bs, KB)) return e;
  const dim3 grid((unsigned)((a->nq + BM - 1) / BM), (unsigned)a->H, (unsigned)a->B);
  launch_pdl(attn_tc_fwd_kernel, grid, dim3(NT), FWD_SMEM, (cudaStream_t)stream, tq, tk, tv, p);
  count_launch();
  return check_launch("attn_tc_fwd_kernel");
}

bool bwd_supported(const bb_flash_args* a) {
  if (!fwd_supported(a) || a->dbias != nullptr) return false;
  const uintptr_t al = reinterpret_cast<uintptr_t>(a->dout) | reinterpret_cast<uintptr_t>(a->dq) |
                       reinterpret_cast<uintptr_t>(a->dk) | reinterpret_cast<uintptr_t>(a->dv);
  if (al & 15) return false;
  if ((a->lddo | a->lddq | a->lddk | a->lddv) % 8) return false;
  if ((a->do_bs | a->dq_bs | a->dk_bs | a->dv_bs) % 8) return false;
  return true;
}

int launch_bwd(const bb_flash_args* a, void* stream) {
  if (int e = init_once()) return e;
  BwdParams p;
  memset(&p, 0, sizeof(p));
  p.o = (const bf16*)a->o; p.dout = (const bf16*)a->dout;
  p.dq = (bf16*)a->dq; p.dk = (bf16*)a->dk; p.dv = (bf16*)a->dv;
  p.o_bs = a->o_bs; p.do_bs = a->do_bs; p.dq_bs = a->dq_bs; p.dk_bs = a->dk_bs; p.dv_bs = a->dv_bs;
  p.ldo = a->ldo; p.lddo = a->lddo; p.lddq = a->lddq; p.lddk = a->lddk; p.lddv = a->lddv;
  p.lse = a->lse; p.dsum = a->dsum; p.kmask = a->kmask;
  p.B = a->B; p.H = a->H; p.nq = a->nq; p.nk = a->nk;
  p.a2 = a->alpha * LOG2E; p.alpha = a->alpha;
  p.seed = a->seed; p.thresh = a->thresh; p.scale = a->scale;
  CUtensorMap tq, tk, tv, tdo, tq64, tk64, tv64, tdo64;
  if (int e = make_tmap_bf16_4d(&tq, a->q, 64, a->nq, a->H, a->B, a->ldq, 64, a->q_bs, BM)) return e;
  if (int e = make_tmap_bf16_4d(&tdo, a->dout, 64, a->nq, a->H, a->B, a->lddo, 64, a->do_bs, BM)) return e;
  if (int e = make_tmap_bf16_4d(&tk, a->k, 64, a->nk, a->H, a->B, a->ldk, 64, a->k_bs, BM)) return e;
  if (int e = make_tmap_bf16_4d(&tv, a->v, 64, a->nk, a->H, a->B, a->ldv, 64, a->v_bs, BM)) return e;
  if (int e = make_tmap_bf16_4d(&tq64, a->q, 64, a->nq, a->H, a->B, a->ldq, 64, a->q_bs, KB)) return e;
  if (int e = make_tmap_bf16_4d(&tdo64, a->dout, 64, a->nq, a->H, a->B, a->lddo, 64, a->do_bs, KB)) return e;
  if (int e = make_tmap_bf16_4d(&tk64, a->k, 64, a->nk, a->H, a->B, a->ldk, 64, a->k_bs, KB)) return e;
  if (int e = make_tmap_bf16_4d(&tv64, a->v, 64, a->nk, a->H, a->B, a->ldv, 64, a->v_bs, KB)) return e;
  const dim3 gq((unsigned)((a->nq + BM - 1) / BM), (unsigned)a->H, (unsigned)a->B);
  const dim3 gk((unsigned)((a->nk + BM - 1) / BM), (unsigned)a->H, (unsigned)a->B);
  launch_pdl(attn_tc_bwd_kernel<0>, gq, dim3(NT), BWD_SMEM, (cudaStream_t)stream, tq, tdo, tk64, tv64, p);
  launch_pdl(attn_tc_bwd_kernel<1>, gk, dim3(NT), BWD_SMEM, (cudaStream_t)stream, tk, tv, tq64, tdo64, p);
  count_launch(2);
  return check_launch("attn_tc_bwd kernels");
}

}  // namespace fat
}  // namespace bb

extern "C" int bb_set_attn_tc(int mode) { return bb::fat::set_tc_mode(mode); }
// kept for the C ABI: the wgmma kernels record no per-CTA trace
extern "C" int bb_attn_tc_trace(long long* device_buf) {
  (void)device_buf;
  return 0;
}

namespace bb { int set_salt_attn_tc(const unsigned long long* p) { return set_drop_salt_ptr_tu(p) == cudaSuccess ? 0 : -1; } }
