// Fused attention core for head dim 64: softmax(alpha Q K^T + kmask + bias) V with probability dropout, forward and
// backward, without ever writing the (nq x nk) score / probability matrices to HBM.
//
// Why a separate kernel next to the wgmma GEMM: on this path the attention products are tiny per (sample, head)
// problems -- 80x80, 36x36, ~23x23, 23x80, 441x80 and 441x441, all with K = 64 -- 384..2148 of them per launch.  As
// batched GEMMs they are one k-block per tile, so the unfused sequence (QK^T -> fp32 scores -> softmax kernel -> P ->
// PV, and five launches in backward) is bound by writing and re-reading the score matrices (0.3 GB per 441-key layer)
// and by per-launch latency, not by tensor throughput (measured 48 TFLOP/s on the 441x441x64 score GEMM).  Here one CTA
// owns 64 queries (or 64 keys) of one (sample, head), streams the other side through shared memory in 64-row tiles
// with cp.async, keeps S / P / dS in registers (warp-level mma.sync m16n8k16 bf16, fp32 accumulate; the tiles are too
// small for a 64-row warpgroup instruction to pay) and uses the online-softmax recurrence, so HBM traffic is Q, K, V,
// O (+ dO, dQ, dK, dV) only.  Backward recomputes P from the saved row log-sum-exp:
//   kernel A (per 64 queries): D = rowsum(dO * O), dQ = alpha * dS K,            dbias += dS
//   kernel B (per 64 keys)   : dV = Pdrop^T dO,    dK = alpha * dS^T Q
// with dS = P * (drop(dP) - D), dP = dO V^T.  No atomics except the (B,nq,nk) bias gradient (summed over heads).
//
// Reference semantics: BertSelfAttention / BertOutAttention (vilmodel.py:103-154, 325-363) and the attention inside
// nn.MultiheadAttention of the panorama encoder (transformer.py:170-182).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../include/bevbert_b200.h"
#include "attn_tc.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {
namespace fa {

typedef __nv_bfloat16 bf16;

constexpr int BM = 64;   // rows owned by a CTA (queries in fwd / kernel A, keys in kernel B)
constexpr int BN = 64;   // rows of a streamed tile
constexpr int DH = 64;   // head dim
constexpr int NT = 128;  // 4 warps, 16 owned rows each
constexpr int TILE_BYTES = 64 * 128;
constexpr float LOG2E = 1.4426950408889634f;

struct Params {
  const bf16 *q, *k, *v, *o, *dout;
  bf16 *out, *dq, *dk, *dv;
  int64_t q_bs, k_bs, v_bs, o_bs, do_bs, dq_bs, dk_bs, dv_bs;  // elements between samples
  int ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv;              // elements between rows
  float* lse;    // (B,H,nq) row log-sum-exp, log2 domain
  float* dsum;   // (B,H,nq) rowsum(dO * O)
  const float* kmask;
  const float* bias;
  float* dbias;
  int64_t dbias_hs;   // deterministic mode: per-head partials dbias + h * dbias_hs, plain stores; 0: fp32 atomics
  int B, H, nq, nk;
  float alpha;
  uint64_t seed;
  uint32_t thresh;
  float scale;
};

// ------------------------------------------------------------------------------------------------ primitives
// 64 x 64 bf16 tile, 128 B per row, 16-byte chunks XOR-swizzled by the row so ldmatrix is conflict-free
__device__ __forceinline__ uint32_t swz(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;   // 0 source bytes -> the 16 destination bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// rows [0, rows_valid) of a (rows x 64) bf16 matrix at g (row stride ld elements) -> swizzled tile; the rest zero
__device__ __forceinline__ void load_tile(uint32_t tile, const bf16* g, int ld, int rows_valid, int tid) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = tid + i * NT, row = c >> 3, ch = c & 7;
    const bool ok = row < rows_valid;
    cp_async16(tile + swz(row, ch), ok ? (const void*)(g + (int64_t)row * ld + ch * 8) : (const void*)g, ok);
  }
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// A-operand fragments of the warp's 16 rows [row0, row0+16) x 64 columns of a [row][col] tile
__device__ __forceinline__ void load_a_frags(uint32_t tile, int row0, int lane, uint32_t (&f)[4][4]) {
  const int row = row0 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) ldsm_x4(tile + swz(row, kk * 2 + (lane >> 4)), f[kk][0], f[kk][1], f[kk][2], f[kk][3]);
}
// acc[nb] (16 x 8 each, nb = 0..7 over the tile's 64 rows) += A(16 x 64) * T^T, T = [n][k] tile (64 x 64)
__device__ __forceinline__ void mma_a_tT(float (&acc)[8][4], const uint32_t (&a)[4][4], uint32_t tile, int lane) {
  const int nrow = (lane & 7) + (lane >> 4) * 8, kc = (lane >> 3) & 1;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b0, b1, b2, b3;
      ldsm_x4(tile + swz(np * 16 + nrow, kk * 2 + kc), b0, b1, b2, b3);
      mma_bf16(acc[2 * np], a[kk], b0, b1);
      mma_bf16(acc[2 * np + 1], a[kk], b2, b3);
    }
  }
}
// acc[nb] (16 x 8 each, nb over the 64 columns of T) += P(16 x 64, given as C-layout fp32 -> bf16) * T, T = [k][n] tile
__device__ __forceinline__ void mma_p_t(float (&acc)[8][4], const float (&p)[8][4], uint32_t tile, int lane) {
  const int krow = (lane & 7) + ((lane >> 3) & 1) * 8, nc = lane >> 4;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t a[4];
    a[0] = pack_bf16(p[2 * kk][0], p[2 * kk][1]);
    a[1] = pack_bf16(p[2 * kk][2], p[2 * kk][3]);
    a[2] = pack_bf16(p[2 * kk + 1][0], p[2 * kk + 1][1]);
    a[3] = pack_bf16(p[2 * kk + 1][2], p[2 * kk + 1][3]);
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b0, b1, b2, b3;
      ldsm_x4_t(tile + swz(kk * 16 + krow, np * 2 + nc), b0, b1, b2, b3);
      mma_bf16(acc[2 * np], a, b0, b1);
      mma_bf16(acc[2 * np + 1], a, b2, b3);
    }
  }
}
// the warp's 16 x 64 fp32 accumulator (C layout) -> bf16 rows of `tile` (its own 16 rows), then coalesced 16-byte stores
__device__ __forceinline__ void store_rows(uint32_t tile, uint8_t* tile_ptr, const float (&acc)[8][4], int row0, int lane,
                                           bf16* g, int ld, int rows_valid) {
  const int gq = lane >> 2, t = lane & 3;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    const int r0 = row0 + gq, r1 = r0 + 8;
    *reinterpret_cast<uint32_t*>(tile_ptr + swz(r0, nb) + t * 4) = pack_bf16(acc[nb][0], acc[nb][1]);
    *reinterpret_cast<uint32_t*>(tile_ptr + swz(r1, nb) + t * 4) = pack_bf16(acc[nb][2], acc[nb][3]);
  }
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = lane + i * 32, row = row0 + (c >> 3), ch = c & 7;
    if (row < rows_valid)
      *reinterpret_cast<uint4*>(g + (int64_t)row * ld + ch * 8) = *reinterpret_cast<const uint4*>(tile_ptr + swz(row, ch));
  }
  (void)tile;
}

// Dropout decisions for the attention probabilities: one full hash per (sample, head, query) row, then one cheap
// two-round mix per PAIR of adjacent keys whose 16-bit halves decide the two elements (keep iff half >= thresh >> 16).
// Forward and both backward kernels evaluate the same function of (seed, b, h, q, k).
__device__ __forceinline__ uint32_t row_hash(uint64_t seed, int64_t row) { return rng_u32(seed, (uint64_t)row); }
__device__ __forceinline__ uint32_t mix_pair(uint32_t rowhash, uint32_t pair) {
  // one multiply-xorshift round on a Weyl step of the (already fully mixed) row hash: 6 integer instructions per
  // PAIR of keys; measured on 20000 x 512 decisions at p = 0.1: drop rate 0.10003, adjacent-key correlation < 1e-4
  uint32_t x = rowhash + pair * 0x9E3779B1u;
  x ^= x >> 15;
  x *= 0x2C1B3C6Du;
  x ^= x >> 16;
  return x;
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// log2-domain additive key mask of tile j (kmask * log2e; -inf beyond nk) -> smem, one float per key
__device__ __forceinline__ void stage_kmask(float* km, const Params& p, int b, int j, int tid) {
  if (tid < BN) {
    const int col = j * BN + tid;
    km[tid] = col < p.nk ? (p.kmask ? p.kmask[(int64_t)b * p.nk + col] * LOG2E : 0.f) : -INFINITY;
  }
}
// s (C layout: rows r0 / r0+8 = queries, cols = keys of tile j) -> log2-domain logits (alpha s + kmask + bias) log2e
__device__ __forceinline__ void logits_qk(float (&s)[8][4], const Params& p, const float* km, int b, int r0, int j, int t) {
  const float a2 = p.alpha * LOG2E;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    const float2 m = *reinterpret_cast<const float2*>(km + nb * 8 + 2 * t);
    s[nb][0] = fmaf(s[nb][0], a2, m.x);
    s[nb][1] = fmaf(s[nb][1], a2, m.y);
    s[nb][2] = fmaf(s[nb][2], a2, m.x);
    s[nb][3] = fmaf(s[nb][3], a2, m.y);
  }
  if (p.bias) {   // graph bias of the global map encoder only (few, small problems)
    const float* bs0 = r0 < p.nq ? p.bias + ((int64_t)b * p.nq + r0) * p.nk : nullptr;
    const float* bs1 = r0 + 8 < p.nq ? p.bias + ((int64_t)b * p.nq + r0 + 8) * p.nk : nullptr;
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = j * BN + nb * 8 + 2 * t + e;
        if (col < p.nk) {
          if (bs0) s[nb][e] = fmaf(bs0[col], LOG2E, s[nb][e]);
          if (bs1) s[nb][2 + e] = fmaf(bs1[col], LOG2E, s[nb][2 + e]);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ forward
__global__ void __launch_bounds__(NT, 4) flash_fwd_kernel(const Params p) {
  __shared__ __align__(128) uint8_t smem[4 * TILE_BYTES];
  __shared__ __align__(16) float s_km[2][BN];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, t = lane & 3;
  const int q0 = blockIdx.x * BM, h = blockIdx.y, b = blockIdx.z;
  const uint32_t sK = smem_u32(smem), sV = sK + 2 * TILE_BYTES, sQ = sK + TILE_BYTES;   // Q staged in K's 2nd buffer
  pdl_wait();
  pdl_trigger();
  const bf16* kg = p.k + b * p.k_bs + h * DH;
  const bf16* vg = p.v + b * p.v_bs + h * DH;
  const int ntile = (p.nk + BN - 1) / BN;
  const bool active = q0 + warp * 16 < p.nq;   // warps whose 16 rows are all padding only help with the loads
  load_tile(sQ, p.q + b * p.q_bs + (int64_t)q0 * p.ldq + h * DH, p.ldq, p.nq - q0, tid);
  load_tile(sK, kg, p.ldk, p.nk, tid);
  load_tile(sV, vg, p.ldv, p.nk, tid);
  stage_kmask(s_km[0], p, b, 0, tid);
  cp_async_commit();

  const int r0 = q0 + warp * 16 + gq;   // this thread's rows: r0 and r0 + 8
  const uint32_t t16 = p.thresh >> 16;
  const uint32_t rh0 = row_hash(p.seed, ((int64_t)b * p.H + h) * p.nq + r0), rh1 = row_hash(p.seed, ((int64_t)b * p.H + h) * p.nq + r0 + 8);
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  uint32_t qf[4][4];
  cp_async_wait<0>();
  __syncthreads();
  load_a_frags(sQ, warp * 16, lane, qf);

  for (int j = 0; j < ntile; ++j) {
    const int buf = j & 1;
    cp_async_wait<0>();
    __syncthreads();   // tile j has landed; every warp is done with tile j-1 (and with Q), so the other buffer is free
    if (j + 1 < ntile) {
      load_tile(sK + (buf ^ 1) * TILE_BYTES, kg + (int64_t)(j + 1) * BN * p.ldk, p.ldk, p.nk - (j + 1) * BN, tid);
      load_tile(sV + (buf ^ 1) * TILE_BYTES, vg + (int64_t)(j + 1) * BN * p.ldv, p.ldv, p.nk - (j + 1) * BN, tid);
      stage_kmask(s_km[buf ^ 1], p, b, j + 1, tid);
      cp_async_commit();
    }
    if (!active) continue;

    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
    mma_a_tT(s, qf, sK + buf * TILE_BYTES, lane);
    logits_qk(s, p, s_km[buf], b, r0, j, t);

    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      mx0 = fmaxf(mx0, fmaxf(s[nb][0], s[nb][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nb][2], s[nb][3]));
    }
    const float mn0 = fmaxf(m0, quad_max(mx0)), mn1 = fmaxf(m1, quad_max(mx1));
    const float ms0 = mn0 == -INFINITY ? 0.f : mn0, ms1 = mn1 == -INFINITY ? 0.f : mn1;
    const float c0 = ex2(m0 - ms0), c1 = ex2(m1 - ms1);
    m0 = mn0;
    m1 = mn1;
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      float p00 = ex2(s[nb][0] - ms0), p01 = ex2(s[nb][1] - ms0), p10 = ex2(s[nb][2] - ms1), p11 = ex2(s[nb][3] - ms1);
      ps0 += p00 + p01;
      ps1 += p10 + p11;
      if (p.thresh) {
        const uint32_t pair = j * (BN / 2) + nb * 4 + t;
        const uint32_t x0 = mix_pair(rh0, pair), x1 = mix_pair(rh1, pair);
        p00 = (x0 & 0xFFFFu) >= t16 ? p00 * p.scale : 0.f;
        p01 = (x0 >> 16) >= t16 ? p01 * p.scale : 0.f;
        p10 = (x1 & 0xFFFFu) >= t16 ? p10 * p.scale : 0.f;
        p11 = (x1 >> 16) >= t16 ? p11 * p.scale : 0.f;
      }
      s[nb][0] = p00;
      s[nb][1] = p01;
      s[nb][2] = p10;
      s[nb][3] = p11;
    }
    l0 = l0 * c0 + ps0;
    l1 = l1 * c1 + ps1;
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      o[nb][0] *= c0;
      o[nb][1] *= c0;
      o[nb][2] *= c1;
      o[nb][3] *= c1;
    }
    mma_p_t(o, s, sV + buf * TILE_BYTES, lane);
  }
  __syncthreads();   // the K buffers double as the output staging tile
  l0 = quad_sum(l0);
  l1 = quad_sum(l1);
  const float i0 = l0 > 0.f ? 1.0f / l0 : 0.f, i1 = l1 > 0.f ? 1.0f / l1 : 0.f;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    o[nb][0] *= i0;
    o[nb][1] *= i0;
    o[nb][2] *= i1;
    o[nb][3] *= i1;
  }
  if (t == 0 && p.lse) {
    float* lse = p.lse + ((int64_t)b * p.H + h) * p.nq;
    if (r0 < p.nq) lse[r0] = l0 > 0.f ? m0 + log2f(l0) : INFINITY;
    if (r0 + 8 < p.nq) lse[r0 + 8] = l1 > 0.f ? m1 + log2f(l1) : INFINITY;
  }
  store_rows(sK, smem, o, warp * 16, lane, p.out + b * p.o_bs + (int64_t)q0 * p.ldo + h * DH, p.ldo, p.nq - q0);
}

// ------------------------------------------------------------------------------------------------ backward A: dQ
__global__ void __launch_bounds__(NT, 3) flash_bwd_dq_kernel(const Params p) {
  __shared__ __align__(128) uint8_t smem[4 * TILE_BYTES];
  __shared__ __align__(16) float s_km[2][BN];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, t = lane & 3;
  const int q0 = blockIdx.x * BM, h = blockIdx.y, b = blockIdx.z;
  const uint32_t sK = smem_u32(smem), sV = sK + 2 * TILE_BYTES, sQ = sK + TILE_BYTES, sdO = sV + TILE_BYTES;
  pdl_wait();
  pdl_trigger();
  const bf16* kg = p.k + b * p.k_bs + h * DH;
  const bf16* vg = p.v + b * p.v_bs + h * DH;
  const bf16* dog = p.dout + b * p.do_bs + (int64_t)q0 * p.lddo + h * DH;
  const bf16* og = p.o + b * p.o_bs + (int64_t)q0 * p.ldo + h * DH;
  const int ntile = (p.nk + BN - 1) / BN;
  const bool active = q0 + warp * 16 < p.nq;
  load_tile(sQ, p.q + b * p.q_bs + (int64_t)q0 * p.ldq + h * DH, p.ldq, p.nq - q0, tid);   // staged in the 2nd buffers
  load_tile(sdO, dog, p.lddo, p.nq - q0, tid);
  load_tile(sK, kg, p.ldk, p.nk, tid);
  load_tile(sV, vg, p.ldv, p.nk, tid);
  stage_kmask(s_km[0], p, b, 0, tid);
  cp_async_commit();

  const int r0 = q0 + warp * 16 + gq;
  const uint32_t t16 = p.thresh >> 16;
  const uint32_t rh0 = row_hash(p.seed, ((int64_t)b * p.H + h) * p.nq + r0), rh1 = row_hash(p.seed, ((int64_t)b * p.H + h) * p.nq + r0 + 8);
  // D = rowsum(dO * O) for rows r0, r0+8: the quad's 4 lanes take 16 columns each
  float d0 = 0.f, d1 = 0.f;
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int r = r0 + rr * 8;
    float acc = 0.f;
    if (r < p.nq) {
      const int lr = r - q0;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const uint4 a = *reinterpret_cast<const uint4*>(dog + (int64_t)lr * p.lddo + t * 16 + c * 8);
        const uint4 o4 = *reinterpret_cast<const uint4*>(og + (int64_t)lr * p.ldo + t * 16 + c * 8);
        const __nv_bfloat162* pa = reinterpret_cast<const __nv_bfloat162*>(&a);
        const __nv_bfloat162* po = reinterpret_cast<const __nv_bfloat162*>(&o4);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 fa = __bfloat1622float2(pa[e]), fo = __bfloat1622float2(po[e]);
          acc += fa.x * fo.x + fa.y * fo.y;
        }
      }
    }
    acc = quad_sum(acc);
    if (rr == 0) d0 = acc; else d1 = acc;
  }
  const float* lseg = p.lse + ((int64_t)b * p.H + h) * p.nq;
  const float lse0 = r0 < p.nq ? lseg[r0] : INFINITY, lse1 = r0 + 8 < p.nq ? lseg[r0 + 8] : INFINITY;
  if (t == 0) {
    float* ds = p.dsum + ((int64_t)b * p.H + h) * p.nq;
    if (r0 < p.nq) ds[r0] = d0;
    if (r0 + 8 < p.nq) ds[r0 + 8] = d1;
  }

  float dq[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
  uint32_t qf[4][4], dof[4][4];
  cp_async_wait<0>();
  __syncthreads();
  load_a_frags(sQ, warp * 16, lane, qf);
  load_a_frags(sdO, warp * 16, lane, dof);

  for (int j = 0; j < ntile; ++j) {
    const int buf = j & 1;
    cp_async_wait<0>();
    __syncthreads();
    if (j + 1 < ntile) {
      load_tile(sK + (buf ^ 1) * TILE_BYTES, kg + (int64_t)(j + 1) * BN * p.ldk, p.ldk, p.nk - (j + 1) * BN, tid);
      load_tile(sV + (buf ^ 1) * TILE_BYTES, vg + (int64_t)(j + 1) * BN * p.ldv, p.ldv, p.nk - (j + 1) * BN, tid);
      stage_kmask(s_km[buf ^ 1], p, b, j + 1, tid);
      cp_async_commit();
    }
    if (!active) continue;
    float s[8][4], dp[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
      dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
    }
    mma_a_tT(s, qf, sK + buf * TILE_BYTES, lane);
    logits_qk(s, p, s_km[buf], b, r0, j, t);
    mma_a_tT(dp, dof, sV + buf * TILE_BYTES, lane);
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      float g00 = dp[nb][0], g01 = dp[nb][1], g10 = dp[nb][2], g11 = dp[nb][3];
      if (p.thresh) {
        const uint32_t pair = j * (BN / 2) + nb * 4 + t;
        const uint32_t x0 = mix_pair(rh0, pair), x1 = mix_pair(rh1, pair);
        g00 = (x0 & 0xFFFFu) >= t16 ? g00 * p.scale : 0.f;
        g01 = (x0 >> 16) >= t16 ? g01 * p.scale : 0.f;
        g10 = (x1 & 0xFFFFu) >= t16 ? g10 * p.scale : 0.f;
        g11 = (x1 >> 16) >= t16 ? g11 * p.scale : 0.f;
      }
      s[nb][0] = ex2(s[nb][0] - lse0) * (g00 - d0);   // -inf logits / +inf lse -> p = 0
      s[nb][1] = ex2(s[nb][1] - lse0) * (g01 - d0);
      s[nb][2] = ex2(s[nb][2] - lse1) * (g10 - d1);
      s[nb][3] = ex2(s[nb][3] - lse1) * (g11 - d1);
    }
    if (p.dbias) {   // graph-bias gradient (global map encoder): sum over heads with fp32 atomics or per-head partials
      float* dbh = p.dbias + h * p.dbias_hs;
      float* db0 = r0 < p.nq ? dbh + ((int64_t)b * p.nq + r0) * p.nk : nullptr;
      float* db1 = r0 + 8 < p.nq ? dbh + ((int64_t)b * p.nq + r0 + 8) * p.nk : nullptr;
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = j * BN + nb * 8 + 2 * t + e;
          if (col < p.nk) {
            if (p.dbias_hs) {
              if (db0) db0[col] = s[nb][e];
              if (db1) db1[col] = s[nb][2 + e];
            } else {
              if (db0) atomicAdd(db0 + col, s[nb][e]);
              if (db1) atomicAdd(db1 + col, s[nb][2 + e]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      s[nb][0] *= p.alpha;
      s[nb][1] *= p.alpha;
      s[nb][2] *= p.alpha;
      s[nb][3] *= p.alpha;
    }
    mma_p_t(dq, s, sK + buf * TILE_BYTES, lane);
  }
  __syncthreads();
  store_rows(sK, smem, dq, warp * 16, lane, p.dq + b * p.dq_bs + (int64_t)q0 * p.lddq + h * DH, p.lddq, p.nq - q0);
}

// ------------------------------------------------------------------------------------------------ backward B: dK, dV
__global__ void __launch_bounds__(NT) flash_bwd_dkv_kernel(const Params p) {
  __shared__ __align__(128) uint8_t smem[4 * TILE_BYTES];
  __shared__ float s_lse[2][BN], s_dsum[2][BN];
  __shared__ uint32_t s_rh[2][BN];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, t = lane & 3;
  const int k0 = blockIdx.x * BM, h = blockIdx.y, b = blockIdx.z;
  const uint32_t sQ = smem_u32(smem), sdO = sQ + 2 * TILE_BYTES;
  pdl_wait();
  pdl_trigger();
  const bf16* qg = p.q + b * p.q_bs + h * DH;
  const bf16* dog = p.dout + b * p.do_bs + h * DH;
  const float* lseg = p.lse + ((int64_t)b * p.H + h) * p.nq;
  const float* dsg = p.dsum + ((int64_t)b * p.H + h) * p.nq;
  const int ntile = (p.nq + BN - 1) / BN;

  // K and V of the owned keys -> A fragments (staged through the second halves of the ring)
  load_tile(sQ + TILE_BYTES, p.k + b * p.k_bs + (int64_t)k0 * p.ldk + h * DH, p.ldk, p.nk - k0, tid);
  load_tile(sdO + TILE_BYTES, p.v + b * p.v_bs + (int64_t)k0 * p.ldv + h * DH, p.ldv, p.nk - k0, tid);
  cp_async_commit();
  load_tile(sQ, qg, p.ldq, p.nq, tid);
  load_tile(sdO, dog, p.lddo, p.nq, tid);
  const int64_t rngb = ((int64_t)b * p.H + h) * p.nq;
  if (tid < BN) {
    s_lse[0][tid] = tid < p.nq ? lseg[tid] : INFINITY;
    s_dsum[0][tid] = tid < p.nq ? dsg[tid] : 0.f;
    if (p.thresh) s_rh[0][tid] = row_hash(p.seed, rngb + tid);
  }
  cp_async_commit();
  cp_async_wait<1>();
  __syncthreads();
  uint32_t kf[4][4], vf[4][4];
  load_a_frags(sQ + TILE_BYTES, warp * 16, lane, kf);
  load_a_frags(sdO + TILE_BYTES, warp * 16, lane, vf);
  const bool active = k0 + warp * 16 < p.nk;

  const int kr0 = k0 + warp * 16 + gq;   // this thread's keys: kr0 and kr0 + 8
  const float km0 = (kr0 < p.nk) ? (p.kmask ? p.kmask[(int64_t)b * p.nk + kr0] : 0.f) : -INFINITY;
  const float km1 = (kr0 + 8 < p.nk) ? (p.kmask ? p.kmask[(int64_t)b * p.nk + kr0 + 8] : 0.f) : -INFINITY;
  const uint32_t t16 = p.thresh >> 16, pair0 = (uint32_t)kr0 >> 1, sh = (kr0 & 1) * 16;
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
    dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
  }

  for (int j = 0; j < ntile; ++j) {
    const int buf = j & 1;
    cp_async_wait<0>();
    __syncthreads();   // tile j landed; all warps hold their K / V fragments and are done with tile j-1
    if (j + 1 < ntile) {
      const int qn = (j + 1) * BN;
      load_tile(sQ + (buf ^ 1) * TILE_BYTES, qg + (int64_t)qn * p.ldq, p.ldq, p.nq - qn, tid);
      load_tile(sdO + (buf ^ 1) * TILE_BYTES, dog + (int64_t)qn * p.lddo, p.lddo, p.nq - qn, tid);
      if (tid < BN) {
        s_lse[buf ^ 1][tid] = qn + tid < p.nq ? lseg[qn + tid] : INFINITY;
        s_dsum[buf ^ 1][tid] = qn + tid < p.nq ? dsg[qn + tid] : 0.f;
        if (p.thresh) s_rh[buf ^ 1][tid] = row_hash(p.seed, rngb + qn + tid);
      }
      cp_async_commit();
    }
    if (!active) continue;

    // S^T (keys x queries) and dP^T
    float s[8][4], dp[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
      dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
    }
    mma_a_tT(s, kf, sQ + buf * TILE_BYTES, lane);
    mma_a_tT(dp, vf, sdO + buf * TILE_BYTES, lane);
    float pd[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int ql = nb * 8 + 2 * t + e, qi = j * BN + ql;   // query (column)
        const float lse = s_lse[buf][ql], dsum = s_dsum[buf][ql];
        float b0 = 0.f, b1 = 0.f;
        if (p.bias && qi < p.nq) {
          const float* bs = p.bias + ((int64_t)b * p.nq + qi) * p.nk;
          if (kr0 < p.nk) b0 = bs[kr0];
          if (kr0 + 8 < p.nk) b1 = bs[kr0 + 8];
        }
        const float p0 = ex2((s[nb][e] * p.alpha + km0 + b0) * LOG2E - lse);
        const float p1 = ex2((s[nb][2 + e] * p.alpha + km1 + b1) * LOG2E - lse);
        float g0 = dp[nb][e], g1 = dp[nb][2 + e], q0v = p0, q1v = p1;
        if (p.thresh) {
          const uint32_t rh = s_rh[buf][ql];
          const bool keep0 = ((mix_pair(rh, pair0) >> sh) & 0xFFFFu) >= t16;
          const bool keep1 = ((mix_pair(rh, pair0 + 4) >> sh) & 0xFFFFu) >= t16;
          g0 = keep0 ? g0 * p.scale : 0.f;
          g1 = keep1 ? g1 * p.scale : 0.f;
          q0v = keep0 ? p0 * p.scale : 0.f;
          q1v = keep1 ? p1 * p.scale : 0.f;
        }
        pd[nb][e] = q0v;
        pd[nb][2 + e] = q1v;
        s[nb][e] = p0 * (g0 - dsum) * p.alpha;
        s[nb][2 + e] = p1 * (g1 - dsum) * p.alpha;
      }
    }
    mma_p_t(dv, pd, sdO + buf * TILE_BYTES, lane);
    mma_p_t(dk, s, sQ + buf * TILE_BYTES, lane);
  }
  __syncthreads();
  store_rows(sQ, smem, dk, warp * 16, lane, p.dk + b * p.dk_bs + (int64_t)k0 * p.lddk + h * DH, p.lddk, p.nk - k0);
  store_rows(sdO, smem + 2 * TILE_BYTES, dv, warp * 16, lane, p.dv + b * p.dv_bs + (int64_t)k0 * p.lddv + h * DH, p.lddv,
             p.nk - k0);
}

static int fill(Params& p, const bb_flash_args* a, bool bwd) {
  if (!a || !a->q || !a->k || !a->v) return set_error("bb_flash: null q / k / v");
  if (a->dh != 64) return set_error("bb_flash: head dim must be 64");
  if (a->B <= 0 || a->H <= 0 || a->nq <= 0 || a->nk <= 0) return set_error("bb_flash: sizes must be positive");
  if ((a->ldq | a->ldk | a->ldv | a->ldo) % 8) return set_error("bb_flash: row strides must be multiples of 8 elements");
  if (a->B > 65535 || a->H > 65535) return set_error("bb_flash: B, H must be <= 65535");
  memset(&p, 0, sizeof(p));
  p.q = (const bf16*)a->q; p.k = (const bf16*)a->k; p.v = (const bf16*)a->v;
  p.q_bs = a->q_bs; p.k_bs = a->k_bs; p.v_bs = a->v_bs; p.ldq = a->ldq; p.ldk = a->ldk; p.ldv = a->ldv;
  p.o = (const bf16*)a->o; p.out = (bf16*)a->o; p.o_bs = a->o_bs; p.ldo = a->ldo;
  p.lse = a->lse; p.kmask = a->kmask; p.bias = a->bias;
  p.B = a->B; p.H = a->H; p.nq = a->nq; p.nk = a->nk; p.alpha = a->alpha;
  p.seed = a->seed; p.thresh = a->thresh; p.scale = a->scale;
  if (!a->o || !a->lse) return set_error("bb_flash: null o / lse");
  // both cores move 16-byte chunks of every row of every sample (cp.async / uint4 here, TMA in attn_tc.cu)
  if ((reinterpret_cast<uintptr_t>(a->q) | reinterpret_cast<uintptr_t>(a->k) | reinterpret_cast<uintptr_t>(a->v) |
       reinterpret_cast<uintptr_t>(a->o)) & 15)
    return set_error("bb_flash: q / k / v / o must be 16-byte aligned");
  if ((a->q_bs | a->k_bs | a->v_bs | a->o_bs) % 8) return set_error("bb_flash: batch strides must be multiples of 8 elements");
  if (bwd) {
    if (!a->dout || !a->dq || !a->dk || !a->dv || !a->dsum) return set_error("bb_flash_bwd: null gradient pointer");
    if ((a->lddo | a->lddq | a->lddk | a->lddv) % 8) return set_error("bb_flash_bwd: row strides must be multiples of 8");
    if ((reinterpret_cast<uintptr_t>(a->dout) | reinterpret_cast<uintptr_t>(a->dq) | reinterpret_cast<uintptr_t>(a->dk) |
         reinterpret_cast<uintptr_t>(a->dv)) & 15)
      return set_error("bb_flash_bwd: dout / dq / dk / dv must be 16-byte aligned");
    if ((a->do_bs | a->dq_bs | a->dk_bs | a->dv_bs) % 8)
      return set_error("bb_flash_bwd: batch strides must be multiples of 8 elements");
    p.dout = (const bf16*)a->dout; p.do_bs = a->do_bs; p.lddo = a->lddo; p.dsum = a->dsum;
    p.dq = (bf16*)a->dq; p.dq_bs = a->dq_bs; p.lddq = a->lddq;
    p.dk = (bf16*)a->dk; p.dk_bs = a->dk_bs; p.lddk = a->lddk;
    p.dv = (bf16*)a->dv; p.dv_bs = a->dv_bs; p.lddv = a->lddv;
    p.dbias = a->dbias;
  }
  return 0;
}

}  // namespace fa
}  // namespace bb

extern "C" int bb_flash_fwd(const bb_flash_args* a, void* stream) {
  using namespace bb;
  fa::Params p;
  if (int e = fa::fill(p, a, false)) return e;
  if (fat::fwd_supported(a)) return fat::launch_fwd(a, stream);   // wgmma / TMA core (attn_tc.cu)
  const dim3 grid((unsigned)((a->nq + fa::BM - 1) / fa::BM), (unsigned)a->H, (unsigned)a->B);
  launch_pdl(fa::flash_fwd_kernel, grid, dim3(fa::NT), 0, (cudaStream_t)stream, p);
  count_launch();
  return check_launch("flash_fwd_kernel");
}

extern "C" int bb_flash_bwd(const bb_flash_args* a, void* stream) {
  using namespace bb;
  fa::Params p;
  if (int e = fa::fill(p, a, true)) return e;
  if (fat::bwd_supported(a)) return fat::launch_bwd(a, stream);   // wgmma / TMA core (attn_tc.cu)
  const dim3 gq((unsigned)((a->nq + fa::BM - 1) / fa::BM), (unsigned)a->H, (unsigned)a->B);
  const dim3 gk((unsigned)((a->nk + fa::BM - 1) / fa::BM), (unsigned)a->H, (unsigned)a->B);
  if (p.dbias && det_on()) {   // per-head partials, then a sum over heads in head order
    p.dbias_hs = (int64_t)a->B * a->nq * a->nk;
    p.dbias = det_partials((cudaStream_t)stream, (size_t)a->H * p.dbias_hs * sizeof(float), "bb_flash_bwd (graph-bias gradient)");
    if (!p.dbias) return -1;
  }
  launch_pdl(fa::flash_bwd_dq_kernel, gq, dim3(fa::NT), 0, (cudaStream_t)stream, p);
  launch_pdl(fa::flash_bwd_dkv_kernel, gk, dim3(fa::NT), 0, (cudaStream_t)stream, p);
  count_launch(2);
  if (int e = check_launch("flash_bwd kernels")) return e;
  return p.dbias_hs ? det_reduce(p.dbias, a->H, p.dbias_hs, 1, a->dbias, nullptr, nullptr, (cudaStream_t)stream) : 0;
}

namespace bb { int set_salt_attn_flash(const unsigned long long* p) { return set_drop_salt_ptr_tu(p) == cudaSuccess ? 0 : -1; } }
