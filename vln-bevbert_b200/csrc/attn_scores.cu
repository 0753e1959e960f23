// Fused attention-score kernels for sm_90a (keys per row <= 512, head dim 64):
//   mode 0:  P  = softmax(alpha * Q K^T + kmask + bias)  (+ dropped copy Pd)         -- forward
//   mode 1:  dS = P o (g - sum_k P g) * out_scale,  g = (dO V^T) o dropout-mask        -- backward
// A CTA owns 128 query rows of one (sample, head); Q and all (<= 512) K rows arrive by TMA in 128B-swizzled shared
// memory (double buffered across tiles).  Each of the two consumer warpgroups forms its 64 x nk product with wgmma,
// 64 keys at a time into registers, and runs the row-wise softmax / softmax-backward on the fragments in two passes
// (statistics, then outputs -- the 64-key block is recomputed, which costs tensor time that is otherwise idle):
// the fp32 score matrix never exists in HBM.
// Replaces the (batched GEMM -> fp32 scores -> bb_softmax_fwd/bwd) pair of the unfused path; same dropout
// counters (row * ld + column), so forward and backward stay interchangeable with the unfused kernels.
//
// Reference: vilmodel.py:117-127 / 335-346 (scores, mask, softmax, attention dropout) and their autograd.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <mutex>
#include <stdio.h>
#include <string.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {

bool act_f32();   // gemm_f32.cu: fp32-activation verification mode (bb_set_act_f32)

constexpr int AS_THREADS = 288;            // warps 0..7: two consumer warpgroups (64 query rows each), warp 8: TMA
constexpr int AS_Q_BYTES = 128 * 64 * 2;   // 16 KB
constexpr int AS_K_BYTES = 512 * 64 * 2;   // 64 KB
constexpr int AS_STAGE = AS_Q_BYTES + AS_K_BYTES;
constexpr int AS_STAGES = 2;

__device__ __forceinline__ float quad_max_f(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum_f(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

struct ScoreParams {
  int B, H, nq, nk, ldp, m_tiles, mode;
  float alpha, out_scale, scale;
  unsigned long long seed;
  unsigned int thresh;
  const float* kmask;
  const float* bias;
  __nv_bfloat16* P;
  __nv_bfloat16* Pd;
  const __nv_bfloat16* Pin;
  __nv_bfloat16* dS;
  float* dbias;
};

// 64 query rows x 64 keys (block c) of the product into this warpgroup's accumulator fragment
__device__ __forceinline__ void score_block(float (&s)[32], uint32_t sq, uint32_t sk, int c) {
#pragma unroll
  for (int i = 0; i < 32; ++i) s[i] = 0.0f;
  fence_regs(s);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k)
    wgmma_m64n64_ss<0, 0>(s, wgmma_desc(sq + k * 32, 16, 1024), wgmma_desc(sk + c * 8192 + k * 32, 16, 1024),
                          k > 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);
}

__global__ void __launch_bounds__(AS_THREADS, 1)
attn_scores_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   const ScoreParams p, int total_tiles) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + AS_STAGES * AS_STAGE);
  uint64_t* empty_bar = full_bar + AS_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < AS_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  const int nkb = (p.nk + 63) / 64;     // 64-key blocks of the product
  const int nkb_out = (p.ldp + 63) / 64;  // 64-column blocks of the output rows (columns >= nk are written as 0)

  if (warp == 8) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int mt = tile % p.m_tiles;
        const int h = (tile / p.m_tiles) % p.H;
        const int b = tile / (p.m_tiles * p.H);
        mbar_wait_relaxed(&empty_bar[stage], phase ^ 1);
        uint8_t* sq = smem + stage * AS_STAGE;
        uint8_t* sk = sq + AS_Q_BYTES;
        mbar_expect_tx(&full_bar[stage], AS_Q_BYTES + nkb * 8192);
        tma_load_4d(sq, &tmap_a, &full_bar[stage], 0, mt * 128, h, b);
        for (int j = 0; j < nkb; ++j) tma_load_4d(sk + j * 8192, &tmap_b, &full_bar[stage], 0, j * 64, h, b);
        if (++stage == AS_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- consumers: row-wise softmax on the fragments
  // Thread t of warpgroup wg holds query rows r0 = 16 (t / 32) + (t % 32) / 4 and r0 + 8 of the tile's 64-row half and,
  // of each 64-key block, columns 8 j + 2 (t % 4) + {0, 1}; a row lives in the 4 threads of a quad.
  const int wg = warp >> 2;
  const int r0 = (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int mt = tile % p.m_tiles;
    const int h = (tile / p.m_tiles) % p.H;
    const int b = tile / (p.m_tiles * p.H);
    int q[2];
    bool row_ok[2];
    long long grow[2];   // global row index of P / dS
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      q[hh] = mt * 128 + wg * 64 + r0 + 8 * hh;
      row_ok[hh] = q[hh] < p.nq;
      grow[hh] = ((long long)b * p.H + h) * p.nq + q[hh];
    }
    const uint32_t sq = smem_u32(smem + stage * AS_STAGE) + wg * 8192;
    const uint32_t sk = smem_u32(smem + stage * AS_STAGE) + AS_Q_BYTES;
    mbar_wait(&full_bar[stage], phase);
    float s[32];
    if (p.mode == 0) {
      // scores with mask and bias, for the 16 columns of block c held by this thread
      auto scores = [&](int c) {
        score_block(s, sq, sk, c);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = c * 64 + 8 * jj + cq + e;
            const float km = col < p.nk ? (p.kmask ? __ldg(p.kmask + (long long)b * p.nk + col) : 0.0f) : -INFINITY;
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              float v = fmaf(s[4 * jj + 2 * hh + e], p.alpha, km);
              if (p.bias && row_ok[hh] && col < p.nk) v += __ldg(p.bias + ((long long)b * p.nq + q[hh]) * p.nk + col);
              s[4 * jj + 2 * hh + e] = v;
            }
          }
      };
      // pass A: online row maximum / sum of exponentials
      float mx[2] = {-INFINITY, -INFINITY}, sum[2] = {0.0f, 0.0f};
      for (int c = 0; c < nkb; ++c) {
        scores(c);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float cm = -INFINITY;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) cm = fmaxf(cm, fmaxf(s[4 * jj + 2 * hh], s[4 * jj + 2 * hh + 1]));
          if (cm > mx[hh]) {
            sum[hh] *= __expf(mx[hh] - cm);   // exp(-inf) = 0 on the first block
            mx[hh] = cm;
          }
          if (mx[hh] > -INFINITY) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) sum[hh] += __expf(s[4 * jj + 2 * hh] - mx[hh]) + __expf(s[4 * jj + 2 * hh + 1] - mx[hh]);
          }
        }
      }
      float m[2], inv[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        m[hh] = quad_max_f(mx[hh]);
        const float part = mx[hh] > -INFINITY ? sum[hh] * __expf(mx[hh] - m[hh]) : 0.0f;
        const float tot = quad_sum_f(part);
        // all keys masked with -inf: P = Pd = 0 (exp(-inf - 0) * 0), as bb_softmax_fwd and the flash cores give, so
        // that dS and the graph-bias gradient of the row are 0 as well
        inv[hh] = tot > 0.0f ? 1.0f / tot : 0.0f;
        if (m[hh] == -INFINITY) m[hh] = 0.0f;
      }
      // pass B: probabilities (and their dropped copy)
      for (int c = 0; c < nkb_out; ++c) {
        if (c < nkb) scores(c);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int col = c * 64 + 8 * jj + cq;
          if (col >= p.ldp) continue;   // ldp is a multiple of 8: both columns of the pair are in the row
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            if (!row_ok[hh]) continue;
            float pr[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) pr[e] = (col + e < p.nk) ? __expf(s[4 * jj + 2 * hh + e] - m[hh]) * inv[hh] : 0.0f;
            const long long off = grow[hh] * p.ldp + col;
            *reinterpret_cast<__nv_bfloat162*>(p.P + off) = __floats2bfloat162_rn(pr[0], pr[1]);
            if (p.Pd) {
              if (p.thresh) {
#pragma unroll
                for (int e = 0; e < 2; ++e) pr[e] = drop_keep(p.seed, (uint64_t)(off + e), p.thresh) ? pr[e] * p.scale : 0.0f;
              }
              *reinterpret_cast<__nv_bfloat162*>(p.Pd + off) = __floats2bfloat162_rn(pr[0], pr[1]);
            }
          }
        }
      }
    } else {
      // backward: g = (dO V^T) o dropout-mask ; dot = sum_k P g ; dS = P o (g - dot) * out_scale
      auto grads = [&](int c) {
        score_block(s, sq, sk, c);
        if (p.thresh) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const uint64_t idx = (uint64_t)(grow[hh] * p.ldp + c * 64 + 8 * jj + cq + e);
                float& g = s[4 * jj + 2 * hh + e];
                g = drop_keep(p.seed, idx, p.thresh) ? g * p.scale : 0.0f;
              }
        }
      };
      auto pin = [&](int hh, int col) {   // P of (row hh, col .. col + 1); col < ldp
        return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.Pin + grow[hh] * p.ldp + col));
      };
      float dot[2] = {0.0f, 0.0f};
      for (int c = 0; c < nkb; ++c) {
        grads(c);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int col = c * 64 + 8 * jj + cq;
          if (col >= p.nk) continue;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            if (!row_ok[hh]) continue;
            const float2 pv = pin(hh, col);
            dot[hh] = fmaf(pv.x, s[4 * jj + 2 * hh], dot[hh]);
            if (col + 1 < p.nk) dot[hh] = fmaf(pv.y, s[4 * jj + 2 * hh + 1], dot[hh]);
          }
        }
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) dot[hh] = quad_sum_f(dot[hh]);
      for (int c = 0; c < nkb_out; ++c) {
        if (c < nkb) grads(c);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int col = c * 64 + 8 * jj + cq;
          if (col >= p.ldp) continue;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            if (!row_ok[hh]) continue;
            const float2 pv = pin(hh, col);
            float ds[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float d = 0.0f;
              if (col + e < p.nk) {
                d = (e ? pv.y : pv.x) * (s[4 * jj + 2 * hh + e] - dot[hh]);
                if (p.dbias) atomicAdd(p.dbias + ((long long)b * p.nq + q[hh]) * p.nk + col + e, d);
              }
              ds[e] = d * p.out_scale;
            }
            *reinterpret_cast<__nv_bfloat162*>(p.dS + grow[hh] * p.ldp + col) = __floats2bfloat162_rn(ds[0], ds[1]);
          }
        }
      }
    }
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
    if (++stage == AS_STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
}

typedef CUresult (*PFN_encodeTiled2)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int make_map_rows(CUtensorMap* map, const void* base, int rows, int H, int B, int64_t ld, int64_t s1, int64_t s2,
                         int box_rows) {
  static PFN_encodeTiled2 enc = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      enc = reinterpret_cast<PFN_encodeTiled2>(fp);
  });
  if (!enc) return set_error("cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15) || ld % 8 || s1 % 8 || s2 % 8)
    return set_error("bb_attn_scores: operands must be 16-byte aligned with strides in multiples of 8 elements");
  if (s1 == 0) s1 = 8;
  if (s2 == 0) s2 = 8;
  cuuint64_t dims[4] = {64, (cuuint64_t)rows, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)s1 * 2, (cuuint64_t)s2 * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("bb_attn_scores: cuTensorMapEncodeTiled failed");
  return 0;
}

}  // namespace bb

extern "C" int bb_attn_scores(const bb_attn_scores_args* a, void* stream_) {
  using namespace bb;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!a || !a->A || !a->Bm) return set_error("bb_attn_scores: null argument");
  if (act_f32())
    return set_error("bb_attn_scores: bf16 operands and outputs only; the fp32 verification mode (bb_set_act_f32) runs "
                     "the unfused GEMM + bb_softmax_fwd/bwd sequence");
  if (a->B <= 0 || a->H <= 0 || a->nq <= 0) return 0;
  if (a->nk < 1 || a->nk > 512) return set_error("bb_attn_scores: needs 1 <= nk <= 512 keys per row");
  if (a->ldp % 8 != 0 || a->ldp < a->nk) return set_error("bb_attn_scores: ldp must be a multiple of 8 and >= nk");
  if (a->mode == 0 && !a->P) return set_error("bb_attn_scores: mode 0 needs P");
  if (a->mode == 1 && (!a->Pin || !a->dS)) return set_error("bb_attn_scores: mode 1 needs Pin and dS");
  // P / Pd / Pin / dS are stored and read as bf16 pairs
  for (const void* t : {(const void*)a->P, (const void*)a->Pd, a->Pin, (const void*)a->dS})
    if (reinterpret_cast<uintptr_t>(t) & 3) return set_error("bb_attn_scores: P, Pd, Pin and dS must be 4-byte aligned");
  if (a->mode == 1 && a->dbias && det_mode() == 1)
    return set_error("bb_attn_scores: the fused-scores (BB_FUSED_SCORES_MAX) graph-bias gradient adds with fp32 atomics "
                     "and has no deterministic implementation");
  static int num_sms = 0;
  if (!num_sms) {
    int dev = 0, optin = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (cudaFuncSetAttribute(attn_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin) != cudaSuccess)
      return set_error("cudaFuncSetAttribute failed for attn_scores_kernel");
  }
  ScoreParams p;
  memset(&p, 0, sizeof(p));
  p.B = a->B; p.H = a->H; p.nq = a->nq; p.nk = a->nk; p.ldp = a->ldp; p.mode = a->mode;
  p.m_tiles = (a->nq + 127) / 128;
  p.alpha = a->alpha; p.out_scale = a->out_scale; p.scale = a->scale; p.seed = a->seed; p.thresh = a->thresh;
  p.kmask = a->kmask; p.bias = a->bias;
  p.P = reinterpret_cast<__nv_bfloat16*>(a->P);
  p.Pd = reinterpret_cast<__nv_bfloat16*>(a->Pd);
  p.Pin = reinterpret_cast<const __nv_bfloat16*>(a->Pin);
  p.dS = reinterpret_cast<__nv_bfloat16*>(a->dS);
  p.dbias = a->dbias;
  CUtensorMap ta, tb;
  int e = make_map_rows(&ta, a->A, a->nq, a->H, a->B, a->lda, a->a_s1, a->a_s2, 128);
  if (e) return e;
  e = make_map_rows(&tb, a->Bm, a->nk, a->H, a->B, a->ldb, a->b_s1, a->b_s2, 64);
  if (e) return e;
  const long long total = (long long)p.m_tiles * a->H * a->B;
  const int grid = total < num_sms ? (int)total : num_sms;
  const size_t smem_bytes = (size_t)AS_STAGES * AS_STAGE + 1024 + 64;
  bb::launch_pdl(attn_scores_kernel, grid, AS_THREADS, smem_bytes, stream, ta, tb, p, (int)total);
  count_launch();
  return check_launch("attn_scores_kernel");
}

namespace bb { int set_salt_attn_scores(const unsigned long long* p) { return set_drop_salt_ptr_tu(p) == cudaSuccess ? 0 : -1; } }
