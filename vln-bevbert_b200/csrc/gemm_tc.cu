// Batched bf16 GEMM for sm_90a: TMA -> 128B-swizzled shared memory -> wgmma (fp32 accumulators in registers) ->
// epilogue with fused bias / GELU / ReLU / gelu' / dropout / residual, staged through shared memory so that global
// accesses are 16-byte row segments and the per-element code is one compact loop.
//
// Persistent, warp-specialised, ping-pong: warpgroup 0 is the TMA producer (one lane issues), warpgroups 1 and 2 are
// consumers that each own whole output tiles and alternate over the CTA's tile sequence.  The two consumers take turns
// in the main loop, so one warpgroup's epilogue runs while the other's MMAs keep the tensor cores busy.  setmaxnreg
// moves registers from the producer to the consumers (a 128 x 128 fp32 accumulator is 128 registers per thread).
// One CTA per SM; the producer runs ahead through a ring of shared-memory stages in tile order.
//
// Tile: 128 (M) x BN (N, 64 or 128) x 64 (K) per pipeline stage. Operands may be K-major or MN-major (transposed in
// memory; wgmma reads either from shared memory), which gives all of  X*W^T (forward), dY*W (dX) and dY^T*X (dW)
// and the batched attention products without any transposition pass over HBM.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <mutex>
#include <unordered_map>
#include <vector>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB
constexpr int CONSUMER_THREADS = 128;             // one warpgroup
constexpr int NUM_THREADS = 3 * CONSUMER_THREADS;  // producer warpgroup + 2 consumer warpgroups
constexpr int PRODUCER_REGS = 40;                  // 128 x 40 + 256 x 232 <= 64 K registers per SM
constexpr int CONSUMER_REGS = 232;
constexpr int MAX_STAGES = 8;

struct GemmKParams {
  int M, N, K;
  int nb1, nb2;
  int block_n;
  int a_mn, b_mn;
  int split_k, kb_total, kb_per_split;
  int m_tiles, n_tiles;
  int stages;
  int out_f32, atomic;
  int vec_ok;
  long long ldd, d_s1, d_s2;
  void* D;
  float alpha;
  const float* bias;
  int act;
  __nv_bfloat16* aux_out;
  const __nv_bfloat16* aux_in;
  int epi_mul;
  const __nv_bfloat16* add_in;
  unsigned long long drop_seed;
  unsigned int drop_thresh;
  float drop_scale;
  int fast_gelu;      // experiment: Abramowitz-Stegun erf on approximate MUFU ops instead of erff()
  float* det_part;     // EPI_SPLIT_DET: fp32 partial tiles, [split][tile][128 x BN]
  unsigned* det_cnt;   // EPI_SPLIT_DET: per-tile arrival counters (zero between launches)
  long long* trace;   // debug: per CTA and local tile 4 globaltimer stamps (mma start/end, epilogue start/end) or null
  unsigned long long* prof;   // measurement: [0] = min over CTAs of the start stamp, [1] = max of the end stamp, or null
};

__device__ __forceinline__ long long gtimer() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

struct TileCoord {
  int split, b1, b2, m_tile, n_tile;
};

__device__ __forceinline__ TileCoord decode_tile(const GemmKParams& p, int tile) {
  TileCoord t;
  t.n_tile = tile % p.n_tiles;
  tile /= p.n_tiles;
  t.m_tile = tile % p.m_tiles;
  tile /= p.m_tiles;
  t.b1 = tile % p.nb1;
  tile /= p.nb1;
  t.b2 = tile % p.nb2;
  tile /= p.nb2;
  t.split = tile;
  return t;
}

__device__ __forceinline__ float bf2f(__nv_bfloat16 v) { return __bfloat162float(v); }

// Epilogue variants.  GENERIC decides every feature at run time (activation, second output, gelu'/relu' multiply,
// dropout, residual add, any store); the others fix at compile time the feature combinations the model launches, so
// their per-element code is short and free of branches.  Dropout and bias stay run-time switches everywhere.
enum : int {
  EPI_GENERIC = 0,
  EPI_PLAIN = 1,       // alpha, bias; bf16 or fp32 store
  EPI_ATOMIC = 2,      // alpha, bias; fp32 atomic accumulate (split-K weight gradients)
  EPI_GELU_PRE = 3,    // bf16 pre-activation to aux_out, GELU, dropout; bf16 store
  EPI_MUL_DGELU = 4,   // * gelu'(aux_in), dropout; bf16 store
  EPI_MUL_DRELU = 5,   // * relu'(aux_in), dropout; bf16 store
  EPI_ADD = 6,         // dropout, + add_in; bf16 store
  EPI_SPLIT_DET = 7,   // alpha, bias; split-K partials summed in split order by the last split (deterministic mode)
  EPI_COUNT = 8
};

template <int EPI>
__device__ __forceinline__ int epi_mul_of(const GemmKParams& p) {
  return EPI == EPI_GENERIC ? p.epi_mul : (EPI == EPI_MUL_DGELU ? 1 : EPI == EPI_MUL_DRELU ? 2 : 0);
}
template <int EPI>
__device__ __forceinline__ bool epi_add_of(const GemmKParams& p) {
  return EPI == EPI_GENERIC ? p.add_in != nullptr : EPI == EPI_ADD;
}

// Epilogues of EPI_ATOMIC (split-K weight gradients) and EPI_SPLIT_DET read the accumulators straight from registers;
// every other variant stages them through shared memory (epilogue_staged).
__host__ __device__ constexpr bool epi_staged(int epi) { return epi != EPI_ATOMIC && epi != EPI_SPLIT_DET; }
// Shared memory of the two staging buffers (64 x BN fp32 each), carved out ahead of the stage ring.
__host__ __device__ constexpr int staging_bytes(int bn, int epi) { return epi_staged(epi) ? 2 * 64 * bn * 4 : 0; }

// Epilogue of EPI_ATOMIC for one 128 x BN tile: alpha, bias, fp32 atomic add of each accumulator pair straight from
// registers.  acc[hh] holds rows 64 hh .. 64 hh + 63 in the wgmma fragment order (thread rows r0, r0 + 8; columns
// 8 j + cq, + 1).  EDGE: the tile may extend past the last row or column, or lack paired-access alignment.
template <int BN, bool EDGE>
__device__ __forceinline__ void epilogue_atomic(const GemmKParams& p, const TileCoord& t, const float (&acc)[2][BN / 2],
                                                int r0, int cq) {
  const int n0 = t.n_tile * BN;
  const bool add_bias = p.bias != nullptr && t.split == 0;
  const long long batch_off = (long long)t.b1 * p.d_s1 + (long long)t.b2 * p.d_s2;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + 8 * j + cq;
    if (EDGE && col >= p.N) continue;
    const bool two = !EDGE || col + 1 < p.N;
    const bool vec = !EDGE || (two && p.vec_ok);
    const float b0 = add_bias ? __ldg(p.bias + col) : 0.0f;
    const float b1 = add_bias && two ? __ldg(p.bias + col + 1) : 0.0f;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int hh = r >> 1, h = r & 1;
      const int row = t.m_tile * BLOCK_M + 64 * hh + r0 + 8 * h;
      if (EDGE && row >= p.M) continue;
      float* D = reinterpret_cast<float*>(p.D) + batch_off + (long long)row * p.ldd + col;
      float v0 = acc[hh][4 * j + 2 * h] * p.alpha, v1 = acc[hh][4 * j + 2 * h + 1] * p.alpha;
      if (add_bias) {
        v0 += b0;
        if (two) v1 += b1;
      }
      if (vec) {
        atomicAdd(reinterpret_cast<float2*>(D), make_float2(v0, v1));
      } else {
        atomicAdd(D, v0);
        if (two) atomicAdd(D + 1, v1);
      }
    }
  }
}

// ---- staged epilogue
// A consumer warpgroup writes one 64-row half of its accumulators to its own 64 x BN fp32 staging buffer in shared
// memory, then walks the half row by row: each thread takes 8 consecutive columns of a row, so every global access is
// a 16-byte vector and a row segment is contiguous across threads.  The per-element code is one rolled loop for interior
// and edge tiles alike, instead of a fully unrolled copy per accumulator register.
constexpr int STAGE_U = 2;   // rows per thread and loop iteration; the next iteration's global inputs are prefetched

// Byte offset of the 16-byte chunk holding columns 4 c .. 4 c + 3 of staged row r.  XOR swizzle: the 8-byte fragment
// stores of a half-warp (rows r0 .. r0 + 3, 8 columns) and the 16-byte row loads of a quarter-warp (8 threads of one
// row, chunks 2 g or 2 g + 1) both touch 32 distinct banks.
template <int BN>
__device__ __forceinline__ uint32_t stage_off(int r, int c) {
  return (uint32_t)(r * BN * 4 + ((c ^ (2 * (r & 3)) ^ ((c >> 3) & 1)) << 4));
}

__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ float bf16_at(const uint4& v, int i) {
  const uint32_t w = i < 2 ? v.x : i < 4 ? v.y : i < 6 ? v.z : v.w;
  return (i & 1) ? bf16_hi(w) : bf16_lo(w);
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return (uint32_t)__bfloat16_as_ushort(h.x) | ((uint32_t)__bfloat16_as_ushort(h.y) << 16);
}

// 8 bf16 at src + off, of which the first n (1 .. 8) exist; vec: all 8 exist and are 16-byte aligned.
__device__ __forceinline__ uint4 load8(const __nv_bfloat16* src, long long off, int n, bool vec) {
  if (vec) return __ldg(reinterpret_cast<const uint4*>(src + off));
  uint32_t w[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t lo = 2 * k < n ? __bfloat16_as_ushort(src[off + 2 * k]) : 0u;
    const uint32_t hi = 2 * k + 1 < n ? __bfloat16_as_ushort(src[off + 2 * k + 1]) : 0u;
    w[k] = lo | (hi << 16);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ void store8_bf16(__nv_bfloat16* dst, long long off, int n, bool vec, const float (&v)[8]) {
  if (vec) {
    *reinterpret_cast<uint4*>(dst + off) =
        make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (i < n) dst[off + i] = __float2bfloat16(v[i]);
  }
}

// The epilogue of 8 consecutive columns of one row at element offset `off`, of which the first n exist.  v: the
// accumulators; b: bias (used when add_bias); mul_in / add_in: the aux_in and add_in values.  The per-element
// arithmetic and its order are those of every earlier version of this kernel, so results are unchanged bit for bit.
template <int EPI>
__device__ __forceinline__ void epi_chunk(const GemmKParams& p, long long off, int n, bool vec, float (&v)[8],
                                          const float (&b)[8], bool add_bias, const uint4& mul_in, const uint4& add_in) {
  const bool generic = EPI == EPI_GENERIC;
  const bool aux_out = generic ? p.aux_out != nullptr : EPI == EPI_GELU_PRE;
  const int act = generic ? p.act : (EPI == EPI_GELU_PRE ? 1 : 0);
  const int mul = epi_mul_of<EPI>(p);
  const bool add = epi_add_of<EPI>(p);
  const bool drop = (generic || EPI >= EPI_GELU_PRE) && p.drop_thresh != 0;
  const bool out_f32 = (generic || EPI == EPI_PLAIN) && p.out_f32 != 0;
  const bool fast_gelu = generic && p.fast_gelu;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[i] *= p.alpha;
    if (add_bias) v[i] += b[i];
  }
  if (aux_out) store8_bf16(p.aux_out, off, n, vec, v);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (act == 1) v[i] = fast_gelu ? gelu_fast(v[i]) : gelu_erf(v[i]);
    else if (act == 2) v[i] = fmaxf(v[i], 0.0f);
    if (mul == 1) v[i] *= fast_gelu ? dgelu_fast(bf16_at(mul_in, i)) : dgelu_erf(bf16_at(mul_in, i));
    else if (mul == 2) v[i] = bf16_at(mul_in, i) > 0.0f ? v[i] : 0.0f;
    if (drop) v[i] = drop_keep(p.drop_seed, (uint64_t)(off + i), p.drop_thresh) ? v[i] * p.drop_scale : 0.0f;
    if (add) v[i] += bf16_at(add_in, i);
  }
  if (out_f32) {
    float* D = reinterpret_cast<float*>(p.D) + off;
    if (vec) {
      reinterpret_cast<float4*>(D)[0] = make_float4(v[0], v[1], v[2], v[3]);
      reinterpret_cast<float4*>(D)[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (i < n) D[i] = v[i];
    }
  } else {
    store8_bf16(reinterpret_cast<__nv_bfloat16*>(p.D), off, n, vec, v);
  }
}

// Staged epilogue of one 128 x BN tile (see above).  stage_buf: this warpgroup's 64 x BN fp32 buffer; barrier 3 + c
// spans the warpgroup only.  Thread tid owns columns 8 g .. 8 g + 7 (g = tid % (BN / 8)) of rows rs, rs + RP, ...
template <int BN, int EPI>
__device__ __forceinline__ void epilogue_staged(const GemmKParams& p, const TileCoord& t, const float (&acc)[2][BN / 2],
                                                uint8_t* stage_buf, int r0, int cq, int c) {
  constexpr int TPR = BN / 8;                     // threads per row
  constexpr int RP = CONSUMER_THREADS / TPR;      // rows per pass of the warpgroup
  constexpr int GROUPS = 64 / (RP * STAGE_U);     // loop iterations per half
  // Prefetch the next iteration's aux_in / add_in; GENERIC (two inputs) loads them in the iteration instead, so that
  // it needs no spills.
  constexpr bool PREFETCH = EPI != EPI_GENERIC;
  const int tid = threadIdx.x % CONSUMER_THREADS;
  const int g = tid % TPR, rs = tid / TPR;
  const int col = t.n_tile * BN + 8 * g;
  const int n = min(8, p.N - col);                // columns of the thread's chunk that exist (<= 0: none)
  const bool vec = p.vec_ok && n == 8;
  const bool add_bias = p.bias != nullptr && t.split == 0;
  const bool mul = epi_mul_of<EPI>(p) != 0;
  const bool add = epi_add_of<EPI>(p);
  float b[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) b[i] = add_bias && i < n ? __ldg(p.bias + col + i) : 0.0f;
  const long long batch_off = (long long)t.b1 * p.d_s1 + (long long)t.b2 * p.d_s2 + col;
  const uint32_t sbuf = smem_u32(stage_buf);
  const int row0 = t.m_tile * BLOCK_M + rs;

  // global inputs of the STAGE_U rows of loop iteration k of half hh
  auto load_inputs = [&](int hh, int k, uint4 (&mi)[STAGE_U], uint4 (&ai)[STAGE_U]) {
#pragma unroll
    for (int u = 0; u < STAGE_U; ++u) {
      const int row = row0 + 64 * hh + (k * STAGE_U + u) * RP;
      const bool ok = n > 0 && row < p.M;
      const long long off = batch_off + (long long)row * p.ldd;
      mi[u] = mul && ok ? load8(p.aux_in, off, n, vec) : make_uint4(0, 0, 0, 0);
      ai[u] = add && ok ? load8(p.add_in, off, n, vec) : make_uint4(0, 0, 0, 0);
    }
  };

#pragma unroll 1
  for (int hh = 0; hh < 2; ++hh) {
    uint4 mi[STAGE_U], ai[STAGE_U];
    if (PREFETCH) load_inputs(hh, 0, mi, ai);
    // phase 1: fragments -> staging buffer, once every thread has read the previous half out of it
    named_bar_sync(3 + c, CONSUMER_THREADS);
    if (hh == 0) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          st_shared_v2(sbuf + stage_off<BN>(r0 + 8 * h, 2 * j + (cq >> 2)) + (cq & 2) * 4, acc[0][4 * j + 2 * h],
                       acc[0][4 * j + 2 * h + 1]);
    } else {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          st_shared_v2(sbuf + stage_off<BN>(r0 + 8 * h, 2 * j + (cq >> 2)) + (cq & 2) * 4, acc[1][4 * j + 2 * h],
                       acc[1][4 * j + 2 * h + 1]);
    }
    named_bar_sync(3 + c, CONSUMER_THREADS);
    // phase 2: rows of the staged half, STAGE_U per iteration, the next iteration's inputs in flight
#pragma unroll 1
    for (int k = 0; k < GROUPS; ++k) {
      uint4 mi_next[STAGE_U] = {}, ai_next[STAGE_U] = {};
      if (!PREFETCH) load_inputs(hh, k, mi, ai);
      else if (k + 1 < GROUPS) load_inputs(hh, k + 1, mi_next, ai_next);
      float v[STAGE_U][8];
#pragma unroll
      for (int u = 0; u < STAGE_U; ++u) {
        const int rl = rs + (k * STAGE_U + u) * RP;
        const float4 x = ld_shared_v4f(sbuf + stage_off<BN>(rl, 2 * g));
        const float4 y = ld_shared_v4f(sbuf + stage_off<BN>(rl, 2 * g + 1));
        v[u][0] = x.x; v[u][1] = x.y; v[u][2] = x.z; v[u][3] = x.w;
        v[u][4] = y.x; v[u][5] = y.y; v[u][6] = y.z; v[u][7] = y.w;
      }
#pragma unroll
      for (int u = 0; u < STAGE_U; ++u) {
        const int row = row0 + 64 * hh + (k * STAGE_U + u) * RP;
        if (n > 0 && row < p.M)
          epi_chunk<EPI>(p, batch_off + (long long)row * p.ldd, n, vec, v[u], b, add_bias, mi[u], ai[u]);
      }
      if (PREFETCH) {
#pragma unroll
        for (int u = 0; u < STAGE_U; ++u) {
          mi[u] = mi_next[u];
          ai[u] = ai_next[u];
        }
      }
    }
  }
}

// Deterministic split-K epilogue of one 128 x BN tile.  Every split stores alpha * acc (+ bias in split 0) to its own
// fp32 partial tile with plain stores; then one thread of the warpgroup takes a ticket from the tile's arrival
// counter, after a fence.  The warpgroup that arrives last adds the S partials in split order 0 .. S-1 to D and resets
// the counter, so the counters are zero again for the next launch or graph replay.  Nobody waits for anybody.
template <int BN, bool EDGE>
__device__ __forceinline__ void epilogue_split_det(const GemmKParams& p, const TileCoord& t, const float (&acc)[2][BN / 2],
                                                   int r0, int cq, int c, int* ticket) {
  const int n0 = t.n_tile * BN;
  const long long tile = (((long long)t.b2 * p.nb1 + t.b1) * p.m_tiles + t.m_tile) * p.n_tiles + t.n_tile;
  const long long tiles = (long long)p.m_tiles * p.n_tiles * p.nb1 * p.nb2;
  constexpr int TILE = BLOCK_M * BN;
  float* mine = p.det_part + ((long long)t.split * tiles + tile) * TILE;
  const bool add_bias = p.bias != nullptr && t.split == 0;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + 8 * j + cq;
    const float b0 = add_bias && (!EDGE || col < p.N) ? __ldg(p.bias + col) : 0.0f;
    const float b1 = add_bias && (!EDGE || col + 1 < p.N) ? __ldg(p.bias + col + 1) : 0.0f;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int hh = r >> 1, h = r & 1;
      const int rl = 64 * hh + r0 + 8 * h;
      float v0 = acc[hh][4 * j + 2 * h] * p.alpha, v1 = acc[hh][4 * j + 2 * h + 1] * p.alpha;
      if (add_bias) {
        v0 += b0;
        v1 += b1;
      }
      __stcg(reinterpret_cast<float2*>(mine + rl * BN + 8 * j + cq), make_float2(v0, v1));
    }
  }
  const int tid = threadIdx.x % CONSUMER_THREADS;
  __threadfence();
  named_bar_sync(3 + c, CONSUMER_THREADS);
  if (tid == 0) *ticket = (int)atomicAdd(p.det_cnt + tile, 1u);
  named_bar_sync(3 + c, CONSUMER_THREADS);
  if (*ticket != p.split_k - 1) return;
  __threadfence();
  const float* first = p.det_part + tile * TILE;
  const long long batch_off = (long long)t.b1 * p.d_s1 + (long long)t.b2 * p.d_s2;
#pragma unroll 1
  for (int r = 0; r < 4; ++r) {
    const int rl = 64 * (r >> 1) + r0 + 8 * (r & 1);
    const int row = t.m_tile * BLOCK_M + rl;
    if (EDGE && row >= p.M) continue;
    float* drow = reinterpret_cast<float*>(p.D) + batch_off + (long long)row * p.ldd;
#pragma unroll 4
    for (int j = 0; j < BN / 8; ++j) {
      const int cl = 8 * j + cq, col = n0 + cl;
      if (EDGE && col >= p.N) continue;
      float2 s = __ldcg(reinterpret_cast<const float2*>(first + rl * BN + cl));
      for (int k = 1; k < p.split_k; ++k) {
        const float2 v = __ldcg(reinterpret_cast<const float2*>(first + (long long)k * tiles * TILE + rl * BN + cl));
        s.x += v.x;
        s.y += v.y;
      }
      if (!EDGE || (col + 1 < p.N && p.vec_ok)) {
        float2* d = reinterpret_cast<float2*>(drow + col);
        const float2 o = *d;
        *d = make_float2(o.x + s.x, o.y + s.y);
      } else {
        drow[col] += s.x;
        if (col + 1 < p.N) drow[col + 1] += s.y;
      }
    }
  }
  if (tid == 0) p.det_cnt[tile] = 0u;
}

template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BN == 64) wgmma_m64n64_ss<TA, TB>(acc, da, db, scale_d);
  else wgmma_m64n128_ss<TA, TB>(acc, da, db, scale_d);
}

// k-blocks [kb0, kb1) of one 128 x BN tile into this warpgroup's accumulators (two m64 wgmma per k16 step; both read
// the same B tile).  TA / TB (operand MN-major) are template parameters so that the whole loop is free of branches
// around the asynchronous MMAs.  Once the last MMAs are issued, the other consumer warpgroup is let into its main loop
// (ordered barrier `next_bar`, when it has a next tile); then the MMAs are drained and the last stage is released.
template <int BN, int TA, int TB>
__device__ __forceinline__ void mainloop(float (&acc)[2][BN / 2], uint8_t* smem, int stage_bytes, uint64_t* full_bar,
                                         uint64_t* empty_bar, int stages, int stage, uint32_t phase, int kb0, int kb1,
                                         int lane, int next_bar) {
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(smem + stage * stage_bytes);
    const uint32_t sb = sa + A_STAGE_BYTES;
    fence_regs(acc[0]);
    fence_regs(acc[1]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / 16; ++k) {
      const uint64_t db = TB ? wgmma_desc(sb + k * 2048, 8192, 1024) : wgmma_desc(sb + k * 32, 16, 1024);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t s = sa + hh * 8192;
        const uint64_t da = TA ? wgmma_desc(s + k * 2048, 8192, 1024) : wgmma_desc(s + k * 32, 16, 1024);
        wgmma_tile<BN, TA, TB>(acc[hh], da, db, (kb > kb0 || k > 0) ? 1u : 0u);
      }
    }
    wgmma_commit();
    fence_regs(acc[0]);
    fence_regs(acc[1]);
    // at most the group just issued is in flight: the previous stage has been read and can be refilled
    wgmma_wait<1>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == stages) {
      stage = 0;
      phase ^= 1;
    }
  }
  if (next_bar >= 0) named_bar_arrive(next_bar, 2 * CONSUMER_THREADS);
  wgmma_wait<0>();
  fence_regs(acc[0]);
  fence_regs(acc[1]);
  if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
}

template <int BN, int EPI>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmKParams p, int total_tiles) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for SWIZZLE_128B atoms.  Layout: [staging buffers of the two consumer warpgroups, staged
  // variants only] [stage ring] [barriers]
  uint8_t* stage_bufs = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem = stage_bufs + staging_bytes(BN, EPI);
  constexpr int B_STAGE_BYTES = BN * BLOCK_K * 2;
  constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + p.stages * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + MAX_STAGES;

  const int wg = threadIdx.x / CONSUMER_THREADS;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);   // lane 0 of each warp of the consumer warpgroup that read the stage
    }
    fence_mbar_init();
  }
  __syncthreads();
  // Everything above (barrier init, descriptor prefetch) overlapped the previous kernel's tail; from here on global
  // memory is read and written.
  pdl_wait();
  pdl_trigger();
  if (p.prof && threadIdx.x == 0) atomicMin(p.prof, (unsigned long long)gtimer());

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer (one lane), stages in tile order
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const TileCoord t = decode_tile(p, tile);
        const int kb0 = t.split * p.kb_per_split;
        const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);
        const int m0 = t.m_tile * BLOCK_M;
        const int n0 = t.n_tile * BN;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait_relaxed(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          const int k0 = kb * BLOCK_K;
          if (!p.a_mn) {
            tma_load_4d(sa, &tmap_a, &full_bar[stage], k0, m0, t.b1, t.b2);
          } else {
            tma_load_4d(sa, &tmap_a, &full_bar[stage], m0, k0, t.b1, t.b2);
            tma_load_4d(sa + 8192, &tmap_a, &full_bar[stage], m0 + 64, k0, t.b1, t.b2);
          }
          if (!p.b_mn) {
            tma_load_4d(sb, &tmap_b, &full_bar[stage], k0, n0, t.b1, t.b2);
          } else {
#pragma unroll
            for (int j = 0; j < BN / 64; ++j)
              tma_load_4d(sb + j * 8192, &tmap_b, &full_bar[stage], n0 + 64 * j, k0, t.b1, t.b2);
          }
          if (++stage == p.stages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: ping-pong over the CTA's tiles
    // Consumer warpgroup c owns the CTA's local tiles lt = c, c + 2, ...  Main loops take turns through two named
    // barriers: before the main loop of tile lt > 0 a warpgroup waits on its own barrier (1 + c) for the other one to
    // have issued all MMAs of tile lt - 1, so each epilogue runs under the other warpgroup's MMAs.  A warpgroup signals
    // only when the other one has a next tile, so no arrival is left pending when the kernel ends.
    setmaxnreg_inc<CONSUMER_REGS>();
    const int c = wg - 1;
    const int r0 = (warp & 3) * 16 + (lane >> 2);   // fragment rows r0 and r0 + 8 of each 64-row half
    const int cq = 2 * (lane & 3);                  // fragment column offset within each 8-column group
    uint32_t kdone = 0;   // k-blocks the producer queued for the CTA's earlier tiles: position in the stage ring
    int lt = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++lt) {
      const TileCoord t = decode_tile(p, tile);
      const int kb0 = t.split * p.kb_per_split;
      const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);
      const uint32_t kpos = kdone;
      kdone += kb1 - kb0;
      if ((lt & 1) != c) continue;
      const int stage = (int)(kpos % (uint32_t)p.stages);
      const uint32_t phase = (kpos / (uint32_t)p.stages) & 1;
      const int next_bar = tile + (int)gridDim.x < total_tiles ? 2 - c : -1;
      if (lt > 0) named_bar_sync(1 + c, 2 * CONSUMER_THREADS);
      const bool stamp = p.trace && lt < 16 && (threadIdx.x % CONSUMER_THREADS) == 0;
      if (stamp) p.trace[((long long)blockIdx.x * 16 + lt) * 4 + 0] = gtimer();
      float acc[2][BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[0][i] = acc[1][i] = 0.0f;
      switch (p.a_mn * 2 + p.b_mn) {
        case 0: mainloop<BN, 0, 0>(acc, smem, STAGE_BYTES, full_bar, empty_bar, p.stages, stage, phase, kb0, kb1, lane, next_bar); break;
        case 1: mainloop<BN, 0, 1>(acc, smem, STAGE_BYTES, full_bar, empty_bar, p.stages, stage, phase, kb0, kb1, lane, next_bar); break;
        case 2: mainloop<BN, 1, 0>(acc, smem, STAGE_BYTES, full_bar, empty_bar, p.stages, stage, phase, kb0, kb1, lane, next_bar); break;
        default: mainloop<BN, 1, 1>(acc, smem, STAGE_BYTES, full_bar, empty_bar, p.stages, stage, phase, kb0, kb1, lane, next_bar); break;
      }
      if (stamp) {
        p.trace[((long long)blockIdx.x * 16 + lt) * 4 + 1] = gtimer();
        p.trace[((long long)blockIdx.x * 16 + lt) * 4 + 2] = gtimer();
      }
      const bool interior = p.vec_ok && (t.m_tile + 1) * BLOCK_M <= p.M && (t.n_tile + 1) * BN <= p.N;
      if constexpr (epi_staged(EPI)) {
        epilogue_staged<BN, EPI>(p, t, acc, stage_bufs + c * (staging_bytes(BN, EPI) / 2), r0, cq, c);
      } else if constexpr (EPI == EPI_SPLIT_DET) {
        int* ticket = reinterpret_cast<int*>(empty_bar + MAX_STAGES) + c;
        if (interior) epilogue_split_det<BN, false>(p, t, acc, r0, cq, c, ticket);
        else epilogue_split_det<BN, true>(p, t, acc, r0, cq, c, ticket);
      } else {
        if (interior) epilogue_atomic<BN, false>(p, t, acc, r0, cq);
        else epilogue_atomic<BN, true>(p, t, acc, r0, cq);
      }
      if (stamp) p.trace[((long long)blockIdx.x * 16 + lt) * 4 + 3] = gtimer();
    }
  }

  __syncthreads();
  if (p.prof && threadIdx.x == 0) atomicMax(p.prof + 1, (unsigned long long)gtimer());
}

// ------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

// 4-D bf16 tensor map: dims (inner, rows, b1, b2) with element strides (1, ld, s1, s2); box (64, box_rows, 1, 1).
// Encoded maps are cached per (base, geometry): a training step re-creates the same ~600 maps every step (the caching
// allocator hands back the same activation addresses), and cuTensorMapEncodeTiled is host work on a host-co-limited
// path.  The map only depends on the key, so a stale entry can never be wrong; the cache is dropped when it grows.
struct MapKey {
  const void* base;
  uint64_t inner, rows, nb1, nb2;
  int64_t ld, s1, s2;
  uint32_t box_rows;
  bool operator==(const MapKey& o) const {
    return base == o.base && inner == o.inner && rows == o.rows && nb1 == o.nb1 && nb2 == o.nb2 && ld == o.ld &&
           s1 == o.s1 && s2 == o.s2 && box_rows == o.box_rows;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = reinterpret_cast<uintptr_t>(k.base) * 0x9E3779B97F4A7C15ull;
    auto mix = [&](uint64_t v) { h = (h ^ v) * 0xBF58476D1CE4E5B9ull; h ^= h >> 29; };
    mix(k.inner); mix(k.rows); mix(k.nb1); mix(k.nb2); mix((uint64_t)k.ld); mix((uint64_t)k.s1); mix((uint64_t)k.s2);
    mix(k.box_rows);
    return (size_t)h;
  }
};
int make_tmap_bf16_4d(CUtensorMap* map, const void* base, uint64_t inner, uint64_t rows, uint64_t nb1, uint64_t nb2,
                      int64_t ld, int64_t s1, int64_t s2, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error("cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error("tensor-map operand base not 16-byte aligned");
  if (ld % 8 != 0) return set_error("tensor-map operand leading dimension must be a multiple of 8 elements");
  // unused batch dims get a harmless 16-byte-multiple stride
  if (nb1 <= 1) s1 = ld * (int64_t)rows;
  if (nb2 <= 1) s2 = s1 * (int64_t)(nb1 > 0 ? nb1 : 1);
  if (s1 % 8 != 0 || s2 % 8 != 0) return set_error("tensor-map operand batch strides must be multiples of 8 elements");
  if (s1 == 0) s1 = 8;
  if (s2 == 0) s2 = 8;
  static thread_local std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  const MapKey key{base, inner, rows, nb1, nb2, ld, s1, s2, box_rows};
  auto it = cache.find(key);
  if (it != cache.end()) {
    *map = it->second;
    return 0;
  }
  cuuint64_t dims[4] = {inner, rows, nb1 ? nb1 : 1, nb2 ? nb2 : 1};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)s1 * 2, (cuuint64_t)s2 * 2};
  cuuint32_t box[4] = {64, box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf),
             "cuTensorMapEncodeTiled failed (%d): dims=(%llu,%llu,%llu,%llu) ld=%lld s1=%lld s2=%lld box_rows=%u",
             (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
             (unsigned long long)dims[3], (long long)ld, (long long)s1, (long long)s2, box_rows);
    return set_error(buf);
  }
  if (cache.size() > 8192) cache.clear();
  cache.emplace(key, *map);
  return 0;
}
static inline int make_map(CUtensorMap* map, const void* base, uint64_t inner, uint64_t rows, uint64_t nb1, uint64_t nb2,
                           int64_t ld, int64_t s1, int64_t s2, uint32_t box_rows) {
  return bb::make_tmap_bf16_4d(map, base, inner, rows, nb1, nb2, ld, s1, s2, box_rows);
}

// ---- optional per-launch timing (bench.py roofline): every launch gets a slot of two 64-bit words in a caller-provided
// device buffer; CTAs stamp %globaltimer into it (min of the starts after griddepcontrol.wait, max of the ends), so the
// measured span is the kernel's own execution -- no events between launches, programmatic dependent launch and CUDA-graph
// replay stay intact (a replay overwrites the slots of its launches).
struct ProfRec {
  long long dims[6];  // M, N, K, batches, a_mn, b_mn
};
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;
static size_t g_prof_used = 0;
static unsigned long long* g_prof_buf = nullptr;
static size_t g_prof_cap = 0;

static long long* g_trace = nullptr;   // bb_gemm_trace(): device buffer of (grid x 16 x 4) timestamps, debug only

typedef void (*GemmKernel)(CUtensorMap, CUtensorMap, GemmKParams, int);
template <int BN>
static GemmKernel gemm_kernel(int epi) {
  switch (epi) {
    case EPI_PLAIN: return gemm_tc_kernel<BN, EPI_PLAIN>;
    case EPI_ATOMIC: return gemm_tc_kernel<BN, EPI_ATOMIC>;
    case EPI_GELU_PRE: return gemm_tc_kernel<BN, EPI_GELU_PRE>;
    case EPI_MUL_DGELU: return gemm_tc_kernel<BN, EPI_MUL_DGELU>;
    case EPI_MUL_DRELU: return gemm_tc_kernel<BN, EPI_MUL_DRELU>;
    case EPI_ADD: return gemm_tc_kernel<BN, EPI_ADD>;
    case EPI_SPLIT_DET: return gemm_tc_kernel<BN, EPI_SPLIT_DET>;
    default: return gemm_tc_kernel<BN, EPI_GENERIC>;
  }
}

static int g_num_sms = 0;
static int g_smem_optin = 0;
static int init_device_info() {
  if (g_num_sms) return 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return set_error("cudaGetDevice failed");
  cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&g_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  bool ok = true;
  auto set = [&](auto kernel) {
    ok = ok && cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, g_smem_optin) == cudaSuccess;
  };
  for (int epi = 0; epi < EPI_COUNT; ++epi) {
    set(gemm_kernel<64>(epi));
    set(gemm_kernel<128>(epi));
  }
  if (!ok) return set_error("cudaFuncSetAttribute(max dynamic smem) failed for gemm_tc_kernel");
  return 0;
}

}  // namespace bb

namespace bb {
bool act_f32();                                                    // gemm_f32.cu
int gemm_f32_launch(const bb_gemm_args* a, cudaStream_t stream);   // fp32 verification arm
}  // namespace bb

extern "C" int bb_gemm_bf16(const bb_gemm_args* a, void* stream_) {
  using namespace bb;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (act_f32()) return gemm_f32_launch(a, stream);
  if (!a || !a->A || !a->B || !a->D) return set_error("bb_gemm_bf16: null argument");
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return set_error("bb_gemm_bf16: M, N, K must be positive");
  if (int e = init_device_info()) return e;
  const int nb1 = a->nb1 > 0 ? a->nb1 : 1, nb2 = a->nb2 > 0 ? a->nb2 : 1;
  const int split_k_req = a->split_k > 1 ? a->split_k : 1;
  const bool atomic = a->accumulate || split_k_req > 1;
  if (atomic && !a->out_f32) return set_error("bb_gemm_bf16: accumulate / split_k need fp32 output");
  if (atomic && (a->act || a->epi_mul || a->aux_out || a->add_in || a->drop_thresh))
    return set_error("bb_gemm_bf16: accumulate / split_k cannot be combined with a non-linear epilogue");
  if (a->block_n > 0 && (a->block_n < 16 || a->block_n > 256 || a->block_n % 16 != 0 || (a->b_mn && a->block_n % 64 != 0)))
    return set_error("bb_gemm_bf16: invalid block_n");

  GemmKParams p;
  memset(&p, 0, sizeof(p));
  p.M = a->M;
  p.N = a->N;
  p.K = a->K;
  p.nb1 = nb1;
  p.nb2 = nb2;
  p.a_mn = a->a_mn ? 1 : 0;
  p.b_mn = a->b_mn ? 1 : 0;
  p.m_tiles = (a->M + BLOCK_M - 1) / BLOCK_M;
  // N tile: the kernel is built for 64- and 128-wide tiles (a 64 x 128 fp32 accumulator is 64 registers per thread).
  // A requested block_n is a width hint: <= 64 selects the narrow tile.  Otherwise narrow tiles are used for narrow
  // products and whenever 128-wide tiles would leave more than half of the SMs idle.
  int bn;
  if (a->block_n > 0) {
    bn = a->block_n <= 64 ? 64 : 128;
  } else if (a->N <= 64) {
    bn = 64;
  } else {
    const long long t128 = (long long)p.m_tiles * ((a->N + 127) / 128) * nb1 * nb2 * split_k_req;
    bn = 2 * t128 < g_num_sms ? 64 : 128;
  }
  p.block_n = bn;
  p.n_tiles = (a->N + bn - 1) / bn;
  p.kb_total = (a->K + BLOCK_K - 1) / BLOCK_K;
  int sk = split_k_req < p.kb_total ? split_k_req : p.kb_total;
  p.kb_per_split = (p.kb_total + sk - 1) / sk;
  sk = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
  p.split_k = sk;
  p.out_f32 = a->out_f32 ? 1 : 0;
  p.atomic = atomic ? 1 : 0;
  p.ldd = a->ldd;
  p.d_s1 = a->d_s1;
  p.d_s2 = a->d_s2;
  p.D = a->D;
  p.alpha = a->alpha;
  p.bias = a->bias;
  p.act = a->act;
  p.aux_out = reinterpret_cast<__nv_bfloat16*>(a->aux_out);
  p.aux_in = reinterpret_cast<const __nv_bfloat16*>(a->aux_in);
  p.epi_mul = a->epi_mul;
  p.add_in = reinterpret_cast<const __nv_bfloat16*>(a->add_in);
  p.drop_seed = a->drop_seed;
  p.drop_thresh = a->drop_thresh;
  p.drop_scale = a->drop_scale;
  p.trace = g_trace;
  {
    static int fg = -1;
    if (fg < 0) {
      const char* e_ = getenv("BB_FAST_GELU");
      fg = (e_ && e_[0] == '1') ? 1 : 0;
    }
    p.fast_gelu = fg;
  }
  if (p.epi_mul && !p.aux_in) return set_error("bb_gemm_bf16: epi_mul needs aux_in");
  // paired (2-element) epilogue accesses only when every row segment is suitably aligned
  {
    const int al = 8;  // elements
    bool ok = (a->ldd % al == 0) && (a->d_s1 % al == 0) && (a->d_s2 % al == 0);
    ok = ok && ((reinterpret_cast<uintptr_t>(a->D) & 15) == 0);
    if (a->aux_out) ok = ok && ((reinterpret_cast<uintptr_t>(a->aux_out) & 15) == 0);
    if (a->aux_in) ok = ok && ((reinterpret_cast<uintptr_t>(a->aux_in) & 15) == 0);
    if (a->add_in) ok = ok && ((reinterpret_cast<uintptr_t>(a->add_in) & 15) == 0);
    p.vec_ok = ok ? 1 : 0;
  }

  // epilogue variant: the compile-time one for the feature combination, else the generic one (which also carries the
  // BB_FAST_GELU experiment)
  int epi = EPI_GENERIC;
  const bool plain = !p.act && !p.aux_out && !p.epi_mul && !p.add_in && !p.drop_thresh;
  if (plain) {
    // accumulate without a split has one writer per element, so its atomic add is already deterministic
    epi = p.atomic ? (det_on() && p.split_k > 1 ? EPI_SPLIT_DET : EPI_ATOMIC) : EPI_PLAIN;
  } else if (!p.out_f32 && !p.fast_gelu) {
    if (p.act == 1 && p.aux_out && !p.epi_mul && !p.add_in) epi = EPI_GELU_PRE;
    else if (!p.act && !p.aux_out && p.epi_mul == 1 && !p.add_in) epi = EPI_MUL_DGELU;
    else if (!p.act && !p.aux_out && p.epi_mul == 2 && !p.add_in) epi = EPI_MUL_DRELU;
    else if (!p.act && !p.aux_out && !p.epi_mul && p.add_in) epi = EPI_ADD;
  }

  const int stage_bytes = A_STAGE_BYTES + bn * BLOCK_K * 2;
  const int staging = staging_bytes(bn, epi);
  int stages = (g_smem_optin - 1024 - 256 - staging) / stage_bytes;
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  {
    static int env_stages = -1;  // BB_GEMM_STAGES: pipeline-depth experiments only
    if (env_stages < 0) {
      const char* e_ = getenv("BB_GEMM_STAGES");
      env_stages = e_ ? atoi(e_) : 0;
    }
    if (env_stages >= 2 && env_stages < stages) stages = env_stages;
  }
  if (stages < 2) return set_error("bb_gemm_bf16: not enough shared memory for 2 stages");
  p.stages = stages;
  const size_t smem_bytes = (size_t)staging + (size_t)stages * stage_bytes + 1024 + 256;

  CUtensorMap ta, tb;
  int e;
  if (!p.a_mn) e = make_map(&ta, a->A, a->K, a->M, nb1, nb2, a->lda, a->a_s1, a->a_s2, BLOCK_M);
  else e = make_map(&ta, a->A, a->M, a->K, nb1, nb2, a->lda, a->a_s1, a->a_s2, BLOCK_K);
  if (e) return e;
  if (!p.b_mn) e = make_map(&tb, a->B, a->K, a->N, nb1, nb2, a->ldb, a->b_s1, a->b_s2, bn);
  else e = make_map(&tb, a->B, a->N, a->K, nb1, nb2, a->ldb, a->b_s1, a->b_s2, BLOCK_K);
  if (e) return e;

  const long long total = (long long)p.m_tiles * p.n_tiles * nb1 * nb2 * p.split_k;
  if (total > 0x7fffffffLL) return set_error("bb_gemm_bf16: too many tiles");
  const int grid = total < g_num_sms ? (int)total : g_num_sms;
  if (epi == EPI_SPLIT_DET) {
    const long long tiles = total / p.split_k;
    if (tiles * 4 > (long long)DET_COUNTER_BYTES) return set_error("bb_gemm_bf16: too many output tiles for deterministic split-K");
    p.det_part = det_partials(stream, (size_t)total * BLOCK_M * bn * sizeof(float), "bb_gemm_bf16 (split-K)");
    if (!p.det_part) return -1;
    p.det_cnt = det_counters(stream);
  }
  if (g_prof_on && g_prof_buf && g_prof_used < g_prof_cap) {
    if (g_prof_used == g_prof.size()) g_prof.push_back(ProfRec());
    ProfRec* rec = &g_prof[g_prof_used];
    rec->dims[0] = a->M; rec->dims[1] = a->N; rec->dims[2] = a->K; rec->dims[3] = (long long)nb1 * nb2;
    rec->dims[4] = p.a_mn; rec->dims[5] = p.b_mn;
    p.prof = g_prof_buf + 2 * g_prof_used;
    ++g_prof_used;
  }
  GemmKernel kernel = bn == 64 ? gemm_kernel<64>(epi) : gemm_kernel<128>(epi);
  bb::launch_pdl(kernel, grid, NUM_THREADS, smem_bytes, stream, ta, tb, p, (int)total);
  count_launch();
  return check_launch("gemm_tc_kernel");
}

extern "C" int bb_gemm_trace(long long* device_buf) {
  bb::g_trace = device_buf;
  return 0;
}

extern "C" int bb_gemm_profile_buffer(unsigned long long* device_buf, int64_t capacity_launches) {
  bb::g_prof_buf = device_buf;
  bb::g_prof_cap = device_buf ? (size_t)capacity_launches : 0;
  return 0;
}
extern "C" int bb_gemm_profile(int enable) {
  if (enable && !bb::g_prof_buf) return bb::set_error("bb_gemm_profile: register a device buffer with bb_gemm_profile_buffer first");
  bb::g_prof_on = enable != 0;
  if (enable) bb::g_prof_used = 0;
  return 0;
}
extern "C" int64_t bb_gemm_profile_count(void) { return (int64_t)bb::g_prof_used; }
extern "C" int bb_gemm_profile_read(int64_t idx, float* ms, int64_t* dims6) {
  using namespace bb;
  if (idx < 0 || (size_t)idx >= g_prof_used) return set_error("bb_gemm_profile_read: index out of range");
  unsigned long long t[2];
  if (cudaMemcpy(t, g_prof_buf + 2 * idx, sizeof(t), cudaMemcpyDeviceToHost) != cudaSuccess)
    return set_error("bb_gemm_profile_read: cudaMemcpy failed");
  *ms = (t[1] > t[0] && t[0] != ~0ull) ? (float)((double)(t[1] - t[0]) * 1e-6) : 0.f;
  for (int i = 0; i < 6; ++i) dims6[i] = g_prof[idx].dims[i];
  return 0;
}

namespace bb { int set_salt_gemm_tc(const unsigned long long* p) { return set_drop_salt_ptr_tu(p) == cudaSuccess ? 0 : -1; } }
