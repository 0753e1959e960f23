// HBM-bound row kernels for the BEVBert encoder stack on sm_90a: casts with dropout, fused
// (dropout + residual +) LayerNorm forward/backward, masked softmax forward/backward with the graph bias,
// bias-gradient column sums, embedding sum / scatter, row gather / scatter-add and fused softmax
// cross-entropy. One warp per row where rows are <= 1024 wide, 16-byte vector accesses, fp32 math,
// bf16 storage, warp-shuffle reductions; parameter-gradient reductions use per-block partials + atomics, or, in the
// deterministic mode, per-block partials in a workspace summed in block order by a second kernel (det_reduce).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <initializer_list>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {

typedef __nv_bfloat16 bf16;
bool act_f32();   // gemm_f32.cu: fp32-activation verification mode (bb_set_act_f32)

// Activation storage type T: bf16 in the product, float in the high-precision verification arm (every kernel that
// reads or writes activations is instantiated for both; the C entry points pick by bb::act_f32()).
__device__ __forceinline__ float tof(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float tof(float v) { return v; }
template <typename T> __device__ __forceinline__ T fromf(float v);
template <> __device__ __forceinline__ bf16 fromf<bf16>(float v) { return __float2bfloat16(v); }
template <> __device__ __forceinline__ float fromf<float>(float v) { return v; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ void load8(const bf16* p, float (&v)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void store8(bf16* p, const float (&v)[8]) {
  __align__(16) __nv_bfloat162 h[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = *reinterpret_cast<uint4*>(h);
}
__device__ __forceinline__ void store8(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}

// ------------------------------------------------------------------------------------- casts
template <typename T>
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, T* __restrict__ dst, long long n, uint64_t seed,
                                     uint32_t thresh, float scale) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long stride = (long long)gridDim.x * blockDim.x * 8;
  for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n) {
      float v[8];
      load8(src + i, v);
      if (thresh) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = drop_keep(seed, i + j, thresh) ? v[j] * scale : 0.f;
      }
      store8(dst + i, v);
    } else {
      for (long long j = i; j < n; ++j) {
        float v = src[j];
        if (thresh) v = drop_keep(seed, j, thresh) ? v * scale : 0.f;
        dst[j] = fromf<T>(v);
      }
    }
  }
}
template <typename T>
__global__ void cast_bf16_f32_kernel(const T* __restrict__ src, float* __restrict__ dst, long long n) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long stride = (long long)gridDim.x * blockDim.x * 8;
  for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n) {
      float v[8];
      load8(src + i, v);
      store8(dst + i, v);
    } else {
      for (long long j = i; j < n; ++j) dst[j] = tof(src[j]);
    }
  }
}
template <typename T>
__global__ void add_bf16_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out,
                                long long n) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long stride = (long long)gridDim.x * blockDim.x * 8;
  for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n) {
      float x[8], y[8];
      load8(a + i, x);
      load8(b + i, y);
#pragma unroll
      for (int j = 0; j < 8; ++j) x[j] += y[j];
      store8(out + i, x);
    } else {
      for (long long j = i; j < n; ++j) out[j] = fromf<T>(tof(a[j]) + tof(b[j]));
    }
  }
}
template <typename T>
__global__ void dropout_bf16_kernel(const T* __restrict__ src, T* __restrict__ dst, long long n, uint64_t seed,
                                    uint32_t thresh, float scale) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long stride = (long long)gridDim.x * blockDim.x * 8;
  for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n) {
      float v[8];
      load8(src + i, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = drop_keep(seed, i + j, thresh) ? v[j] * scale : 0.f;
      store8(dst + i, v);
    } else {
      for (long long j = i; j < n; ++j)
        dst[j] = fromf<T>(drop_keep(seed, j, thresh) ? tof(src[j]) * scale : 0.f);
    }
  }
}
template <typename T>
__global__ void act_bwd_bf16_kernel(const T* __restrict__ dy, const T* __restrict__ aux, int mode,
                                    T* __restrict__ out, long long n) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long stride = (long long)gridDim.x * blockDim.x * 8;
  for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n) {
      float g[8], a[8];
      load8(dy + i, g);
      load8(aux + i, a);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = (mode == 1) ? g[j] * dgelu_erf(a[j]) : (a[j] > 0.f ? g[j] : 0.f);
      store8(out + i, g);
    } else {
      for (long long j = i; j < n; ++j) {
        const float a = tof(aux[j]), g = tof(dy[j]);
        out[j] = fromf<T>((mode == 1) ? g * dgelu_erf(a) : (a > 0.f ? g : 0.f));
      }
    }
  }
}
// out = a (+ b) (+ table[idx[r]]) (+ vec)
template <typename T>
__global__ void add_rows_kernel(const T* __restrict__ a, const T* __restrict__ b, const float* __restrict__ table,
                                const int64_t* __restrict__ idx, const float* __restrict__ vec, long long rows, int H,
                                T* __restrict__ out) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const int h8 = H / 8;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= rows * h8) return;
  const long long r = i / h8;
  const int c = (i % h8) * 8;
  float v[8];
  load8(a + r * H + c, v);
  if (b) {
    float t[8];
    load8(b + r * H + c, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] += t[j];
  }
  if (table) {
    float t[8];
    load8(table + idx[r] * H + c, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] += t[j];
  }
  if (vec) {
    float t[8];
    load8(vec + c, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] += t[j];
  }
  store8(out + r * H + c, v);
}
// out = ((a + b) + c) (+ table[idx[r]]) (+ vec), each row operand with its own row stride: the VLN-CE view embedding
// (image + depth + location terms, bevbert_ce/pretrain/pretrain_src/model/vilmodel.py:506-533) in one pass
template <typename T>
__global__ void add_rows3_kernel(const T* __restrict__ a, long long lda, const T* __restrict__ b, long long ldb,
                                 const T* __restrict__ c3, long long ldc, const float* __restrict__ table,
                                 const int64_t* __restrict__ idx, const float* __restrict__ vec, long long rows, int H,
                                 T* __restrict__ out, long long ldo) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const int h8 = H / 8;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= rows * h8) return;
  const long long r = i / h8;
  const int c = (i % h8) * 8;
  float v[8], t[8];
  load8(a + r * lda + c, v);
  load8(b + r * ldb + c, t);
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] += t[j];
  load8(c3 + r * ldc + c, t);
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] += t[j];
  if (table) {
    load8(table + idx[r] * H + c, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] += t[j];
  }
  if (vec) {
    load8(vec + c, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] += t[j];
  }
  store8(out + r * ldo + c, v);
}
template <typename T>
__global__ void scale_rows_bf16_kernel(T* __restrict__ x, const float* __restrict__ g, long long rows, long long ld) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= rows * ld) return;
  x[i] = fromf<T>(tof(x[i]) * g[i / ld]);
}
// one warp per segment; lanes stride over H in 8-wide chunks
template <typename T>
__global__ void segment_wsum_kernel(const T* __restrict__ src, const int32_t* __restrict__ seg_off,
                                    const int32_t* __restrict__ idx, const float* __restrict__ w, long long nseg, int H,
                                    T* __restrict__ out) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const int lane = threadIdx.x & 31;
  const long long s = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (s >= nseg) return;
  const int e0 = seg_off[s], e1 = seg_off[s + 1];
  for (int c = lane * 8; c < H; c += 256) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int e = e0; e < e1; ++e) {
      float v[8];
      load8(src + (long long)idx[e] * H + c, v);
      const float ww = w[e];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += ww * v[j];
    }
    store8(out + s * H + c, acc);
  }
}
template <typename T>
__global__ void segment_wsum_bwd_kernel(const T* __restrict__ dout, const int32_t* __restrict__ seg_off,
                                        const int32_t* __restrict__ idx, const float* __restrict__ w, long long nseg,
                                        int H, float* __restrict__ dsrc) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const int lane = threadIdx.x & 31;
  const long long s = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (s >= nseg) return;
  const int e0 = seg_off[s], e1 = seg_off[s + 1];
  for (int c = lane * 8; c < H; c += 256) {
    float g[8];
    load8(dout + s * H + c, g);
    for (int e = e0; e < e1; ++e) {
      const float ww = w[e];
      float* d = dsrc + (long long)idx[e] * H + c;
#pragma unroll
      for (int j = 0; j < 8; ++j) atomicAdd(d + j, ww * g[j]);
    }
  }
}
template <typename T>
__global__ void axpy_f32_from_bf16_kernel(const T* __restrict__ x, float* __restrict__ y, long long n) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += stride)
    y[i] += tof(x[i]);
}

// ------------------------------------------------------------------------------------- LayerNorm
constexpr int LN_MAXCH = 4;  // 4 chunks of 256 columns -> H <= 1024
constexpr int LN_WARPS = 8;

// Dropout decisions of the LayerNorm sites, one 8-bit keep mask per 8-element vector: a full hash of (seed, vector
// index) and four cheap mixes whose 16-bit halves decide two elements each (keep iff half >= thresh >> 16) -- 4.5
// integer instructions per element instead of a 12-instruction hash each (the backward kernel executed 70 instructions
// per element in round 1, most of them the two per-element hashes).  Forward and backward evaluate the same function.
__device__ __forceinline__ uint32_t ln_keep8(uint64_t seed, long long elem0, uint32_t thresh) {
  const uint32_t h = rng_u32(seed, (uint64_t)(elem0 >> 3));
  const uint32_t t16s = thresh & 0xFFFF0000u;
  uint32_t bits = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    uint32_t x = h + (uint32_t)(k + 1) * 0x9E3779B1u;
    x ^= x >> 15;
    x *= 0x2C1B3C6Du;
    x ^= x >> 16;
    bits |= ((x << 16) >= t16s ? 1u : 0u) << (2 * k);
    bits |= (x >= t16s ? 1u : 0u) << (2 * k + 1);
  }
  return bits;
}
// raw 8-element vectors (kept packed while they wait in registers for the next row)
template <typename T> struct Raw8;
template <> struct Raw8<bf16> {
  uint4 v;
  __device__ __forceinline__ void load(const bf16* p) { v = __ldg(reinterpret_cast<const uint4*>(p)); }
  __device__ __forceinline__ void unpack(float (&f)[8]) const {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = __bfloat1622float2(h[i]);
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
  }
};
template <> struct Raw8<float> {
  float4 a, b;
  __device__ __forceinline__ void load(const float* p) {
    a = __ldg(reinterpret_cast<const float4*>(p));
    b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  }
  __device__ __forceinline__ void unpack(float (&f)[8]) const {
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
    f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
};

template <typename XT, typename T>
__global__ void __launch_bounds__(LN_WARPS * 32)
layernorm_fwd_kernel(const XT* __restrict__ x, const T* __restrict__ res, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, long long rows, int H, uint64_t seed_in,
                     uint32_t thresh_in, float scale_in, uint64_t seed_out, uint32_t thresh_out, float scale_out,
                     T* __restrict__ y, float* __restrict__ y_f32, float* __restrict__ mean_out,
                     float* __restrict__ rstd_out) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * (long long)LN_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const long long base = row * H;
  float z[LN_MAXCH][8];
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < LN_MAXCH; ++c) {
    const int col = c * 256 + lane * 8;
    if (col < H) {
      load8(x + base + col, z[c]);
      if (thresh_in) {
        const uint32_t keep = ln_keep8(seed_in, base + col, thresh_in);
#pragma unroll
        for (int j = 0; j < 8; ++j) z[c][j] = (keep >> j) & 1u ? z[c][j] * scale_in : 0.f;
      }
      if (res) {
        float r[8];
        load8(res + base + col, r);
#pragma unroll
        for (int j = 0; j < 8; ++j) z[c][j] += r[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s += z[c][j];
    }
  }
  const float mean = warp_sum(s) / (float)H;
  float q = 0.f;
#pragma unroll
  for (int c = 0; c < LN_MAXCH; ++c) {
    const int col = c * 256 + lane * 8;
    if (col < H) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = z[c][j] - mean;
        q += d * d;
      }
    }
  }
  const float var = warp_sum(q) / (float)H;
  const float rstd = 1.0f / sqrtf(var + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
#pragma unroll
  for (int c = 0; c < LN_MAXCH; ++c) {
    const int col = c * 256 + lane * 8;
    if (col < H) {
      float g[8], b[8], o[8];
      load8(gamma + col, g);
      load8(beta + col, b);
      const uint32_t keep = thresh_out ? ln_keep8(seed_out, base + col, thresh_out) : 0xFFu;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j] = (z[c][j] - mean) * rstd * g[j] + b[j];
        if (thresh_out) o[j] = (keep >> j) & 1u ? o[j] * scale_out : 0.f;
      }
      if (y) store8(y + base + col, o);
      if (y_f32) store8(y_f32 + base + col, o);
    }
  }
}

// Backward.  Grid-stride over rows, one warp per row; each lane keeps per-column dgamma / dbeta / dxsum partials in
// registers (reduced through shared memory, one atomicAdd per column per block).  NCH = 256-column chunks per row (3 for
// H <= 768).  The three input vectors of the NEXT row are loaded (kept packed) before the current row is processed, so
// every warp has two rows of loads in flight: the round-1 kernel stalled on the load -> reduce -> store chain of a
// single row (ncu: long-scoreboard stalls on the first use of each loaded vector, 0.24 of the HBM peak).
template <typename DYT, typename XT, typename DXT, typename T, int NCH>
__global__ void __launch_bounds__(LN_WARPS * 32)
layernorm_bwd_kernel(const DYT* __restrict__ dy, const XT* __restrict__ x, const T* __restrict__ res,
                     const float* __restrict__ gamma, const float* __restrict__ mean_in,
                     const float* __restrict__ rstd_in, long long rows, int H, uint64_t seed_in, uint32_t thresh_in,
                     float scale_in, uint64_t seed_out, uint32_t thresh_out, float scale_out, DXT* __restrict__ dx,
                     T* __restrict__ dres, float* __restrict__ dgamma, float* __restrict__ dbeta,
                     float* __restrict__ dxsum, float* __restrict__ det_part) {
  bb::pdl_wait();
  bb::pdl_trigger();
  extern __shared__ float ln_part[];  // [3][LN_WARPS][H] per-warp partial dgamma / dbeta / dxsum
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float pg[NCH][8], pb[NCH][8], px[NCH][8];
#pragma unroll
  for (int c = 0; c < NCH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) pg[c][j] = pb[c][j] = px[c][j] = 0.f;
  float gm[NCH][8];
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int col = c * 256 + lane * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) gm[c][j] = 0.f;
    if (col < H) load8(gamma + col, gm[c]);
  }

  const long long rstep = (long long)gridDim.x * LN_WARPS;
  long long row = blockIdx.x * (long long)LN_WARPS + warp;
  Raw8<XT> nx[NCH];
  Raw8<T> nr[NCH];
  Raw8<DYT> nd[NCH];
  float nmean = 0.f, nrstd = 0.f;
  auto fetch = [&](long long r) {
    const long long b = r * H;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = c * 256 + lane * 8;
      if (col < H) {
        nx[c].load(x + b + col);
        if (res) nr[c].load(res + b + col);
        nd[c].load(dy + b + col);
      }
    }
    nmean = mean_in[r];
    nrstd = rstd_in[r];
  };
  if (row < rows) fetch(row);
  for (; row < rows; row += rstep) {
    const long long base = row * H;
    const float mean = nmean, rstd = nrstd;
    float xh[NCH][8], g[NCH][8];
    uint32_t keep_in[NCH];
    float c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = c * 256 + lane * 8;
      keep_in[c] = 0xFFu;
      if (col < H) {
        float z[8], d[8];
        nx[c].unpack(z);
        if (thresh_in) {
          keep_in[c] = ln_keep8(seed_in, base + col, thresh_in);
#pragma unroll
          for (int j = 0; j < 8; ++j) z[j] = (keep_in[c] >> j) & 1u ? z[j] * scale_in : 0.f;
        }
        if (res) {
          float r[8];
          nr[c].unpack(r);
#pragma unroll
          for (int j = 0; j < 8; ++j) z[j] += r[j];
        }
        nd[c].unpack(d);
        const uint32_t keep_out = thresh_out ? ln_keep8(seed_out, base + col, thresh_out) : 0xFFu;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (thresh_out) d[j] = (keep_out >> j) & 1u ? d[j] * scale_out : 0.f;
          xh[c][j] = (z[j] - mean) * rstd;
          g[c][j] = d[j] * gm[c][j];
          c1 += g[c][j];
          c2 += g[c][j] * xh[c][j];
          pg[c][j] += d[j] * xh[c][j];
          pb[c][j] += d[j];
        }
      }
    }
    if (row + rstep < rows) fetch(row + rstep);      // next row's loads fly during the reductions and stores below
    c1 = warp_sum(c1) / (float)H;
    c2 = warp_sum(c2) / (float)H;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = c * 256 + lane * 8;
      if (col < H) {
        float dz[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) dz[j] = rstd * (g[c][j] - c1 - xh[c][j] * c2);
        if (dres) store8(dres + base + col, dz);
        if (dx || dxsum) {
          if (thresh_in) {
#pragma unroll
            for (int j = 0; j < 8; ++j) dz[j] = (keep_in[c] >> j) & 1u ? dz[j] * scale_in : 0.f;
          }
          if (dx) store8(dx + base + col, dz);
#pragma unroll
          for (int j = 0; j < 8; ++j) px[c][j] += dz[j];
        }
      }
    }
  }
  if (dgamma || dbeta || dxsum) {
    float* sg = ln_part;
    float* sb = ln_part + LN_WARPS * H;
    float* sx = ln_part + 2 * LN_WARPS * H;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col = c * 256 + lane * 8;
      if (col < H) {
        store8(sg + warp * H + col, pg[c]);
        store8(sb + warp * H + col, pb[c]);
        store8(sx + warp * H + col, px[c]);
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
      float a = 0.f, b = 0.f, x_ = 0.f;
#pragma unroll
      for (int w = 0; w < LN_WARPS; ++w) {
        a += sg[w * H + i];
        b += sb[w * H + i];
        x_ += sx[w * H + i];
      }
      if (det_part) {   // deterministic mode: this block's partials, summed in block order by det_reduce
        float* pp = det_part + (long long)blockIdx.x * 3 * H;
        pp[i] = a;
        pp[H + i] = b;
        pp[2 * H + i] = x_;
        continue;
      }
      if (dgamma) atomicAdd(dgamma + i, a);
      if (dbeta) atomicAdd(dbeta + i, b);
      if (dxsum) atomicAdd(dxsum + i, x_);
    }
  }
}

// ------------------------------------------------------------------------------------- column sums
template <typename T>
__global__ void __launch_bounds__(256)
colsum_bf16_kernel(const T* __restrict__ x, long long rows, int N, long long ld, float* __restrict__ out,
                   float* __restrict__ det_part) {
  bb::pdl_wait();
  bb::pdl_trigger();
  // blockDim = (32, 8): 32 lanes x 8 columns each = 256 columns per block in x; rows strided over y and grid.y
  __shared__ float part[8][256];
  const int col = blockIdx.x * 256 + threadIdx.x * 8;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (col < N) {
    const bool vec = (col + 8 <= N) && (ld % 8 == 0);
    const long long rstep = (long long)gridDim.y * 8;
    long long r = blockIdx.y * 8 + threadIdx.y;
    if (vec) {
      for (; r + 3 * rstep < rows; r += 4 * rstep) {      // four independent 16-byte loads in flight per lane
        float v0[8], v1[8], v2[8], v3[8];
        load8(x + r * ld + col, v0);
        load8(x + (r + rstep) * ld + col, v1);
        load8(x + (r + 2 * rstep) * ld + col, v2);
        load8(x + (r + 3 * rstep) * ld + col, v3);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += (v0[j] + v1[j]) + (v2[j] + v3[j]);
      }
    }
    for (; r < rows; r += rstep) {
      if (vec) {
        float v[8];
        load8(x + r * ld + col, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += v[j];
      } else {
        for (int j = 0; j < 8; ++j)
          if (col + j < N) acc[j] += tof(x[r * ld + col + j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[threadIdx.y][threadIdx.x * 8 + j] = acc[j];
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;
  float s = 0.f;
#pragma unroll
  for (int yy = 0; yy < 8; ++yy) s += part[yy][t];
  const int c = blockIdx.x * 256 + t;
  if (c >= N) return;
  if (det_part) det_part[(long long)blockIdx.y * N + c] = s;   // deterministic mode: summed by det_reduce
  else atomicAdd(out + c, s);
}

// o_k[i] += sum of the partials part[p][k][i] over p in ascending order (see common.h)
__global__ void det_reduce_kernel(const float* __restrict__ part, int nparts, long long n, int nout, float* o0,
                                  float* o1, float* o2) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n * nout; i += stride) {
    const int k = (int)(i / n);
    const long long e = i - (long long)k * n;
    float* o = k == 0 ? o0 : (k == 1 ? o1 : o2);
    if (!o) continue;
    float s = part[i];
    for (int p = 1; p < nparts; ++p) s += part[(long long)p * nout * n + i];
    o[e] += s;
  }
}

// ------------------------------------------------------------------------------------- softmax
template <int MAXE, typename T>
__global__ void __launch_bounds__(256)
softmax_fwd_kernel(const float* __restrict__ scores, const float* __restrict__ kmask, const float* __restrict__ bias,
                   long long nrows, int H, int nq, int nk, int ld, uint64_t seed, uint32_t thresh, float scale,
                   T* __restrict__ probs, T* __restrict__ probs_drop) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (row >= nrows) return;
  const int q = row % nq;
  const long long b = row / ((long long)nq * H);
  const float* s = scores + row * ld;
  const float* km = kmask ? kmask + b * nk : nullptr;
  const float* bs = bias ? bias + (b * nq + q) * nk : nullptr;
  float v[MAXE];
  float mx = -INFINITY;
#pragma unroll
  for (int e = 0; e < MAXE; ++e) {
    const int k = e * 32 + lane;
    float t = -INFINITY;
    if (k < nk) {
      t = s[k];
      if (km) t += km[k];
      if (bs) t += bs[k];
    }
    v[e] = t;
    mx = fmaxf(mx, t);
  }
  mx = warp_max(mx);
  // every key masked with -inf: exp(-inf - 0) = 0 and P = Pd = 0, as the flash cores give, instead of -inf - -inf = NaN
  if (mx == -INFINITY) mx = 0.f;
  float sum = 0.f;
#pragma unroll
  for (int e = 0; e < MAXE; ++e) {
    const int k = e * 32 + lane;
    const float ex = (k < nk) ? __expf(v[e] - mx) : 0.f;
    v[e] = ex;
    sum += ex;
  }
  sum = warp_sum(sum);
  const float inv = sum > 0.f ? 1.0f / sum : 0.f;
  T* p = probs + row * ld;
  T* pd = probs_drop ? probs_drop + row * ld : nullptr;
#pragma unroll
  for (int e = 0; e < MAXE; ++e) {
    const int k = e * 32 + lane;
    if (k < ld) {
      const float pr = (k < nk) ? v[e] * inv : 0.f;
      p[k] = fromf<T>(pr);
      if (pd) {
        float t = pr;
        if (thresh) t = drop_keep(seed, row * ld + k, thresh) ? pr * scale : 0.f;
        pd[k] = fromf<T>(t);
      }
    }
  }
}

template <int MAXE, typename T>
__global__ void __launch_bounds__(256)
softmax_bwd_kernel(const T* __restrict__ probs, const float* __restrict__ dprobs, long long nrows, int H, int nq,
                   int nk, int ld, uint64_t seed, uint32_t thresh, float scale, float out_scale, T* __restrict__ ds,
                   float* __restrict__ dbias, long long dbias_hs) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (row >= nrows) return;
  const int q = row % nq;
  const long long b = row / ((long long)nq * H);
  const T* p = probs + row * ld;
  const float* dp = dprobs + row * ld;
  float pv[MAXE], g[MAXE];
  float dot = 0.f;
#pragma unroll
  for (int e = 0; e < MAXE; ++e) {
    const int k = e * 32 + lane;
    pv[e] = 0.f;
    g[e] = 0.f;
    if (k < nk) {
      pv[e] = tof(p[k]);
      float t = dp[k];
      if (thresh) t = drop_keep(seed, row * ld + k, thresh) ? t * scale : 0.f;
      g[e] = t;
      dot += pv[e] * t;
    }
  }
  dot = warp_sum(dot);
  T* o = ds + row * ld;
  // dbias_hs != 0 (deterministic mode): per-head partials dbias[h] at a stride of dbias_hs, one plain store each
  float* db = dbias ? dbias + (dbias_hs ? (row / nq % H) * dbias_hs : 0) + (b * nq + q) * nk : nullptr;
#pragma unroll
  for (int e = 0; e < MAXE; ++e) {
    const int k = e * 32 + lane;
    if (k < ld) {
      const float d = (k < nk) ? pv[e] * (g[e] - dot) : 0.f;
      o[k] = fromf<T>(d * out_scale);
      if (db && k < nk) {
        if (dbias_hs) db[k] = d;
        else atomicAdd(db + k, d);
      }
    }
  }
}

// ------------------------------------------------------------------------------------- embeddings
__global__ void embed_sum_kernel(const int64_t* __restrict__ ids, const float* __restrict__ word,
                                 const float* __restrict__ pos, const float* __restrict__ type0, long long ntok, int L,
                                 int H, float* __restrict__ out) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;  // over ntok * H/4
  const int h4 = H / 4;
  if (i >= ntok * h4) return;
  const long long tok = i / h4;
  const int c = (i % h4) * 4;
  const int l = tok % L;
  const float4 w = __ldg(reinterpret_cast<const float4*>(word + ids[tok] * H + c));
  const float4 p = __ldg(reinterpret_cast<const float4*>(pos + (long long)l * H + c));
  const float4 t = __ldg(reinterpret_cast<const float4*>(type0 + c));
  float4 o;
  o.x = (w.x + p.x) + t.x;
  o.y = (w.y + p.y) + t.y;
  o.z = (w.z + p.z) + t.z;
  o.w = (w.w + p.w) + t.w;
  *reinterpret_cast<float4*>(out + tok * H + c) = o;
}
__global__ void embed_scatter_grad_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dz, long long ntok,
                                          int L, int H, int64_t padding_idx, float* __restrict__ dword,
                                          float* __restrict__ dpos, float* __restrict__ dtype0) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= ntok * H) return;
  const long long tok = i / H;
  const int c = i % H;
  const int l = tok % L;
  const float g = dz[i];
  const int64_t id = ids[tok];
  if (dword && id != padding_idx) atomicAdd(dword + id * H + c, g);
  if (dpos) atomicAdd(dpos + (long long)l * H + c, g);
  if (dtype0) atomicAdd(dtype0 + c, g);
}

// ------------------------------------------------------------------------------------- gather / scatter rows
template <typename T>
__global__ void gather_rows_bf16_kernel(const T* __restrict__ in, const int64_t* __restrict__ idx, long long nout,
                                        int H, T* __restrict__ out) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const int h8 = H / 8;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= nout * h8) return;
  const long long r = i / h8;
  const int c = (i % h8) * 8;
  const int64_t src = idx[r];
  float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (src >= 0) load8(in + src * H + c, v);
  store8(out + r * H + c, v);
}
template <typename T>
__global__ void scatter_add_rows_kernel(const T* __restrict__ in, const int64_t* __restrict__ idx, long long nin,
                                        int H, float* __restrict__ out) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= nin * H) return;
  const long long r = i / H;
  const int c = i % H;
  const int64_t dst = idx[r];
  if (dst >= 0) atomicAdd(out + dst * H + c, tof(in[i]));
}
// Deterministic scatter-add by destination: entries e = 0 .. n-1 are sorted by destination dst[e] (stably, so equal
// destinations keep ascending source order); out[d] += ((t_e1 + t_e2) + ...) over the run of entries with dst == d,
// t_e = w[e] * src[src_row[e]] (one rounded product, no FMA) or src[src_row[e]] without w.  dst < 0 is dropped.  The
// thread of a run's first entry walks the run, 8 columns at a time.
template <typename S>
__global__ void scatter_rows_sorted_kernel(const S* __restrict__ src, const int64_t* __restrict__ src_row,
                                           const float* __restrict__ w, const int64_t* __restrict__ dst, long long n,
                                           int H, float* __restrict__ out) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const int h8 = H / 8;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n * h8) return;
  const long long e0 = i / h8;
  const int c = (int)(i % h8) * 8;
  const int64_t d = dst[e0];
  if (d < 0 || (e0 > 0 && dst[e0 - 1] == d)) return;
  float acc[8];
  for (long long e = e0; e < n && dst[e] == d; ++e) {
    float v[8];
    load8(src + src_row[e] * H + c, v);
    if (w) {
      const float ww = w[e];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = __fmul_rn(ww, v[j]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = e == e0 ? v[j] : __fadd_rn(acc[j], v[j]);
  }
  float o[8];
  float* po = out + d * H + c;
  load8(po, o);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = __fadd_rn(o[j], acc[j]);
  store8(po, o);
}

// ------------------------------------------------------------------------------------- softmax cross entropy
template <typename T>
__global__ void __launch_bounds__(256)
softmax_xent_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels, int V, long long ld,
                    float* __restrict__ loss, const float* __restrict__ gscale, T* __restrict__ dlogits) {
  bb::pdl_wait();
  bb::pdl_trigger();
  __shared__ float red[8];
  __shared__ float bcast;
  const long long row = blockIdx.x;
  const float* x = logits + row * ld;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t lab = labels[row];
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < V; i += 256) mx = fmaxf(mx, x[i]);
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = red[0];
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    bcast = m;
  }
  __syncthreads();
  mx = bcast;
  float s = 0.f;
  for (int i = threadIdx.x; i < V; i += 256) s += __expf(x[i] - mx);
  s = warp_sum(s);
  __syncthreads();
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    bcast = t;
  }
  __syncthreads();
  s = bcast;
  const bool valid = lab >= 0 && lab < V;
  if (threadIdx.x == 0) loss[row] = valid ? (logf(s) + mx - x[lab]) : 0.f;
  if (dlogits) {
    const float gs = valid ? (gscale ? gscale[row] : 1.f) : 0.f;
    const float inv = 1.0f / s;
    T* d = dlogits + row * ld;
    for (int i = threadIdx.x; i < ld; i += 256) {
      float g = 0.f;
      if (i < V) g = (__expf(x[i] - mx) * inv - (i == lab ? 1.f : 0.f)) * gs;
      d[i] = fromf<T>(g);
    }
  }
}

static int device_sms() {   // grid caps of the grid-strided kernels: the SM count of the device this library runs on
  static int n = 0;
  if (!n) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;   // H100 SXM
  }
  return n;
}
static inline unsigned grid1d(long long n, int per_block, int cap = 0) {
  if (cap <= 0) cap = device_sms() * 16;
  long long g = (n + per_block - 1) / per_block;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (unsigned)g;
}

// every pointer of an entry point whose kernel reads or writes it in 16-byte vectors (NULL counts as aligned)
static inline bool aligned16(std::initializer_list<const void*> ps) {
  for (const void* p : ps)
    if (reinterpret_cast<uintptr_t>(p) & 15) return false;
  return true;
}

}  // namespace bb

using namespace bb;
#define STREAM ((cudaStream_t)stream)
// run the statement with T = float in the fp32 verification mode, T = bf16 otherwise
#define ACT_T(...)              \
  do {                          \
    if (bb::act_f32()) {        \
      typedef float T;          \
      __VA_ARGS__;              \
    } else {                    \
      typedef bf16 T;           \
      __VA_ARGS__;              \
    }                           \
  } while (0)

extern "C" int bb_cast_f32_bf16(const float* src, void* dst, int64_t n, uint64_t seed, uint32_t thresh, float scale,
                                void* stream) {
  if (n <= 0) return 0;
  if (((uintptr_t)src & 15) || ((uintptr_t)dst & 15)) return set_error("bb_cast_f32_bf16: pointers must be 16B aligned");
  ACT_T(bb::launch_pdl(cast_f32_bf16_kernel<T>, grid1d(n, 256 * 8), 256, 0, STREAM, src, (T*)dst, n, seed, thresh, scale));
  count_launch();
  return check_launch("cast_f32_bf16_kernel");
}
extern "C" int bb_cast_bf16_f32(const void* src, float* dst, int64_t n, void* stream) {
  if (n <= 0) return 0;
  if (((uintptr_t)src & 15) || ((uintptr_t)dst & 15)) return set_error("bb_cast_bf16_f32: pointers must be 16B aligned");
  ACT_T(bb::launch_pdl(cast_bf16_f32_kernel<T>, grid1d(n, 256 * 8), 256, 0, STREAM, (const T*)src, dst, n));
  count_launch();
  return check_launch("cast_bf16_f32_kernel");
}
extern "C" int bb_add_bf16(const void* a, const void* b, void* out, int64_t n, void* stream) {
  if (n <= 0) return 0;
  if (((uintptr_t)a & 15) || ((uintptr_t)b & 15) || ((uintptr_t)out & 15))
    return set_error("bb_add_bf16: pointers must be 16B aligned");
  ACT_T(bb::launch_pdl(add_bf16_kernel<T>, grid1d(n, 256 * 8), 256, 0, STREAM, (const T*)a, (const T*)b, (T*)out, n));
  count_launch();
  return check_launch("add_bf16_kernel");
}
extern "C" int bb_dropout_bf16(const void* src, void* dst, int64_t n, uint64_t seed, uint32_t thresh, float scale,
                               void* stream) {
  if (n <= 0) return 0;
  if (((uintptr_t)src & 15) || ((uintptr_t)dst & 15)) return set_error("bb_dropout_bf16: pointers must be 16B aligned");
  ACT_T(bb::launch_pdl(dropout_bf16_kernel<T>, grid1d(n, 256 * 8), 256, 0, STREAM, (const T*)src, (T*)dst, n, seed, thresh, scale));
  count_launch();
  return check_launch("dropout_bf16_kernel");
}
extern "C" int bb_act_bwd_bf16(const void* dy, const void* aux, int mode, void* out, int64_t n, void* stream) {
  if (n <= 0) return 0;
  if (mode != 1 && mode != 2) return set_error("bb_act_bwd_bf16: mode must be 1 (gelu) or 2 (relu)");
  if (((uintptr_t)dy & 15) || ((uintptr_t)aux & 15) || ((uintptr_t)out & 15))
    return set_error("bb_act_bwd_bf16: pointers must be 16B aligned");
  ACT_T(bb::launch_pdl(act_bwd_bf16_kernel<T>, grid1d(n, 256 * 8), 256, 0, STREAM, (const T*)dy, (const T*)aux, mode, (T*)out, n));
  count_launch();
  return check_launch("act_bwd_bf16_kernel");
}
extern "C" int bb_add_rows(const void* a, const void* b, const float* table, const int64_t* idx, const float* vec,
                           int64_t rows, int H, void* out, void* stream) {
  if (rows <= 0) return 0;
  if (H % 8 != 0) return set_error("bb_add_rows: H must be a multiple of 8");
  if (table && !idx) return set_error("bb_add_rows: table needs idx");
  if (!aligned16({a, b, table, vec, out})) return set_error("bb_add_rows: a / b / table / vec / out must be 16-byte aligned");
  const long long n = rows * (H / 8);
  ACT_T(bb::launch_pdl(add_rows_kernel<T>, (unsigned)((n + 255) / 256), 256, 0, STREAM, (const T*)a, (const T*)b, table, idx, vec,
                                                                   rows, H, (T*)out));
  count_launch();
  return check_launch("add_rows_kernel");
}
extern "C" int bb_add_rows3(const void* a, int64_t lda, const void* b, int64_t ldb, const void* c, int64_t ldc,
                            const float* table, const int64_t* idx, const float* vec, int64_t rows, int H, void* out,
                            int64_t ldo, void* stream) {
  if (rows <= 0) return 0;
  if (H <= 0 || H % 8 != 0) return set_error("bb_add_rows3: H must be a positive multiple of 8");
  if (!a || !b || !c || !out) return set_error("bb_add_rows3: a / b / c / out must not be NULL");
  if (table && !idx) return set_error("bb_add_rows3: table needs idx");
  for (int64_t ld : {lda, ldb, ldc, ldo})
    if (ld < H || ld % 8 != 0) return set_error("bb_add_rows3: every row stride must be >= H and a multiple of 8");
  if (!aligned16({a, b, c, table, vec, out}))
    return set_error("bb_add_rows3: a / b / c / table / vec / out must be 16-byte aligned");
  const long long n = rows * (H / 8);
  ACT_T(bb::launch_pdl(add_rows3_kernel<T>, (unsigned)((n + 255) / 256), 256, 0, STREAM, (const T*)a, (long long)lda,
                       (const T*)b, (long long)ldb, (const T*)c, (long long)ldc, table, idx, vec, (long long)rows, H,
                       (T*)out, (long long)ldo));
  count_launch();
  return check_launch("add_rows3_kernel");
}
extern "C" int bb_scale_rows_bf16(void* x, const float* g, int64_t rows, int64_t ld, void* stream) {
  if (rows <= 0) return 0;
  const long long n = rows * ld;
  ACT_T(bb::launch_pdl(scale_rows_bf16_kernel<T>, (unsigned)((n + 255) / 256), 256, 0, STREAM, (T*)x, g, rows, ld));
  count_launch();
  return check_launch("scale_rows_bf16_kernel");
}
extern "C" int bb_segment_wsum(const void* src, const int32_t* seg_off, const int32_t* idx, const float* w,
                               int64_t nseg, int H, void* out, void* stream) {
  if (nseg <= 0) return 0;
  if (H % 8 != 0) return set_error("bb_segment_wsum: H must be a multiple of 8");
  if (!aligned16({src, out})) return set_error("bb_segment_wsum: src / out must be 16-byte aligned");
  ACT_T(bb::launch_pdl(segment_wsum_kernel<T>, (unsigned)((nseg + 7) / 8), 256, 0, STREAM, (const T*)src, seg_off, idx, w, nseg, H,
                                                                      (T*)out));
  count_launch();
  return check_launch("segment_wsum_kernel");
}
extern "C" int bb_segment_wsum_bwd(const void* dout, const int32_t* seg_off, const int32_t* idx, const float* w,
                                   int64_t nseg, int H, float* dsrc_f32, void* stream) {
  if (nseg <= 0) return 0;
  if (H % 8 != 0) return set_error("bb_segment_wsum_bwd: H must be a multiple of 8");
  if (!aligned16({dout})) return set_error("bb_segment_wsum_bwd: dout must be 16-byte aligned");
  if (det_on()) return set_error("bb_segment_wsum_bwd adds with atomics; in deterministic mode use bb_scatter_rows_sorted");
  ACT_T(bb::launch_pdl(segment_wsum_bwd_kernel<T>, (unsigned)((nseg + 7) / 8), 256, 0, STREAM, (const T*)dout, seg_off, idx, w, nseg, H,
                                                                          dsrc_f32));
  count_launch();
  return check_launch("segment_wsum_bwd_kernel");
}
extern "C" int bb_axpy_f32_from_bf16(const void* x, float* y, int64_t n, void* stream) {
  if (n <= 0) return 0;
  ACT_T(bb::launch_pdl(axpy_f32_from_bf16_kernel<T>, grid1d(n, 256), 256, 0, STREAM, (const T*)x, y, n));
  count_launch();
  return check_launch("axpy_f32_from_bf16_kernel");
}

extern "C" int bb_layernorm_fwd(const void* x, int x_f32, const void* residual, const float* gamma, const float* beta,
                                float eps, int64_t rows, int H, uint64_t seed_in, uint32_t thresh_in, float scale_in,
                                uint64_t seed_out, uint32_t thresh_out, float scale_out, void* y, float* y_f32,
                                float* mean, float* rstd, void* stream) {
  if (rows <= 0) return 0;
  if (H % 8 != 0 || H > LN_MAXCH * 256) return set_error("bb_layernorm_fwd: H must be a multiple of 8 and <= 1024");
  if (!aligned16({x, residual, gamma, beta, y, y_f32}))
    return set_error("bb_layernorm_fwd: x / residual / gamma / beta / y / y_f32 must be 16-byte aligned");
  const unsigned grid = (unsigned)((rows + LN_WARPS - 1) / LN_WARPS);
  if (x_f32)
    ACT_T(bb::launch_pdl(layernorm_fwd_kernel<float, T>, grid, LN_WARPS * 32, 0, STREAM, 
        (const float*)x, (const T*)residual, gamma, beta, eps, rows, H, seed_in, thresh_in, scale_in, seed_out,
        thresh_out, scale_out, (T*)y, y_f32, mean, rstd));
  else
    ACT_T(bb::launch_pdl(layernorm_fwd_kernel<bf16, T>, grid, LN_WARPS * 32, 0, STREAM, 
        (const bf16*)x, (const T*)residual, gamma, beta, eps, rows, H, seed_in, thresh_in, scale_in, seed_out,
        thresh_out, scale_out, (T*)y, y_f32, mean, rstd));
  count_launch();
  return check_launch("layernorm_fwd_kernel");
}

extern "C" int bb_layernorm_bwd(const void* dy, int dy_f32, const void* x, int x_f32, const void* residual,
                                const float* gamma, const float* mean, const float* rstd, int64_t rows, int H,
                                uint64_t seed_in, uint32_t thresh_in, float scale_in, uint64_t seed_out,
                                uint32_t thresh_out, float scale_out, void* dx, int dx_f32, void* dres, float* dgamma,
                                float* dbeta, float* dxsum, void* stream) {
  if (rows <= 0) return 0;
  if (H % 8 != 0 || H > LN_MAXCH * 256) return set_error("bb_layernorm_bwd: H must be a multiple of 8 and <= 1024");
  if (!aligned16({dy, x, residual, gamma, dx, dres}))
    return set_error("bb_layernorm_bwd: dy / x / residual / gamma / dx / dres must be 16-byte aligned");
  long long g = (rows + LN_WARPS - 1) / LN_WARPS;
  if (g > device_sms()) g = device_sms();   // one resident block per SM (233 registers), rows grid-strided
  const unsigned grid = (unsigned)g;
  const size_t ln_smem = (size_t)3 * LN_WARPS * H * sizeof(float);
  float* part = nullptr;
  if (det_on() && (dgamma || dbeta || dxsum)) {
    part = det_partials(STREAM, (size_t)grid * 3 * H * sizeof(float), "bb_layernorm_bwd");
    if (!part) return -1;
  }
#define LN_BWD(DYT, XT, DXT, AT)                                                                                    \
  do {                                                                                                              \
    static bool attr_done = false;                                                                                  \
    if (!attr_done) {                                                                                               \
      cudaFuncSetAttribute(layernorm_bwd_kernel<DYT, XT, DXT, AT, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 98304); \
      cudaFuncSetAttribute(layernorm_bwd_kernel<DYT, XT, DXT, AT, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 98304); \
      attr_done = true;                                                                                             \
    }                                                                                                               \
    if (H <= 768)                                                                                                   \
      bb::launch_pdl(layernorm_bwd_kernel<DYT, XT, DXT, AT, 3>, grid, LN_WARPS * 32, ln_smem, STREAM, (const DYT*)dy, \
                     (const XT*)x, (const AT*)residual, gamma, mean, rstd, rows, H, seed_in, thresh_in, scale_in,   \
                     seed_out, thresh_out, scale_out, (DXT*)dx, (AT*)dres, dgamma, dbeta, dxsum, part);             \
    else                                                                                                            \
      bb::launch_pdl(layernorm_bwd_kernel<DYT, XT, DXT, AT, 4>, grid, LN_WARPS * 32, ln_smem, STREAM, (const DYT*)dy, \
                     (const XT*)x, (const AT*)residual, gamma, mean, rstd, rows, H, seed_in, thresh_in, scale_in,   \
                     seed_out, thresh_out, scale_out, (DXT*)dx, (AT*)dres, dgamma, dbeta, dxsum, part);             \
  } while (0)
  if (bb::act_f32()) {
    if (dy_f32 && x_f32 && dx_f32) LN_BWD(float, float, float, float);
    else return set_error("bb_layernorm_bwd: the fp32 verification mode needs fp32 dy / x / dx");
  } else if (!dy_f32 && !x_f32 && !dx_f32) LN_BWD(bf16, bf16, bf16, bf16);
  else if (!dy_f32 && x_f32 && dx_f32) LN_BWD(bf16, float, float, bf16);
  else if (dy_f32 && !x_f32 && !dx_f32) LN_BWD(float, bf16, bf16, bf16);
  else if (dy_f32 && x_f32 && dx_f32) LN_BWD(float, float, float, bf16);
  else if (!dy_f32 && !x_f32 && dx_f32) LN_BWD(bf16, bf16, float, bf16);
  else if (!dy_f32 && x_f32 && !dx_f32) LN_BWD(bf16, float, bf16, bf16);
  else return set_error("bb_layernorm_bwd: unsupported dtype combination");
#undef LN_BWD
  count_launch();
  if (int e = check_launch("layernorm_bwd_kernel")) return e;
  return part ? det_reduce(part, (int)grid, H, 3, dgamma, dbeta, dxsum, STREAM) : 0;
}

namespace bb {
template <typename T>
static int colsum_run(const T* x, long long rows, int N, long long ld, float* out, cudaStream_t stream) {
  if (rows <= 0 || N <= 0) return 0;
  if (ld % 8 == 0 && !aligned16({x}))      // the kernel reads 16-byte vectors exactly when ld % 8 == 0
    return set_error("bb_colsum_bf16: x must be 16-byte aligned when ld is a multiple of 8");
  long long gy = (rows + 63) / 64;
  if (gy > 64) gy = 64;
  dim3 grid((N + 255) / 256, (unsigned)gy);
  float* part = nullptr;
  if (det_on()) {
    part = det_partials(stream, (size_t)gy * N * sizeof(float), "bb_colsum_bf16");
    if (!part) return -1;
  }
  bb::launch_pdl(colsum_bf16_kernel<T>, grid, dim3(32, 8), 0, stream, x, rows, N, ld, out, part);
  count_launch();
  if (int e = check_launch("colsum_bf16_kernel")) return e;
  return part ? det_reduce(part, (int)gy, N, 1, out, nullptr, nullptr, stream) : 0;
}

int det_reduce(const float* part, int nparts, long long n, int nout, float* o0, float* o1, float* o2,
               cudaStream_t stream) {
  if (n <= 0 || nparts <= 0) return 0;
  bb::launch_pdl(det_reduce_kernel, grid1d(n * nout, 256), 256, 0, stream, part, nparts, n, nout, o0, o1, o2);
  count_launch();
  return check_launch("det_reduce_kernel");
}
}  // namespace bb

extern "C" int bb_colsum_bf16(const void* x, int64_t rows, int N, int64_t ld, float* out, void* stream) {
  int rc = 0;
  ACT_T(rc = colsum_run((const T*)x, rows, N, ld, out, STREAM));
  return rc;
}

extern "C" int bb_softmax_fwd(const float* scores, const float* kmask, const float* bias, int nbatch, int H, int nq,
                              int nk, int ld, uint64_t seed, uint32_t thresh, float scale, void* probs,
                              void* probs_drop, void* stream) {
  const long long nrows = (long long)nbatch * H * nq;
  if (nrows <= 0) return 0;
  if (ld < nk || ld > 1024) return set_error("bb_softmax_fwd: need nk <= ld <= 1024");
  const unsigned grid = (unsigned)((nrows + 7) / 8);
  if (ld <= 128)
    ACT_T(bb::launch_pdl(softmax_fwd_kernel<4, T>, grid, 256, 0, STREAM, scores, kmask, bias, nrows, H, nq, nk, ld, seed, thresh, scale,
                                                    (T*)probs, (T*)probs_drop));
  else if (ld <= 512)
    ACT_T(bb::launch_pdl(softmax_fwd_kernel<16, T>, grid, 256, 0, STREAM, scores, kmask, bias, nrows, H, nq, nk, ld, seed, thresh, scale,
                                                     (T*)probs, (T*)probs_drop));
  else
    ACT_T(bb::launch_pdl(softmax_fwd_kernel<32, T>, grid, 256, 0, STREAM, scores, kmask, bias, nrows, H, nq, nk, ld, seed, thresh, scale,
                                                     (T*)probs, (T*)probs_drop));
  count_launch();
  return check_launch("softmax_fwd_kernel");
}

extern "C" int bb_softmax_bwd(const void* probs, const float* dprobs, int nbatch, int H, int nq, int nk, int ld,
                              uint64_t seed, uint32_t thresh, float scale, float out_scale, void* ds, float* dbias,
                              void* stream) {
  const long long nrows = (long long)nbatch * H * nq;
  if (nrows <= 0) return 0;
  if (ld < nk || ld > 1024) return set_error("bb_softmax_bwd: need nk <= ld <= 1024");
  const unsigned grid = (unsigned)((nrows + 7) / 8);
  float* dbias_out = dbias;
  long long hs = 0;   // deterministic mode: per-head bias-gradient partials, then a sum over heads in head order
  if (dbias && det_on()) {
    hs = (long long)nbatch * nq * nk;
    dbias = det_partials(STREAM, (size_t)H * hs * sizeof(float), "bb_softmax_bwd (graph-bias gradient)");
    if (!dbias) return -1;
  }
  if (ld <= 128)
    ACT_T(bb::launch_pdl(softmax_bwd_kernel<4, T>, grid, 256, 0, STREAM, (const T*)probs, dprobs, nrows, H, nq, nk, ld, seed, thresh,
                                                    scale, out_scale, (T*)ds, dbias, hs));
  else if (ld <= 512)
    ACT_T(bb::launch_pdl(softmax_bwd_kernel<16, T>, grid, 256, 0, STREAM, (const T*)probs, dprobs, nrows, H, nq, nk, ld, seed, thresh,
                                                     scale, out_scale, (T*)ds, dbias, hs));
  else
    ACT_T(bb::launch_pdl(softmax_bwd_kernel<32, T>, grid, 256, 0, STREAM, (const T*)probs, dprobs, nrows, H, nq, nk, ld, seed, thresh,
                                                     scale, out_scale, (T*)ds, dbias, hs));
  count_launch();
  if (int e = check_launch("softmax_bwd_kernel")) return e;
  return hs ? det_reduce(dbias, H, hs, 1, dbias_out, nullptr, nullptr, STREAM) : 0;
}

extern "C" int bb_embed_sum(const int64_t* ids, const float* word, const float* pos, const float* type0, int64_t ntok,
                            int L, int H, float* out, void* stream) {
  if (ntok <= 0) return 0;
  if (H % 4 != 0) return set_error("bb_embed_sum: H must be a multiple of 4");
  if (!aligned16({word, pos, type0, out})) return set_error("bb_embed_sum: word / pos / type0 / out must be 16-byte aligned");
  const long long n = ntok * (H / 4);
  bb::launch_pdl(embed_sum_kernel, (unsigned)((n + 255) / 256), 256, 0, STREAM, ids, word, pos, type0, ntok, L, H, out);
  count_launch();
  return check_launch("embed_sum_kernel");
}
extern "C" int bb_embed_scatter_grad(const int64_t* ids, const float* dz, int64_t ntok, int L, int H,
                                     int64_t padding_idx, float* dword, float* dpos, float* dtype0, void* stream) {
  if (ntok <= 0) return 0;
  if (det_on()) {
    // word table: by destination through bb_scatter_rows_sorted; position table: dpos[l] += sum over b, in b order, of
    // dz[b, l]; type row: a column sum
    if (dword) return set_error("bb_embed_scatter_grad: in deterministic mode the word-table gradient goes through "
                                "bb_scatter_rows_sorted (pass dword = NULL)");
    if (dpos && ntok % L) return set_error("bb_embed_scatter_grad: ntok must be a multiple of L");
    if (dpos) {
      if (int e = det_reduce(dz, (int)(ntok / L), (long long)L * H, 1, dpos, nullptr, nullptr, STREAM)) return e;
    }
    return dtype0 ? colsum_run(dz, ntok, H, H, dtype0, STREAM) : 0;
  }
  const long long n = ntok * H;
  bb::launch_pdl(embed_scatter_grad_kernel, (unsigned)((n + 255) / 256), 256, 0, STREAM, ids, dz, ntok, L, H, padding_idx, dword,
                                                                             dpos, dtype0);
  count_launch();
  return check_launch("embed_scatter_grad_kernel");
}

extern "C" int bb_gather_rows_bf16(const void* in, const int64_t* idx, int64_t nout, int H, void* out, void* stream) {
  if (nout <= 0) return 0;
  if (H % 8 != 0) return set_error("bb_gather_rows_bf16: H must be a multiple of 8");
  if (!aligned16({in, out})) return set_error("bb_gather_rows_bf16: in / out must be 16-byte aligned");
  const long long n = nout * (H / 8);
  ACT_T(bb::launch_pdl(gather_rows_bf16_kernel<T>, (unsigned)((n + 255) / 256), 256, 0, STREAM, (const T*)in, idx, nout, H, (T*)out));
  count_launch();
  return check_launch("gather_rows_bf16_kernel");
}
extern "C" int bb_scatter_add_rows(const void* in_bf16, const int64_t* idx, int64_t nin, int H, float* out_f32,
                                   void* stream) {
  if (nin <= 0) return 0;
  if (det_on()) return set_error("bb_scatter_add_rows adds with atomics; in deterministic mode use bb_scatter_rows_sorted");
  const long long n = nin * H;
  ACT_T(bb::launch_pdl(scatter_add_rows_kernel<T>, (unsigned)((n + 255) / 256), 256, 0, STREAM, (const T*)in_bf16, idx, nin, H, out_f32));
  count_launch();
  return check_launch("scatter_add_rows_kernel");
}

extern "C" int bb_scatter_rows_sorted(const void* src, int src_f32, const int64_t* src_row, const float* w,
                                      const int64_t* dst_sorted, int64_t n, int H, float* out_f32, void* stream) {
  if (n <= 0) return 0;
  if (H % 8 != 0) return set_error("bb_scatter_rows_sorted: H must be a multiple of 8");
  if ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(out_f32)) & 15)
    return set_error("bb_scatter_rows_sorted: src and out must be 16-byte aligned");
  const long long nt = n * (H / 8);
  const unsigned grid = (unsigned)((nt + 255) / 256);
  if (src_f32)
    bb::launch_pdl(scatter_rows_sorted_kernel<float>, grid, 256, 0, STREAM, (const float*)src, src_row, w, dst_sorted,
                   n, H, out_f32);
  else if (bb::act_f32())
    return set_error("bb_scatter_rows_sorted: the fp32 verification mode needs fp32 src");
  else
    bb::launch_pdl(scatter_rows_sorted_kernel<bf16>, grid, 256, 0, STREAM, (const bf16*)src, src_row, w, dst_sorted,
                   n, H, out_f32);
  count_launch();
  return check_launch("scatter_rows_sorted_kernel");
}

extern "C" int bb_softmax_xent(const float* logits, const int64_t* labels, int64_t rows, int V, int64_t ld, float* loss,
                               const float* gscale, void* dlogits, void* stream) {
  if (rows <= 0) return 0;
  ACT_T(bb::launch_pdl(softmax_xent_kernel<T>, (unsigned)rows, 256, 0, STREAM, logits, labels, V, ld, loss, gscale, (T*)dlogits));
  count_launch();
  return check_launch("softmax_xent_kernel");
}

namespace bb { int set_salt_rowops(const unsigned long long* p) { return set_drop_salt_ptr_tu(p) == cudaSuccess ? 0 : -1; } }
