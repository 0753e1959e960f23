// Multi-tensor kernels over a device table of tensors: global gradient norm, AdamW update (+ bf16 weight shadow),
// fp32 -> bf16 shadow refresh.  One launch covers every parameter of the model (568 tensors, 239 M elements) instead
// of ~6 small launches per tensor.
//
// Reference semantics: pretrain_src/optim/adamw.py:53-112 (per-parameter step counter, m/v update, bias-corrected
// step size computed on the host, p -= step_size * m / (sqrt(v) + eps), then decoupled decay p -= lr*wd*p computed
// from the UPDATED p) and torch.nn.utils.clip_grad_norm_ as called at pretrain_src/train_r2r.py:298
// (coef = min(1, max_norm / (||g||_2 + 1e-6)) applied to every gradient).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace {
constexpr int MT_THREADS = 256;
constexpr int MT_CHUNK = 4096;   // elements per CTA: 16 per thread, 4 x 16-byte accesses in flight per operand

// the tensor whose chunk range contains `chunk` (table sorted by chunk0; chunk0[0] == 0)
__device__ __forceinline__ int find_tensor(const bb_mt_tensor* __restrict__ t, int nt, long long chunk) {
  int lo = 0, hi = nt - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&t[mid].chunk0) <= chunk) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ float block_sum(float v, float* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x < 32) {
    r = threadIdx.x < MT_THREADS / 32 ? sh[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  }
  return r;
}

__global__ void __launch_bounds__(MT_THREADS) mt_sumsq_kernel(const bb_mt_tensor* __restrict__ table, int nt,
                                                             float* __restrict__ out, float* __restrict__ det_part) {
  __shared__ float sh[MT_THREADS / 32];
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long chunk = blockIdx.x;
  const int ti = find_tensor(table, nt, chunk);
  const float* g = table[ti].g;
  const long long n = table[ti].n;
  const long long base = (chunk - table[ti].chunk0) * MT_CHUNK;
  float acc = 0.f;
  if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
#pragma unroll
    for (int k = 0; k < MT_CHUNK / (MT_THREADS * 4); ++k) {
      const long long i = base + (k * MT_THREADS + threadIdx.x) * 4;
      if (i + 4 <= n) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(g + i));
        acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      } else {
        for (long long j = i; j < n; ++j) acc += g[j] * g[j];
      }
    }
  } else {
    for (long long i = base + threadIdx.x; i < n && i < base + MT_CHUNK; i += MT_THREADS) acc += g[i] * g[i];
  }
  const float s = block_sum(acc, sh);
  if (threadIdx.x == 0) {
    if (det_part) det_part[chunk] = s;   // deterministic mode: summed in chunk order by mt_sumsq_det_kernel
    else atomicAdd(out, s);
  }
}

// Deterministic mode: one block sums the per-chunk partials; thread t adds chunks t, t + MT_THREADS, ... in order, and
// block_sum combines the threads in a fixed tree.
__global__ void __launch_bounds__(MT_THREADS) mt_sumsq_det_kernel(const float* __restrict__ part, long long n,
                                                                 float* __restrict__ out) {
  __shared__ float sh[MT_THREADS / 32];
  bb::pdl_wait();
  bb::pdl_trigger();
  float acc = 0.f;
  for (long long i = threadIdx.x; i < n; i += MT_THREADS) acc += part[i];
  const float s = block_sum(acc, sh);
  if (threadIdx.x == 0) *out = s;
}

struct AdamParams {
  float beta1, beta2, eps, max_norm, grad_scale;
  const float* sumsq;
};

__device__ __forceinline__ void adam1(float& p, float g, float& m, float& v, const AdamParams& a, float coef,
                                      float step_size, float decay) {
  g *= coef;
  m = a.beta1 * m + (1.0f - a.beta1) * g;
  v = a.beta2 * v + (1.0f - a.beta2) * g * g;
  p = p - step_size * (m / (sqrtf(v) + a.eps));
  p = p - decay * p;            // decoupled decay on the updated value (adamw.py:110)
}

__global__ void __launch_bounds__(MT_THREADS) mt_adamw_kernel(const bb_mt_tensor* __restrict__ table, int nt,
                                                             AdamParams a) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long chunk = blockIdx.x;
  const int ti = find_tensor(table, nt, chunk);
  const bb_mt_tensor t = table[ti];
  float coef = a.grad_scale;
  if (a.sumsq != nullptr && a.max_norm > 0.f) {
    const float norm = sqrtf(__ldg(a.sumsq)) * a.grad_scale;
    coef *= fminf(1.0f, a.max_norm / (norm + 1e-6f));
  }
  const long long base = (chunk - t.chunk0) * MT_CHUNK;
  __nv_bfloat16* p16 = reinterpret_cast<__nv_bfloat16*>(t.p16);
  const bool vec = ((reinterpret_cast<uintptr_t>(t.p) | reinterpret_cast<uintptr_t>(t.g) | reinterpret_cast<uintptr_t>(t.m) |
                     reinterpret_cast<uintptr_t>(t.v)) & 15) == 0 && (reinterpret_cast<uintptr_t>(t.p16) & 7) == 0;
  if (vec) {
#pragma unroll
    for (int k = 0; k < MT_CHUNK / (MT_THREADS * 4); ++k) {
      const long long i = base + (k * MT_THREADS + threadIdx.x) * 4;
      if (i + 4 <= t.n) {
        float4 p = *reinterpret_cast<const float4*>(t.p + i);
        const float4 g = __ldg(reinterpret_cast<const float4*>(t.g + i));
        float4 m = *reinterpret_cast<const float4*>(t.m + i);
        float4 v = *reinterpret_cast<const float4*>(t.v + i);
        adam1(p.x, g.x, m.x, v.x, a, coef, t.step_size, t.decay);
        adam1(p.y, g.y, m.y, v.y, a, coef, t.step_size, t.decay);
        adam1(p.z, g.z, m.z, v.z, a, coef, t.step_size, t.decay);
        adam1(p.w, g.w, m.w, v.w, a, coef, t.step_size, t.decay);
        *reinterpret_cast<float4*>(t.p + i) = p;
        *reinterpret_cast<float4*>(t.m + i) = m;
        *reinterpret_cast<float4*>(t.v + i) = v;
        if (p16) {
          const __nv_bfloat162 lo = __floats2bfloat162_rn(p.x, p.y), hi = __floats2bfloat162_rn(p.z, p.w);
          uint2 pk;
          pk.x = *reinterpret_cast<const uint32_t*>(&lo);
          pk.y = *reinterpret_cast<const uint32_t*>(&hi);
          *reinterpret_cast<uint2*>(p16 + i) = pk;
        }
      } else {
        for (long long j = i; j < t.n; ++j) {
          float p = t.p[j], m = t.m[j], v = t.v[j];
          adam1(p, t.g[j], m, v, a, coef, t.step_size, t.decay);
          t.p[j] = p; t.m[j] = m; t.v[j] = v;
          if (p16) p16[j] = __float2bfloat16(p);
        }
      }
    }
  } else {
    for (long long j = base + threadIdx.x; j < t.n && j < base + MT_CHUNK; j += MT_THREADS) {
      float p = t.p[j], m = t.m[j], v = t.v[j];
      adam1(p, t.g[j], m, v, a, coef, t.step_size, t.decay);
      t.p[j] = p; t.m[j] = m; t.v[j] = v;
      if (p16) p16[j] = __float2bfloat16(p);
    }
  }
}

__global__ void __launch_bounds__(MT_THREADS) mt_cast_kernel(const bb_mt_tensor* __restrict__ table, int nt) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long chunk = blockIdx.x;
  const int ti = find_tensor(table, nt, chunk);
  const float* src = table[ti].p;
  __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(table[ti].p16);
  const long long n = table[ti].n;
  const long long base = (chunk - table[ti].chunk0) * MT_CHUNK;
  if (((reinterpret_cast<uintptr_t>(src) & 15) | (reinterpret_cast<uintptr_t>(dst) & 7)) == 0) {
#pragma unroll
    for (int k = 0; k < MT_CHUNK / (MT_THREADS * 4); ++k) {
      const long long i = base + (k * MT_THREADS + threadIdx.x) * 4;
      if (i + 4 <= n) {
        const float4 p = __ldg(reinterpret_cast<const float4*>(src + i));
        const __nv_bfloat162 lo = __floats2bfloat162_rn(p.x, p.y), hi = __floats2bfloat162_rn(p.z, p.w);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&lo);
        pk.y = *reinterpret_cast<const uint32_t*>(&hi);
        *reinterpret_cast<uint2*>(dst + i) = pk;
      } else {
        for (long long j = i; j < n; ++j) dst[j] = __float2bfloat16(src[j]);
      }
    }
  } else {
    for (long long j = base + threadIdx.x; j < n && j < base + MT_CHUNK; j += MT_THREADS) dst[j] = __float2bfloat16(src[j]);
  }
}
}  // namespace

using namespace bb;

extern "C" int bb_mt_chunk_elems(void) { return MT_CHUNK; }

extern "C" int bb_mt_sumsq(const bb_mt_tensor* table_dev, int ntensors, int64_t total_chunks, float* out, void* stream) {
  if (!table_dev || !out) return set_error("bb_mt_sumsq: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemsetAsync(out, 0, sizeof(float), s) != cudaSuccess) return set_error("bb_mt_sumsq: memset failed");
  if (ntensors <= 0 || total_chunks <= 0) return 0;
  if (total_chunks > 0x7fffffffLL) return set_error("bb_mt_sumsq: too many chunks");
  float* part = nullptr;
  if (det_on()) {
    part = det_partials(s, (size_t)total_chunks * sizeof(float), "bb_mt_sumsq");
    if (!part) return -1;
  }
  bb::launch_pdl(mt_sumsq_kernel, (unsigned)total_chunks, MT_THREADS, 0, s, table_dev, ntensors, out, part);
  count_launch();
  if (int e = check_launch("mt_sumsq_kernel")) return e;
  if (!part) return 0;
  bb::launch_pdl(mt_sumsq_det_kernel, 1, MT_THREADS, 0, s, (const float*)part, (long long)total_chunks, out);
  count_launch();
  return check_launch("mt_sumsq_det_kernel");
}

extern "C" int bb_adamw_step(const bb_mt_tensor* table_dev, int ntensors, int64_t total_chunks, float beta1, float beta2,
                             float eps, const float* sumsq, float max_norm, float grad_scale, void* stream) {
  if (!table_dev) return set_error("bb_adamw_step: null table");
  if (ntensors <= 0 || total_chunks <= 0) return 0;
  if (total_chunks > 0x7fffffffLL) return set_error("bb_adamw_step: too many chunks");
  AdamParams a;
  a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.max_norm = max_norm; a.grad_scale = grad_scale; a.sumsq = sumsq;
  bb::launch_pdl(mt_adamw_kernel, (unsigned)total_chunks, MT_THREADS, 0, (cudaStream_t)stream, table_dev, ntensors, a);
  count_launch();
  return check_launch("mt_adamw_kernel");
}

extern "C" int bb_mt_cast_bf16(const bb_mt_tensor* table_dev, int ntensors, int64_t total_chunks, void* stream) {
  if (!table_dev) return set_error("bb_mt_cast_bf16: null table");
  if (ntensors <= 0 || total_chunks <= 0) return 0;
  if (total_chunks > 0x7fffffffLL) return set_error("bb_mt_cast_bf16: too many chunks");
  bb::launch_pdl(mt_cast_kernel, (unsigned)total_chunks, MT_THREADS, 0, (cudaStream_t)stream, table_dev, ntensors);
  count_launch();
  return check_launch("mt_cast_kernel");
}
