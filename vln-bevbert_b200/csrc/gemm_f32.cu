// High-precision verification arm of the GEMM entry point: when the library is in fp32-activation mode
// (bb_set_act_f32(1)), bb_gemm_bf16 dispatches here.  Same argument struct, same operand-major / batch-stride /
// epilogue semantics as the wgmma kernel (gemm_tc.cu), but A, B, aux, add_in and D are fp32 and every product is an
// fp32 FMA on the CUDA cores.  It exists to separate kernel LOGIC from bf16 PRECISION in the parity tests (north_star
// "1e-3 rel fp32"): throughput is irrelevant here (a plain 64 x 64 shared-memory tiling), results are deterministic.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {

static int g_act_f32 = 0;
bool act_f32() { return g_act_f32 != 0; }

namespace {
constexpr int TM = 64, TN = 64, TK = 16;

struct F32Params {
  const float *A, *B, *aux_in, *add_in, *bias;
  float *D, *aux_out;
  int M, N, K, nb1;
  int a_mn, b_mn;
  long long lda, a_s1, a_s2, ldb, b_s1, b_s2, ldd, d_s1, d_s2;
  float alpha;
  int act, epi_mul, accumulate;
  uint64_t drop_seed;
  uint32_t drop_thresh;
  float drop_scale;
};

__global__ void __launch_bounds__(256) gemm_f32_kernel(const F32Params p) {
  __shared__ float As[TK][TM + 1];
  __shared__ float Bs[TK][TN + 1];
  pdl_wait();
  pdl_trigger();
  const int b1 = blockIdx.z % p.nb1, b2 = blockIdx.z / p.nb1;
  const float* A = p.A + b1 * p.a_s1 + b2 * p.a_s2;
  const float* B = p.B + b1 * p.b_s1 + b2 * p.b_s2;
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < p.K; k0 += TK) {
    for (int e = threadIdx.x; e < TM * TK; e += 256) {
      // consecutive threads walk the contiguous dimension of the operand
      const int mm = p.a_mn ? (e % TM) : (e / TK), kk = p.a_mn ? (e / TM) : (e % TK);
      const int m = m0 + mm, k = k0 + kk;
      As[kk][mm] = (m < p.M && k < p.K) ? A[p.a_mn ? (long long)k * p.lda + m : (long long)m * p.lda + k] : 0.f;
    }
    for (int e = threadIdx.x; e < TN * TK; e += 256) {
      const int nn = p.b_mn ? (e % TN) : (e / TK), kk = p.b_mn ? (e / TN) : (e % TK);
      const int n = n0 + nn, k = k0 + kk;
      Bs[kk][nn] = (n < p.N && k < p.K) ? B[p.b_mn ? (long long)k * p.ldb + n : (long long)n * p.ldb + k] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  const long long boff = b1 * p.d_s1 + b2 * p.d_s2;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= p.N) continue;
      const long long off = boff + (long long)m * p.ldd + n;
      float v = acc[i][j] * p.alpha;
      if (p.bias) v += p.bias[n];
      if (p.aux_out) p.aux_out[off] = v;
      if (p.act == 1) v = gelu_erf(v);
      else if (p.act == 2) v = fmaxf(v, 0.f);
      else if (p.act == 3) v = qgelu(v);
      if (p.epi_mul == 1) v *= dgelu_erf(p.aux_in[off]);
      else if (p.epi_mul == 2) v = p.aux_in[off] > 0.f ? v : 0.f;
      if (p.drop_thresh) v = drop_keep(p.drop_seed, (uint64_t)off, p.drop_thresh) ? v * p.drop_scale : 0.f;
      if (p.add_in) v += p.add_in[off];
      if (p.accumulate) p.D[off] += v;     // one CTA owns the element: no atomics needed (no split-K here)
      else p.D[off] = v;
    }
  }
}
}  // namespace

int gemm_f32_launch(const bb_gemm_args* a, cudaStream_t stream) {
  if (!a || !a->A || !a->B || !a->D) return set_error("bb_gemm (fp32 arm): null argument");
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return set_error("bb_gemm (fp32 arm): M, N, K must be positive");
  F32Params p;
  memset(&p, 0, sizeof(p));
  p.A = (const float*)a->A; p.B = (const float*)a->B; p.D = (float*)a->D;
  p.aux_in = (const float*)a->aux_in; p.add_in = (const float*)a->add_in; p.aux_out = (float*)a->aux_out;
  p.bias = a->bias;
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.nb1 = a->nb1 > 0 ? a->nb1 : 1;
  const int nb2 = a->nb2 > 0 ? a->nb2 : 1;
  p.a_mn = a->a_mn ? 1 : 0; p.b_mn = a->b_mn ? 1 : 0;
  p.lda = a->lda; p.a_s1 = a->a_s1; p.a_s2 = a->a_s2;
  p.ldb = a->ldb; p.b_s1 = a->b_s1; p.b_s2 = a->b_s2;
  p.ldd = a->ldd; p.d_s1 = a->d_s1; p.d_s2 = a->d_s2;
  p.alpha = a->alpha; p.act = a->act; p.epi_mul = a->epi_mul;
  p.accumulate = (a->accumulate || a->split_k > 1) ? 1 : 0;
  p.drop_seed = a->drop_seed; p.drop_thresh = a->drop_thresh; p.drop_scale = a->drop_scale;
  const dim3 grid((unsigned)((a->N + TN - 1) / TN), (unsigned)((a->M + TM - 1) / TM), (unsigned)(p.nb1 * nb2));
  if (grid.y > 65535 || grid.z > 65535) return set_error("bb_gemm (fp32 arm): problem too large for the verification kernel");
  launch_pdl(gemm_f32_kernel, grid, dim3(256), 0, stream, p);
  count_launch();
  return check_launch("gemm_f32_kernel");
}

}  // namespace bb

extern "C" int bb_set_act_f32(int on) {
  const int prev = bb::g_act_f32;
  bb::g_act_f32 = on ? 1 : 0;
  return prev;
}
extern "C" int bb_get_act_f32(void) { return bb::g_act_f32; }

namespace bb { int set_salt_gemm_f32(const unsigned long long* p) { return set_drop_salt_ptr_tu(p) == cudaSuccess ? 0 : -1; } }
