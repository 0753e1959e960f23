// Standalone GPU self-test for bb_gemm_bf16 (links against the C ABI objects). One case per process
// invocation so a hang in one configuration cannot mask the others:  selftest_gemm <case|all|list>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../include/bevbert_b200.h"

#define CK(x)                                                                  \
  do {                                                                         \
    cudaError_t e_ = (x);                                                      \
    if (e_ != cudaSuccess) {                                                   \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      exit(2);                                                                 \
    }                                                                          \
  } while (0)

struct Case {
  const char* name;
  int M, N, K, nb1, nb2, a_mn, b_mn;
  long long lda, a_s1, a_s2, ldb, b_s1, b_s2, ldd, d_s1, d_s2;
  int out_f32, split_k, act, use_bias, use_aux_out, epi_mul, use_add, block_n;
  float alpha;
  int timing_iters;
};

__global__ void ref_gemm(const __nv_bfloat16* A, const __nv_bfloat16* B, float* Dref, Case c, const float* bias,
                         const __nv_bfloat16* aux_in, const __nv_bfloat16* add_in, float* pre_ref) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long per = (long long)c.M * c.N;
  long long total = per * c.nb1 * c.nb2;
  if (idx >= total) return;
  int n = idx % c.N;
  int m = (idx / c.N) % c.M;
  int b = idx / per;
  int b1 = b % c.nb1, b2 = b / c.nb1;
  const __nv_bfloat16* a = A + b1 * c.a_s1 + b2 * c.a_s2;
  const __nv_bfloat16* bb_ = B + b1 * c.b_s1 + b2 * c.b_s2;
  float acc = 0.f;
  for (int k = 0; k < c.K; ++k) {
    float av = __bfloat162float(c.a_mn ? a[(long long)k * c.lda + m] : a[(long long)m * c.lda + k]);
    float bv = __bfloat162float(c.b_mn ? bb_[(long long)k * c.ldb + n] : bb_[(long long)n * c.ldb + k]);
    acc += av * bv;
  }
  float v = acc * c.alpha;
  if (bias) v += bias[n];
  long long off = b1 * c.d_s1 + b2 * c.d_s2 + (long long)m * c.ldd + n;
  pre_ref[off] = v;
  if (c.act == 1) v = v * 0.5f * (1.0f + erff(v * 0.70710678f));
  if (c.act == 2) v = fmaxf(v, 0.f);
  if (c.epi_mul == 1) {
    float x = __bfloat162float(aux_in[off]);
    float cdf = 0.5f * (1.0f + erff(x * 0.70710678f));
    float pdf = 0.39894228f * expf(-0.5f * x * x);
    v *= cdf + x * pdf;
  } else if (c.epi_mul == 2) {
    v = __bfloat162float(aux_in[off]) > 0.f ? v : 0.f;
  }
  if (add_in) v += __bfloat162float(add_in[off]);
  Dref[off] = v;
}

static float frand() { return (float)rand() / RAND_MAX * 2.f - 1.f; }

// FNV-1a over raw output bytes: two builds of the library computed the same bits iff the hashes agree
static unsigned long long fnv1a(const void* data, size_t n) {
  const unsigned char* b = static_cast<const unsigned char*>(data);
  unsigned long long h = 0xcbf29ce484222325ull;
  for (size_t i = 0; i < n; ++i) h = (h ^ b[i]) * 0x100000001b3ull;
  return h;
}

static int run_case(const Case& c) {
  const int nb = c.nb1 * c.nb2;
  // buffer extents (elements)
  long long a_ext = (c.nb1 - 1) * c.a_s1 + (c.nb2 - 1) * c.a_s2 + (c.a_mn ? (long long)(c.K - 1) * c.lda + c.M
                                                                         : (long long)(c.M - 1) * c.lda + c.K);
  long long b_ext = (c.nb1 - 1) * c.b_s1 + (c.nb2 - 1) * c.b_s2 + (c.b_mn ? (long long)(c.K - 1) * c.ldb + c.N
                                                                         : (long long)(c.N - 1) * c.ldb + c.K);
  long long d_ext = (c.nb1 - 1) * c.d_s1 + (c.nb2 - 1) * c.d_s2 + (long long)(c.M - 1) * c.ldd + c.N;
  a_ext += 64; b_ext += 64; d_ext += 64;
  std::vector<__nv_bfloat16> hA(a_ext), hB(b_ext), hAux(d_ext), hAdd(d_ext);
  for (auto& v : hA) v = __float2bfloat16(frand());
  for (auto& v : hB) v = __float2bfloat16(frand());
  for (auto& v : hAux) v = __float2bfloat16(frand() * 2.f);
  for (auto& v : hAdd) v = __float2bfloat16(frand());
  std::vector<float> hBias(c.N);
  for (auto& v : hBias) v = frand();
  __nv_bfloat16 *dA, *dB, *dAux, *dAdd, *dAuxOut;
  float *dBias, *dRef, *dPre;
  void* dD;
  CK(cudaMalloc(&dA, a_ext * 2));
  CK(cudaMalloc(&dB, b_ext * 2));
  CK(cudaMalloc(&dAux, d_ext * 2));
  CK(cudaMalloc(&dAdd, d_ext * 2));
  CK(cudaMalloc(&dAuxOut, d_ext * 2));
  CK(cudaMalloc(&dBias, c.N * 4));
  CK(cudaMalloc(&dRef, d_ext * 4));
  CK(cudaMalloc(&dPre, d_ext * 4));
  CK(cudaMalloc(&dD, d_ext * 4));
  CK(cudaMemcpy(dA, hA.data(), a_ext * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dB, hB.data(), b_ext * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dAux, hAux.data(), d_ext * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dAdd, hAdd.data(), d_ext * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dBias, hBias.data(), c.N * 4, cudaMemcpyHostToDevice));
  CK(cudaMemset(dRef, 0, d_ext * 4));
  CK(cudaMemset(dPre, 0, d_ext * 4));
  CK(cudaMemset(dD, 0, d_ext * 4));
  CK(cudaMemset(dAuxOut, 0, d_ext * 2));

  long long total = (long long)c.M * c.N * nb;
  ref_gemm<<<(unsigned)((total + 255) / 256), 256>>>(dA, dB, dRef, c, c.use_bias ? dBias : nullptr,
                                                     c.epi_mul ? dAux : nullptr, c.use_add ? dAdd : nullptr, dPre);
  CK(cudaDeviceSynchronize());

  bb_gemm_args g;
  memset(&g, 0, sizeof(g));
  g.A = dA; g.B = dB; g.D = dD;
  g.M = c.M; g.N = c.N; g.K = c.K; g.nb1 = c.nb1; g.nb2 = c.nb2; g.a_mn = c.a_mn; g.b_mn = c.b_mn;
  g.lda = c.lda; g.a_s1 = c.a_s1; g.a_s2 = c.a_s2;
  g.ldb = c.ldb; g.b_s1 = c.b_s1; g.b_s2 = c.b_s2;
  g.ldd = c.ldd; g.d_s1 = c.d_s1; g.d_s2 = c.d_s2;
  g.out_f32 = c.out_f32; g.split_k = c.split_k; g.alpha = c.alpha;
  g.bias = c.use_bias ? dBias : nullptr;
  g.act = c.act;
  g.aux_out = c.use_aux_out ? dAuxOut : nullptr;
  g.aux_in = c.epi_mul ? dAux : nullptr;
  g.epi_mul = c.epi_mul;
  g.add_in = c.use_add ? dAdd : nullptr;
  g.block_n = c.block_n;
  int rc = bb_gemm_bf16(&g, nullptr);
  if (rc) {
    printf("CASE %-22s ERROR rc=%d: %s\n", c.name, rc, bb_last_error());
    return 1;
  }
  cudaError_t se = cudaDeviceSynchronize();
  if (se != cudaSuccess) {
    printf("CASE %-22s CUDA-ERROR after kernel: %s\n", c.name, cudaGetErrorString(se));
    return 1;
  }
  std::vector<float> hRef(d_ext), hPre(d_ext), hOut(d_ext);
  CK(cudaMemcpy(hRef.data(), dRef, d_ext * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hPre.data(), dPre, d_ext * 4, cudaMemcpyDeviceToHost));
  unsigned long long hash_d;
  if (c.out_f32) {
    CK(cudaMemcpy(hOut.data(), dD, d_ext * 4, cudaMemcpyDeviceToHost));
    hash_d = fnv1a(hOut.data(), d_ext * 4);
  } else {
    std::vector<__nv_bfloat16> t(d_ext);
    CK(cudaMemcpy(t.data(), dD, d_ext * 2, cudaMemcpyDeviceToHost));
    for (long long i = 0; i < d_ext; ++i) hOut[i] = __bfloat162float(t[i]);
    hash_d = fnv1a(t.data(), d_ext * 2);
  }
  std::vector<__nv_bfloat16> hAuxOut(d_ext);
  CK(cudaMemcpy(hAuxOut.data(), dAuxOut, d_ext * 2, cudaMemcpyDeviceToHost));
  const unsigned long long hash_aux = fnv1a(hAuxOut.data(), d_ext * 2);
  double max_err = 0, max_ref = 0, max_aux_err = 0;
  long long bad_i = -1;
  // compare only addressed outputs; everything else must still be zero (catches stray writes)
  std::vector<char> touched(d_ext, 0);
  for (int b2 = 0; b2 < c.nb2; ++b2)
    for (int b1 = 0; b1 < c.nb1; ++b1)
      for (int m = 0; m < c.M; ++m)
        for (int n = 0; n < c.N; ++n) {
          long long off = b1 * c.d_s1 + b2 * c.d_s2 + (long long)m * c.ldd + n;
          touched[off] = 1;
          double e = fabs((double)hOut[off] - hRef[off]);
          if (e > max_err) { max_err = e; bad_i = off; }
          if (fabs(hRef[off]) > max_ref) max_ref = fabs(hRef[off]);
          if (c.use_aux_out) {
            double ea = fabs((double)__bfloat162float(hAuxOut[off]) - hPre[off]);
            if (ea > max_aux_err) max_aux_err = ea;
          }
        }
  long long stray = 0;
  for (long long i = 0; i < d_ext; ++i)
    if (!touched[i] && hOut[i] != 0.f) ++stray;
  const double tol = (c.out_f32 ? 2e-3 : 1.2e-2) * (max_ref > 1 ? max_ref : 1);
  bool ok = max_err <= tol && stray == 0 && (!c.use_aux_out || max_aux_err <= 1.2e-2 * (max_ref > 1 ? max_ref : 1));
  float ms = 0;
  if (c.timing_iters > 0 && ok) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int i = 0; i < 3; ++i) bb_gemm_bf16(&g, nullptr);
    cudaEventRecord(e0);
    for (int i = 0; i < c.timing_iters; ++i) bb_gemm_bf16(&g, nullptr);
    cudaEventRecord(e1);
    CK(cudaEventSynchronize(e1));
    cudaEventElapsedTime(&ms, e0, e1);
    ms /= c.timing_iters;
  }
  if (getenv("BB_GEMM_TRACE") && c.timing_iters > 0 && ok) {
    // per-tile timeline of one warm launch: MMA issue window and epilogue window of the first tiles of a few CTAs
    const int ncta = 160;
    long long* dT;
    CK(cudaMalloc(&dT, (size_t)ncta * 16 * 4 * 8));
    CK(cudaMemset(dT, 0, (size_t)ncta * 16 * 4 * 8));
    bb_gemm_trace(dT);
    bb_gemm_bf16(&g, nullptr);
    CK(cudaDeviceSynchronize());
    bb_gemm_trace(nullptr);
    std::vector<long long> hT((size_t)ncta * 16 * 4);
    CK(cudaMemcpy(hT.data(), dT, hT.size() * 8, cudaMemcpyDeviceToHost));
    long long t0 = 0;
    for (long long v : hT) if (v && (!t0 || v < t0)) t0 = v;
    for (int cta : {0, 1, 2, 73, 147}) {
      printf("   trace cta %3d:", cta);
      for (int i = 0; i < 16; ++i) {
        const long long* r = &hT[((size_t)cta * 16 + i) * 4];
        if (!r[0] && !r[2]) break;
        printf(" [mma %.2f-%.2f epi %.2f-%.2f]", (r[0] - t0) * 1e-3, (r[1] - t0) * 1e-3, (r[2] - t0) * 1e-3, (r[3] - t0) * 1e-3);
      }
      printf("\n");
    }
    cudaFree(dT);
  }
  double tflops = ms > 0 ? 2.0 * c.M * c.N * c.K * nb / (ms * 1e-3) / 1e12 : 0;
  printf("CASE %-22s %s max_err=%.4g (at %lld) max_ref=%.4g aux_err=%.4g stray=%lld  %.3f ms %.1f TFLOP/s  "
         "hash D=%016llx aux=%016llx\n", c.name, ok ? "PASS" : "FAIL", max_err, bad_i, max_ref, max_aux_err, stray, ms,
         tflops, hash_d, hash_aux);
  if (!ok && bad_i >= 0) {
    // print a small window of outputs around the first row for diagnosis
    printf("   first 8 outputs: ");
    for (int i = 0; i < 8; ++i) printf("%.3f/%.3f ", hOut[i], hRef[i]);
    printf("\n");
  }
  cudaFree(dA); cudaFree(dB); cudaFree(dAux); cudaFree(dAdd); cudaFree(dAuxOut); cudaFree(dBias);
  cudaFree(dRef); cudaFree(dPre); cudaFree(dD);
  return ok ? 0 : 1;
}

int main(int argc, char** argv) {
  // name, M,N,K, nb1,nb2, a_mn,b_mn, lda,a_s1,a_s2, ldb,b_s1,b_s2, ldd,d_s1,d_s2, f32, splitk, act,bias,auxout,epimul,add, block_n, alpha, iters
  const int H = 12, Bs = 3, nq = 441, nkp = 448;
  std::vector<Case> cases = {
      {"nt_exact", 256, 256, 128, 1, 1, 0, 0, 128, 0, 0, 128, 0, 0, 256, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 1.f, 0},
      {"nt_exact_bf16", 256, 256, 128, 1, 1, 0, 0, 128, 0, 0, 128, 0, 0, 256, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1.f, 0},
      {"nt_bn64", 128, 64, 64, 1, 1, 0, 0, 64, 0, 0, 64, 0, 0, 64, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 1.f, 0},
      {"nt_tails", 300, 200, 136, 1, 1, 0, 0, 136, 0, 0, 136, 0, 0, 200, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 1.f, 0},
      {"nt_gelu_aux", 1000, 3072, 768, 1, 1, 0, 0, 768, 0, 0, 768, 0, 0, 3072, 0, 0, 0, 1, 1, 1, 1, 0, 0, 0, 1.f, 0},
      {"nt_dgelu_add", 515, 768, 3072, 1, 1, 0, 0, 3072, 0, 0, 3072, 0, 0, 768, 0, 0, 0, 1, 0, 0, 0, 1, 1, 0, 1.f, 0},
      {"nt_drelu", 200, 768, 768, 1, 1, 0, 0, 768, 0, 0, 768, 0, 0, 768, 0, 0, 0, 1, 0, 0, 0, 2, 0, 0, 1.f, 0},
      {"nn_dx", 300, 768, 3072, 1, 1, 0, 1, 3072, 0, 0, 768, 0, 0, 768, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1.f, 0},
      {"nn_small", 128, 64, 64, 1, 1, 0, 1, 64, 0, 0, 64, 0, 0, 64, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 1.f, 0},
      {"tn_small", 128, 64, 64, 1, 1, 1, 0, 128, 0, 0, 64, 0, 0, 64, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 1.f, 0},
      {"tt_small", 128, 64, 64, 1, 1, 1, 1, 128, 0, 0, 64, 0, 0, 64, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 1.f, 0},
      {"tt_dw_splitk", 768, 3072, 5000, 1, 1, 1, 1, 768, 0, 0, 3072, 0, 0, 3072, 0, 0, 1, 8, 0, 0, 0, 0, 0, 0, 1.f, 0},
      {"tt_dw_tails", 1000, 40, 777 + 7, 1, 1, 1, 1, 1000, 0, 0, 40, 0, 0, 40, 0, 0, 1, 3, 0, 0, 0, 0, 0, 0, 1.f, 0},
      // attention-shaped batched products on a packed (B, n, 3*768) QKV buffer
      {"attn_qk", nq, nq, 64, H, Bs, 0, 0, 2304, 64, (long long)nq * 2304, 2304, 64, (long long)nq * 2304, nkp,
       (long long)nq * nkp, (long long)H * nq * nkp, 1, 1, 0, 0, 0, 0, 0, 0, 0.125f, 0},
      {"attn_pv", nq, 64, nq, H, Bs, 0, 1, nkp, (long long)nq * nkp, (long long)H * nq * nkp, 2304, 64,
       (long long)nq * 2304, 768, 64, (long long)nq * 768, 0, 1, 0, 0, 0, 0, 0, 0, 1.f, 0},
      {"attn_dv", nq, 64, nq, H, Bs, 1, 1, nkp, (long long)nq * nkp, (long long)H * nq * nkp, 768, 64,
       (long long)nq * 768, 2304, 64, (long long)nq * 2304, 0, 1, 0, 0, 0, 0, 0, 0, 1.f, 0},
      {"attn_small", 20, 80, 64, H, Bs, 0, 0, 768, 64, 20 * 768, 1536, 64, 80 * 1536, 80, 20 * 80, H * 20 * 80, 1, 1,
       0, 0, 0, 0, 0, 0, 0.125f, 0},
      // throughput probes (forward-shaped)
      {"perf_qkv", 14112, 2304, 768, 1, 1, 0, 0, 768, 0, 0, 768, 0, 0, 2304, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 1.f, 20},
      {"perf_ffn1", 14112, 3072, 768, 1, 1, 0, 0, 768, 0, 0, 768, 0, 0, 3072, 0, 0, 0, 1, 1, 1, 1, 0, 0, 0, 1.f, 20},
      {"perf_ffn2", 14112, 768, 3072, 1, 1, 0, 0, 3072, 0, 0, 3072, 0, 0, 768, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 1.f, 20},
      {"perf_sq8k", 8192, 8192, 8192, 1, 1, 0, 0, 8192, 0, 0, 8192, 0, 0, 8192, 0, 0, 0, 1, 0, 0, 0, 0, 0, 256, 1.f, 5},
      {"perf_lang_ffn1", 2560, 3072, 768, 1, 1, 0, 0, 768, 0, 0, 768, 0, 0, 3072, 0, 0, 0, 1, 1, 1, 1, 0, 0, 0, 1.f, 50},
      {"perf_lang_dx", 2560, 768, 3072, 1, 1, 0, 1, 3072, 0, 0, 768, 0, 0, 768, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 1.f, 50},
      {"perf_lang_dw", 3072, 768, 2560, 1, 1, 1, 1, 3072, 0, 0, 768, 0, 0, 768, 0, 0, 1, 1, 0, 0, 0, 0, 0, 128, 1.f, 50},
      {"perf_attn_s441", 441, 441, 64, 12, 32, 0, 0, 2304, 64, 441LL * 2304, 2304, 64, 441LL * 2304, 448, 441LL * 448,
       12LL * 441 * 448, 1, 1, 0, 0, 0, 0, 0, 0, 0.125f, 20},
      {"perf_dw", 768, 3072, 14112, 1, 1, 1, 1, 768, 0, 0, 3072, 0, 0, 3072, 0, 0, 1, 8, 0, 0, 0, 0, 0, 0, 1.f, 20},
      // FFN up-projection backward dX: (dY W2) * gelu'(pre)
      {"perf_dgelu", 14112, 3072, 768, 1, 1, 0, 1, 768, 0, 0, 3072, 0, 0, 3072, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 1.f, 20},
      // QKV backward dX with the residual gradient added
      {"perf_qkv_dx", 14112, 768, 2304, 1, 1, 0, 1, 2304, 0, 0, 768, 0, 0, 768, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 1.f, 20},
      // ping-pong tile schedules (tile counts for a 132-SM H100): 3 tiles per CTA, so the first consumer warpgroup
      // takes one tile more than the second; a single tile; one tile more than the grid (one CTA runs two)
      {"pp_odd_tiles", 4224, 1536, 256, 1, 1, 0, 0, 256, 0, 0, 256, 0, 0, 1536, 0, 0, 0, 1, 1, 1, 1, 0, 0, 0, 1.f, 0},
      {"pp_one_tile", 100, 60, 512, 1, 1, 0, 0, 512, 0, 0, 512, 0, 0, 60, 0, 0, 0, 1, 0, 1, 0, 0, 1, 0, 1.f, 0},
      {"pp_grid_plus_1", 17024, 128, 192, 1, 1, 0, 1, 192, 0, 0, 128, 0, 0, 128, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 1.f, 0},
  };
  if (argc < 2 || !strcmp(argv[1], "list")) {
    for (auto& c : cases) printf("%s\n", c.name);
    return 0;
  }
  srand(1234);
  int fails = 0;
  for (auto& c : cases)
    if (!strcmp(argv[1], "all") || !strcmp(argv[1], c.name)) fails += run_case(c);
  return fails ? 1 : 0;
}
