// Input side of a ViT image tower (OpenAI CLIP's VisionTransformer, the VLN-CE policy's RGB encoder): the patch rows of
// its stride-P convolution with the image preprocessing fused in, and the token rows of its first block (class token,
// positional embedding, ln_pre).  The convolution itself is a GEMM of the patch rows with the flattened conv1 weight.
// Both kernels have bf16 (product) and fp32 (verification arm, bb_set_act_f32) output instantiations.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {
bool act_f32();   // gemm_f32.cu

namespace {
typedef __nv_bfloat16 bf16;

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

__device__ __forceinline__ void store8(bf16* p, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]),
                                            pack_bf16(v[6], v[7]));
}
__device__ __forceinline__ void store8(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}

struct Norm3 {
  float mean[3], std[3];
};

// One thread per 8 consecutive columns of a patch row.  Row r = (n, py, px) in token order (n * gh + py) * gw + px;
// column (c, ky, kx) = c * P * P + ky * P + kx, the flatten order of a (width, 3, P, P) convolution weight.  The value is
// torchvision's ConvertImageDtype(float) then Normalize, in torch's own fp32 operations on the device: a uint8 pixel is
// converted and multiplied by the fp32 reciprocal of 255 (torch divides by a scalar that way on CUDA), then
// (v - mean[c]) / std[c] with a correctly rounded subtraction and division.  Float pixels skip the conversion.
template <typename In, typename Out>
__global__ void __launch_bounds__(256) image_patches_kernel(const In* __restrict__ img, long long sn, long long sh,
                                                            long long sw, long long sc, int gh, int gw, int P,
                                                            float scale, Norm3 nm, long long rows, Out* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const int KP = 3 * P * P, cpr = KP / 8;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= rows * cpr) return;
  const long long r = i / cpr;
  const int j = (int)(i % cpr) * 8;
  const long long n = r / (gh * gw);
  const int t = (int)(r % (gh * gw)), py = t / gw, px = t % gw;
  const In* base = img + n * sn + (long long)(py * P) * sh + (long long)(px * P) * sw;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int col = j + e, c = col / (P * P), rem = col % (P * P), ky = rem / P, kx = rem % P;
    float x = static_cast<float>(base[ky * sh + kx * sw + c * sc]);
    if (sizeof(In) == 1) x = __fmul_rn(x, scale);
    const float m = c == 0 ? nm.mean[0] : c == 1 ? nm.mean[1] : nm.mean[2];   // selects keep nm out of local memory
    const float sd = c == 0 ? nm.std[0] : c == 1 ? nm.std[1] : nm.std[2];
    v[e] = __fdiv_rn(__fsub_rn(x, m), sd);
  }
  store8(out + r * KP + j, v);
}

// One warp per token row of the (N, T, H) block input: row (n, 0) = cls + pos[0], row (n, t) = patch[n (T-1) + t-1] +
// pos[t]; then LayerNorm over H in fp32 (two-pass mean and variance, rstd = rsqrt(var + eps)), scaled and shifted.
template <typename Out>
__global__ void __launch_bounds__(256) vit_tokens_kernel(const float* __restrict__ patch, const float* __restrict__ cls,
                                                         const float* __restrict__ pos, const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, float eps, long long rows,
                                                         int T, int H, Out* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  constexpr int MAXC = 4;   // 8-wide chunks per lane: H <= 1024
  const int lane = threadIdx.x & 31;
  const long long r = blockIdx.x * (long long)(blockDim.x / 32) + threadIdx.x / 32;
  if (r >= rows) return;
  const long long n = r / T;
  const int t = (int)(r % T);
  const float* src = t == 0 ? cls : patch + (n * (T - 1) + t - 1) * H;
  const float* pr = pos + (long long)t * H;
  float v[MAXC][8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < MAXC; ++k) {
    const int col = (lane + 32 * k) * 8;
    if (col < H) {
      const float4* a = reinterpret_cast<const float4*>(src + col);
      const float4* b = reinterpret_cast<const float4*>(pr + col);
      const float4 a0 = a[0], a1 = a[1], b0 = __ldg(b), b1 = __ldg(b + 1);
      v[k][0] = a0.x + b0.x; v[k][1] = a0.y + b0.y; v[k][2] = a0.z + b0.z; v[k][3] = a0.w + b0.w;
      v[k][4] = a1.x + b1.x; v[k][5] = a1.y + b1.y; v[k][6] = a1.z + b1.z; v[k][7] = a1.w + b1.w;
#pragma unroll
      for (int e = 0; e < 8; ++e) s += v[k][e];
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / H;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < MAXC; ++k)
    if ((lane + 32 * k) * 8 < H)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = v[k][e] - mean;
        q += d * d;
      }
#pragma unroll
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / H + eps);
#pragma unroll
  for (int k = 0; k < MAXC; ++k) {
    const int col = (lane + 32 * k) * 8;
    if (col < H) {
      float y[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] = (v[k][e] - mean) * rstd * __ldg(gamma + col + e) + __ldg(beta + col + e);
      store8(out + r * H + col, y);
    }
  }
}
}  // namespace
}  // namespace bb

using namespace bb;

extern "C" int bb_image_patches(const void* img, int img_u8, int N, int H, int W, int64_t sn, int64_t sh, int64_t sw,
                                int64_t sc, int P, const float* mean, const float* std_, void* out, void* stream) {
  if (!img || !out || !mean || !std_) return set_error("bb_image_patches: img / out / mean / std must not be NULL");
  if (N <= 0 || H <= 0 || W <= 0 || P <= 0) return set_error("bb_image_patches: N, H, W and P must be positive");
  if (H % P || W % P) return set_error("bb_image_patches: the image height and width must be multiples of the patch size");
  if ((3 * P * P) % 8) return set_error("bb_image_patches: 3 * P * P must be a multiple of 8");
  if (sn < 0 || sh < 0 || sw < 0 || sc < 0) return set_error("bb_image_patches: strides must be non-negative");
  if (((uintptr_t)out & 15) || (!img_u8 && ((uintptr_t)img & 3)))
    return set_error("bb_image_patches: out must be 16-byte aligned and a float image 4-byte aligned");
  Norm3 nm;
  for (int c = 0; c < 3; ++c) {
    nm.mean[c] = mean[c];
    nm.std[c] = std_[c];
  }
  const int gh = H / P, gw = W / P;
  const long long rows = (long long)N * gh * gw, n = rows * (3 * P * P / 8);
  const float scale = 1.0f / 255.0f;
  const dim3 grid((unsigned)((n + 255) / 256));
  cudaStream_t st = (cudaStream_t)stream;
  if (img_u8) {
    if (act_f32())
      launch_pdl(image_patches_kernel<uint8_t, float>, grid, dim3(256), 0, st, (const uint8_t*)img, (long long)sn,
                     (long long)sh, (long long)sw, (long long)sc, gh, gw, P, scale, nm, rows, (float*)out);
    else
      launch_pdl(image_patches_kernel<uint8_t, bf16>, grid, dim3(256), 0, st, (const uint8_t*)img, (long long)sn,
                     (long long)sh, (long long)sw, (long long)sc, gh, gw, P, scale, nm, rows, (bf16*)out);
  } else {
    if (act_f32())
      launch_pdl(image_patches_kernel<float, float>, grid, dim3(256), 0, st, (const float*)img, (long long)sn,
                     (long long)sh, (long long)sw, (long long)sc, gh, gw, P, scale, nm, rows, (float*)out);
    else
      launch_pdl(image_patches_kernel<float, bf16>, grid, dim3(256), 0, st, (const float*)img, (long long)sn,
                     (long long)sh, (long long)sw, (long long)sc, gh, gw, P, scale, nm, rows, (bf16*)out);
  }
  count_launch();
  return check_launch("image_patches_kernel");
}

extern "C" int bb_vit_tokens(const float* patch, const float* cls, const float* pos, const float* gamma,
                             const float* beta, float eps, int N, int T, int H, void* out, void* stream) {
  if (!patch || !cls || !pos || !gamma || !beta || !out)
    return set_error("bb_vit_tokens: patch / cls / pos / gamma / beta / out must not be NULL");
  if (N <= 0 || T < 2) return set_error("bb_vit_tokens: N must be positive and T >= 2");
  if (H <= 0 || H % 8 || H > 1024) return set_error("bb_vit_tokens: H must be a positive multiple of 8, at most 1024");
  for (const void* p : {(const void*)patch, (const void*)cls, (const void*)pos, (const void*)gamma, (const void*)beta, (const void*)out})
    if ((uintptr_t)p & 15) return set_error("bb_vit_tokens: every pointer must be 16-byte aligned");
  const long long rows = (long long)N * T;
  const dim3 grid((unsigned)((rows + 7) / 8));
  cudaStream_t st = (cudaStream_t)stream;
  if (act_f32())
    launch_pdl(vit_tokens_kernel<float>, grid, dim3(256), 0, st, patch, cls, pos, gamma, beta, eps, rows, T, H,
               (float*)out);
  else
    launch_pdl(vit_tokens_kernel<bf16>, grid, dim3(256), 0, st, patch, cls, pos, gamma, beta, eps, rows, T, H,
               (bf16*)out);
  count_launch();
  return check_launch("vit_tokens_kernel");
}
