// The VLN-CE policy's depth encoder (bevbert_ce/vlnce_baselines/models/encoders/resnet_encoders.py:13-107 over
// habitat-lab v0.1.7's DD-PPO ResNetEncoder with a GroupNorm ResNet-50): NHWC convolutions with GroupNorm statistics
// written by the producer, the fused 2x2 average-pool + 7x7 stem, and the GroupNorm apply with its residual and
// max-pool variants.
//
// GroupNorm partial statistics.  A kernel that writes a (N, H, W, C) map (rows m = (n, h, w) flattened) also writes, for
// each stat tile of `tm` consecutive rows, each image the tile touches (its segment j = n - first image of the tile) and
// each channel block of cb = min(C / G, 32) channels, one float4 {count, mean, M2, 0} of the values as STORED (fp16
// rounded in the product path), at index (tile * SEG + j) * (C / cb) + channel / cb, SEG = (tm + H W - 2) / (H W) + 1
// (the most images tm consecutive rows can touch).  Each float4 is computed by one warp with two passes over the staged
// tile in a fixed order and written with a plain store, so the statistics are deterministic.  bb_groupnorm_apply
// combines the partials of (image, group) tile by tile and block by block with Chan's parallel rule.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {
bool act_f32();   // gemm_f32.cu: fp32-activation verification mode (bb_set_act_f32)

namespace {
constexpr int CONV_BM = 128;        // output pixels per CTA (two consumer warpgroups of 64 rows)
constexpr int CONV_THREADS = 256;
constexpr int CONV_STAGES = 4;      // smem ring; loads run two k-chunks ahead of the MMAs, one MMA group in flight
constexpr int STEM_BAND = 8;        // output rows per stem CTA
constexpr int STEM_MAX_WO = 256;
constexpr int GN_MAX_C = 1024, GN_MAX_G = 32;
constexpr int GN_VECS_PER_CTA = 4096;   // 8-channel vectors of one image per apply CTA

__host__ __device__ inline int stat_cb(int C, int G) { return C / G < 32 ? C / G : 32; }
__host__ __device__ inline int stat_seg(int tm, long long hw) { return (int)((tm + hw - 2) / hw) + 1; }

// ------------------------------------------------------------------------------------------ fp16 wgmma, cp.async
template <int BN>
__device__ void wgmma_f16(float (&d)[BN / 2], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d);
template <>
__device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}

// K-major operand tile of rows of KC fp16 (RB = 2 KC bytes: 128, 64 or 32), stored with the matching wgmma swizzle
// (128B / 64B / 32B): the 16-byte chunk at byte offset o of the dense tile goes to o ^ (((o >> 7) & (RB/16 - 1)) << 4),
// so a repeat of 8 rows (8 RB bytes, the descriptor's stride offset) is conflict-free.  Tiles are 1024-byte aligned.
template <int KC>
__device__ __forceinline__ uint32_t swz(int row, int chunk) {
  constexpr int RB = 2 * KC, MASK = RB / 16 - 1;
  const uint32_t o = row * RB + chunk * 16;
  return o ^ (((o >> 7) & MASK) << 4);
}
template <int KC>
__device__ __forceinline__ uint64_t conv_desc(uint32_t addr) {
  constexpr uint64_t layout = KC == 64 ? 1 : KC == 32 ? 2 : 3;   // SWIZZLE_128B / 64B / 32B
  uint64_t d = (addr & 0x3FFFF) >> 4;
  d |= (uint64_t)1 << 16;                                      // leading offset: unused by swizzled K-major tiles
  d |= (uint64_t)(((16 * KC) >> 4) & 0x3FFF) << 32;            // stride offset: 8 rows of 2 KC bytes
  d |= layout << 62;
  return d;
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ------------------------------------------------------------------------------------------ 8-channel vectors
__device__ __forceinline__ void ld8(const __half* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __half22float2(h[i]);
    v[2 * i] = f.x, v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void ld8(const float* p, float (&v)[8]) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = b.x, v[5] = b.y, v[6] = b.z, v[7] = b.w;
}
__device__ __forceinline__ void st8(__half* p, const float (&v)[8]) {
  uint4 u;
  __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ void st8(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void cp8(__half* dst, const __half* src) {
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
}
__device__ __forceinline__ void cp8(float* dst, const float* src) {
  reinterpret_cast<float4*>(dst)[0] = reinterpret_cast<const float4*>(src)[0];
  reinterpret_cast<float4*>(dst)[1] = reinterpret_cast<const float4*>(src)[1];
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Store a staged output tile (rows x bn, row stride ld elements; tile column 0 is output channel n0) and write its
// GroupNorm partials (file comment).  Stat tile index `st`, stat tile height `tm`; hw = H W of the output map.
template <typename T>
__device__ void store_tile_stats(const T* tile, int ld, long long m0, int rows, int n0, int bn, T* __restrict__ y,
                                 int C, long long hw, int cb, int seg, long long st, float4* __restrict__ stats) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int vpr = bn / 8;
  for (int i = tid; i < rows * vpr; i += blockDim.x) {
    const int r = i / vpr, v = i - r * vpr;
    cp8(y + (m0 + r) * C + n0 + v * 8, tile + r * ld + v * 8);
  }
  const long long first = m0 / hw, last = (m0 + rows - 1) / hw;
  const int nb = bn / cb, units = (int)(last - first + 1) * nb;
  for (int u = warp; u < units; u += nwarps) {
    const int j = u / nb, b = u - j * nb;
    const long long img = first + j;
    const long long lo = (img * hw > m0 ? img * hw : m0) - m0;
    const long long hi = ((img + 1) * hw < m0 + rows ? (img + 1) * hw : m0 + rows) - m0;
    const int cnt = (int)(hi - lo) * cb;
    const T* t = tile + lo * ld + b * cb;
    float s = 0.f;
    for (int e = lane; e < cnt; e += 32) s += (float)t[(e / cb) * ld + e % cb];
    const float mean = warp_sum(s) / (float)cnt;
    float q = 0.f;
    for (int e = lane; e < cnt; e += 32) {
      const float d = (float)t[(e / cb) * ld + e % cb] - mean;
      q = fmaf(d, d, q);
    }
    q = warp_sum(q);
    if (lane == 0) stats[(st * seg + j) * (C / cb) + n0 / cb + b] = make_float4((float)cnt, mean, q, 0.f);
  }
}

struct ConvArgs {
  const void* x;   // (N, H, W, Cin)
  const void* w;   // (Cout, R, R, Cin)
  void* y;         // (N, Ho, Wo, Cout)
  float4* stats;
  int N, H, W, Cin, Ho, Wo, Cout, R, stride, pad, cb, seg;
  long long M;
};

// Implicit GEMM: D (M x Cout) = A (M x K) B^T, M = output pixels (n, oh, ow), K = (r, s, cin) in chunks of KC channels
// of one filter tap.  All 256 threads gather the A rows of a chunk (one 16-byte cp.async per row piece; zero fill for
// padding taps and rows past M) and the B rows, into the swizzled ring; each warpgroup runs m64nBNk16 wgmmas on its 64
// rows.  The fp32 accumulators are rounded to fp16 into a staged tile, stored and reduced to the GroupNorm partials.
template <int BN, int KC>
__global__ void __launch_bounds__(CONV_THREADS, 1) conv_wgmma_kernel(ConvArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int A_BYTES = CONV_BM * KC * 2, B_BYTES = BN * KC * 2, STAGE = A_BYTES + B_BYTES;
  constexpr int CPR = KC / 8, A_IT = CONV_BM * CPR / CONV_THREADS, ROWS_PER_IT = CONV_THREADS / CPR;
  static_assert(A_BYTES % 1024 == 0 && B_BYTES % 1024 == 0, "tiles must keep 1024-byte alignment");
  const int tid = threadIdx.x, wg = tid >> 7;
  const long long m0 = (long long)blockIdx.x * CONV_BM;
  const int n0 = blockIdx.y * BN;
  const __half* __restrict__ x = static_cast<const __half*>(a.x);
  const __half* __restrict__ w = static_cast<const __half*>(a.w);
  const int hwo = a.Ho * a.Wo, cch = a.Cin / KC, KT = a.R * a.R * cch, Ktot = a.R * a.R * a.Cin;

  const int ac = tid % CPR;
  int a_img[A_IT], a_ih[A_IT], a_iw[A_IT];
#pragma unroll
  for (int i = 0; i < A_IT; ++i) {
    const long long m = m0 + tid / CPR + i * ROWS_PER_IT;
    const int n = (int)(m / hwo), rem = (int)(m - (long long)n * hwo), oh = rem / a.Wo, ow = rem - oh * a.Wo;
    a_img[i] = m < a.M ? n : -1;
    a_ih[i] = oh * a.stride - a.pad;
    a_iw[i] = ow * a.stride - a.pad;
  }
  const uint32_t sbase = smem_u32(smem);
  auto load = [&](int kt, int st) {
    const uint32_t sa = sbase + st * STAGE, sb = sa + A_BYTES;
    const int tap = kt / cch, c0 = (kt - tap * cch) * KC;
    const int r = tap / a.R, s = tap - r * a.R;
#pragma unroll
    for (int i = 0; i < A_IT; ++i) {
      const int ih = a_ih[i] + r, iw = a_iw[i] + s;
      const bool ok = a_img[i] >= 0 && (unsigned)ih < (unsigned)a.H && (unsigned)iw < (unsigned)a.W;
      const __half* src = ok ? x + (((long long)a_img[i] * a.H + ih) * a.W + iw) * a.Cin + c0 + ac * 8 : x;
      cp_async16(sa + swz<KC>(tid / CPR + i * ROWS_PER_IT, ac), src, ok ? 16 : 0);
    }
    for (int i = tid; i < BN * CPR; i += CONV_THREADS) {
      const int row = i / CPR, c = i - row * CPR;
      cp_async16(sb + swz<KC>(row, c), w + (long long)(n0 + row) * Ktot + (long long)kt * KC + c * 8, 16);
    }
  };

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  pdl_wait();
#pragma unroll
  for (int s = 0; s < CONV_STAGES - 2; ++s) {
    if (s < KT) load(s, s);
    cp_async_commit();
  }
  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<CONV_STAGES - 3>();
    fence_proxy_async();   // this thread's cp.async writes, visible to the async proxy (wgmma)
    __syncthreads();       // ... and every thread's; also: every warpgroup has retired the MMAs of chunk kt - 2
    const uint32_t sa = sbase + (kt % CONV_STAGES) * STAGE + wg * 64 * KC * 2, sb = sbase + (kt % CONV_STAGES) * STAGE + A_BYTES;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KC / 16; ++kk) wgmma_f16<BN>(acc, conv_desc<KC>(sa + kk * 32), conv_desc<KC>(sb + kk * 32), 1);
    wgmma_commit();
    wgmma_wait<1>();
    if (kt + CONV_STAGES - 2 < KT) load(kt + CONV_STAGES - 2, (kt + CONV_STAGES - 2) % CONV_STAGES);
    cp_async_commit();
  }
  wgmma_wait<0>();
  fence_regs(acc);
  pdl_trigger();
  __syncthreads();   // every warpgroup's MMAs are done: the ring becomes the staging tile

  constexpr int LD = BN + 8;
  __half* tile = reinterpret_cast<__half*>(smem);
  const int warp = tid >> 5, lane = tid & 31;
  const int r0 = wg * 64 + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = 8 * j + 2 * (lane & 3);
    *reinterpret_cast<__half2*>(tile + r0 * LD + col) = __floats2half2_rn(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<__half2*>(tile + (r0 + 8) * LD + col) = __floats2half2_rn(acc[4 * j + 2], acc[4 * j + 3]);
  }
  __syncthreads();
  const int rows = (int)(a.M - m0 < CONV_BM ? a.M - m0 : CONV_BM);
  store_tile_stats<__half>(tile, LD, m0, rows, n0, BN, static_cast<__half*>(a.y), a.Cout, hwo, a.cb, a.seg,
                           blockIdx.x, a.stats);
}

// fp32 verification arm of the same entry: CUDA-core direct convolution in a fixed (r, s, cin) order, same tiles
// (128 rows x 32 channels per CTA), same staged store and statistics.
__global__ void __launch_bounds__(CONV_THREADS) conv_f32_kernel(ConvArgs a) {
  __shared__ __align__(16) float tile[CONV_BM * 36];
  const float* __restrict__ x = static_cast<const float*>(a.x);
  const float* __restrict__ w = static_cast<const float*>(a.w);
  const int tid = threadIdx.x, row = tid & (CONV_BM - 1), cg = tid >> 7;
  const long long m0 = (long long)blockIdx.x * CONV_BM, m = m0 + row;
  const int n0 = blockIdx.y * 32, co0 = n0 + cg * 16;
  const int hwo = a.Ho * a.Wo, Ktot = a.R * a.R * a.Cin;
  pdl_wait();
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  if (m < a.M) {
    const int n = (int)(m / hwo), rem = (int)(m - (long long)n * hwo), oh = rem / a.Wo, ow = rem - oh * a.Wo;
    for (int r = 0; r < a.R; ++r) {
      const int ih = oh * a.stride - a.pad + r;
      if ((unsigned)ih >= (unsigned)a.H) continue;
      for (int s = 0; s < a.R; ++s) {
        const int iw = ow * a.stride - a.pad + s;
        if ((unsigned)iw >= (unsigned)a.W) continue;
        const float* xp = x + (((long long)n * a.H + ih) * a.W + iw) * a.Cin;
        const float* wp = w + (long long)co0 * Ktot + (r * a.R + s) * a.Cin;
        for (int ci = 0; ci < a.Cin; ++ci) {
          const float xv = xp[ci];
#pragma unroll
          for (int j = 0; j < 16; ++j) acc[j] = fmaf(xv, __ldg(wp + (long long)j * Ktot + ci), acc[j]);
        }
      }
    }
  }
  pdl_trigger();
#pragma unroll
  for (int j = 0; j < 16; ++j) tile[row * 36 + cg * 16 + j] = acc[j];
  __syncthreads();
  const int rows = (int)(a.M - m0 < CONV_BM ? a.M - m0 : CONV_BM);
  store_tile_stats<float>(tile, 36, m0, rows, n0, 32, static_cast<float*>(a.y), a.Cout, hwo, a.cb, a.seg, blockIdx.x,
                          a.stats);
}

// avg_pool2d(depth, 2) then the 7x7 / 2, pad 3 convolution with one input channel and 32 outputs, on CUDA cores.  One
// CTA per band of STEM_BAND output rows of one image: the band's pooled rows (2 BAND + 5, zero outside the map) are
// computed once into shared memory from the raw depth (each pooled value ((a + b) + c) + d, times 1/4, avg_pool2d's own
// order), then each output row is a fixed-order 49-tap sum per (pixel, channel), staged, stored and reduced to the
// GroupNorm partials with one stat tile per output row (tm = Wo).
template <typename T>
__global__ void __launch_bounds__(CONV_THREADS) depth_stem_kernel(const float* __restrict__ depth, long long sn,
                                                                  long long sh, long long sw, int Hp, int Wp, int Ho,
                                                                  int Wo, const float* __restrict__ wt, int cb,
                                                                  int seg, T* __restrict__ y, float4* __restrict__ stats) {
  extern __shared__ __align__(16) float sm[];
  constexpr int PR = 2 * STEM_BAND + 5;
  const int pw = Wp + 6, ld = 40;
  float* ws = sm;                        // 32 x 49
  float* pool = ws + 32 * 49;            // PR x (Wp + 6)
  T* tile = reinterpret_cast<T*>(pool + ((PR * pw + 3) & ~3));   // Wo x ld
  const int bands = (Ho + STEM_BAND - 1) / STEM_BAND;
  const int n = blockIdx.x / bands, oh0 = (blockIdx.x - n * bands) * STEM_BAND;
  const int tid = threadIdx.x;
  pdl_wait();
  for (int i = tid; i < 32 * 49; i += CONV_THREADS) ws[i] = wt[i];
  const float* img = depth + n * sn;
  for (int i = tid; i < PR * pw; i += CONV_THREADS) {
    const int r = i / pw, ph = 2 * oh0 - 3 + r, pc = i - r * pw - 3;
    float v = 0.f;
    if ((unsigned)ph < (unsigned)Hp && (unsigned)pc < (unsigned)Wp) {
      const float* p = img + 2 * ph * sh + 2 * pc * sw;
      v = (((p[0] + p[sw]) + p[sh]) + p[sh + sw]) * 0.25f;
    }
    pool[i] = v;
  }
  __syncthreads();
  pdl_trigger();
  const long long hw = (long long)Ho * Wo;
  for (int o = 0; o < STEM_BAND && oh0 + o < Ho; ++o) {
    for (int i = tid; i < Wo * 32; i += CONV_THREADS) {
      const int ow = i >> 5, co = i & 31;
      const float* pp = pool + 2 * o * pw + 2 * ow;
      const float* wp = ws + co * 49;
      float acc = 0.f;
#pragma unroll
      for (int r = 0; r < 7; ++r)
#pragma unroll
        for (int s = 0; s < 7; ++s) acc = fmaf(pp[r * pw + s], wp[r * 7 + s], acc);
      tile[ow * ld + co] = (T)acc;
    }
    __syncthreads();
    const long long row = (long long)n * Ho + oh0 + o;
    store_tile_stats<T>(tile, ld, row * Wo, Wo, 0, 32, y, 32, hw, cb, seg, row, stats);
    __syncthreads();
  }
}

struct GnIn {
  const void* x;
  const float4* stats;
  const float* gamma;
  const float* beta;
  int tm;
};

// Per-channel mean and gamma * rstd of image n from the partials: thread g < G combines its group's partials tile by
// tile (the tiles that touch image n, in order) and block by block with Chan's rule; variance = M2 / count (biased,
// as GroupNorm), rstd = 1 / sqrt(var + eps).
__device__ void gn_stats(const GnIn& s, int n, long long hw, int C, int G, float eps, float* mean_c, float* scale_c,
                         float* gm, float* gr) {
  const int tid = threadIdx.x, cpg = C / G, cb = stat_cb(C, G), bpg = cpg / cb, nblk = C / cb;
  const int seg = stat_seg(s.tm, hw);
  if (tid < G) {
    const long long t0 = (long long)n * hw / s.tm, t1 = ((long long)(n + 1) * hw - 1) / s.tm;
    float cnt = 0.f, mean = 0.f, m2 = 0.f;
    for (long long t = t0; t <= t1; ++t) {
      const int j = (int)(n - t * s.tm / hw);
      const float4* p = s.stats + (t * seg + j) * nblk + tid * bpg;
      for (int k = 0; k < bpg; ++k) {
        const float4 q = p[k];
        const float nt = cnt + q.x, d = q.y - mean;
        mean = fmaf(d, q.x / nt, mean);
        m2 = m2 + q.z + d * d * (cnt * q.x / nt);
        cnt = nt;
      }
    }
    gm[tid] = mean;
    gr[tid] = 1.0f / sqrtf(m2 / cnt + eps);
  }
  __syncthreads();
  for (int c = tid; c < C; c += blockDim.x) {
    mean_c[c] = gm[c / cpg];
    scale_c[c] = gr[c / cpg] * __ldg(s.gamma + c);
  }
}

// y = relu(gamma (x - mean) rstd + beta  [+ identity | + gamma2 (x2 - mean2) rstd2 + beta2]) with MODE 0 / 1 / 2, or
// MODE 3: the 3x3 / 2, pad 1 max-pool of relu(gamma (x - mean) rstd + beta).  One CTA per GN_VECS_PER_CTA 8-channel
// output vectors of one image (blockIdx.y).  nchw: the output is (N, C, Ho, Wo) instead of NHWC.
template <typename T, typename TO, int MODE>
__global__ void __launch_bounds__(CONV_THREADS) gn_apply_kernel(GnIn a, GnIn b, const T* __restrict__ idn, int H,
                                                                int W, int C, int G, float eps, int Ho, int Wo,
                                                                int nchw, TO* __restrict__ out) {
  __shared__ float mean_a[GN_MAX_C], scale_a[GN_MAX_C], mean_b[MODE == 2 ? GN_MAX_C : 1],
      scale_b[MODE == 2 ? GN_MAX_C : 1];
  __shared__ float gm[GN_MAX_G], gr[GN_MAX_G];
  const int n = blockIdx.y, tid = threadIdx.x;
  const long long hw = (long long)H * W;
  pdl_wait();
  gn_stats(a, n, hw, C, G, eps, mean_a, scale_a, gm, gr);
  if (MODE == 2) {
    __syncthreads();
    gn_stats(b, n, hw, C, G, eps, mean_b, scale_b, gm, gr);
  }
  __syncthreads();
  pdl_trigger();
  const int vpp = C / 8;
  const long long nv = (long long)Ho * Wo * vpp, v0 = (long long)blockIdx.x * GN_VECS_PER_CTA;
  const long long v1 = v0 + GN_VECS_PER_CTA < nv ? v0 + GN_VECS_PER_CTA : nv;
  const T* xa = static_cast<const T*>(a.x) + n * hw * C;
  for (long long v = v0 + tid; v < v1; v += CONV_THREADS) {
    const long long pix = v / vpp;
    const int c = (int)(v - pix * vpp) * 8;
    float y[8];
    if (MODE == 3) {
      const int oh = (int)(pix / Wo), ow = (int)(pix - (long long)oh * Wo);
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] = 0.f;    // every window holds a valid pixel and relu(.) >= 0
      for (int dh = 0; dh < 3; ++dh) {
        const int ih = 2 * oh - 1 + dh;
        if ((unsigned)ih >= (unsigned)H) continue;
        for (int dw = 0; dw < 3; ++dw) {
          const int iw = 2 * ow - 1 + dw;
          if ((unsigned)iw >= (unsigned)W) continue;
          float xv[8];
          ld8(xa + ((long long)ih * W + iw) * C + c, xv);
#pragma unroll
          for (int e = 0; e < 8; ++e)
            y[e] = fmaxf(y[e], fmaxf(fmaf(xv[e] - mean_a[c + e], scale_a[c + e], __ldg(a.beta + c + e)), 0.f));
        }
      }
    } else {
      float xv[8];
      ld8(xa + pix * C + c, xv);
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] = fmaf(xv[e] - mean_a[c + e], scale_a[c + e], __ldg(a.beta + c + e));
      if (MODE == 1) {
        float r[8];
        ld8(idn + (n * hw + pix) * C + c, r);
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] += r[e];
      } else if (MODE == 2) {
        float r[8];
        ld8(static_cast<const T*>(b.x) + (n * hw + pix) * C + c, r);
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] += fmaf(r[e] - mean_b[c + e], scale_b[c + e], __ldg(b.beta + c + e));
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] = fmaxf(y[e], 0.f);
    }
    if (nchw) {
#pragma unroll
      for (int e = 0; e < 8; ++e) out[((long long)n * C + c + e) * Ho * Wo + pix] = (TO)y[e];
    } else {
      st8(out + ((long long)n * Ho * Wo + pix) * C + c, y);
    }
  }
}

template <typename K>
void allow_smem(K* kernel, int bytes) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

template <int BN, int KC>
int launch_conv(const ConvArgs& a, cudaStream_t st) {
  constexpr int smem = CONV_STAGES * (CONV_BM + BN) * KC * 2 + 1024;
  static bool init = false;
  if (!init) {
    allow_smem(conv_wgmma_kernel<BN, KC>, smem);
    init = true;
  }
  const dim3 grid((unsigned)((a.M + CONV_BM - 1) / CONV_BM), (unsigned)(a.Cout / BN));
  launch_pdl(conv_wgmma_kernel<BN, KC>, grid, dim3(CONV_THREADS), smem, st, a);
  return 0;
}

template <int KC>
int launch_conv_kc(const ConvArgs& a, cudaStream_t st) {
  if (a.Cout % 128 == 0) return launch_conv<128, KC>(a, st);
  if (a.Cout % 64 == 0) return launch_conv<64, KC>(a, st);
  return launch_conv<32, KC>(a, st);
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }
}  // namespace
}  // namespace bb

using namespace bb;

extern "C" int bb_conv2d(const void* x, const void* w, int N, int H, int W, int Cin, int Cout, int R, int stride,
                         int groups, void* y, void* stats, void* stream) {
  if (!x || !w || !y || !stats) return set_error("bb_conv2d: x / w / y / stats must not be NULL");
  if (N <= 0 || H <= 0 || W <= 0) return set_error("bb_conv2d: N, H and W must be positive");
  if (R != 1 && R != 3) return set_error("bb_conv2d: the filter must be 1x1 or 3x3");
  if (stride != 1 && stride != 2) return set_error("bb_conv2d: stride must be 1 or 2");
  if (Cin <= 0 || Cin % 16) return set_error("bb_conv2d: Cin must be a positive multiple of 16");
  if (Cout <= 0 || Cout % 32) return set_error("bb_conv2d: Cout must be a positive multiple of 32");
  if (groups <= 0 || Cout % groups) return set_error("bb_conv2d: groups must divide Cout");
  const int cpg = Cout / groups, cb = stat_cb(Cout, groups);
  if (cpg % cb || 32 % cb) return set_error("bb_conv2d: Cout / groups must divide 32 or be a multiple of 32");
  if (!aligned16(x) || !aligned16(w) || !aligned16(y) || !aligned16(stats))
    return set_error("bb_conv2d: x, w, y and stats must be 16-byte aligned");
  ConvArgs a;
  a.x = x, a.w = w, a.y = y, a.stats = static_cast<float4*>(stats);
  a.N = N, a.H = H, a.W = W, a.Cin = Cin, a.Cout = Cout, a.R = R, a.stride = stride, a.pad = (R - 1) / 2;
  a.Ho = (H + 2 * a.pad - R) / stride + 1;
  a.Wo = (W + 2 * a.pad - R) / stride + 1;
  a.M = (long long)N * a.Ho * a.Wo;
  a.cb = cb;
  a.seg = stat_seg(CONV_BM, (long long)a.Ho * a.Wo);
  if ((a.M + CONV_BM - 1) / CONV_BM > 0x7fffffffLL) return set_error("bb_conv2d: too many output pixels");
  cudaStream_t st = (cudaStream_t)stream;
  if (act_f32()) {
    const dim3 grid((unsigned)((a.M + CONV_BM - 1) / CONV_BM), (unsigned)(Cout / 32));
    launch_pdl(conv_f32_kernel, grid, dim3(CONV_THREADS), 0, st, a);
  } else if (Cin % 64 == 0) {
    launch_conv_kc<64>(a, st);
  } else if (Cin % 32 == 0) {
    launch_conv_kc<32>(a, st);
  } else {
    launch_conv_kc<16>(a, st);
  }
  count_launch();
  return check_launch("conv2d");
}

extern "C" int bb_depth_stem(const float* depth, int N, int Hd, int Wd, int64_t sn, int64_t sh, int64_t sw,
                             const float* w, int groups, void* y, void* stats, void* stream) {
  if (!depth || !w || !y || !stats) return set_error("bb_depth_stem: depth / w / y / stats must not be NULL");
  if (N <= 0 || Hd < 2 || Wd < 2) return set_error("bb_depth_stem: N must be positive and the depth at least 2 x 2");
  if (sn < 0 || sh < 0 || sw < 0) return set_error("bb_depth_stem: strides must be non-negative");
  if (groups <= 0 || 32 % groups) return set_error("bb_depth_stem: groups must divide 32");
  if (((uintptr_t)depth & 3) || !aligned16(y) || !aligned16(stats) || ((uintptr_t)w & 3))
    return set_error("bb_depth_stem: y and stats must be 16-byte aligned, depth and w 4-byte aligned");
  const int Hp = Hd / 2, Wp = Wd / 2, Ho = (Hp - 1) / 2 + 1, Wo = (Wp - 1) / 2 + 1;
  if (Wo > STEM_MAX_WO) return set_error("bb_depth_stem: the output may be at most 256 pixels wide (depth width 1024)");
  const int cb = stat_cb(32, groups), seg = stat_seg(Wo, (long long)Ho * Wo);
  const int pool_floats = ((2 * STEM_BAND + 5) * (Wp + 6) + 3) & ~3;
  const bool f32 = act_f32();
  const int smem = (32 * 49 + pool_floats) * 4 + Wo * 40 * (f32 ? 4 : 2);
  const dim3 grid((unsigned)(N * ((Ho + STEM_BAND - 1) / STEM_BAND)));
  static bool init = false;
  if (!init) {   // once, for the widest map accepted
    const int most = (32 * 49 + (((2 * STEM_BAND + 5) * (2 * STEM_MAX_WO + 6) + 3) & ~3)) * 4 + STEM_MAX_WO * 40 * 4;
    allow_smem(depth_stem_kernel<float>, most);
    allow_smem(depth_stem_kernel<__half>, most);
    init = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (f32) {
    launch_pdl(depth_stem_kernel<float>, grid, dim3(CONV_THREADS), smem, st, depth, (long long)sn, (long long)sh,
               (long long)sw, Hp, Wp, Ho, Wo, w, cb, seg, (float*)y, (float4*)stats);
  } else {
    launch_pdl(depth_stem_kernel<__half>, grid, dim3(CONV_THREADS), smem, st, depth, (long long)sn, (long long)sh,
               (long long)sw, Hp, Wp, Ho, Wo, w, cb, seg, (__half*)y, (float4*)stats);
  }
  count_launch();
  return check_launch("depth_stem_kernel");
}

namespace {
template <typename T, typename TO>
void launch_gn(int mode, const GnIn& a, const GnIn& b, const void* idn, int N, int H, int W, int C, int G, float eps,
               int Ho, int Wo, int nchw, void* out, cudaStream_t st) {
  const long long nv = (long long)Ho * Wo * (C / 8);
  const dim3 grid((unsigned)((nv + GN_VECS_PER_CTA - 1) / GN_VECS_PER_CTA), (unsigned)N);
  const T* id = static_cast<const T*>(idn);
  TO* o = static_cast<TO*>(out);
  switch (mode) {
    case 0: launch_pdl(gn_apply_kernel<T, TO, 0>, grid, dim3(CONV_THREADS), 0, st, a, b, id, H, W, C, G, eps, Ho, Wo, nchw, o); break;
    case 1: launch_pdl(gn_apply_kernel<T, TO, 1>, grid, dim3(CONV_THREADS), 0, st, a, b, id, H, W, C, G, eps, Ho, Wo, nchw, o); break;
    case 2: launch_pdl(gn_apply_kernel<T, TO, 2>, grid, dim3(CONV_THREADS), 0, st, a, b, id, H, W, C, G, eps, Ho, Wo, nchw, o); break;
    default: launch_pdl(gn_apply_kernel<T, TO, 3>, grid, dim3(CONV_THREADS), 0, st, a, b, id, H, W, C, G, eps, Ho, Wo, nchw, o); break;
  }
}
}  // namespace

extern "C" int bb_groupnorm_apply(const void* x, const void* stats, int tm, const float* gamma, const float* beta,
                                  const void* x2, const void* stats2, int tm2, const float* gamma2, const float* beta2,
                                  const void* identity, int N, int H, int W, int C, int groups, float eps, int mode,
                                  int out_f32, void* out, void* stream) {
  if (!x || !stats || !gamma || !beta || !out) return set_error("bb_groupnorm_apply: x / stats / gamma / beta / out must not be NULL");
  if (N <= 0 || H <= 0 || W <= 0 || tm <= 0) return set_error("bb_groupnorm_apply: N, H, W and tm must be positive");
  if (C <= 0 || C % 8 || C > GN_MAX_C) return set_error("bb_groupnorm_apply: C must be a positive multiple of 8, at most 1024");
  if (groups <= 0 || groups > GN_MAX_G || C % groups) return set_error("bb_groupnorm_apply: groups must divide C and be at most 32");
  if ((C / groups) % stat_cb(C, groups) || 32 % stat_cb(C, groups))
    return set_error("bb_groupnorm_apply: C / groups must divide 32 or be a multiple of 32");
  if (mode < 0 || mode > 3) return set_error("bb_groupnorm_apply: mode must be 0 (relu), 1 (+identity), 2 (+second norm) or 3 (max-pool)");
  if (mode == 1 && !identity) return set_error("bb_groupnorm_apply: mode 1 needs identity");
  if (mode == 2 && (!x2 || !stats2 || !gamma2 || !beta2 || tm2 <= 0))
    return set_error("bb_groupnorm_apply: mode 2 needs x2, stats2, gamma2, beta2 and tm2");
  if (out_f32 && mode != 0) return set_error("bb_groupnorm_apply: an fp32 output is only offered with mode 0");
  for (const void* p : {x, stats, (const void*)out, identity, x2, stats2})
    if (p && !aligned16(p)) return set_error("bb_groupnorm_apply: tensors must be 16-byte aligned");
  const int Ho = mode == 3 ? (H - 1) / 2 + 1 : H, Wo = mode == 3 ? (W - 1) / 2 + 1 : W;
  const GnIn a{x, static_cast<const float4*>(stats), gamma, beta, tm};
  const GnIn b{x2, static_cast<const float4*>(stats2), gamma2, beta2, tm2};
  cudaStream_t st = (cudaStream_t)stream;
  if (act_f32())
    launch_gn<float, float>(mode, a, b, identity, N, H, W, C, groups, eps, Ho, Wo, out_f32, out, st);
  else if (out_f32)
    launch_gn<__half, float>(mode, a, b, identity, N, H, W, C, groups, eps, Ho, Wo, 1, out, st);
  else
    launch_gn<__half, __half>(mode, a, b, identity, N, H, W, C, groups, eps, Ho, Wo, 0, out, st);
  count_launch();
  return check_launch("gn_apply_kernel");
}
