// Heatmap non-maximum suppression of the VLN-CE waypoint predictor (bevbert_ce/vlnce_baselines/waypoint_pred/utils.py:
// nms with gaussian=False, called at models/Policy_ViewSelection_BEV.py:221 on the softmaxed, wrapped heatmap).
// One CTA per batch row; the row's map lives in shared memory and is suppressed in place, round after round, with the
// reference's own fp32 arithmetic, so every output is bit-identical to the reference on the CPU.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {
namespace {
constexpr int NMS_THREADS = 256;
constexpr int NMS_MAX_CELLS = 8192;   // H * W of one map: 32 KB of shared memory; the policy's map is 122 x 12

// True when (a, ia) ranks above (b, ib) under torch.max's rules: NaN above every number (the lowest index among NaNs),
// otherwise the larger value, and on equal values (-0.0 == +0.0) the lower index.  A strict total order on distinct
// indices, so every lane of a butterfly reduction ends with the same winner.
__device__ __forceinline__ bool beats(float a, int ia, float b, int ib) {
  const bool na = a != a, nb = b != b;
  if (na || nb) return na && (!nb || ia < ib);
  return a > b || (a == b && ia < ib);
}

__device__ __forceinline__ void warp_best(float& v, int& i) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (beats(ov, oi, v, i)) v = ov, i = oi;
  }
}

// Round r: ix = argmax of the suppressed map; out[ix] = pred[ix] (the unsuppressed value, < 0 clamped to +0 as the
// reference's final `output[output < 0] = 0` does); then every cell is multiplied by (1 - g), g = 1 inside the
// neighbourhood of ix and 0 outside.  The neighbourhood is utils.py's `neighborhoods` in fp32: x_mu = ix % W,
// y_mu = ix / W (true division, correctly rounded), rows kept where |y - y_mu| <= sigma_y and columns where
// min(|x - x_mu|, |x - x_mu + W|) <= sigma_x.  A literal multiply, not a flag: a suppressed negative becomes -0.0, a NaN
// or an infinity becomes NaN, and a later round may pick an already-suppressed cell, as in the reference.  Each thread
// owns the cells i = tid + k * NMS_THREADS for the scan and the suppression alike, so the map needs no barrier between
// them.
__global__ void __launch_bounds__(NMS_THREADS) waypoint_nms_kernel(const float* __restrict__ pred, int H, int W,
                                                                    float sigma_x, float sigma_y, int rounds,
                                                                    float* __restrict__ out) {
  __shared__ float map[NMS_MAX_CELLS];
  __shared__ float warp_v[NMS_THREADS / 32];
  __shared__ int warp_i[NMS_THREADS / 32];
  __shared__ int pick;
  pdl_wait();
  pdl_trigger();
  const int n = H * W, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* src = pred + (long long)blockIdx.x * n;
  float* dst = out + (long long)blockIdx.x * n;
  for (int i = tid; i < n; i += NMS_THREADS) {
    map[i] = src[i];
    dst[i] = 0.f;
  }
  __syncthreads();
  const float fw = (float)W;
  for (int r = 0; r < rounds; ++r) {
    float bv = -__int_as_float(0x7f800000);   // -inf at an index past every cell: any cell beats it
    int bi = 0x7fffffff;
    for (int i = tid; i < n; i += NMS_THREADS)
      if (beats(map[i], i, bv, bi)) bv = map[i], bi = i;
    warp_best(bv, bi);
    if (lane == 0) warp_v[warp] = bv, warp_i[warp] = bi;
    __syncthreads();
    if (warp == 0) {
      bv = lane < NMS_THREADS / 32 ? warp_v[lane] : -__int_as_float(0x7f800000);
      bi = lane < NMS_THREADS / 32 ? warp_i[lane] : 0x7fffffff;
      warp_best(bv, bi);
      if (lane == 0) {
        pick = bi;
        const float v = src[bi];
        dst[bi] = v < 0.f ? 0.f : v;
      }
    }
    __syncthreads();
    const int ix = pick;
    const float x_mu = (float)(ix % W), y_mu = __fdiv_rn((float)ix, fw);
    for (int i = tid; i < n; i += NMS_THREADS) {
      const int row = i / W, col = i - row * W;
      const float xd = __fsub_rn((float)col, x_mu), yd = __fsub_rn((float)row, y_mu);
      const float xc = fminf(fabsf(xd), fabsf(__fadd_rn(xd, fw)));
      const float g = (xc <= sigma_x && fabsf(yd) <= sigma_y) ? 1.f : 0.f;
      map[i] = __fmul_rn(map[i], __fsub_rn(1.f, g));
    }
  }
}
}  // namespace
}  // namespace bb

using namespace bb;

extern "C" int bb_waypoint_nms(const float* pred, int B, int H, int W, float sigma_x, float sigma_y,
                               int max_predictions, float* out, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return set_error("bb_waypoint_nms: B, H and W must be positive");
  if (!pred || !out) return set_error("bb_waypoint_nms: pred / out must not be NULL");
  if ((long long)H * W > NMS_MAX_CELLS) return set_error("bb_waypoint_nms: H * W must be at most 8192");
  if (max_predictions < 0) return set_error("bb_waypoint_nms: max_predictions must be non-negative");
  if (((uintptr_t)pred & 3) || ((uintptr_t)out & 3)) return set_error("bb_waypoint_nms: pred / out must be 4-byte aligned");
  const long long cells = (long long)B * H * W;
  if (pred < out + cells && out < pred + cells) return set_error("bb_waypoint_nms: pred and out must not overlap");
  launch_pdl(waypoint_nms_kernel, dim3((unsigned)B), dim3(NMS_THREADS), 0, (cudaStream_t)stream, pred, H, W, sigma_x,
             sigma_y, max_predictions, out);
  count_launch();
  return check_launch("waypoint_nms_kernel");
}
