// Heatmap non-maximum suppression of the VLN-CE waypoint predictor (bevbert_ce/vlnce_baselines/waypoint_pred/utils.py:
// nms with gaussian=False, called at models/Policy_ViewSelection_BEV.py:221 on the softmaxed, wrapped heatmap).
// One CTA per batch row; the row's map lives in shared memory and is suppressed in place, round after round, with the
// reference's own fp32 arithmetic, so every output is bit-identical to the reference on the CPU.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"
#include "waypoint_nms.cuh"

namespace bb {
namespace {
constexpr int NMS_THREADS = 256;
constexpr int NMS_MAX_CELLS = 8192;   // H * W of one map: 32 KB of shared memory; the policy's map is 122 x 12

// One CTA per map: the map is copied into shared memory and suppressed there by nms::rounds (waypoint_nms.cuh).
__global__ void __launch_bounds__(NMS_THREADS) waypoint_nms_kernel(const float* __restrict__ pred, int H, int W,
                                                                    float sigma_x, float sigma_y, int rounds,
                                                                    float* __restrict__ out) {
  __shared__ float map[NMS_MAX_CELLS];
  __shared__ nms::Scratch<NMS_THREADS> scratch;
  pdl_wait();
  pdl_trigger();
  const int n = H * W, tid = threadIdx.x;
  const float* src = pred + (long long)blockIdx.x * n;
  float* dst = out + (long long)blockIdx.x * n;
  for (int i = tid; i < n; i += NMS_THREADS) {
    map[i] = src[i];
    dst[i] = 0.f;
  }
  __syncthreads();
  nms::rounds<NMS_THREADS>(map, src, dst, nullptr, H, W, sigma_x, sigma_y, rounds, scratch);
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
