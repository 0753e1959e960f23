// Device code of the waypoint heatmap NMS (waypoint_pred/utils.py nms, gaussian=False), shared by bb_waypoint_nms
// (waypoint.cu) and the candidate pass of the CE waypoint step (ce_step.cu), so both pick with the same rules.
#pragma once
#include <cuda_runtime.h>

namespace bb {
namespace nms {

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

// Shared memory of one CTA's rounds.
template <int THREADS>
struct Scratch {
  float warp_v[THREADS / 32];
  int warp_i[THREADS / 32];
  int pick;
};

// `rounds` rounds over the H x W map `map` (shared memory, suppressed in place); `src` holds the unsuppressed values
// and `dst` the output, zeroed by the caller.  Round r: ix = argmax of the suppressed map; dst[ix] = src[ix] (< 0
// clamped to +0, as the reference's final `output[output < 0] = 0` does); picks[r] = ix when picks is not NULL; then
// every cell is multiplied by (1 - g), g = 1 inside the neighbourhood of ix and 0 outside.  The neighbourhood is
// utils.py's `neighborhoods` in fp32: x_mu = ix % W, y_mu = ix / W (true division, correctly rounded), rows kept where
// |y - y_mu| <= sigma_y and columns where min(|x - x_mu|, |x - x_mu + W|) <= sigma_x.  A literal multiply, not a flag: a
// suppressed negative becomes -0.0, a NaN or an infinity becomes NaN, and a later round may pick an already-suppressed
// cell, as in the reference.  Each thread owns the cells i = tid + k * THREADS for the scan and the suppression alike,
// so the map needs no barrier between them.  All THREADS threads of the CTA must call it; it ends on a barrier-free
// suppression pass, so a caller that reads the map or dst afterwards synchronises first.
template <int THREADS>
__device__ __forceinline__ void rounds(float* map, const float* src, float* dst, int* picks, int H, int W,
                                       float sigma_x, float sigma_y, int n_rounds, Scratch<THREADS>& s) {
  const int n = H * W, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float fw = (float)W;
  for (int r = 0; r < n_rounds; ++r) {
    float bv = -__int_as_float(0x7f800000);   // -inf at an index past every cell: any cell beats it
    int bi = 0x7fffffff;
    for (int i = tid; i < n; i += THREADS)
      if (beats(map[i], i, bv, bi)) bv = map[i], bi = i;
    warp_best(bv, bi);
    if (lane == 0) s.warp_v[warp] = bv, s.warp_i[warp] = bi;
    __syncthreads();
    if (warp == 0) {
      bv = lane < THREADS / 32 ? s.warp_v[lane] : -__int_as_float(0x7f800000);
      bi = lane < THREADS / 32 ? s.warp_i[lane] : 0x7fffffff;
      warp_best(bv, bi);
      if (lane == 0) {
        s.pick = bi;
        const float v = src[bi];
        dst[bi] = v < 0.f ? 0.f : v;
        if (picks) picks[r] = bi;
      }
    }
    __syncthreads();
    const int ix = s.pick;
    const float x_mu = (float)(ix % W), y_mu = __fdiv_rn((float)ix, fw);
    for (int i = tid; i < n; i += THREADS) {
      const int row = i / W, col = i - row * W;
      const float xd = __fsub_rn((float)col, x_mu), yd = __fsub_rn((float)row, y_mu);
      const float xc = fminf(fabsf(xd), fabsf(__fadd_rn(xd, fw)));
      const float g = (xc <= sigma_x && fabsf(yd) <= sigma_y) ? 1.f : 0.f;
      map[i] = __fmul_rn(map[i], __fsub_rn(1.f, g));
    }
  }
}

}  // namespace nms
}  // namespace bb
