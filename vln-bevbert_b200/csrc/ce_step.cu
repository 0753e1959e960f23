// The glue of the VLN-CE policy's `waypoint` call (bevbert_ce/vlnce_baselines/models/Policy_ViewSelection_BEV.py:166-
// 321, in_train=False) and of the trainer's _vp_feature_variable (ss_trainer_BEV.py:347-384), as two kernels that run
// inside the call's CUDA graph: no host memory is read and nothing synchronises with the host.
//   bb_ce_view_stack: the 12 + 12 per-heading observations -> the encoders' clockwise image batches and the 14 x 14
//     depth grid (AdaptiveAvgPool2d((14, 14)) in the CUDA device's own arithmetic).
//   bb_ce_waypoint_candidates: heatmap logits -> softmax, one-row wrap, NMS (waypoint_nms.cuh), strip, the nonzero
//     cells as (angle, distance) picks, and every feature array the `panorama` call takes.
//   bb_ce_waypoint_candidates_aug: the same with in_train=True (waypoint augmentation, lines 229-264): each pick is
//     replaced by a cell sampled from its image's regional softmax, given the caller's Exp(1) noise.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"
#include "waypoint_nms.cuh"

namespace bb {
namespace {
constexpr int VIEWS = 12, GRID = 14, GRID_CELLS = GRID * GRID;
constexpr int STACK_THREADS = 256, STACK_TILE = STACK_THREADS * 16;

// One image slot n = 12 b + s per blockIdx.y.  Slot s holds the k-th view in the observation dict's order,
// s = (12 - k) % 12 (the reference's reversal to clockwise order), read from table[k] (rgb) and table[12 + k] (depth).
// blockIdx.x < rgb_tiles copies rgb bytes, the next depth_tiles blocks copy depth values, and the last block writes the
// slot's 196 grid cells.  The grid is the arithmetic of the CUDA AdaptiveAvgPool2d((14, 14)) on the reference's permuted
// (N, 1, H, W) batch, confirmed against the device on order-sensitive inputs: bins [floor(i H / 14), ceil((i + 1) H /
// 14)), an fp32 sum from +0 in row-major order, times the fp32 reciprocal of kH * kW.
__global__ void __launch_bounds__(STACK_THREADS) ce_view_stack_kernel(const bb_ce_view* __restrict__ table, int Hr,
                                                                      int Wr, int Hd, int Wd, int rgb_tiles,
                                                                      int depth_tiles, uint8_t* __restrict__ rgb_out,
                                                                      float* __restrict__ depth_out,
                                                                      float* __restrict__ grid_out) {
  pdl_wait();
  pdl_trigger();
  const int n = blockIdx.y, b = n / VIEWS, s = n - b * VIEWS, k = (VIEWS - s) % VIEWS;
  const int tile = blockIdx.x, tid = threadIdx.x;
  if (tile < rgb_tiles) {
    const bb_ce_view v = table[k];
    const uint8_t* src = (const uint8_t*)v.ptr + b * v.sb;
    const long long count = (long long)Hr * Wr * 3;
    uint8_t* dst = rgb_out + (long long)n * count;
    const long long end = min(count, (long long)(tile + 1) * STACK_TILE);
    for (long long e = (long long)tile * STACK_TILE + tid; e < end; e += STACK_THREADS) {
      const int c = (int)(e % 3), hw = (int)(e / 3), w = hw % Wr, h = hw / Wr;
      dst[e] = src[h * v.sh + w * v.sw + c * v.sc];
    }
    return;
  }
  const bb_ce_view v = table[VIEWS + k];
  const float* src = (const float*)v.ptr + b * v.sb;
  if (tile < rgb_tiles + depth_tiles) {
    const long long count = (long long)Hd * Wd;
    float* dst = depth_out + (long long)n * count;
    const long long end = min(count, (long long)(tile - rgb_tiles + 1) * STACK_TILE);
    for (long long e = (long long)(tile - rgb_tiles) * STACK_TILE + tid; e < end; e += STACK_THREADS) {
      const int w = (int)(e % Wd), h = (int)(e / Wd);
      dst[e] = src[h * v.sh + w * v.sw];
    }
    return;
  }
  if (tid >= GRID_CELLS) return;
  const int i = tid / GRID, j = tid - i * GRID;
  const int h0 = i * Hd / GRID, h1 = ((i + 1) * Hd + GRID - 1) / GRID;
  const int w0 = j * Wd / GRID, w1 = ((j + 1) * Wd + GRID - 1) / GRID;
  float sum = 0.f;
  for (int h = h0; h < h1; ++h)
    for (int w = w0; w < w1; ++w) sum = __fadd_rn(sum, src[h * v.sh + w * v.sw]);
  grid_out[(long long)n * GRID_CELLS + tid] = __fmul_rn(sum, __fdiv_rn(1.f, (float)((h1 - h0) * (w1 - w0))));
}

constexpr int CAND_THREADS = 256;
constexpr int ANGLES = 120, DISTS = 12, CELLS = ANGLES * DISTS, WRAP_ROWS = ANGLES + 2, WRAP_CELLS = WRAP_ROWS * DISTS;
constexpr int MAX_PRED = 5, RGB_DIM = 512, DEP_DIM = 128, DEP_HW = 16, VIEW_ROWS = MAX_PRED + VIEWS;
constexpr float SIGMA_X = 7.f, SIGMA_Y = 5.f;   // nms(..., sigma=(7.0, 5.0)) at Policy_ViewSelection_BEV.py:221

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, ov) : __fadd_rn(v, ov);
  }
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = red[0];
  for (int w = 1; w < CAND_THREADS / 32; ++w) v = is_max ? fmaxf(v, red[w]) : __fadd_rn(v, red[w]);
  __syncthreads();
  return v;
}

// the clockwise image of counter-clockwise view j: view 0 stays, views 1..11 are flipped
__device__ __forceinline__ int cw_image(int j) { return (VIEWS - j) % VIEWS; }

// Writes one environment's picks row (pairs, count, view length) from cnt (angle, distance) pairs, and row_view: the
// counter-clockwise view of each panorama input row (the candidates' views, then the views without a candidate in
// ascending order, then -1).
__device__ void write_picks(int* pk, const int* ang, const int* dist, int cnt, int* row_view) {
  bool cand_view[VIEWS] = {};
  for (int q = 0; q < MAX_PRED; ++q) {
    const int a = q < cnt ? ang[q] : 0, d = q < cnt ? dist[q] : 0;
    pk[2 * q] = a;
    pk[2 * q + 1] = d;
    int img = VIEWS - (a + 5) / 10;
    if (img == VIEWS) img = 0;
    if (q < cnt) cand_view[img] = true, row_view[q] = img;
  }
  int len = cnt;
  for (int j = 0; j < VIEWS; ++j)
    if (!cand_view[j]) row_view[len++] = j;
  for (int t = len; t < VIEW_ROWS; ++t) row_view[t] = -1;
  pk[2 * MAX_PRED] = cnt;
  pk[2 * MAX_PRED + 1] = len;
}

// Waypoint augmentation of one pick at angle a, by one warp: the 120 regional logits of its clockwise image
// img = (a + 5) / 10 (12 -> 0), logits[(10 img + r - 5) mod 120, d] at s = 12 r + d; their softmax in the arithmetic of
// torch's CUDA softmax for rows of 120 (lane l holds s = l + 32 it; a sequential ternary max and sum per lane, then a
// butterfly); Categorical's renormalisation p / sum(p), the sum in this kernel's own order (per lane, then a
// butterfly); and torch.multinomial's single draw argmax(p / q) over the noise row q, under torch.argmax's rules.  The
// sample s becomes angle s / 12 + ((img - 1) * 10 + 5, or 0 for image 0) and distance s % 12.
__device__ __forceinline__ void sample_pick(const float* __restrict__ x, const float* __restrict__ q, int a, int* ang,
                                            int* dist) {
  constexpr int IT = 4, REGION = ANGLES;   // 120 = 10 angles x 12 distances, 4 x 32 lanes
  const int lane = threadIdx.x & 31;
  int img = (a + 5) / 10;
  if (img == VIEWS) img = 0;
  float e[IT];
#pragma unroll
  for (int it = 0; it < IT; ++it) {
    const int s = lane + 32 * it, r = s / DISTS, d = s - r * DISTS;
    e[it] = s < REGION ? x[((10 * img + r - 5 + ANGLES) % ANGLES) * DISTS + d] : -__int_as_float(0x7f800000);
  }
  float m = e[0];
#pragma unroll
  for (int it = 1; it < IT; ++it) m = m > e[it] ? m : e[it];
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    m = m < om ? om : m;
  }
  float sum = 0.f;
#pragma unroll
  for (int it = 0; it < IT; ++it) {
    e[it] = expf(__fsub_rn(e[it], m));
    sum = __fadd_rn(sum, e[it]);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) sum = __fadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, o));
  float norm = 0.f;
#pragma unroll
  for (int it = 0; it < IT; ++it) {
    e[it] = __fdiv_rn(e[it], sum);
    if (lane + 32 * it < REGION) norm = __fadd_rn(norm, e[it]);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) norm = __fadd_rn(norm, __shfl_xor_sync(0xffffffffu, norm, o));
  float bv = -__int_as_float(0x7f800000);
  int bi = 0x7fffffff;
#pragma unroll
  for (int it = 0; it < IT; ++it) {
    const int s = lane + 32 * it;
    if (s >= REGION) continue;
    const float v = __fdiv_rn(__fdiv_rn(e[it], norm), q[s]);
    if (nms::beats(v, s, bv, bi)) bv = v, bi = s;
  }
  nms::warp_best(bv, bi);
  if (lane == 0) {
    *ang = bi / DISTS + (img != 0 ? (img - 1) * 10 + 5 : 0);
    *dist = bi % DISTS;
  }
}

// One CTA per environment b.  AUG: in_train=True, `noise` (B, 5, 120) holds pick k's Exp(1) row at [b, k]; picks gets
// the sampled pairs, nms_picks (may be NULL) the pre-sampling ones, and the features follow the sampled views.
template <bool AUG>
__global__ void __launch_bounds__(CAND_THREADS) ce_waypoint_candidates_kernel(
    const float* __restrict__ logits, const float* __restrict__ noise, const float* __restrict__ rgb_vec,
    const float* __restrict__ depth_feat, int* __restrict__ picks, int* __restrict__ nms_picks,
    float* __restrict__ prob, float* __restrict__ pano_rgb, float* __restrict__ pano_depth,
    float* __restrict__ cand_rgb, float* __restrict__ cand_depth, float* __restrict__ rgb_fts,
    float* __restrict__ dep_fts) {
  __shared__ float heat[WRAP_CELLS];     // the wrapped softmax map, unsuppressed
  __shared__ float work[WRAP_CELLS];     // the same, suppressed round by round
  __shared__ float out_map[WRAP_CELLS];  // nms's output
  __shared__ float dep_mean[VIEWS * DEP_DIM];
  __shared__ float red[CAND_THREADS / 32];
  __shared__ nms::Scratch<CAND_THREADS> scratch;
  __shared__ int round_pick[MAX_PRED];
  __shared__ int pick_ang[MAX_PRED], pick_dist[MAX_PRED];
  __shared__ int row_view[VIEW_ROWS];    // counter-clockwise view of each panorama input row, -1: zeros
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* x = logits + (long long)b * CELLS;

  // 1. softmax over the 1440 cells: expf(x - max) / sum, the sum in this kernel's own order (within 16 fp32 ulps of
  // torch's values; the NMS picks, which compare cells of one map under one divisor, are torch's)
  float m = -__int_as_float(0x7f800000);
  for (int i = tid; i < CELLS; i += CAND_THREADS) m = fmaxf(m, x[i]);
  m = block_reduce(m, true, red);
  float sum = 0.f;
  for (int i = tid; i < CELLS; i += CAND_THREADS) {
    const float e = expf(__fsub_rn(x[i], m));
    work[i] = e;
    sum = __fadd_rn(sum, e);
  }
  sum = block_reduce(sum, false, red);
  // 2. wrap: row 0 is angle 119, rows 1..120 are angles 0..119, row 121 is angle 0
  for (int i = tid; i < CELLS; i += CAND_THREADS) {
    const float p = __fdiv_rn(work[i], sum);
    if (prob) prob[(long long)b * CELLS + i] = p;
    heat[i + DISTS] = p;
    if (i < DISTS) heat[(WRAP_ROWS - 1) * DISTS + i] = p;
    if (i >= CELLS - DISTS) heat[i - (CELLS - DISTS)] = p;
  }
  __syncthreads();
  for (int i = tid; i < WRAP_CELLS; i += CAND_THREADS) {
    work[i] = heat[i];
    out_map[i] = 0.f;
  }
  __syncthreads();
  // 3. NMS, bb_waypoint_nms's rounds
  nms::rounds<CAND_THREADS>(work, heat, out_map, round_pick, WRAP_ROWS, DISTS, SIGMA_X, SIGMA_Y, MAX_PRED, scratch);
  __syncthreads();

  // 4 + 5. strip the wrap rows and compact the nonzero cells in row-major order: every nonzero cell of nms's output is
  // a pick, so the picks that survive the strip and are nonzero, sorted and without repeats, are `nonzero`'s rows.
  if (tid == 0) {
    int cells[MAX_PRED], cnt = 0;
    for (int r = 0; r < MAX_PRED; ++r) {
      const int ix = round_pick[r], row = ix / DISTS;
      if (row < 1 || row > ANGLES || !(out_map[ix] != 0.f)) continue;
      int at = cnt;
      bool seen = false;
      for (int q = 0; q < cnt; ++q) seen |= cells[q] == ix;
      if (seen) continue;
      while (at > 0 && cells[at - 1] > ix) cells[at] = cells[at - 1], --at;
      cells[at] = ix;
      ++cnt;
    }
    for (int q = 0; q < cnt; ++q) pick_ang[q] = cells[q] / DISTS - 1, pick_dist[q] = cells[q] % DISTS;
    int* out = AUG ? nms_picks : picks;
    if (out) write_picks(out + b * BB_CE_PICK_COLS, pick_ang, pick_dist, cnt, row_view);
    scratch.pick = cnt;
  }
  if (AUG) {
    __syncthreads();
    const int warp = tid >> 5;
    if (warp < scratch.pick)
      sample_pick(x, noise + ((long long)b * MAX_PRED + warp) * ANGLES, pick_ang[warp], &pick_ang[warp],
                  &pick_dist[warp]);
    __syncthreads();
    if (tid == 0) write_picks(picks + b * BB_CE_PICK_COLS, pick_ang, pick_dist, scratch.pick, row_view);
  }
  // 6. features.  pano_depth: torch's CUDA mean over the 4 x 4 cells as the device computes it (confirmed on order-
  // sensitive inputs): each cell from +0, a halving tree (cell q += cell q + 8, then + 4, + 2, + 1), then times 1/16.
  const float* dep = depth_feat + (long long)b * VIEWS * DEP_DIM * DEP_HW;
  for (int o = tid; o < VIEWS * DEP_DIM; o += CAND_THREADS) {
    const int j = o / DEP_DIM, c = o - j * DEP_DIM;
    const float* p = dep + ((long long)cw_image(j) * DEP_DIM + c) * DEP_HW;
    float t[DEP_HW];
#pragma unroll
    for (int q = 0; q < DEP_HW; ++q) t[q] = __fadd_rn(0.f, p[q]);
#pragma unroll
    for (int q = 0; q < 8; ++q) t[q] = __fadd_rn(t[q], t[q + 8]);
#pragma unroll
    for (int q = 0; q < 4; ++q) t[q] = __fadd_rn(t[q], t[q + 4]);
    t[0] = __fadd_rn(t[0], t[2]);
    t[1] = __fadd_rn(t[1], t[3]);
    t[0] = __fadd_rn(t[0], t[1]);
    const float mean = __fmul_rn(t[0], 1.f / DEP_HW);
    dep_mean[o] = mean;
    pano_depth[(long long)b * VIEWS * DEP_DIM + o] = mean;
  }
  const float* rgb = rgb_vec + (long long)b * VIEWS * RGB_DIM;
  for (int o = tid; o < VIEWS * RGB_DIM; o += CAND_THREADS) {
    const int j = o / RGB_DIM, c = o - j * RGB_DIM;
    pano_rgb[(long long)b * VIEWS * RGB_DIM + o] = rgb[cw_image(j) * RGB_DIM + c];
  }
  __syncthreads();
  const int cnt = scratch.pick;
  for (int o = tid; o < MAX_PRED * RGB_DIM; o += CAND_THREADS) {
    const int q = o / RGB_DIM, c = o - q * RGB_DIM;
    cand_rgb[(long long)b * MAX_PRED * RGB_DIM + o] = q < cnt ? rgb[cw_image(row_view[q]) * RGB_DIM + c] : 0.f;
  }
  for (int o = tid; o < MAX_PRED * DEP_DIM; o += CAND_THREADS) {
    const int q = o / DEP_DIM, c = o - q * DEP_DIM;
    cand_depth[(long long)b * MAX_PRED * DEP_DIM + o] = q < cnt ? dep_mean[row_view[q] * DEP_DIM + c] : 0.f;
  }
  for (int o = tid; o < VIEW_ROWS * RGB_DIM; o += CAND_THREADS) {
    const int t = o / RGB_DIM, c = o - t * RGB_DIM, j = row_view[t];
    rgb_fts[(long long)b * VIEW_ROWS * RGB_DIM + o] = j >= 0 ? rgb[cw_image(j) * RGB_DIM + c] : 0.f;
  }
  for (int o = tid; o < VIEW_ROWS * DEP_DIM; o += CAND_THREADS) {
    const int t = o / DEP_DIM, c = o - t * DEP_DIM, j = row_view[t];
    dep_fts[(long long)b * VIEW_ROWS * DEP_DIM + o] = j >= 0 ? dep_mean[j * DEP_DIM + c] : 0.f;
  }
}

bool overlaps(const void* a, long long na, const void* b, long long nb) {
  const char *pa = (const char*)a, *pb = (const char*)b;
  return pa < pb + nb && pb < pa + na;
}
}  // namespace
}  // namespace bb

using namespace bb;

extern "C" int bb_ce_view_stack(const bb_ce_view* table, int B, int rgb_h, int rgb_w, int depth_h, int depth_w,
                                uint8_t* rgb_out, float* depth_out, float* grid_out, void* stream) {
  if (B <= 0 || rgb_h <= 0 || rgb_w <= 0 || depth_h <= 0 || depth_w <= 0)
    return set_error("bb_ce_view_stack: B and the image sizes must be positive");
  if (depth_h < GRID || depth_w < GRID) return set_error("bb_ce_view_stack: the depth images must be at least 14 x 14");
  if ((long long)rgb_h * rgb_w * 3 > (1LL << 30) || (long long)depth_h * depth_w > (1LL << 28))
    return set_error("bb_ce_view_stack: image too large");
  if ((long long)B * VIEWS > 65535) return set_error("bb_ce_view_stack: 12 B must be at most 65535");
  if (!table || !rgb_out || !depth_out || !grid_out)
    return set_error("bb_ce_view_stack: table / rgb_out / depth_out / grid_out must not be NULL");
  if (((uintptr_t)table & 7) || ((uintptr_t)depth_out & 3) || ((uintptr_t)grid_out & 3))
    return set_error("bb_ce_view_stack: table must be 8-byte and depth_out / grid_out 4-byte aligned");
  const long long n = (long long)B * VIEWS, rgb_bytes = n * rgb_h * rgb_w * 3, depth_bytes = n * depth_h * depth_w * 4,
                  grid_bytes = n * GRID_CELLS * 4;
  if (overlaps(rgb_out, rgb_bytes, depth_out, depth_bytes) || overlaps(rgb_out, rgb_bytes, grid_out, grid_bytes) ||
      overlaps(depth_out, depth_bytes, grid_out, grid_bytes))
    return set_error("bb_ce_view_stack: the outputs must not overlap");
  const int rgb_tiles = (int)((3LL * rgb_h * rgb_w + STACK_TILE - 1) / STACK_TILE);
  const int depth_tiles = (int)(((long long)depth_h * depth_w + STACK_TILE - 1) / STACK_TILE);
  launch_pdl(ce_view_stack_kernel, dim3((unsigned)(rgb_tiles + depth_tiles + 1), (unsigned)n), dim3(STACK_THREADS), 0,
             (cudaStream_t)stream, table, rgb_h, rgb_w, depth_h, depth_w, rgb_tiles, depth_tiles, rgb_out, depth_out,
             grid_out);
  count_launch();
  return check_launch("ce_view_stack_kernel");
}

namespace bb {
namespace {
// The argument checks of both candidate entry points: NULL, alignment, and no output overlapping another output or an
// input.  noise (AUG only) and the optional prob / nms_picks join the lists when given.
int check_candidates(const char* name, const float* logits, const float* noise, const float* rgb_vec,
                     const float* depth_feat, int B, int* picks, int* nms_picks, float* prob, float* pano_rgb,
                     float* pano_depth, float* cand_rgb, float* cand_depth, float* rgb_fts, float* dep_fts, bool aug) {
  char msg[160];
  if (B <= 0 || B > 65535) {
    snprintf(msg, sizeof msg, "%s: B must be in [1, 65535]", name);
    return set_error(msg);
  }
  const void* ptrs[] = {logits, rgb_vec, depth_feat, picks, pano_rgb, pano_depth, cand_rgb, cand_depth, rgb_fts,
                        dep_fts, aug ? (const void*)noise : (const void*)logits};
  for (const void* p : ptrs)
    if (!p) {
      snprintf(msg, sizeof msg, "%s: only %s may be NULL", name, aug ? "nms_picks" : "prob");
      return set_error(msg);
    }
  for (const void* p : ptrs)
    if ((uintptr_t)p & 3) {
      snprintf(msg, sizeof msg, "%s: pointers must be 4-byte aligned", name);
      return set_error(msg);
    }
  if (((uintptr_t)prob & 3) || ((uintptr_t)nms_picks & 3)) {
    snprintf(msg, sizeof msg, "%s: pointers must be 4-byte aligned", name);
    return set_error(msg);
  }
  const long long f = 4LL * B;
  const struct { const void* p; long long n; } outs[] = {
      {picks, f * BB_CE_PICK_COLS}, {prob, prob ? f * CELLS : 0}, {nms_picks, nms_picks ? f * BB_CE_PICK_COLS : 0},
      {pano_rgb, f * VIEWS * RGB_DIM}, {pano_depth, f * VIEWS * DEP_DIM}, {cand_rgb, f * MAX_PRED * RGB_DIM},
      {cand_depth, f * MAX_PRED * DEP_DIM}, {rgb_fts, f * VIEW_ROWS * RGB_DIM}, {dep_fts, f * VIEW_ROWS * DEP_DIM}};
  const struct { const void* p; long long n; } ins[] = {{logits, f * CELLS},
                                                        {rgb_vec, f * VIEWS * RGB_DIM},
                                                        {depth_feat, f * VIEWS * DEP_DIM * DEP_HW},
                                                        {noise, aug ? f * MAX_PRED * ANGLES : 0}};
  const int n_out = (int)(sizeof(outs) / sizeof(outs[0])), n_in = (int)(sizeof(ins) / sizeof(ins[0]));
  for (int i = 0; i < n_out; ++i) {
    for (int j = i + 1; j < n_out; ++j)
      if (overlaps(outs[i].p, outs[i].n, outs[j].p, outs[j].n)) {
        snprintf(msg, sizeof msg, "%s: the outputs must not overlap", name);
        return set_error(msg);
      }
    for (int j = 0; j < n_in; ++j)
      if (overlaps(outs[i].p, outs[i].n, ins[j].p, ins[j].n)) {
        snprintf(msg, sizeof msg, "%s: an output overlaps an input", name);
        return set_error(msg);
      }
  }
  return 0;
}
}  // namespace
}  // namespace bb

extern "C" int bb_ce_waypoint_candidates(const float* logits, const float* rgb_vec, const float* depth_feat, int B,
                                         int* picks, float* prob, float* pano_rgb, float* pano_depth, float* cand_rgb,
                                         float* cand_depth, float* rgb_fts, float* dep_fts, void* stream) {
  if (check_candidates("bb_ce_waypoint_candidates", logits, nullptr, rgb_vec, depth_feat, B, picks, nullptr, prob,
                       pano_rgb, pano_depth, cand_rgb, cand_depth, rgb_fts, dep_fts, false))
    return -1;
  launch_pdl(ce_waypoint_candidates_kernel<false>, dim3((unsigned)B), dim3(CAND_THREADS), 0, (cudaStream_t)stream,
             logits, (const float*)nullptr, rgb_vec, depth_feat, picks, (int*)nullptr, prob, pano_rgb, pano_depth,
             cand_rgb, cand_depth, rgb_fts, dep_fts);
  count_launch();
  return check_launch("ce_waypoint_candidates_kernel");
}

extern "C" int bb_ce_waypoint_candidates_aug(const float* logits, const float* noise, const float* rgb_vec,
                                             const float* depth_feat, int B, int* picks, int* nms_picks,
                                             float* pano_rgb, float* pano_depth, float* cand_rgb, float* cand_depth,
                                             float* rgb_fts, float* dep_fts, void* stream) {
  if (check_candidates("bb_ce_waypoint_candidates_aug", logits, noise, rgb_vec, depth_feat, B, picks, nms_picks,
                       nullptr, pano_rgb, pano_depth, cand_rgb, cand_depth, rgb_fts, dep_fts, true))
    return -1;
  launch_pdl(ce_waypoint_candidates_kernel<true>, dim3((unsigned)B), dim3(CAND_THREADS), 0, (cudaStream_t)stream,
             logits, noise, rgb_vec, depth_feat, picks, nms_picks, (float*)nullptr, pano_rgb, pano_depth, cand_rgb,
             cand_depth, rgb_fts, dep_fts);
  count_launch();
  return check_launch("ce_waypoint_candidates_aug_kernel");
}
