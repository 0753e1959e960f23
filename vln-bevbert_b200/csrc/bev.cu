// BEV grid lifting for sm_90a: depth un-projection + camera->world->ego transforms + integer cell index
// (one pass, bit-exact arithmetic order), then a deterministic scatter-mean pool of 768-wide patch
// features (and float64 semantic one-hots) into the D x D metric map.
//
// Reference: pretrain_src/model/pretrain_cmt.py:114-167 (lift_splat), bev_utils.py:139-172,198,349-378
// (PointCloud.forward) and :381-430 (project_bev); torch_scatter.scatter_mean call sites :407,417.
// These are HBM-bound kernels: coalesced 16-byte row loads, no atomics, no intermediate point cloud in HBM.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {

// ---------------------------------------------------------------------------------------------
// Point arithmetic shared by every kernel that places points into the map. All of it uses explicit round-to-nearest
// single operations (no FMA contraction) in a fixed order so that the CPU oracles (oracle/bevbert_ref.py: lift_points,
// cell_index; tests/nav_bev_oracle.py: nav_splat_nodes) reproduce every bit.
// ---------------------------------------------------------------------------------------------
// world -> ego: (w - S) then [p, 1] * T_w2c^T, each 4-term dot product left to right (pretrain_cmt.py:133-137,
// map_nav_src/r2r/agent.py:162-166). S (3), E = T_w2c (4x4 row major).
__device__ __forceinline__ void ego_transform(float w0, float w1, float w2, const float* S, const float* E, float e[3]) {
  const float p0 = __fsub_rn(w0, S[0]), p1 = __fsub_rn(w1, S[1]), p2 = __fsub_rn(w2, S[2]);
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    float acc = __fmul_rn(p0, E[j * 4 + 0]);
    acc = __fadd_rn(acc, __fmul_rn(p1, E[j * 4 + 1]));
    acc = __fadd_rn(acc, __fmul_rn(p2, E[j * 4 + 2]));
    acc = __fadd_rn(acc, E[j * 4 + 3]);
    e[j] = acc;
  }
}

// discretise an ego-frame point (bev_utils.py:393-406): round half to even, bounds, height clip -> D*z+x or -1.
// NaN coordinates compare false everywhere in the reference and then index out of range; we drop them.
__device__ __forceinline__ int32_t bev_cell(float e0, float e1, float e2, bool no_depth, int D, float res, float half,
                                            float y_clip) {
  const float gx = rintf(__fadd_rn(__fdiv_rn(e0, res), half));
  const float gz = rintf(__fadd_rn(__fdiv_rn(e2, res), half));
  const float Df = (float)D;
  const bool outside = (gx >= Df) || (gz >= Df) || (gx < 0.0f) || (gz < 0.0f);
  const bool bad = no_depth || outside || (e1 > y_clip) || !(gx == gx) || !(gz == gz);
  return bad ? -1 : (int32_t)(Df * gz + gx);
}

// depth pixel -> world point (bev_utils.py:130-131,167-172,198): z = d * depth_scale, x = z * ((col + 0.5 - cx) / fx),
// y = z * ((row + 0.5 - cy) / fy), then each row of T (4x4 row major) dotted with (x, y, z, 1) left to right.
// Returns the no-depth flag, z == 0 after the scale (bev_utils.py:371).
__device__ __forceinline__ bool camera_to_world(float d, int row, int col, float depth_scale, float fx, float fy,
                                                float cx, float cy, const float* T, float w[3]) {
  const float z = __fmul_rn(d, depth_scale);  // depths * 10   (pretrain_cmt.py:125, ss_trainer_BEV.py:402)
  const float xs = __fdiv_rn(__fsub_rn(__fadd_rn((float)col, 0.5f), cx), fx);  // bev_utils.py:130
  const float ys = __fdiv_rn(__fsub_rn(__fadd_rn((float)row, 0.5f), cy), fy);  // bev_utils.py:131
  const float x = __fmul_rn(z, xs);
  const float y = __fmul_rn(z, ys);
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    float acc = __fmul_rn(T[j * 4 + 0], x);
    acc = __fadd_rn(acc, __fmul_rn(T[j * 4 + 1], y));
    acc = __fadd_rn(acc, __fmul_rn(T[j * 4 + 2], z));
    acc = __fadd_rn(acc, T[j * 4 + 3]);
    w[j] = acc;
  }
  return z == 0.0f;
}

// One thread per point.
__global__ void lift_index_kernel(const float* __restrict__ depths, const float* __restrict__ T_c2w,
                                  const float* __restrict__ S_w2c, const float* __restrict__ T_w2c, int B, int V, int Hf,
                                  int Wf, float depth_scale, float fx, float fy, float cx, float cy, int D, float res,
                                  float half, float y_clip, int32_t* __restrict__ cell_idx, float* __restrict__ pc_out) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const int P = V * Hf * Wf;
  const long long gid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (gid >= (long long)B * P) return;
  const int b = gid / P;
  const int pidx = gid % P;
  const int v = pidx / (Hf * Wf);
  const int pix = pidx % (Hf * Wf);
  const int row = pix / Wf, col = pix % Wf;

  float w[3];
  const bool no_depth = camera_to_world(depths[gid], row, col, depth_scale, fx, fy, cx, cy,
                                        T_c2w + ((long long)b * V + v) * 16, w);
  float e[3];
  ego_transform(w[0], w[1], w[2], S_w2c + (long long)b * 3, T_w2c + (long long)b * 16, e);
  if (pc_out) {
    pc_out[gid * 3 + 0] = e[0];
    pc_out[gid * 3 + 1] = e[1];
    pc_out[gid * 3 + 2] = e[2];
  }
  cell_idx[gid] = bev_cell(e[0], e[1], e[2], no_depth, D, res, half, y_clip);
}

// World points and no-depth mask of N depth views (PointCloud.forward, bev_utils.py:349-378, as the VLN-CE trainer's
// `lift` calls it, ss_trainer_BEV.py:386-410): one thread per point, world point minus world_shift (3 floats).
// The block's points are staged in shared memory so that the (n, 3) rows leave as consecutive floats.
constexpr int LP_THREADS = 256;

__global__ void __launch_bounds__(LP_THREADS)
lift_points_kernel(const float* __restrict__ depths, const float* __restrict__ T_c2w, long long n, int HW, int Wf,
                   float depth_scale, float fx, float fy, float cx, float cy, const float* __restrict__ world_shift,
                   float* __restrict__ pts, uint8_t* __restrict__ no_depth) {
  __shared__ float spts[LP_THREADS * 3];
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long base = (long long)blockIdx.x * LP_THREADS;
  const long long gid = base + threadIdx.x;
  if (gid < n) {
    const long long view = gid / HW;
    const int pix = (int)(gid - view * HW);
    float w[3];
    no_depth[gid] = camera_to_world(__ldg(depths + gid), pix / Wf, pix % Wf, depth_scale, fx, fy, cx, cy,
                                    T_c2w + view * 16, w);
#pragma unroll
    for (int j = 0; j < 3; ++j) spts[threadIdx.x * 3 + j] = __fsub_rn(w[j], __ldg(world_shift + j));  // :243
  }
  __syncthreads();
  const long long nf = (n - base) * 3;  // floats this block owns
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int i = k * LP_THREADS + threadIdx.x;
    if (i < nf) pts[base * 3 + i] = spts[i];
  }
}

// Cell index of an ego-frame point cloud (PointCloud.project_bev called with a ready-made cloud: the agents gather
// the clouds of neighbouring panoramas first, map_nav_src/r2r/agent.py:115-192): same discretisation as above.
__global__ void cell_index_kernel(const float* __restrict__ pc, const uint8_t* __restrict__ no_depth, long long n, int D,
                                  float res, float half, float y_clip, int32_t* __restrict__ cell_idx) {
  bb::pdl_wait();
  bb::pdl_trigger();
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= n) return;
  cell_idx[gid] = bev_cell(pc[gid * 3 + 0], pc[gid * 3 + 1], pc[gid * 3 + 2], no_depth && no_depth[gid], D, res, half,
                           y_clip);
}

// ---------------------------------------------------------------------------------------------
// Scatter-mean: block = 8 warps = 8 cells of one sample; the sample's cell indices are staged once in
// shared memory; each warp scans them 32 at a time (ballot) and accumulates matching rows in
// ascending point order -> deterministic, equals a sequential index_add_.
// ---------------------------------------------------------------------------------------------
constexpr int SC_WARPS = 8;
constexpr int SC_MAXV = 6;  // float4 per lane per pass -> 768 columns per pass

// 4 consecutive features of a point row: fp32 (the reference's collate dtype) or bf16 (16-bit wire format: the grid
// features are stored as 16-bit floats on disk and used as bf16 GEMM operands right after the pooling anyway)
__device__ __forceinline__ float4 load_feat4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 load_feat4(const __nv_bfloat16* p) {
  const uint2 raw = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.x));
  const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.y));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}

template <typename FT>
__global__ void __launch_bounds__(SC_WARPS * 32)
scatter_mean_f32_kernel(const FT* __restrict__ feats, const int32_t* __restrict__ cell_idx, int P, int C, int ncell,
                        float* __restrict__ bev_f32, __nv_bfloat16* __restrict__ bev_bf16,
                        uint8_t* __restrict__ ob_mask, int32_t* __restrict__ counts) {
  bb::pdl_wait();
  bb::pdl_trigger();
  extern __shared__ int32_t sidx[];
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int32_t* idx = cell_idx + (long long)b * P;
  for (int i = threadIdx.x; i < P; i += blockDim.x) sidx[i] = idx[i];
  __syncthreads();
  const int cell = blockIdx.x * SC_WARPS + warp;
  if (cell >= ncell) return;
  const FT* fb = feats + (long long)b * P * C;
  const long long orow = ((long long)b * ncell + cell) * C;

  float vmax = -INFINITY, vmin = INFINITY;
  int cnt = 0;
  for (int c0 = 0; c0 < C; c0 += SC_MAXV * 128) {
    float4 acc[SC_MAXV];
#pragma unroll
    for (int i = 0; i < SC_MAXV; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    cnt = 0;
    for (int base = 0; base < P; base += 32) {
      const int my = (base + lane < P) ? sidx[base + lane] : -1;
      unsigned m = __ballot_sync(0xffffffffu, my == cell);
      while (m) {
        const int j = __ffs(m) - 1;
        m &= m - 1;
        const FT* rowp = fb + (long long)(base + j) * C + c0;
        float4 t[SC_MAXV];
#pragma unroll
        for (int i = 0; i < SC_MAXV; ++i) {
          const int col = i * 128 + lane * 4;
          t[i] = (c0 + col < C) ? load_feat4(rowp + col) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int i = 0; i < SC_MAXV; ++i) {
          acc[i].x = __fadd_rn(acc[i].x, t[i].x);
          acc[i].y = __fadd_rn(acc[i].y, t[i].y);
          acc[i].z = __fadd_rn(acc[i].z, t[i].z);
          acc[i].w = __fadd_rn(acc[i].w, t[i].w);
        }
        ++cnt;
      }
    }
    const float denom = (float)(cnt < 1 ? 1 : cnt);  // count.clamp(min=1)
#pragma unroll
    for (int i = 0; i < SC_MAXV; ++i) {
      const int col = c0 + i * 128 + lane * 4;
      if (col < C) {
        float4 mval;
        mval.x = __fdiv_rn(acc[i].x, denom);
        mval.y = __fdiv_rn(acc[i].y, denom);
        mval.z = __fdiv_rn(acc[i].z, denom);
        mval.w = __fdiv_rn(acc[i].w, denom);
        vmax = fmaxf(vmax, fmaxf(fmaxf(mval.x, mval.y), fmaxf(mval.z, mval.w)));
        vmin = fminf(vmin, fminf(fminf(mval.x, mval.y), fminf(mval.z, mval.w)));
        if (bev_f32) *reinterpret_cast<float4*>(bev_f32 + orow + col) = mval;
        if (bev_bf16) {
          __nv_bfloat162 lo = __floats2bfloat162_rn(mval.x, mval.y), hi = __floats2bfloat162_rn(mval.z, mval.w);
          uint2 pk;
          pk.x = *reinterpret_cast<uint32_t*>(&lo);
          pk.y = *reinterpret_cast<uint32_t*>(&hi);
          *reinterpret_cast<uint2*>(bev_bf16 + orow + col) = pk;
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
  }
  if (lane == 0) {
    if (ob_mask) ob_mask[(long long)b * ncell + cell] = !((vmax == 0.0f) && (vmin == 0.0f));
    if (counts) counts[(long long)b * ncell + cell] = cnt;
  }
}

// float64 semantic labels: S <= 64 classes, lane l owns classes l and l+32.
__global__ void __launch_bounds__(SC_WARPS * 32)
scatter_sem_f64_kernel(const double* __restrict__ sems, const int32_t* __restrict__ cell_idx, int P, int S, int ncell,
                       double* __restrict__ bev_sem, uint8_t* __restrict__ sem_mask) {
  bb::pdl_wait();
  bb::pdl_trigger();
  extern __shared__ int32_t sidx[];
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int32_t* idx = cell_idx + (long long)b * P;
  for (int i = threadIdx.x; i < P; i += blockDim.x) sidx[i] = idx[i];
  __syncthreads();
  const int cell = blockIdx.x * SC_WARPS + warp;
  if (cell >= ncell) return;
  const double* sb = sems + (long long)b * P * S;
  double a0 = 0.0, a1 = 0.0;
  int cnt = 0;
  for (int base = 0; base < P; base += 32) {
    const int my = (base + lane < P) ? sidx[base + lane] : -1;
    unsigned m = __ballot_sync(0xffffffffu, my == cell);
    while (m) {
      const int j = __ffs(m) - 1;
      m &= m - 1;
      const double* rowp = sb + (long long)(base + j) * S;
      if (lane < S) a0 = __dadd_rn(a0, rowp[lane]);
      if (lane + 32 < S) a1 = __dadd_rn(a1, rowp[lane + 32]);
      ++cnt;
    }
  }
  const double denom = (double)(cnt < 1 ? 1 : cnt);
  double m0 = __ddiv_rn(a0, denom), m1 = __ddiv_rn(a1, denom);
  m0 = m0 > 0.0 ? 1.0 : m0;  // sem[sem>0] = 1 (bev_utils.py:422)
  m1 = m1 > 0.0 ? 1.0 : m1;
  const long long orow = ((long long)b * ncell + cell) * S;
  if (lane < S) bev_sem[orow + lane] = m0;
  if (lane + 32 < S) bev_sem[orow + lane + 32] = m1;
  double tot = (lane < S ? m0 : 0.0) + (lane + 32 < S ? m1 : 0.0);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
  if (lane == 0 && sem_mask) sem_mask[(long long)b * ncell + cell] = tot > 0.0;
}

// ---------------------------------------------------------------------------------------------
// Agent-side BEV straight from the node point clouds (map_nav_src/r2r/agent.py:293-337: gather_node_pc -> pad_sequence
// -> splat -> project_bev). Block = 8 warps = 8 cells of one sample, as in scatter_mean_f32_kernel. The block walks
// the sample's nodes in table order and, inside them, the points in row order, SN_CHUNK at a time: all threads
// ego-transform and discretise a chunk into shared memory (cell index + feature row pointer per point), then each warp
// ballot-scans the chunk for its cell and adds the matching rows. The sums and counts stay in registers across chunks
// and nodes, so the points of a cell are added in ascending order of the concatenated cloud, with no limit on the
// number of points. Columns beyond SC_MAXV * 128 take further passes over the whole walk.
// ---------------------------------------------------------------------------------------------
constexpr int SN_CHUNK = 2048;

template <typename FT>
__global__ void __launch_bounds__(SC_WARPS * 32)
splat_nodes_kernel(const bb_bev_node* __restrict__ nodes, const int32_t* __restrict__ sample_nodes,
                   const float* __restrict__ S_w2c, const float* __restrict__ T_w2c, int C, int D, float res, float half,
                   float y_clip, float* __restrict__ bev, uint8_t* __restrict__ ob_mask) {
  __shared__ int32_t scell[SN_CHUNK];
  __shared__ const FT* srow[SN_CHUNK];
  bb::pdl_wait();
  bb::pdl_trigger();
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ncell = D * D;
  const int cell = blockIdx.x * SC_WARPS + warp;  // a warp past the last cell still stages points
  const int k0 = sample_nodes[b], k1 = sample_nodes[b + 1];
  float S[3], E[12];
#pragma unroll
  for (int i = 0; i < 3; ++i) S[i] = __ldg(S_w2c + b * 3 + i);
#pragma unroll
  for (int i = 0; i < 12; ++i) E[i] = __ldg(T_w2c + b * 16 + i);
  const long long orow = ((long long)b * ncell + cell) * C;

  float vmax = -INFINITY, vmin = INFINITY;
  for (int c0 = 0; c0 < C; c0 += SC_MAXV * 128) {
    float4 acc[SC_MAXV];
#pragma unroll
    for (int i = 0; i < SC_MAXV; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    int cnt = 0;
    int k = k0;
    long long r = 0;  // next row of node k
    while (k < k1) {
      int filled = 0;
      while (k < k1 && filled < SN_CHUNK) {  // block-uniform: every thread walks the same cursor
        const long long n = nodes[k].n;
        const int take = (int)min(n - r, (long long)(SN_CHUNK - filled));
        if (take > 0) {
          const float* pc = nodes[k].pc;
          const uint8_t* nod = nodes[k].no_depth;
          const FT* ft = reinterpret_cast<const FT*>(nodes[k].feat);
          for (int i = threadIdx.x; i < take; i += blockDim.x) {
            const long long row = r + i;
            float e[3];
            ego_transform(pc[row * 3 + 0], pc[row * 3 + 1], pc[row * 3 + 2], S, E, e);
            scell[filled + i] = bev_cell(e[0], e[1], e[2], nod && nod[row], D, res, half, y_clip);
            srow[filled + i] = ft + row * C;
          }
          filled += take;
          r += take;
        }
        if (r >= n) {
          ++k;
          r = 0;
        }
      }
      __syncthreads();
      if (cell < ncell) {
        for (int base = 0; base < filled; base += 32) {
          const int my = (base + lane < filled) ? scell[base + lane] : -1;
          unsigned m = __ballot_sync(0xffffffffu, my == cell);
          while (m) {
            const int j = __ffs(m) - 1;
            m &= m - 1;
            const FT* rowp = srow[base + j] + c0;
            float4 t[SC_MAXV];
#pragma unroll
            for (int i = 0; i < SC_MAXV; ++i) {
              const int col = i * 128 + lane * 4;
              t[i] = (c0 + col < C) ? load_feat4(rowp + col) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int i = 0; i < SC_MAXV; ++i) {
              acc[i].x = __fadd_rn(acc[i].x, t[i].x);
              acc[i].y = __fadd_rn(acc[i].y, t[i].y);
              acc[i].z = __fadd_rn(acc[i].z, t[i].z);
              acc[i].w = __fadd_rn(acc[i].w, t[i].w);
            }
            ++cnt;
          }
        }
      }
      __syncthreads();  // the next chunk overwrites the staging arrays
    }
    if (cell < ncell) {
      const float denom = (float)(cnt < 1 ? 1 : cnt);  // count.clamp(min=1)
#pragma unroll
      for (int i = 0; i < SC_MAXV; ++i) {
        const int col = c0 + i * 128 + lane * 4;
        if (col < C) {
          float4 mval;
          mval.x = __fdiv_rn(acc[i].x, denom);
          mval.y = __fdiv_rn(acc[i].y, denom);
          mval.z = __fdiv_rn(acc[i].z, denom);
          mval.w = __fdiv_rn(acc[i].w, denom);
          vmax = fmaxf(vmax, fmaxf(fmaxf(mval.x, mval.y), fmaxf(mval.z, mval.w)));
          vmin = fminf(vmin, fminf(fminf(mval.x, mval.y), fminf(mval.z, mval.w)));
          *reinterpret_cast<float4*>(bev + orow + col) = mval;
        }
      }
    }
  }
  if (cell >= ncell) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
  }
  if (lane == 0) ob_mask[(long long)b * ncell + cell] = !((vmax == 0.0f) && (vmin == 0.0f));
}

}  // namespace bb

extern "C" int bb_bev_lift_index(const float* depths, const float* T_c2w, const float* S_w2c, const float* T_w2c, int B,
                                 int V, int Hf, int Wf, float depth_scale, float fx, float fy, float cx, float cy,
                                 int map_dim, float map_res, float y_clip, int32_t* cell_idx, float* pc_out,
                                 void* stream) {
  using namespace bb;
  if (!depths || !T_c2w || !S_w2c || !T_w2c || !cell_idx) return set_error("bb_bev_lift_index: null argument");
  if (B <= 0) return 0;
  const long long n = (long long)B * V * Hf * Wf;
  const float half = (float)((map_dim - 1) / 2.0);  // (map_dim-1)/2 as in bev_utils.py:393
  bb::launch_pdl(lift_index_kernel, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, 
      depths, T_c2w, S_w2c, T_w2c, B, V, Hf, Wf, depth_scale, fx, fy, cx, cy, map_dim, map_res, half, y_clip, cell_idx,
      pc_out);
  count_launch();
  return check_launch("lift_index_kernel");
}

extern "C" int bb_bev_lift_points(const float* depths, const float* T_c2w, int N, int Hf, int Wf, float depth_scale,
                                  float fx, float fy, float cx, float cy, const float* world_shift, float* pts,
                                  uint8_t* no_depth, void* stream) {
  using namespace bb;
  if (!depths || !T_c2w || !world_shift || !pts || !no_depth) return set_error("bb_bev_lift_points: null argument");
  if (((uintptr_t)depths | (uintptr_t)T_c2w | (uintptr_t)world_shift | (uintptr_t)pts) % 4 != 0)
    return set_error("bb_bev_lift_points: float arguments must be 4-byte aligned");
  if (N <= 0) return set_error("bb_bev_lift_points: N must be > 0");
  if (Hf <= 0 || Wf <= 0 || (long long)Hf * Wf > INT32_MAX)
    return set_error("bb_bev_lift_points: Hf * Wf must be positive and fit in 32 bits");
  const long long n = (long long)N * Hf * Wf;
  const long long blocks = (n + LP_THREADS - 1) / LP_THREADS;
  if (blocks > INT32_MAX) return set_error("bb_bev_lift_points: too many points for one launch");
  bb::launch_pdl(lift_points_kernel, (unsigned)blocks, LP_THREADS, 0, (cudaStream_t)stream, depths, T_c2w, n, Hf * Wf,
                 Wf, depth_scale, fx, fy, cx, cy, world_shift, pts, no_depth);
  count_launch();
  return check_launch("lift_points_kernel");
}

extern "C" int bb_bev_cell_index(const float* pc, const uint8_t* no_depth, int64_t npoints, int map_dim, float map_res,
                                 float y_clip, int32_t* cell_idx, void* stream) {
  using namespace bb;
  if (!pc || !cell_idx) return set_error("bb_bev_cell_index: null argument");
  if (npoints <= 0) return 0;
  const float half = (float)((map_dim - 1) / 2.0);
  bb::launch_pdl(cell_index_kernel, (unsigned)((npoints + 255) / 256), 256, 0, (cudaStream_t)stream, pc, no_depth,
                 (long long)npoints, map_dim, map_res, half, y_clip, cell_idx);
  count_launch();
  return check_launch("cell_index_kernel");
}

template <typename FT>
static int scatter_mean_launch(const FT* feats, const int32_t* cell_idx, int B, int P, int C, int ncell, float* bev_f32,
                               void* bev_bf16, uint8_t* ob_mask, int32_t* counts, void* stream) {
  using namespace bb;
  if (!feats || !cell_idx) return set_error("bb_bev_scatter_mean: null argument");
  if (C % 4 != 0) return set_error("bb_bev_scatter_mean: C must be a multiple of 4");
  if ((size_t)P * 4 > 200 * 1024) return set_error("bb_bev_scatter_mean: too many points per sample for smem");
  if (B <= 0) return 0;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(scatter_mean_f32_kernel<FT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    attr_set = true;
  }
  dim3 grid((ncell + SC_WARPS - 1) / SC_WARPS, B);
  bb::launch_pdl(scatter_mean_f32_kernel<FT>, grid, SC_WARPS * 32, (size_t)P * 4, (cudaStream_t)stream,
      feats, cell_idx, P, C, ncell, bev_f32, reinterpret_cast<__nv_bfloat16*>(bev_bf16), ob_mask, counts);
  count_launch();
  return check_launch("scatter_mean_f32_kernel");
}

extern "C" int bb_bev_scatter_mean_f32(const float* feats, const int32_t* cell_idx, int B, int P, int C, int ncell,
                                       float* bev_f32, void* bev_bf16, uint8_t* ob_mask, int32_t* counts,
                                       void* stream) {
  return scatter_mean_launch(feats, cell_idx, B, P, C, ncell, bev_f32, bev_bf16, ob_mask, counts, stream);
}
extern "C" int bb_bev_scatter_mean_bf16(const void* feats, const int32_t* cell_idx, int B, int P, int C, int ncell,
                                        float* bev_f32, void* bev_bf16, uint8_t* ob_mask, int32_t* counts,
                                        void* stream) {
  return scatter_mean_launch(reinterpret_cast<const __nv_bfloat16*>(feats), cell_idx, B, P, C, ncell, bev_f32, bev_bf16,
                             ob_mask, counts, stream);
}

// Semantic labels as stored on disk: one uint8 class id per point (the reference expands them to float64 one-hots on
// the host, pretrain_src/data/dataset.py:117,402, and ships 24 MB per 32-sample batch across PCIe).  The pooled label
// map is binary (mean of one-hots, then sem[sem > 0] = 1, bev_utils.py:417-423): class c is set in a cell iff at least
// one kept point of class c falls into it -- one 64-bit presence mask per cell, built with shared-memory atomicOr.
__global__ void __launch_bounds__(256)
scatter_sem_u8_kernel(const uint8_t* __restrict__ sem_ids, const int32_t* __restrict__ cell_idx, int P, int S, int ncell,
                      double* __restrict__ bev_sem, uint8_t* __restrict__ sem_mask) {
  bb::pdl_wait();
  bb::pdl_trigger();
  extern __shared__ unsigned long long bits[];
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < ncell; i += blockDim.x) bits[i] = 0ull;
  __syncthreads();
  const uint8_t* ids = sem_ids + (long long)b * P;
  const int32_t* idx = cell_idx + (long long)b * P;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const int c = idx[i];
    const int k = ids[i];
    if (c >= 0 && c < ncell && k < S) atomicOr(&bits[c], 1ull << k);
  }
  __syncthreads();
  double* out = bev_sem + (long long)b * ncell * S;
  for (int i = threadIdx.x; i < ncell * S; i += blockDim.x) {
    const int cell = i / S, k = i - cell * S;
    out[i] = (bits[cell] >> k) & 1ull ? 1.0 : 0.0;
  }
  if (sem_mask)
    for (int i = threadIdx.x; i < ncell; i += blockDim.x) sem_mask[(long long)b * ncell + i] = bits[i] != 0ull;
}

extern "C" int bb_bev_scatter_sem_u8(const uint8_t* sem_ids, const int32_t* cell_idx, int B, int P, int S, int ncell,
                                     double* bev_sem, uint8_t* sem_mask, void* stream) {
  using namespace bb;
  if (!sem_ids || !cell_idx || !bev_sem) return set_error("bb_bev_scatter_sem_u8: null argument");
  if (S > 64) return set_error("bb_bev_scatter_sem_u8: at most 64 classes");
  if ((size_t)ncell * 8 > 48 * 1024) return set_error("bb_bev_scatter_sem_u8: too many cells for shared memory");
  if (B <= 0) return 0;
  bb::launch_pdl(scatter_sem_u8_kernel, (unsigned)B, 256, (size_t)ncell * 8, (cudaStream_t)stream, sem_ids, cell_idx, P, S,
                 ncell, bev_sem, sem_mask);
  count_launch();
  return check_launch("scatter_sem_u8_kernel");
}

extern "C" int bb_bev_scatter_sem_f64(const double* sems, const int32_t* cell_idx, int B, int P, int S, int ncell,
                                      double* bev_sem, uint8_t* sem_mask, void* stream) {
  using namespace bb;
  if (!sems || !cell_idx || !bev_sem) return set_error("bb_bev_scatter_sem_f64: null argument");
  if (S > 64) return set_error("bb_bev_scatter_sem_f64: at most 64 classes");
  if ((size_t)P * 4 > 200 * 1024) return set_error("bb_bev_scatter_sem_f64: too many points per sample for smem");
  if (B <= 0) return 0;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(scatter_sem_f64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    attr_set = true;
  }
  dim3 grid((ncell + SC_WARPS - 1) / SC_WARPS, B);
  bb::launch_pdl(scatter_sem_f64_kernel, grid, SC_WARPS * 32, (size_t)P * 4, (cudaStream_t)stream, sems, cell_idx, P, S, ncell,
                                                                                    bev_sem, sem_mask);
  count_launch();
  return check_launch("scatter_sem_f64_kernel");
}

extern "C" int bb_bev_splat_nodes(const bb_bev_node* nodes, int n_nodes, const int32_t* sample_nodes, int B,
                                  void* table_dev, const float* S_w2c, const float* T_w2c, int C, int feat_bf16,
                                  int map_dim, float map_res, float y_clip, float* bev, uint8_t* ob_mask, void* stream) {
  using namespace bb;
  if (B < 0 || n_nodes < 0) return set_error("bb_bev_splat_nodes: B and n_nodes must be >= 0");
  if (B > 65535) return set_error("bb_bev_splat_nodes: at most 65535 samples per call");
  if (!sample_nodes || !table_dev || !S_w2c || !T_w2c || !bev || !ob_mask || (n_nodes > 0 && !nodes))
    return set_error("bb_bev_splat_nodes: null argument");
  if (C <= 0 || C % 4 != 0) return set_error("bb_bev_splat_nodes: C must be a positive multiple of 4");
  if (map_dim <= 0 || map_dim > 46340) return set_error("bb_bev_splat_nodes: map_dim out of range");
  if ((uintptr_t)table_dev % 8 != 0) return set_error("bb_bev_splat_nodes: table_dev must be 8-byte aligned");
  if (sample_nodes[0] < 0 || sample_nodes[B] > n_nodes)
    return set_error("bb_bev_splat_nodes: sample_nodes must lie in [0, n_nodes]");
  for (int b = 0; b < B; ++b)
    if (sample_nodes[b + 1] < sample_nodes[b]) return set_error("bb_bev_splat_nodes: sample_nodes must be non-decreasing");
  const uintptr_t feat_align = feat_bf16 ? 8 : 16;  // 4 features per load: one 8- or 16-byte access
  for (int i = 0; i < n_nodes; ++i) {
    const bb_bev_node& nd = nodes[i];
    if (nd.n < 0) return set_error("bb_bev_splat_nodes: negative node size");
    if (nd.n == 0) continue;
    if (!nd.pc || !nd.feat) return set_error("bb_bev_splat_nodes: null point or feature pointer in a node");
    if ((uintptr_t)nd.pc % 4 != 0) return set_error("bb_bev_splat_nodes: misaligned point rows");
    if ((uintptr_t)nd.feat % feat_align != 0) return set_error("bb_bev_splat_nodes: misaligned feature rows");
  }
  if (B == 0) return 0;
  const cudaStream_t st = (cudaStream_t)stream;
  char* tab = static_cast<char*>(table_dev);
  const size_t rows_bytes = (size_t)n_nodes * sizeof(bb_bev_node);
  if (rows_bytes && cudaMemcpyAsync(tab, nodes, rows_bytes, cudaMemcpyHostToDevice, st) != cudaSuccess)
    return check_launch("bb_bev_splat_nodes: table copy");
  if (cudaMemcpyAsync(tab + rows_bytes, sample_nodes, (size_t)(B + 1) * 4, cudaMemcpyHostToDevice, st) != cudaSuccess)
    return check_launch("bb_bev_splat_nodes: offsets copy");
  const int ncell = map_dim * map_dim;
  const float half = (float)((map_dim - 1) / 2.0);
  dim3 grid((ncell + SC_WARPS - 1) / SC_WARPS, B);
  const bb_bev_node* dnodes = reinterpret_cast<const bb_bev_node*>(tab);
  const int32_t* doffs = reinterpret_cast<const int32_t*>(tab + rows_bytes);
  if (feat_bf16)
    bb::launch_pdl(splat_nodes_kernel<__nv_bfloat16>, grid, SC_WARPS * 32, 0, st, dnodes, doffs, S_w2c, T_w2c, C,
                   map_dim, map_res, half, y_clip, bev, ob_mask);
  else
    bb::launch_pdl(splat_nodes_kernel<float>, grid, SC_WARPS * 32, 0, st, dnodes, doffs, S_w2c, T_w2c, C, map_dim,
                   map_res, half, y_clip, bev, ob_mask);
  count_launch();
  return check_launch("splat_nodes_kernel");
}
