// The VLN-CE trainer's global-map image input (ss_trainer_BEV.py rollout lines 1032-1033 and 1060-1066,
// GraphMap.update_graph / get_node_embeds in models/graph_utils.py:198-281, and _nav_gmap_variable's stack and
// pad_tensors_wgrad, ss_trainer_BEV.py:534-611) from the episode's stored `panorama` outputs, one launch per
// `navigation` call, and its gradient with respect to every stored step, one launch per backward.  Both read an int32
// table staged by one host-to-device copy; nothing synchronises with the host and nothing adds with atomics.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bevbert_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace bb {
namespace {
constexpr int GMAP_THREADS = 192;   // one float4 column group per thread for H = 768

struct StepRec {
  const float* pano;                // forward: pano_embeds (Bs, Vs, H); backward: its gradient (written)
  const int64_t* nav;               // nav_types (Bs, Vs)
  const uint8_t* mask;              // pano_masks (Bs, Vs)
  int Bs, Vs;
};

__device__ __forceinline__ StepRec step_rec(const int32_t* t, int s) {
  const int32_t* r = t + s * BB_CE_GMAP_STEP_WORDS;
  auto ptr = [&](int w) { return (uintptr_t)(uint32_t)r[w] | ((uintptr_t)(uint32_t)r[w + 1] << 32); };
  return StepRec{(const float*)ptr(0), (const int64_t*)ptr(2), (const uint8_t*)ptr(4), r[6], r[7]};
}

// view index of the k-th entry with nav_types == 1 in one row (the order of the boolean index), -1 if there is none
__device__ __forceinline__ int cand_view(const int64_t* nav, int V, int k) {
  for (int v = 0; v < V; ++v)
    if (nav[v] == 1 && k-- == 0) return v;
  return -1;
}

__device__ __forceinline__ float4 f4(float x) { return make_float4(x, x, x, x); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) {
  return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}
__device__ __forceinline__ float4 mul4(float4 a, float b) {
  return make_float4(__fmul_rn(a.x, b), __fmul_rn(a.y, b), __fmul_rn(a.z, b), __fmul_rn(a.w, b));
}
__device__ __forceinline__ float4 div4(float4 a, float b) {
  return make_float4(__fdiv_rn(a.x, b), __fdiv_rn(a.y, b), __fdiv_rn(a.z, b), __fdiv_rn(a.w, b));
}

// One CTA per output row (blockIdx.x = r < G, blockIdx.y = b), each thread a float4 column group.
__global__ void __launch_bounds__(GMAP_THREADS) ce_gmap_features_kernel(const int32_t* __restrict__ table, int S,
                                                                        int G, int H, float* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const int r = blockIdx.x, b = blockIdx.y;
  const int32_t* rows = table + S * BB_CE_GMAP_STEP_WORDS;
  const int32_t* terms = rows + gridDim.y * G * 3;
  const int32_t* row = rows + (b * G + r) * 3;
  const int kind = row[0];
  float4* o = reinterpret_cast<float4*>(out + ((long long)b * G + r) * H);
  const int h4 = H / 4;
  if (kind == 1) {
    // node: torch's CUDA sum(pano * mask, 1) for fewer than 64 views (one thread per output, four accumulators from
    // +0 taking views v = j mod 4 in ascending order, then ((a0 + a1) + a2) + a3), over the true count sum(mask)
    const StepRec st = step_rec(table, row[1]);
    const int i = row[2];
    const float* p = st.pano + (long long)i * st.Vs * H;
    const uint8_t* m = st.mask + (long long)i * st.Vs;
    int cnt = 0;
    for (int v = 0; v < st.Vs; ++v) cnt += m[v] != 0;
    for (int c = threadIdx.x; c < h4; c += GMAP_THREADS) {
      float4 acc[4] = {f4(0.f), f4(0.f), f4(0.f), f4(0.f)};
      for (int v0 = 0; v0 < st.Vs; v0 += 4) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int v = v0 + j;
          if (v < st.Vs)
            acc[j] = add4(acc[j], mul4(reinterpret_cast<const float4*>(p + (long long)v * H)[c], m[v] ? 1.f : 0.f));
        }
      }
      o[c] = div4(add4(add4(add4(acc[0], acc[1]), acc[2]), acc[3]), (float)cnt);
    }
  } else if (kind == 2) {
    // ghost: ((e1 + e2) + e3) ... in merge order, times the fp32 reciprocal of the count (torch's CUDA division of a
    // tensor by a Python number).  A term whose candidate the row's nav_types does not hold gives NaN.
    const int32_t* tm = terms + row[1] * 3;
    const int n = row[2];
    const float inv = __fdiv_rn(1.f, (float)n);
    for (int c = threadIdx.x; c < h4; c += GMAP_THREADS) {
      float4 acc = f4(0.f);
      for (int j = 0; j < n; ++j) {
        const StepRec st = step_rec(table, tm[3 * j]);
        const int i = tm[3 * j + 1];
        const int v = cand_view(st.nav + (long long)i * st.Vs, st.Vs, tm[3 * j + 2]);
        const float4 x = v < 0 ? f4(__int_as_float(0x7fc00000))
                               : reinterpret_cast<const float4*>(st.pano + ((long long)i * st.Vs + v) * H)[c];
        acc = j == 0 ? x : add4(acc, x);
      }
      o[c] = mul4(acc, inv);
    }
  } else {
    for (int c = threadIdx.x; c < h4; c += GMAP_THREADS) o[c] = f4(0.f);
  }
}

// One CTA per stored row (blockIdx.x = view v, blockIdx.y = record (s, i)): d pano[s][i][v] = node part + ghost part,
// each present or not: node part dout[nb, nr] / sum(mask) where mask[v] (DivBackward with a tensor divisor, then
// MulBackward by the mask), ghost part dout[gb, gr] * fp32(1 / count) when v is the k-th candidate and k merged into
// that ghost (DivBackward with a Python-number divisor).  A row with neither part is +0.
__global__ void __launch_bounds__(GMAP_THREADS) ce_gmap_features_bwd_kernel(const int32_t* __restrict__ table, int S,
                                                                            int G, int H,
                                                                            const float* __restrict__ dout) {
  pdl_wait();
  pdl_trigger();
  const int v = blockIdx.x;
  const int32_t* rec = table + S * BB_CE_GMAP_STEP_WORDS + blockIdx.y * 6;
  const StepRec st = step_rec(table, rec[0]);
  if (v >= st.Vs) return;
  const int i = rec[1], nb = rec[2], nr = rec[3], ncand = rec[5];
  const int32_t* cands = table + S * BB_CE_GMAP_STEP_WORDS + gridDim.y * 6 + rec[4] * 3;
  const uint8_t* m = st.mask + (long long)i * st.Vs;
  const int64_t* nav = st.nav + (long long)i * st.Vs;
  int cnt = 0;
  for (int u = 0; u < st.Vs; ++u) cnt += m[u] != 0;
  int k = -1;
  if (nav[v] == 1) {
    k = 0;
    for (int u = 0; u < v; ++u) k += nav[u] == 1;
  }
  const bool node = nb >= 0 && m[v];
  const int32_t* cd = k >= 0 && k < ncand ? cands + k * 3 : nullptr;
  const bool ghost = cd && cd[0] >= 0;
  const float inv = ghost ? __fdiv_rn(1.f, (float)cd[2]) : 0.f;
  const float4* gn = node ? reinterpret_cast<const float4*>(dout + ((long long)nb * G + nr) * H) : nullptr;
  const float4* gg = ghost ? reinterpret_cast<const float4*>(dout + ((long long)cd[0] * G + cd[1]) * H) : nullptr;
  float4* o = reinterpret_cast<float4*>(const_cast<float*>(st.pano) + ((long long)i * st.Vs + v) * H);
  for (int c = threadIdx.x; c < H / 4; c += GMAP_THREADS) {
    float4 x = f4(0.f);
    if (node) x = div4(gn[c], (float)cnt);
    if (ghost) x = node ? add4(x, mul4(gg[c], inv)) : mul4(gg[c], inv);
    o[c] = x;
  }
}
}  // namespace
}  // namespace bb

using namespace bb;

extern "C" int bb_ce_gmap_features(const int32_t* table, int S, int B, int G, int H, float* out, void* stream) {
  if (!table || !out || S < 0 || B <= 0 || G <= 0 || B > 65535) return set_error("bb_ce_gmap_features: bad arguments");
  if (H <= 0 || H % 4 || (reinterpret_cast<uintptr_t>(out) & 15))
    return set_error("bb_ce_gmap_features: H must be a positive multiple of 4 and out 16-byte aligned");
  launch_pdl(ce_gmap_features_kernel, dim3((unsigned)G, (unsigned)B), dim3(GMAP_THREADS), 0, (cudaStream_t)stream,
             table, S, G, H, out);
  count_launch();
  return check_launch("ce_gmap_features_kernel");
}

extern "C" int bb_ce_gmap_features_bwd(const int32_t* table, int S, int R, int Vmax, int G, int H, const float* dout,
                                       void* stream) {
  if (R == 0) return 0;
  if (!table || !dout || S <= 0 || R < 0 || R > 65535 || Vmax <= 0 || G <= 0)
    return set_error("bb_ce_gmap_features_bwd: bad arguments");
  if (H <= 0 || H % 4 || (reinterpret_cast<uintptr_t>(dout) & 15))
    return set_error("bb_ce_gmap_features_bwd: H must be a positive multiple of 4 and dout 16-byte aligned");
  launch_pdl(ce_gmap_features_bwd_kernel, dim3((unsigned)Vmax, (unsigned)R), dim3(GMAP_THREADS), 0,
             (cudaStream_t)stream, table, S, G, H, dout);
  count_launch();
  return check_launch("ce_gmap_features_bwd_kernel");
}
