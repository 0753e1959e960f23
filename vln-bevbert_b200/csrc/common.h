// Host-side helpers shared by the C-ABI translation units: thread-local error string, launch counter.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace bb {
int set_error(const char* msg);          // stores msg, returns -1
int check_launch(const char* what);      // cudaGetLastError -> 0 / -1 (+message)
void count_launch(int n = 1);
bool pdl_enabled();                      // BB_PDL env (default on)
// 4-D bf16 TMA descriptor: dims (inner, rows, b1, b2), element strides (1, ld, s1, s2), box (64, box_rows, 1, 1),
// 128-byte swizzle, zero fill out of bounds; cached per (base, geometry) (gemm_tc.cu)
int make_tmap_bf16_4d(CUtensorMap* map, const void* base, uint64_t inner, uint64_t rows, uint64_t nb1, uint64_t nb2,
                      int64_t ld, int64_t s1, int64_t s2, uint32_t box_rows);

// Deterministic mode (bb_set_deterministic): every reduction across CTAs adds in a fixed order instead of with fp32
// atomics.  Contributors store partials to a workspace with plain stores; the last-arriving CTA or a following kernel
// sums them in order.  No CTA ever waits on another.
int det_mode();                               // 0 off, 1 on, 2 on but paths without a deterministic kernel still run
inline bool det_on() { return det_mode() != 0; }
constexpr size_t DET_COUNTER_BYTES = 65536;   // split-K tile arrival counters at the start of each workspace
cudaStream_t side_stream();                   // layers.cu: the registered side stream (bb_set_side_stream) or null
// The workspace of a launch on `stream` (the side-stream buffer for the registered side stream, else the main one):
// its partial-sum area after the counters, or null with the error set when it is missing or smaller than `bytes`.
float* det_partials(cudaStream_t stream, size_t bytes, const char* who);
unsigned* det_counters(cudaStream_t stream);  // the zeroed counters of the same workspace
// o_k[i] += part[0][k][i] + part[1][k][i] + ... + part[nparts-1][k][i] (left to right) for k < nout, i < n; null
// outputs are skipped.  part[p][k][i] lives at part + (p * nout + k) * n + i (rowops.cu).
int det_reduce(const float* part, int nparts, long long n, int nout, float* o0, float* o1, float* o2,
               cudaStream_t stream);

// Launch with programmatic dependent launch allowed: the kernel may become resident while the previous kernel on
// the stream drains; every kernel launched this way executes griddepcontrol.wait (bb::pdl_wait) before it touches
// global memory, so ordering is unchanged and only launch latency / prologue overlap the predecessor's tail.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
}  // namespace bb
