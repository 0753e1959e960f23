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
