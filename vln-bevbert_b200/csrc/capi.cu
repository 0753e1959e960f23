// Error reporting and launch accounting for the C ABI (include/bevbert_b200.h).
#include <atomic>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>

#include "../../include/bevbert_b200.h"
#include "common.h"

namespace bb {
static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

int set_error(const char* msg) {
  strncpy(g_err, msg, sizeof(g_err) - 1);
  g_err[sizeof(g_err) - 1] = 0;
  return -1;
}
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return 0;
  char buf[400];
  snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  return set_error(buf);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("BB_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}
}  // namespace bb

namespace bb {
static int g_det = 0;
static char* g_det_ws[2] = {nullptr, nullptr};   // main, side
static int64_t g_det_bytes = 0;

int det_mode() { return g_det; }

static char* det_ws(cudaStream_t stream) { return g_det_ws[stream && stream == side_stream() ? 1 : 0]; }

float* det_partials(cudaStream_t stream, size_t bytes, const char* who) {
  char* ws = det_ws(stream);
  const size_t need = DET_COUNTER_BYTES + bytes;
  if (!ws || (size_t)g_det_bytes < need) {
    char buf[300];
    snprintf(buf, sizeof(buf),
             "%s: deterministic mode needs a workspace of at least %zu bytes on this stream (registered: %lld); "
             "see bb_set_det_workspace", who, need, ws ? (long long)g_det_bytes : 0LL);
    set_error(buf);
    return nullptr;
  }
  return reinterpret_cast<float*>(ws + DET_COUNTER_BYTES);
}
unsigned* det_counters(cudaStream_t stream) { return reinterpret_cast<unsigned*>(det_ws(stream)); }
}  // namespace bb

extern "C" int bb_set_deterministic(int on) {
  if (on < 0 || on > 2) return bb::set_error("bb_set_deterministic: mode must be 0, 1 or 2");
  bb::g_det = on;
  return 0;
}
extern "C" int bb_set_det_workspace(void* main_ws, void* side_ws, int64_t bytes) {
  if ((main_ws || side_ws) && bytes < (int64_t)bb::DET_COUNTER_BYTES)
    return bb::set_error("bb_set_det_workspace: a workspace must hold at least the 64 KB of split-K counters");
  if ((reinterpret_cast<uintptr_t>(main_ws) | reinterpret_cast<uintptr_t>(side_ws)) & 255)
    return bb::set_error("bb_set_det_workspace: workspaces must be 256-byte aligned");
  bb::g_det_ws[0] = static_cast<char*>(main_ws);
  bb::g_det_ws[1] = static_cast<char*>(side_ws);
  bb::g_det_bytes = (main_ws || side_ws) ? bytes : 0;
  return 0;
}

extern "C" const char* bb_last_error(void) { return bb::g_err; }
extern "C" int bb_abi_version(void) { return 1; }
extern "C" int64_t bb_launch_count(void) { return bb::g_launches.load(); }
extern "C" void bb_reset_launch_count(void) { bb::g_launches.store(0); }

namespace bb {
int set_salt_gemm_tc(const unsigned long long*);
int set_salt_rowops(const unsigned long long*);
int set_salt_attn_flash(const unsigned long long*);
int set_salt_attn_tc(const unsigned long long*);
int set_salt_attn_scores(const unsigned long long*);
int set_salt_gemm_f32(const unsigned long long*);
}  // namespace bb
extern "C" int bb_set_drop_salt_ptr(const uint64_t* device_word) {
  const unsigned long long* p = reinterpret_cast<const unsigned long long*>(device_word);
  int rc = bb::set_salt_gemm_tc(p) | bb::set_salt_rowops(p) | bb::set_salt_attn_flash(p) | bb::set_salt_attn_tc(p) |
           bb::set_salt_attn_scores(p) | bb::set_salt_gemm_f32(p);
  return rc ? bb::set_error("bb_set_drop_salt_ptr: cudaMemcpyToSymbol failed") : 0;
}
