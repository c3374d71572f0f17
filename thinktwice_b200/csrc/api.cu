// Library-level entry points: version, last error, launch counter, conv dispatcher.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

static thread_local char g_err[512] = "";
long long g_tt_launches = 0;
int g_tt_debug = 0;   // diagnosis knobs for kernel micro-benchmarks (tools/conv_bench.py); 0 in normal operation

void tt_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int tt_conv2d_simt(const tt_conv_desc* d, const float* x, const float* w, const float* bias, const float* res,
                   const float* res2, const int* gather, const int* m_count, float* y, void* workspace, cudaStream_t st);
int tt_conv2d_tc(const tt_conv_desc* d, const float* x, const float* w, const float* bias, const float* res,
                 const float* res2, float* y, void* workspace, cudaStream_t st, bool allow_split_k = true);
bool tt_conv2d_tc_supported(const tt_conv_desc* d, const void* x, const void* w, const void* y);

extern "C" {

int tt_version(void) { return 100; }
const char* tt_last_error(void) { return g_err; }
long long tt_launch_count(void) { return g_tt_launches; }
int tt_debug_set(int flags) {
  // the knobs the kernels read (include/tt_b200.h); anything else is refused so that no experiment silently measures the default path
  const int known = 128 | 0xFF00 | 0x20000 | 0x40000 | 0x200000 | 0x400000;
  if (flags & ~known) {
    tt_set_error("tt_debug_set: unknown knob bits 0x%x", flags & ~known);
    return TT_ERR_INVALID;
  }
  g_tt_debug = flags;
  return TT_OK;
}

int tt_conv2d(const tt_conv_desc* d, const float* x, const float* w, const float* bias, const float* res,
              const float* res2, const int* gather, const int* m_count, float* y, void* workspace, tt_stream_t stream) {
  TT_REQUIRE(d && x && w && y, "tt_conv2d", "null argument");
  TT_REQUIRE(d->groups >= 1 && d->Cin % d->groups == 0 && d->Cout % d->groups == 0, "tt_conv2d", "bad groups");
  TT_REQUIRE(d->res_mode == TT_RES_NONE || res != nullptr, "tt_conv2d", "res_mode set without a residual");
  if (gather) TT_REQUIRE(d->groups == 1 && d->taps >= 1, "tt_conv2d", "gather mode needs groups == 1 and taps");
  cudaStream_t st = (cudaStream_t)stream;
  int impl = d->impl;
  if (impl >= 2) {
    if (gather || m_count || !tt_conv2d_tc_supported(d, x, w, y) || ((reinterpret_cast<uintptr_t>(res) | reinterpret_cast<uintptr_t>(res2) |
                                                                       reinterpret_cast<uintptr_t>(bias)) & 15)) {
      tt_set_error("tt_conv2d: tensor-core path does not support this shape / alignment");
      return TT_ERR_UNSUPPORTED;
    }
    return tt_conv2d_tc(d, x, w, bias, res, res2, y, workspace, st);
  }
  return tt_conv2d_simt(d, x, w, bias, res, res2, gather, m_count, y, workspace, st);
}

}  // extern "C"
