// Shared helpers for the tt_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/tt_b200.h"

#define TT_DEVICE __device__ __forceinline__

// Every entry point returns 0 or a negative tt_status; nothing in this library calls exit()
// (the reference's launcher does: voxel_pooling_forward_cuda.cu:51-54).
void tt_set_error(const char* fmt, ...);

#define TT_CHECK_LAUNCH(name)                                                     \
  do {                                                                            \
    cudaError_t e__ = cudaGetLastError();                                         \
    if (e__ != cudaSuccess) {                                                     \
      tt_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));       \
      return TT_ERR_CUDA;                                                         \
    }                                                                             \
  } while (0)

#define TT_REQUIRE(cond, name, msg)                                               \
  do {                                                                            \
    if (!(cond)) {                                                                \
      tt_set_error("%s: %s", name, msg);                                          \
      return TT_ERR_INVALID;                                                      \
    }                                                                             \
  } while (0)

static inline int tt_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// SM count of the current device (cached): the CTA count of the persistent kernels and the grid cap of the grid-stride ones
static inline int tt_num_sms() {
  static int n = 0;
  if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); }
  return n;
}

// Activations.  NONE / RELU are inlined; everything with a transcendental (erff, expf, log1pf are ~100 SASS
// instructions each) lives in ONE out-of-line copy per translation unit: inlining it into fully unrolled GEMM
// epilogues blows a tensor-core kernel up by hundreds of KB of SASS and makes its epilogue instruction-cache bound.
static __device__ __noinline__ float tt_act_slow(float v, int act) {
  switch (act) {
    case TT_ACT_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
    case TT_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case TT_ACT_SOFTPLUS: return v > 20.f ? v : log1pf(expf(v));
    case TT_ACT_SOFTPLUS_CLAMP: return fmaxf(v > 20.f ? v : log1pf(expf(v)), 1e-3f);
    default: return v;
  }
}
TT_DEVICE float tt_act(float v, int act) {
  if (act == TT_ACT_NONE) return v;
  if (act == TT_ACT_RELU) return fmaxf(v, 0.f);
  return tt_act_slow(v, act);
}

// 16-byte vector reduction into global memory (sm_90+): the sparse convolutions accumulate taps into an output row
TT_DEVICE void tt_red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

TT_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
TT_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
