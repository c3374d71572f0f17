// Open-loop validation losses (thinktwice_decoder.py:536-620): every term of ThinkTwiceDecoder.loss reduced by one launch.
// CTA (chunk, term) sums a fixed element range of its term in fp64 (fixed per-thread order, fixed shared-memory tree); the last
// CTA to arrive adds the range sums term by term in a fixed order.  No floating-point atomics: the result is bitwise reproducible.
#include "common.cuh"

#include <math_constants.h>

extern long long g_tt_launches;

namespace {

constexpr int LOSS_TPB = 256;
constexpr int LOSS_CHUNKS = 16;         // element ranges per term (CTAs per term)

size_t terms_bytes(int n) { return ((size_t)n * sizeof(tt_loss_term) + 255) / 256 * 256; }

// digamma for finite x > 0: the upward recurrence psi(x) = psi(x + 1) - 1/x to x >= 6 (at most 6 steps), then the asymptotic series.
// Any other x gives NaN, so the loop is bounded whatever the caller passes.
__device__ double digamma_pos(double x) {
  if (!(x > 0.0) || isinf(x)) return CUDART_NAN;
  double r = 0.0;
  while (x < 6.0) { r -= 1.0 / x; x += 1.0; }
  const double f = 1.0 / (x * x);
  return r + log(x) - 0.5 / x
         - f * (1.0 / 12 - f * (1.0 / 120 - f * (1.0 / 252 - f * (1.0 / 240 - f * (1.0 / 132)))));
}

__device__ bool beta_param(double v) { return v > 0.0 && !isinf(v); }

// torch.distributions.kl._kl_beta_beta(p = Beta(a1, b1), q = Beta(a2, b2)) in fp64; NaN outside the Beta domain (finite, > 0)
__device__ double beta_kl(double a1, double b1, double a2, double b2) {
  if (!(beta_param(a1) && beta_param(b1) && beta_param(a2) && beta_param(b2))) return CUDART_NAN;
  const double s1 = a1 + b1, s2 = a2 + b2;
  const double t1 = lgamma(a2) + lgamma(b2) + lgamma(s1);
  const double t2 = lgamma(a1) + lgamma(b1) + lgamma(s2);
  return t1 - t2 + (a1 - a2) * digamma_pos(a1) + (b1 - b2) * digamma_pos(b1) + (s2 - s1) * digamma_pos(s1);
}

// thinktwice_decoder.py:623-636 for one component (fp32 like the reference); the default 0.5 of column 1 survives only NaN inputs
__device__ float action_beta(float a, float b, int comp) {
  float x = comp == 1 ? 0.5f : 0.f;
  if (a > 1.f && b > 1.f) x = (a - 1.f) / (a + b - 2.f);
  else if (a <= 1.f && b > 1.f) x = 0.f;
  else if (a > 1.f && b <= 1.f) x = 1.f;
  else if (a <= 1.f && b <= 1.f) x = a / fmaxf(a + b, 1e-5f);
  return x * 2.f - 1.f;
}

__device__ double term_value(const tt_loss_term& t, long long i) {
  long long po = 0, go = 0;
  for (int d = t.ndim - 1; d >= 0; --d) {
    const long long n = t.shape[d], id = i % n;
    i /= n;
    po += id * t.pred_stride[d];
    go += id * t.gt_stride[d];
  }
  const float p = t.pred[po];
  const float g = t.gt ? t.gt[go] : 0.f;
  switch (t.kind) {
    case TT_LOSS_SMOOTH_L1:
    case TT_LOSS_SMOOTH_L1_CLAMP: {
      const double a = fabs((double)p - (double)g);
      const double v = a < 1.0 ? 0.5 * a * a : a - 0.5;
      return t.kind == TT_LOSS_SMOOTH_L1 || !(v > 5.0) ? v : 5.0;   // clamp(., -5, 5) of a value >= 0; NaN passes through
    }
    case TT_LOSS_L1: return fabs((double)p - (double)g);
    case TT_LOSS_BETA_KL: return beta_kl(g, t.gt2[go], p, t.pred2[po]);
    default: return fabs((double)action_beta(p, t.pred2[po], t.aux) - (double)action_beta(g, t.gt2[go], t.aux));
  }
}

__global__ void __launch_bounds__(LOSS_TPB) loss_reduce_kernel(const tt_loss_term* __restrict__ terms, int n_terms,
                                                               double* __restrict__ partial, unsigned* counter, float* __restrict__ out,
                                                               int n_slots) {
  __shared__ double red[LOSS_TPB];
  __shared__ bool last;
  const tt_loss_term& t = terms[blockIdx.y];
  long long count = 1;
  for (int d = 0; d < t.ndim; ++d) count *= t.shape[d];
  const long long per = (count + LOSS_CHUNKS - 1) / LOSS_CHUNKS;
  const long long lo = blockIdx.x * per, hi = min(count, lo + per);
  double s = 0.0;
  for (long long i = lo + threadIdx.x; i < hi; i += LOSS_TPB) s += term_value(t, i);
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = LOSS_TPB / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    partial[(long long)blockIdx.y * LOSS_CHUNKS + blockIdx.x] = red[0];
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x * gridDim.y - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int slot = threadIdx.x; slot < n_slots; slot += LOSS_TPB) {
    double acc = 0.0;
    for (int k = 0; k < n_terms; ++k) {
      if (terms[k].slot != slot) continue;
      double ts = 0.0;
      for (int c = 0; c < LOSS_CHUNKS; ++c) ts += __ldcg(&partial[(long long)k * LOSS_CHUNKS + c]);
      acc += terms[k].scale * ts;
    }
    out[slot] = (float)acc;
  }
  if (threadIdx.x == 0) *counter = 0u;
}

}  // namespace

extern "C" {

size_t tt_loss_workspace_bytes(int n_terms) {
  return terms_bytes(n_terms) + (size_t)n_terms * LOSS_CHUNKS * sizeof(double) + 256;
}

int tt_loss_reduce(const tt_loss_term* terms, int n_terms, float* out, int n_slots, void* ws, size_t ws_bytes, tt_stream_t stream) {
  TT_REQUIRE(terms && out && ws && n_terms > 0 && n_terms <= 65535 && n_slots > 0, "tt_loss_reduce", "bad arguments");
  TT_REQUIRE(ws_bytes >= tt_loss_workspace_bytes(n_terms), "tt_loss_reduce", "workspace too small");
  for (int k = 0; k < n_terms; ++k) {
    const tt_loss_term& t = terms[k];
    TT_REQUIRE(t.pred && t.ndim >= 1 && t.ndim <= TT_LOSS_MAX_DIM && t.kind >= TT_LOSS_SMOOTH_L1 && t.kind <= TT_LOSS_ACTION_L1 &&
               t.slot >= 0 && t.slot < n_slots, "tt_loss_reduce", "bad term");
    TT_REQUIRE(t.kind < TT_LOSS_BETA_KL || (t.pred2 && t.gt && t.gt2), "tt_loss_reduce", "BETA_KL / ACTION_L1 need pred2, gt and gt2");
    for (int d = 0; d < t.ndim; ++d) TT_REQUIRE(t.shape[d] >= 1, "tt_loss_reduce", "empty dimension");
  }
  cudaStream_t s = (cudaStream_t)stream;
  char* base = (char*)ws;
  tt_loss_term* dterms = (tt_loss_term*)base;
  double* partial = (double*)(base + terms_bytes(n_terms));
  unsigned* counter = (unsigned*)(base + terms_bytes(n_terms) + (size_t)n_terms * LOSS_CHUNKS * sizeof(double));
  if (cudaMemcpyAsync(dterms, terms, (size_t)n_terms * sizeof(tt_loss_term), cudaMemcpyHostToDevice, s) != cudaSuccess ||
      cudaMemsetAsync(counter, 0, sizeof(unsigned), s) != cudaSuccess) {
    tt_set_error("tt_loss_reduce: staging the term table failed: %s", cudaGetErrorString(cudaGetLastError()));
    return TT_ERR_CUDA;
  }
  loss_reduce_kernel<<<dim3(LOSS_CHUNKS, n_terms), LOSS_TPB, 0, s>>>(dterms, n_terms, partial, counter, out, n_slots);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_loss_reduce");
  return TT_OK;
}

}  // extern "C"
