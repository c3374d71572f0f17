// Training-side batch normalization (include/tt_b200.h section 18) on rows x[M][C], C contiguous, float4 over channels.
//   Row passes (stats, forward, backward reduce, backward apply) share one tiling: a CTA of 256 threads covers `ct` float4 columns
//   x `rb` row lanes (ct = C / 4 split into at most 256-column tiles, rb = 256 / ct), so every thread keeps the same four channels
//   and holds their per-channel operands in registers.  The reducing passes give each CTA one fixed chunk of rows (the chunking
//   depends on M and C only), add their row lanes in lane order, and a second kernel folds the chunks of each channel in a fixed
//   tree: no atomics, bitwise reproducible.
//   Statistics: every lane of a chunk sums x - K and (x - K)^2 in fp64 with K the chunk's first row (a shifted sum, so the M2 of a
//   chunk does not cancel), the chunk becomes (n, mean, M2), and chunks and ranks are combined by Chan's formula.
#include "common.cuh"

extern long long g_tt_launches;

namespace {

constexpr int THREADS = 256;
constexpr int MAX_CHUNKS = 1024;    // row chunks of a reducing pass (the chunk fold has one thread per 4 chunks per channel)

struct Tiling {
  int C4, ct, rb, ntile;
  long long rows_per, chunks;       // reducing passes
};

Tiling tiling(long long M, int C) {
  Tiling t;
  t.C4 = C / 4;
  t.ntile = tt_cdiv(t.C4, THREADS);
  t.ct = tt_cdiv(t.C4, t.ntile);
  t.rb = THREADS / t.ct;
  long long rp = (M + MAX_CHUNKS - 1) / MAX_CHUNKS;
  rp = rp < t.rb ? t.rb : rp;
  t.rows_per = rp;
  t.chunks = M > 0 ? (M + rp - 1) / rp : 0;
  return t;
}

// z = weight * ((x - mean) * invstd) + bias (+ r), rounded step by step: the forward and both backward passes compute it alike
TT_DEVICE float bn_xhat(float x, float mean, float invstd) { return __fmul_rn(__fsub_rn(x, mean), invstd); }
template <bool kRes>
TT_DEVICE float bn_z(float x, float r, float mean, float invstd, float w, float b) {
  const float z = __fmaf_rn(w, bn_xhat(x, mean, invstd), b);
  return kRes ? __fadd_rn(z, r) : z;
}
TT_DEVICE float relu(float z) { return z <= 0.f ? 0.f : z; }

TT_DEVICE float f4_get(const float4& v, int k) { return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w; }
TT_DEVICE void f4_set(float4& v, int k, float s) {
  if (k == 0) v.x = s; else if (k == 1) v.y = s; else if (k == 2) v.z = s; else v.w = s;
}

// eval mode takes running_var in the invstd slot
template <bool kTrain>
TT_DEVICE float4 load_invstd(const float* s, int c4, float eps) {
  float4 v = __ldg(reinterpret_cast<const float4*>(s) + c4);
  if (!kTrain) {
    v.x = 1.f / sqrtf(v.x + eps); v.y = 1.f / sqrtf(v.y + eps); v.z = 1.f / sqrtf(v.z + eps); v.w = 1.f / sqrtf(v.w + eps);
  }
  return v;
}

struct Stat {
  double n, mean, m2;
};

// Chan's parallel combination of (count, mean, M2)
TT_DEVICE Stat chan(Stat a, Stat b) {
  const double n = a.n + b.n;
  if (n == 0.0) return a;
  const double delta = b.mean - a.mean, fb = b.n / n;
  return Stat{n, a.mean + delta * fb, a.m2 + b.m2 + delta * delta * a.n * fb};
}

// pass 1 of the statistics: part[g][3][C] = (n, mean, M2) of chunk g's rows
__global__ void __launch_bounds__(THREADS) bn_stats_part_kernel(const float* __restrict__ x, long long M, int C, int ct, int rb,
                                                                long long rows_per, double* __restrict__ part) {
  __shared__ double s1[THREADS][4], s2[THREADS][4];
  const int tx = threadIdx.x % ct, ty = threadIdx.x / ct, c4 = blockIdx.y * ct + tx, C4 = C / 4;
  const long long g = blockIdx.x, r0 = g * rows_per, r1 = min(M, r0 + rows_per);
  const bool on = ty < rb && c4 < C4;
  double a1[4] = {0, 0, 0, 0}, a2[4] = {0, 0, 0, 0};
  float4 K = make_float4(0.f, 0.f, 0.f, 0.f);
  if (on) {
    K = __ldg(reinterpret_cast<const float4*>(x + r0 * C) + c4);
    for (long long m = r0 + ty; m < r1; m += rb) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + m * C) + c4);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const double dv = (double)f4_get(v, k) - (double)f4_get(K, k);
        a1[k] += dv;
        a2[k] = fma(dv, dv, a2[k]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) { s1[threadIdx.x][k] = a1[k]; s2[threadIdx.x][k] = a2[k]; }
  __syncthreads();
  if (ty == 0 && c4 < C4) {
    const double n = (double)(r1 - r0);
    for (int q = 1; q < rb; ++q)
#pragma unroll
      for (int k = 0; k < 4; ++k) { a1[k] += s1[q * ct + tx][k]; a2[k] += s2[q * ct + tx][k]; }
    double* p = part + g * 3 * C + 4 * c4;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      p[k] = n;
      p[C + k] = (double)f4_get(K, k) + a1[k] / n;
      p[2 * C + k] = a2[k] - a1[k] * (a1[k] / n);
    }
  }
}

// pass 2: record[3][C] = the chunks of each channel combined in a fixed tree (one CTA per channel)
__global__ void __launch_bounds__(THREADS) bn_stats_fold_kernel(const double* __restrict__ part, int chunks, int C, double* __restrict__ record) {
  __shared__ Stat red[THREADS];
  const int c = blockIdx.x, t = threadIdx.x;
  Stat s{0.0, 0.0, 0.0};
  for (int g = t; g < chunks; g += THREADS) s = chan(s, Stat{part[(long long)g * 3 * C + c], part[(long long)g * 3 * C + C + c],
                                                               part[(long long)g * 3 * C + 2 * C + c]});
  red[t] = s;
  __syncthreads();
  for (int h = THREADS / 2; h > 0; h >>= 1) {
    if (t < h) red[t] = chan(red[t], red[t + h]);
    __syncthreads();
  }
  if (t == 0) { record[c] = red[0].n; record[C + c] = red[0].mean; record[2 * C + c] = red[0].m2; }
}

// the R ranks' records in rank order -> mean, invstd and the running update
__global__ void bn_rank_fold_kernel(const double* __restrict__ rec, int R, int C, double eps, double f, float* running_mean,
                                    float* running_var, float* __restrict__ mean, float* __restrict__ invstd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  Stat s{0.0, 0.0, 0.0};
  for (int q = 0; q < R; ++q) s = chan(s, Stat{rec[(long long)q * 3 * C + c], rec[(long long)q * 3 * C + C + c], rec[(long long)q * 3 * C + 2 * C + c]});
  mean[c] = (float)s.mean;
  invstd[c] = (float)(1.0 / sqrt(s.m2 / s.n + eps));
  running_mean[c] = (float)((1.0 - f) * (double)running_mean[c] + f * s.mean);
  running_var[c] = (float)((1.0 - f) * (double)running_var[c] + f * (s.m2 / (s.n - 1.0)));
}

template <bool kRes, bool kRelu, bool kTrain>
__global__ void __launch_bounds__(THREADS) bn_forward_kernel(const float* __restrict__ x, const float* __restrict__ r,
                                                             const float* __restrict__ w, const float* __restrict__ b,
                                                             const float* __restrict__ mean, const float* __restrict__ invstd, float eps,
                                                             float* __restrict__ y, long long M, int C, int ct, int rb) {
  const int tx = threadIdx.x % ct, ty = threadIdx.x / ct, c4 = blockIdx.y * ct + tx, C4 = C / 4;
  if (ty >= rb || c4 >= C4) return;
  const float4 mu = __ldg(reinterpret_cast<const float4*>(mean) + c4), is = load_invstd<kTrain>(invstd, c4, eps);
  const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + c4), bv = __ldg(reinterpret_cast<const float4*>(b) + c4);
  for (long long m = (long long)blockIdx.x * rb + ty; m < M; m += (long long)gridDim.x * rb) {
    const long long e = m * C4 + c4;
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + e);
    const float4 rv = kRes ? __ldg(reinterpret_cast<const float4*>(r) + e) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 o;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float z = bn_z<kRes>(f4_get(xv, k), f4_get(rv, k), f4_get(mu, k), f4_get(is, k), f4_get(wv, k), f4_get(bv, k));
      f4_set(o, k, kRelu ? relu(z) : z);
    }
    reinterpret_cast<float4*>(y)[e] = o;
  }
}

// backward pass 1: part[g][2][C] = (sum dz, sum dz (x - mean)) over chunk g's rows
template <bool kRes, bool kRelu, bool kTrain>
__global__ void __launch_bounds__(THREADS) bn_bwd_part_kernel(const float* __restrict__ x, const float* __restrict__ r,
                                                              const float* __restrict__ w, const float* __restrict__ b,
                                                              const float* __restrict__ mean, const float* __restrict__ invstd, float eps,
                                                              const float* __restrict__ gy, long long M, int C, int ct, int rb,
                                                              long long rows_per, double* __restrict__ part) {
  __shared__ double s1[THREADS][4], s2[THREADS][4];
  const int tx = threadIdx.x % ct, ty = threadIdx.x / ct, c4 = blockIdx.y * ct + tx, C4 = C / 4;
  const long long g = blockIdx.x, r0 = g * rows_per, r1 = min(M, r0 + rows_per);
  double a1[4] = {0, 0, 0, 0}, a2[4] = {0, 0, 0, 0};
  if (ty < rb && c4 < C4) {
    const float4 mu = __ldg(reinterpret_cast<const float4*>(mean) + c4), is = load_invstd<kTrain>(invstd, c4, eps);
    const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + c4), bv = __ldg(reinterpret_cast<const float4*>(b) + c4);
    for (long long m = r0 + ty; m < r1; m += rb) {
      const long long e = m * C4 + c4;
      const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + e), g4 = __ldg(reinterpret_cast<const float4*>(gy) + e);
      const float4 rv = kRes && kRelu ? __ldg(reinterpret_cast<const float4*>(r) + e) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float dz = f4_get(g4, k);
        if (kRelu && bn_z<kRes>(f4_get(xv, k), f4_get(rv, k), f4_get(mu, k), f4_get(is, k), f4_get(wv, k), f4_get(bv, k)) <= 0.f) dz = 0.f;
        a1[k] += (double)dz;
        a2[k] = fma((double)dz, (double)f4_get(xv, k) - (double)f4_get(mu, k), a2[k]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) { s1[threadIdx.x][k] = a1[k]; s2[threadIdx.x][k] = a2[k]; }
  __syncthreads();
  if (ty == 0 && c4 < C4) {
    for (int q = 1; q < rb; ++q)
#pragma unroll
      for (int k = 0; k < 4; ++k) { a1[k] += s1[q * ct + tx][k]; a2[k] += s2[q * ct + tx][k]; }
    double* p = part + g * 2 * C + 4 * c4;
#pragma unroll
    for (int k = 0; k < 4; ++k) { p[k] = a1[k]; p[C + k] = a2[k]; }
  }
}

// backward pass 2: record[0][c] = sum dz, record[1][c] = invstd sum dz (x - mean), in a fixed tree; grad_bias / grad_weight from them
template <bool kTrain>
__global__ void __launch_bounds__(THREADS) bn_bwd_fold_kernel(const double* __restrict__ part, int chunks, int C,
                                                              const float* __restrict__ invstd, float eps, double* __restrict__ record,
                                                              float* grad_weight, float* grad_bias) {
  __shared__ double r1[THREADS], r2[THREADS];
  const int c = blockIdx.x, t = threadIdx.x;
  double a = 0.0, s = 0.0;
  for (int g = t; g < chunks; g += THREADS) { a += part[(long long)g * 2 * C + c]; s += part[(long long)g * 2 * C + C + c]; }
  r1[t] = a;
  r2[t] = s;
  __syncthreads();
  for (int h = THREADS / 2; h > 0; h >>= 1) {
    if (t < h) { r1[t] += r1[t + h]; r2[t] += r2[t + h]; }
    __syncthreads();
  }
  if (t == 0) {
    const double is = kTrain ? (double)invstd[c] : (double)(1.f / sqrtf(invstd[c] + eps));
    const double sx = r2[0] * is;
    record[c] = r1[0];
    record[C + c] = sx;
    if (grad_bias) grad_bias[c] = (float)r1[0];
    if (grad_weight) grad_weight[c] = (float)sx;
  }
}

// backward pass 3: grad_x (and grad_r = dz), the R ranks' records folded in rank order by every thread for its four channels
template <bool kRes, bool kRelu, bool kTrain>
__global__ void __launch_bounds__(THREADS) bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ r,
                                                               const float* __restrict__ w, const float* __restrict__ b,
                                                               const float* __restrict__ mean, const float* __restrict__ invstd, float eps,
                                                               const float* __restrict__ gy, const double* __restrict__ rec, int R,
                                                               double n, float* __restrict__ gx, float* __restrict__ gr, long long M,
                                                               int C, int ct, int rb) {
  const int tx = threadIdx.x % ct, ty = threadIdx.x / ct, c4 = blockIdx.y * ct + tx, C4 = C / 4;
  if (ty >= rb || c4 >= C4) return;
  const float4 mu = __ldg(reinterpret_cast<const float4*>(mean) + c4), is = load_invstd<kTrain>(invstd, c4, eps);
  const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + c4), bv = __ldg(reinterpret_cast<const float4*>(b) + c4);
  float4 kx, mdz = make_float4(0.f, 0.f, 0.f, 0.f), mdx = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    f4_set(kx, k, __fmul_rn(f4_get(wv, k), f4_get(is, k)));
    if (kTrain) {
      double s1 = 0.0, s2 = 0.0;
      for (int q = 0; q < R; ++q) { s1 += rec[(long long)q * 2 * C + 4 * c4 + k]; s2 += rec[(long long)q * 2 * C + C + 4 * c4 + k]; }
      f4_set(mdz, k, (float)(s1 / n));
      f4_set(mdx, k, (float)(s2 / n));
    }
  }
  for (long long m = (long long)blockIdx.x * rb + ty; m < M; m += (long long)gridDim.x * rb) {
    const long long e = m * C4 + c4;
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + e), g4 = __ldg(reinterpret_cast<const float4*>(gy) + e);
    const float4 rv = kRes && kRelu ? __ldg(reinterpret_cast<const float4*>(r) + e) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 dz4, gx4;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float dz = f4_get(g4, k);
      if (kRelu && bn_z<kRes>(f4_get(xv, k), f4_get(rv, k), f4_get(mu, k), f4_get(is, k), f4_get(wv, k), f4_get(bv, k)) <= 0.f) dz = 0.f;
      f4_set(dz4, k, dz);
      if (kTrain) {
        const float xh = bn_xhat(f4_get(xv, k), f4_get(mu, k), f4_get(is, k));
        f4_set(gx4, k, f4_get(kx, k) * (dz - f4_get(mdz, k) - xh * f4_get(mdx, k)));
      } else {
        f4_set(gx4, k, f4_get(kx, k) * dz);
      }
    }
    if (gx) reinterpret_cast<float4*>(gx)[e] = gx4;
    if (kRes && gr) reinterpret_cast<float4*>(gr)[e] = dz4;
  }
}

int check(const tt_batch_norm_train_desc* d, const char* name) {
  if (!d) {
    tt_set_error("%s: null descriptor", name);
    return TT_ERR_INVALID;
  }
  const char* bad = nullptr;
  if (d->affine != 1) bad = "affine: only affine=True is supported";
  else if (d->track_running_stats != 1) bad = "track_running_stats: only track_running_stats=True is supported";
  else if (d->C <= 0 || d->C % 4) bad = "C: must be a positive multiple of 4";
  else if (d->M < 0) bad = "M: must be >= 0";
  else if (d->R < 1) bad = "R: must be >= 1";
  else if (!(d->eps > 0.0)) bad = "eps: must be > 0";
  else if (d->act != TT_ACT_NONE && d->act != TT_ACT_RELU) bad = "act: only TT_ACT_NONE and TT_ACT_RELU";
  else if (d->residual != 0 && d->residual != 1) bad = "residual: must be 0 or 1";
  else if (d->training != 0 && d->training != 1) bad = "training: must be 0 or 1";
  if (bad) {
    tt_set_error("%s: unsupported %s", name, bad);
    return TT_ERR_UNSUPPORTED;
  }
  return TT_OK;
}

size_t ws_need(const tt_batch_norm_train_desc* d) {
  const size_t n = (size_t)tiling(d->M, d->C).chunks * 3 * d->C * sizeof(double);
  return n < 256 ? 256 : n;
}

int check_ws(const tt_batch_norm_train_desc* d, size_t ws_bytes, const char* name) {
  const int rc = check(d, name);
  if (rc != TT_OK) return rc;
  if (ws_bytes < ws_need(d)) {
    tt_set_error("%s: unsupported ws_bytes %zu (tt_batch_norm_train_workspace_bytes: %zu)", name, ws_bytes, ws_need(d));
    return TT_ERR_UNSUPPORTED;
  }
  return TT_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

dim3 row_grid(const Tiling& t, long long M) {
  const long long nb = (M + t.rb - 1) / t.rb, cap = (long long)tt_num_sms() * 16 / t.ntile + 1;
  return dim3((unsigned)(nb < cap ? nb : cap), t.ntile);
}

template <template <bool, bool, bool> class K, typename... A>
void launch3(bool res, bool relu, bool train, dim3 grid, cudaStream_t st, A... a) {
  if (res) {
    if (relu) train ? K<true, true, true>::go(grid, st, a...) : K<true, true, false>::go(grid, st, a...);
    else train ? K<true, false, true>::go(grid, st, a...) : K<true, false, false>::go(grid, st, a...);
  } else {
    if (relu) train ? K<false, true, true>::go(grid, st, a...) : K<false, true, false>::go(grid, st, a...);
    else train ? K<false, false, true>::go(grid, st, a...) : K<false, false, false>::go(grid, st, a...);
  }
}

template <bool A, bool B, bool T>
struct Fwd {
  template <typename... X>
  static void go(dim3 g, cudaStream_t st, X... x) { bn_forward_kernel<A, B, T><<<g, THREADS, 0, st>>>(x...); }
};
template <bool A, bool B, bool T>
struct BwdPart {
  template <typename... X>
  static void go(dim3 g, cudaStream_t st, X... x) { bn_bwd_part_kernel<A, B, T><<<g, THREADS, 0, st>>>(x...); }
};
template <bool A, bool B, bool T>
struct BwdApply {
  template <typename... X>
  static void go(dim3 g, cudaStream_t st, X... x) { bn_bwd_apply_kernel<A, B, T><<<g, THREADS, 0, st>>>(x...); }
};

}  // namespace

extern "C" size_t tt_batch_norm_train_workspace_bytes(const tt_batch_norm_train_desc* d) {
  return check(d, "tt_batch_norm_train_workspace_bytes") == TT_OK ? ws_need(d) : 0;
}

extern "C" int tt_batch_norm_train_stats(const tt_batch_norm_train_desc* d, const float* x, double* record, void* ws, size_t ws_bytes,
                                         tt_stream_t stream) {
  static const char* name = "tt_batch_norm_train_stats";
  const int rc = check_ws(d, ws_bytes, name);
  if (rc != TT_OK) return rc;
  TT_REQUIRE(record && ws && (d->M == 0 || (x && aligned16(x))), name, "x (16-byte aligned), record and ws must be non-NULL");
  cudaStream_t st = (cudaStream_t)stream;
  if (d->M == 0) {
    if (cudaMemsetAsync(record, 0, sizeof(double) * 3 * d->C, st) != cudaSuccess) { tt_set_error("%s: memset failed", name); return TT_ERR_CUDA; }
    return TT_OK;
  }
  const Tiling t = tiling(d->M, d->C);
  double* part = static_cast<double*>(ws);
  bn_stats_part_kernel<<<dim3((unsigned)t.chunks, t.ntile), THREADS, 0, st>>>(x, d->M, d->C, t.ct, t.rb, t.rows_per, part);
  bn_stats_fold_kernel<<<d->C, THREADS, 0, st>>>(part, (int)t.chunks, d->C, record);
  g_tt_launches += 2;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}

extern "C" int tt_batch_norm_train_fold(const tt_batch_norm_train_desc* d, const double* records, float* running_mean, float* running_var,
                                        float* mean, float* invstd, tt_stream_t stream) {
  static const char* name = "tt_batch_norm_train_fold";
  const int rc = check(d, name);
  if (rc != TT_OK) return rc;
  TT_REQUIRE(records && running_mean && running_var && mean && invstd, name, "records, running stats, mean and invstd must be non-NULL");
  bn_rank_fold_kernel<<<tt_cdiv(d->C, 128), 128, 0, (cudaStream_t)stream>>>(records, d->R, d->C, d->eps, d->factor, running_mean,
                                                                            running_var, mean, invstd);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}

extern "C" int tt_batch_norm_train_forward(const tt_batch_norm_train_desc* d, const float* x, const float* r, const float* weight,
                                           const float* bias, const float* mean, const float* invstd, float* y, tt_stream_t stream) {
  static const char* name = "tt_batch_norm_train_forward";
  const int rc = check(d, name);
  if (rc != TT_OK) return rc;
  if (d->M == 0) return TT_OK;
  TT_REQUIRE(x && y && aligned16(x) && aligned16(y) && (!d->residual || (r && aligned16(r))), name,
             "x, y (and r with residual) must be non-NULL and 16-byte aligned");
  TT_REQUIRE(weight && bias && mean && invstd, name, "weight, bias, mean and invstd must be non-NULL");
  const Tiling t = tiling(d->M, d->C);
  launch3<Fwd>(d->residual, d->act == TT_ACT_RELU, d->training, row_grid(t, d->M), (cudaStream_t)stream, x, r, weight, bias, mean, invstd,
               (float)d->eps, y, d->M, d->C, t.ct, t.rb);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}

extern "C" int tt_batch_norm_train_backward_reduce(const tt_batch_norm_train_desc* d, const float* x, const float* r, const float* weight,
                                                   const float* bias, const float* mean, const float* invstd, const float* grad_y,
                                                   double* record, float* grad_weight, float* grad_bias, void* ws, size_t ws_bytes,
                                                   tt_stream_t stream) {
  static const char* name = "tt_batch_norm_train_backward_reduce";
  const int rc = check_ws(d, ws_bytes, name);
  if (rc != TT_OK) return rc;
  TT_REQUIRE(record && ws && weight && bias && mean && invstd, name, "record, ws, weight, bias, mean and invstd must be non-NULL");
  cudaStream_t st = (cudaStream_t)stream;
  if (d->M == 0) {
    bool ok = cudaMemsetAsync(record, 0, sizeof(double) * 2 * d->C, st) == cudaSuccess;
    if (grad_weight) ok = ok && cudaMemsetAsync(grad_weight, 0, sizeof(float) * d->C, st) == cudaSuccess;
    if (grad_bias) ok = ok && cudaMemsetAsync(grad_bias, 0, sizeof(float) * d->C, st) == cudaSuccess;
    if (!ok) { tt_set_error("%s: memset failed", name); return TT_ERR_CUDA; }
    return TT_OK;
  }
  TT_REQUIRE(x && grad_y && aligned16(x) && aligned16(grad_y) && (!d->residual || d->act != TT_ACT_RELU || (r && aligned16(r))), name,
             "x, grad_y (and r with residual and ReLU) must be non-NULL and 16-byte aligned");
  const Tiling t = tiling(d->M, d->C);
  double* part = static_cast<double*>(ws);
  launch3<BwdPart>(d->residual, d->act == TT_ACT_RELU, d->training, dim3((unsigned)t.chunks, t.ntile), st, x, r, weight, bias, mean, invstd,
                   (float)d->eps, grad_y, d->M, d->C, t.ct, t.rb, t.rows_per, part);
  if (d->training)
    bn_bwd_fold_kernel<true><<<d->C, THREADS, 0, st>>>(part, (int)t.chunks, d->C, invstd, (float)d->eps, record, grad_weight, grad_bias);
  else
    bn_bwd_fold_kernel<false><<<d->C, THREADS, 0, st>>>(part, (int)t.chunks, d->C, invstd, (float)d->eps, record, grad_weight, grad_bias);
  g_tt_launches += 2;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}

extern "C" int tt_batch_norm_train_backward(const tt_batch_norm_train_desc* d, const float* x, const float* r, const float* weight,
                                            const float* bias, const float* mean, const float* invstd, const float* grad_y,
                                            const double* records, float* grad_x, float* grad_r, tt_stream_t stream) {
  static const char* name = "tt_batch_norm_train_backward";
  const int rc = check(d, name);
  if (rc != TT_OK) return rc;
  if (d->training && d->count < 1) {
    tt_set_error("%s: unsupported count %lld: the global row count must be >= 1", name, d->count);
    return TT_ERR_UNSUPPORTED;
  }
  if (d->M == 0 || (!grad_x && !(d->residual && grad_r))) return TT_OK;
  TT_REQUIRE(x && grad_y && aligned16(x) && aligned16(grad_y) && (!d->residual || d->act != TT_ACT_RELU || (r && aligned16(r))), name,
             "x, grad_y (and r with residual and ReLU) must be non-NULL and 16-byte aligned");
  TT_REQUIRE(weight && bias && mean && invstd && (!d->training || records), name, "weight, bias, mean, invstd and records must be non-NULL");
  TT_REQUIRE((!grad_x || aligned16(grad_x)) && (!grad_r || aligned16(grad_r)), name, "grad_x / grad_r must be 16-byte aligned");
  const Tiling t = tiling(d->M, d->C);
  launch3<BwdApply>(d->residual, d->act == TT_ACT_RELU, d->training, row_grid(t, d->M), (cudaStream_t)stream, x, r, weight, bias, mean,
                    invstd, (float)d->eps, grad_y, records, d->R, (double)d->count, grad_x, d->residual ? grad_r : nullptr, d->M, d->C,
                    t.ct, t.rb);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}
