// Open-loop validation losses (thinktwice_decoder.py:536-620): every term of ThinkTwiceDecoder.loss reduced by one launch.
// CTA (chunk, term) sums a fixed element range of its term in fp64 (fixed per-thread order, fixed shared-memory tree); the last
// CTA to arrive adds the range sums term by term in a fixed order.  No floating-point atomics: the result is bitwise reproducible.
#include "common.cuh"

#include <math_constants.h>

#include <vector>

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

// ---------------------------------------------------------------------------------------------- the camera branch's supervision
// encoder_decoder_framework.py:171-190, 442-491, utils.py:31-47.  CTAs [0, gs) take pixels of the segmentation map (one thread per pixel),
// CTAs [gs, gs + gd) take cells of the depth map (one warp per cell: the 16x16 min-pool, then the D logits).  Each CTA writes fp64 sums
// and integer counts; the last CTA to arrive folds them in CTA order and applies the non-linear finish.
constexpr int CAM_TPB = 256;
constexpr int CAM_WARPS = CAM_TPB / 32;
constexpr int CAM_CTAS_PER_SM = 8;

struct CamPartial {
  double seg, bce;                      // sum of the cross entropies / of the BCE terms
  long long nseg, nfg, bad;             // non-ignored pixels / foreground cells / labels torch rejects
};

// ATen's nearest source index (UpSample.h nearest_idx) for an output of `out` pixels over an input of `in`, scale (float)in / out
__device__ __forceinline__ long long nearest_src(long long k, int in, int out) {
  if (out == in) return k;
  if (out == 2 * in) return k >> 1;
  const long long s = (long long)floorf(__fmul_rn((float)k, (float)in / (float)out));
  return s < in - 1 ? s : in - 1;
}

__device__ __forceinline__ float nan_min(float a, float b) { return (isnan(a) || isnan(b)) ? CUDART_NAN_F : fminf(a, b); }   // torch.min

// log(1 + exp(-|x|)) + max(x, 0) - x * y: BCE with logits for a 0 / 1 target, overflow-free
__device__ __forceinline__ double bce_logit(double x, bool y) { return fmax(x, 0.0) - (y ? x : 0.0) + log1p(exp(-fabs(x))); }

__device__ void seg_pixels(const tt_camera_loss_desc& d, int cta, int n_ctas, CamPartial& p) {
  const long long hw = (long long)d.seg_h * d.seg_w, n = (long long)d.BN * hw;
  for (long long i = (long long)cta * CAM_TPB + threadIdx.x; i < n; i += (long long)n_ctas * CAM_TPB) {
    const long long bn = i / hw, r = i - bn * hw, y = r / d.seg_w, x = r - y * d.seg_w;
    const float lab = __ldg(&d.seg_gt[(bn * d.seg_H + nearest_src(y, d.seg_H, d.seg_h)) * d.seg_W + nearest_src(x, d.seg_W, d.seg_w)]);
    if (!(fabsf(lab) < 2147483648.f)) { ++p.bad; continue; }      // NaN / inf / no int: torch's .long() gives garbage, its CE raises
    const int l = (int)lab;                                        // .long() truncates toward zero
    if (l == d.seg_ignore) continue;
    if (l < 0 || l >= d.seg_classes) { ++p.bad; continue; }
    const float* q = d.seg_logits + i * d.seg_ld + d.seg_coff;
    float m = __ldg(q);
    for (int c = 1; c < d.seg_classes; ++c) m = fmaxf(m, __ldg(q + c));   // a NaN logit still reaches the sum below
    double s = 0.0;
    for (int c = 0; c < d.seg_classes; ++c) s += exp((double)__ldg(q + c) - (double)m);
    p.seg += (double)m + log(s) - (double)__ldg(q + l);
    ++p.nseg;
  }
}

__device__ void depth_cells(const tt_camera_loss_desc& d, int cta, int n_ctas, CamPartial& p) {
  const int lane = threadIdx.x & 31, f = d.depth_factor, ff = f * f;
  const long long hw = (long long)d.depth_h * d.depth_w, n = (long long)d.BN * hw;
  const long long W = (long long)d.depth_w * f, H = (long long)d.depth_h * f;
  const float top = (float)(d.depth_bins + 1);
  for (long long i = (long long)cta * CAM_WARPS + (threadIdx.x >> 5); i < n; i += (long long)n_ctas * CAM_WARPS) {
    const long long bn = i / hw, r = i - bn * hw, cy = r / d.depth_w, cx = r - cy * d.depth_w;
    const float* g = d.depth_gt + (bn * H + cy * f) * W + cx * f;
    float mn = CUDART_INF_F;
    for (int k = lane; k < ff; k += 32) {
      float v = __ldg(&g[(long long)(k / f) * W + k % f]);
      mn = nan_min(mn, v == 0.f ? 1e5f : v);
    }
    for (int o = 16; o > 0; o >>= 1) mn = nan_min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    const float v = __fdiv_rn(__fsub_rn(mn, d.depth_offset), d.depth_step);
    const int bin = (v >= 0.f && v < top) ? (int)v : 0;           // NaN / out of range -> class 0, dropped with the one-hot's column 0
    if (bin < 1) continue;
    const float* q = d.depth_logits + i * d.depth_ld + d.depth_coff;
    for (int c = lane; c < d.depth_bins; c += 32) p.bce += bce_logit((double)__ldg(q + c), c == bin - 1);
    if (lane == 0) ++p.nfg;
  }
}

template <typename T>
__device__ T block_sum(T v, T* red) {                             // fixed shared-memory tree: the same order on every call
  red[threadIdx.x] = v;
  __syncthreads();
  for (int w = CAM_TPB / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  const T s = red[0];
  __syncthreads();
  return s;
}

__device__ CamPartial block_fold(CamPartial p, double* rd, long long* rl) {
  CamPartial s;
  s.seg = block_sum(p.seg, rd);
  s.bce = block_sum(p.bce, rd);
  s.nseg = block_sum(p.nseg, rl);
  s.nfg = block_sum(p.nfg, rl);
  s.bad = block_sum(p.bad, rl);
  return s;
}

__global__ void __launch_bounds__(CAM_TPB) camera_loss_kernel(const tt_camera_loss_desc d, int gs, int gd, CamPartial* __restrict__ part,
                                                              unsigned* counter, float* __restrict__ out) {
  __shared__ double rd[CAM_TPB];
  __shared__ long long rl[CAM_TPB];
  __shared__ bool last;
  CamPartial p{0.0, 0.0, 0, 0, 0};
  if ((int)blockIdx.x < gs) seg_pixels(d, blockIdx.x, gs, p);
  else depth_cells(d, blockIdx.x - gs, gd, p);
  const CamPartial s = block_fold(p, rd, rl);
  if (threadIdx.x == 0) {
    part[blockIdx.x] = s;
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  CamPartial a{0.0, 0.0, 0, 0, 0};
  for (int b = threadIdx.x; b < (int)gridDim.x; b += CAM_TPB) {
    const CamPartial* q = &part[b];
    a.seg += __ldcg(&q->seg); a.bce += __ldcg(&q->bce);
    a.nseg += __ldcg(&q->nseg); a.nfg += __ldcg(&q->nfg); a.bad += __ldcg(&q->bad);
  }
  const CamPartial t = block_fold(a, rd, rl);
  if (threadIdx.x == 0) {
    if (gs > 0) {
      const double ce = t.bad ? CUDART_NAN : t.seg / (double)t.nseg;              // no pixel left: 0 / 0 = NaN, as torch's mean
      const double logpt = -ce;                                                     // utils.py:43-46, on the batch-mean CE
      out[0] = (float)(-pow(1.0 - exp(logpt), (double)d.seg_gamma) * (double)d.seg_alpha * logpt * (double)d.seg_weight);
    }
    if (gd > 0) out[1] = (float)(t.bce / (double)(t.nfg > 0 ? t.nfg : 1));
    *counter = 0u;
  }
}

// CTAs of each half: enough for the work, the SMs' worth shared out by the bytes each half reads per unit of work
void camera_grid(const tt_camera_loss_desc& d, int& gs, int& gd) {
  const long long ns = d.seg_logits ? (long long)d.BN * d.seg_h * d.seg_w : 0;
  const long long nd = d.depth_logits ? (long long)d.BN * d.depth_h * d.depth_w : 0;
  const double bs = (double)ns * (d.seg_classes + 1), bd = (double)nd * ((double)d.depth_factor * d.depth_factor + d.depth_bins);
  const int budget = tt_num_sms() * CAM_CTAS_PER_SM;
  const long long want_s = (ns + CAM_TPB - 1) / CAM_TPB, want_d = (nd + CAM_WARPS - 1) / CAM_WARPS;
  long long cap_s = bs + bd > 0 ? (long long)(budget * bs / (bs + bd)) : 0;
  if (ns && cap_s < 1) cap_s = 1;
  long long cap_d = budget - cap_s;
  if (nd && cap_d < 1) cap_d = 1;
  gs = (int)(want_s < cap_s ? want_s : cap_s);
  gd = (int)(want_d < cap_d ? want_d : cap_d);
}

// ------------------------------------------------------------------------------- training side: the camera supervision's gradient
// The forward is the inference kernel's arithmetic on NCHW logits: one thread per seg pixel and one thread per depth cell, so for a
// fixed class / bin a warp reads 32 consecutive floats of the plane.  It records each pixel's target as a byte for the backward.  The
// backward is element-wise: a thread per seg pixel with its classes in registers, a thread per (cell, bin) of the depth logits.
constexpr int CAMT_TPB = 256;
constexpr int CAMT_CTAS = 1024;         // forward grid (fixed: the fold order does not depend on the device)
constexpr int CAMT_MAX_CLASSES = 32;    // seg classes the backward holds in registers
constexpr int CAMT_MAX_BINS = 255;      // depth bins a byte target holds (0 = background)
constexpr unsigned char SEG_SKIP = 255; // seg target of an ignored pixel, or of a label torch rejects

__device__ void train_seg_pixels(const tt_camera_loss_train_desc& d, int cta, int n_ctas, CamPartial& p, unsigned char* tgt) {
  const int hw = d.seg_h * d.seg_w, n = d.BN * hw, C = d.seg_classes;
  const long long cs = d.seg_stride[1];
  for (int i = cta * CAMT_TPB + threadIdx.x; i < n; i += n_ctas * CAMT_TPB) {
    const int bn = i / hw, r = i - bn * hw, y = r / d.seg_w, x = r - y * d.seg_w;
    const float lab = __ldg(&d.seg_gt[((long long)bn * d.seg_H + nearest_src(y, d.seg_H, d.seg_h)) * d.seg_W + nearest_src(x, d.seg_W, d.seg_w)]);
    unsigned char t = SEG_SKIP;
    if (!(fabsf(lab) < 2147483648.f)) {
      ++p.bad;                                                     // NaN / inf / no int: torch's CE raises
    } else if ((int)lab != d.seg_ignore) {
      const int l = (int)lab;
      if (l < 0 || l >= C) {
        ++p.bad;
      } else {
        const float* q = d.seg_logits + bn * d.seg_stride[0] + r;
        float m = __ldg(q);
        for (int c = 1; c < C; ++c) m = fmaxf(m, __ldg(q + c * cs));
        double s = 0.0;
        for (int c = 0; c < C; ++c) s += exp((double)__ldg(q + c * cs) - (double)m);
        p.seg += (double)m + log(s) - (double)__ldg(q + l * cs);
        ++p.nseg;
        t = (unsigned char)l;
      }
    }
    if (tgt) tgt[i] = t;
  }
}

__device__ void train_depth_cells(const tt_camera_loss_train_desc& d, int cta, int n_ctas, CamPartial& p, unsigned char* tgt, bool vec4) {
  const int f = d.depth_factor, hw = d.depth_h * d.depth_w, n = d.BN * hw;
  const long long W = (long long)d.depth_w * f, H = (long long)d.depth_h * f, cs = d.depth_stride[1];
  const float top = (float)(d.depth_bins + 1);
  for (int i = cta * CAMT_TPB + threadIdx.x; i < n; i += n_ctas * CAMT_TPB) {
    const int bn = i / hw, r = i - bn * hw, cy = r / d.depth_w, cx = r - cy * d.depth_w;
    const float* g = d.depth_gt + ((long long)bn * H + (long long)cy * f) * W + (long long)cx * f;
    float mn = CUDART_INF_F;                                       // min is exact: any order gives the inference kernel's value
    for (int ky = 0; ky < f; ++ky) {
      const float* row = g + ky * W;
      if (vec4) {
        for (int kx = 0; kx < f; kx += 4) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(row + kx));
          mn = nan_min(mn, v.x == 0.f ? 1e5f : v.x); mn = nan_min(mn, v.y == 0.f ? 1e5f : v.y);
          mn = nan_min(mn, v.z == 0.f ? 1e5f : v.z); mn = nan_min(mn, v.w == 0.f ? 1e5f : v.w);
        }
      } else {
        for (int kx = 0; kx < f; ++kx) {
          const float v = __ldg(row + kx);
          mn = nan_min(mn, v == 0.f ? 1e5f : v);
        }
      }
    }
    const float v = __fdiv_rn(__fsub_rn(mn, d.depth_offset), d.depth_step);
    const int bin = (v >= 0.f && v < top) ? (int)v : 0;           // NaN / out of range -> background
    if (tgt) tgt[i] = (unsigned char)bin;
    if (bin < 1) continue;
    const float* q = d.depth_logits + bn * d.depth_stride[0] + r;
    for (int c = 0; c < d.depth_bins; ++c) p.bce += bce_logit((double)__ldg(q + c * cs), c == bin - 1);
    ++p.nfg;
  }
}

__global__ void __launch_bounds__(CAMT_TPB) camera_loss_train_kernel(const tt_camera_loss_train_desc d, int gs, int gd, bool vec4,
                                                                     CamPartial* __restrict__ part, unsigned* counter, float* __restrict__ out,
                                                                     tt_camera_loss_stats* __restrict__ stats, unsigned char* seg_tgt,
                                                                     unsigned char* depth_tgt) {
  __shared__ double rd[CAM_TPB];
  __shared__ long long rl[CAM_TPB];
  __shared__ bool last;
  CamPartial p{0.0, 0.0, 0, 0, 0};
  if ((int)blockIdx.x < gs) train_seg_pixels(d, blockIdx.x, gs, p, seg_tgt);
  else train_depth_cells(d, blockIdx.x - gs, gd, p, depth_tgt, vec4);
  const CamPartial s = block_fold(p, rd, rl);
  if (threadIdx.x == 0) {
    part[blockIdx.x] = s;
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  CamPartial a{0.0, 0.0, 0, 0, 0};
  for (int b = threadIdx.x; b < (int)gridDim.x; b += CAMT_TPB) {
    const CamPartial* q = &part[b];
    a.seg += __ldcg(&q->seg); a.bce += __ldcg(&q->bce);
    a.nseg += __ldcg(&q->nseg); a.nfg += __ldcg(&q->nfg); a.bad += __ldcg(&q->bad);
  }
  const CamPartial t = block_fold(a, rd, rl);
  if (threadIdx.x == 0) {
    tt_camera_loss_stats st{0.0, 0.0, t.nseg, t.nfg, t.bad};
    if (gs > 0) {
      const double ce = t.bad ? CUDART_NAN : t.seg / (double)t.nseg;
      const double logpt = -ce, al = d.seg_alpha, ga = d.seg_gamma;
      out[0] = (float)(-pow(1.0 - exp(logpt), ga) * al * logpt * (double)d.seg_weight);
      const double e = exp(-ce), u = 1.0 - e;                      // f'(ce) = alpha [u^gamma + gamma ce e^-ce u^(gamma - 1)]
      st.ce = ce;
      st.seg_factor = (double)d.seg_weight * al * (pow(u, ga) + ga * ce * e * pow(u, ga - 1.0)) / (double)t.nseg;
    }
    if (gd > 0) out[1] = (float)(t.bce / (double)(t.nfg > 0 ? t.nfg : 1));
    *stats = st;
    *counter = 0u;
  }
}

// CTAs [0, gs): 256 seg pixels each, (image, pixel tile); CTAs [gs, gs + gd): 256 depth cells of one bin each, (image, bin, cell tile)
__global__ void __launch_bounds__(CAMT_TPB) camera_loss_grad_kernel(const tt_camera_loss_train_desc d, int gs, const tt_camera_loss_stats* stats,
                                                                    const unsigned char* __restrict__ seg_tgt,
                                                                    const unsigned char* __restrict__ depth_tgt,
                                                                    const float* __restrict__ grad_loss, float* __restrict__ grad_seg,
                                                                    float* __restrict__ grad_depth) {
  if ((int)blockIdx.x < gs) {
    const int hw = d.seg_h * d.seg_w, tiles = (hw + CAMT_TPB - 1) / CAMT_TPB;
    const int bn = blockIdx.x / tiles, r = (blockIdx.x - bn * tiles) * CAMT_TPB + threadIdx.x;
    if (r >= hw) return;
    const int C = d.seg_classes, t = seg_tgt[bn * hw + r];
    float* o = grad_seg + (long long)bn * C * hw + r;
    if (t == SEG_SKIP) {
#pragma unroll
      for (int c = 0; c < CAMT_MAX_CLASSES; ++c)
        if (c < C) o[c * hw] = 0.f;
      return;
    }
    const float k = (float)((double)__ldg(grad_loss) * stats->seg_factor);
    const float* q = d.seg_logits + bn * d.seg_stride[0] + r;
    float v[CAMT_MAX_CLASSES], m = -CUDART_INF_F, s = 0.f;
#pragma unroll
    for (int c = 0; c < CAMT_MAX_CLASSES; ++c)
      if (c < C) { v[c] = __ldg(q + c * d.seg_stride[1]); m = fmaxf(m, v[c]); }
#pragma unroll
    for (int c = 0; c < CAMT_MAX_CLASSES; ++c)
      if (c < C) { v[c] = expf(v[c] - m); s += v[c]; }
    const float inv = 1.f / s;
#pragma unroll
    for (int c = 0; c < CAMT_MAX_CLASSES; ++c)
      if (c < C) o[c * hw] = k * (v[c] * inv - (c == t ? 1.f : 0.f));
    return;
  }
  const int hw = d.depth_h * d.depth_w, tiles = (hw + CAMT_TPB - 1) / CAMT_TPB;
  const int b = blockIdx.x - gs, img = b / (tiles * d.depth_bins), rest = b - img * tiles * d.depth_bins;
  const int c = rest / tiles, r = (rest - c * tiles) * CAMT_TPB + threadIdx.x;
  if (r >= hw) return;
  const int t = depth_tgt[img * hw + r];
  float g = 0.f;
  if (t > 0) {
    const long long nfg = stats->nfg;
    const float k = (float)((double)__ldg(grad_loss + 1) / (double)(nfg > 0 ? nfg : 1));
    const float x = __ldg(d.depth_logits + img * d.depth_stride[0] + c * d.depth_stride[1] + r);
    g = k * (1.f / (1.f + expf(-x)) - (c == t - 1 ? 1.f : 0.f));
  }
  grad_depth[((long long)img * d.depth_bins + c) * hw + r] = g;
}

// refuses what the kernels cannot index, naming the parameter; touches no pointer but d
int check_camera_train(const tt_camera_loss_train_desc* d, const char* name) {
  TT_REQUIRE(d && d->BN >= 0 && (d->seg_logits || d->depth_logits), name, "bad arguments");
  TT_REQUIRE(!d->seg_logits || (d->seg_h > 0 && d->seg_w > 0 && d->seg_H > 0 && d->seg_W > 0 && d->seg_classes > 0), name,
             "bad segmentation half");
  TT_REQUIRE(!d->depth_logits || (d->depth_h > 0 && d->depth_w > 0 && d->depth_factor > 0 && d->depth_bins > 0 && d->depth_step > 0.f),
             name, "bad depth half");
  const long long lim = 1ll << 31, BN = d->BN;
  const char* bad = nullptr;
  if (d->seg_logits) {
    if (d->seg_classes > CAMT_MAX_CLASSES) bad = "seg_classes: at most 32 classes";
    else if (d->seg_stride[3] != 1 || d->seg_stride[2] != d->seg_w) bad = "seg_stride: the h x w plane must be dense (x stride 1, y stride w)";
    else if (BN * d->seg_h * d->seg_w * d->seg_classes >= lim) bad = "BN, seg_classes, seg_h, seg_w: logits past 32-bit indexing";
    else if (BN * d->seg_H * d->seg_W >= lim) bad = "BN, seg_H, seg_W: labels past 32-bit indexing";
  }
  if (!bad && d->depth_logits) {
    if (d->depth_bins > CAMT_MAX_BINS) bad = "depth_bins: at most 255 bins";
    else if (d->depth_stride[3] != 1 || d->depth_stride[2] != d->depth_w) bad = "depth_stride: the h x w plane must be dense (x stride 1, y stride w)";
    else if (BN * d->depth_h * d->depth_w * d->depth_bins >= lim) bad = "BN, depth_bins, depth_h, depth_w: logits past 32-bit indexing";
    else if (BN * d->depth_h * d->depth_w * d->depth_factor * d->depth_factor >= lim) bad = "BN, depth_factor: depths past 32-bit indexing";
  }
  if (bad) {
    tt_set_error("%s: unsupported %s", name, bad);
    return TT_ERR_UNSUPPORTED;
  }
  return TT_OK;
}

// forward CTAs of each half out of CAMT_CTAS, shared by the bytes each half reads per unit of work
void camera_train_grid(const tt_camera_loss_train_desc& d, int& gs, int& gd) {
  const long long ns = d.seg_logits ? (long long)d.BN * d.seg_h * d.seg_w : 0;
  const long long nd = d.depth_logits ? (long long)d.BN * d.depth_h * d.depth_w : 0;
  const double bs = (double)ns * (d.seg_classes + 1), bd = (double)nd * ((double)d.depth_factor * d.depth_factor + d.depth_bins);
  const long long want_s = (ns + CAMT_TPB - 1) / CAMT_TPB, want_d = (nd + CAMT_TPB - 1) / CAMT_TPB;
  long long cap_s = bs + bd > 0 ? (long long)(CAMT_CTAS * bs / (bs + bd)) : 0;
  if (ns && cap_s < 1) cap_s = 1;
  long long cap_d = CAMT_CTAS - cap_s;
  if (nd && cap_d < 1) cap_d = 1;
  gs = (int)(want_s < cap_s ? want_s : cap_s);
  gd = (int)(want_d < cap_d ? want_d : cap_d);
}

// ------------------------------------------------------------------------------------------------ the decoder terms' gradient
constexpr int GRAD_PER_CTA = LOSS_TPB * 8;   // elements per CTA of the gradient kernel
constexpr int GRAD_MAX_CTAS = 4096;          // CTAs of one term

__device__ double sl1_grad(double d) { return d < -1.0 ? -1.0 : (d > 1.0 ? 1.0 : d); }   // NaN passes through

__global__ void __launch_bounds__(LOSS_TPB) loss_grad_kernel(const tt_loss_term* __restrict__ terms, const tt_loss_grad* __restrict__ grads,
                                                             const int* __restrict__ first, int n_terms, const float* __restrict__ grad_out) {
  int k = 0;
  while (k + 1 < n_terms && first[k + 1] <= (int)blockIdx.x) ++k;
  const tt_loss_term& t = terms[k];
  const tt_loss_grad& g = grads[k];
  long long count = 1;
  for (int j = 0; j < t.ndim; ++j) count *= t.shape[j];
  const int ctas = first[k + 1] - first[k];
  const long long per = (count + ctas - 1) / ctas;
  const long long lo = (long long)(blockIdx.x - first[k]) * per, hi = min(count, lo + per);
  double up = 0.0;
  for (int j = 0; j < g.up_count; ++j) up += (double)__ldg(&grad_out[g.up_slot + j]);
  const double u = up * t.scale;
  for (long long i = lo + threadIdx.x; i < hi; i += LOSS_TPB) {
    long long po = 0, go = 0, qo = 0, e = i;
    for (int j = t.ndim - 1; j >= 0; --j) {
      const long long n = t.shape[j], id = e % n;
      e /= n;
      po += id * t.pred_stride[j];
      go += id * t.gt_stride[j];
      qo += id * g.grad_stride[j];
    }
    const double p = t.pred[po], q = t.gt ? t.gt[go] : 0.0;
    if (t.kind == TT_LOSS_BETA_KL) {
      const double a1 = q, b1 = t.gt2[go], a2 = p, b2 = t.pred2[po];
      const double common = digamma_pos(a1 + b1) - digamma_pos(a2 + b2);
      g.grad_pred[qo] = (float)(u * (digamma_pos(a2) - digamma_pos(a1) + common));
      if (g.grad_pred2) g.grad_pred2[qo] = (float)(u * (digamma_pos(b2) - digamma_pos(b1) + common));
      continue;
    }
    const double d = p - q;
    double w = u;
    if (t.kind == TT_LOSS_SMOOTH_L1_CLAMP) {
      const double a = fabs(d), v = a < 1.0 ? 0.5 * a * a : a - 0.5;
      w = (v >= -5.0 && v <= 5.0) ? u : 0.0;                       // torch.clamp's backward: the gradient passes on [min, max]
    }
    g.grad_pred[qo] = (float)(w * sl1_grad(d));
  }
}

size_t grads_bytes(int n) { return ((size_t)n * sizeof(tt_loss_grad) + 255) / 256 * 256; }

// the lowest and one past the highest byte a gradient view over `t`'s shape touches; false when two elements share an address
bool grad_range(const tt_loss_term& t, const float* p, const long long* st, uintptr_t& lo, uintptr_t& hi) {
  long long neg = 0, pos = 0;
  int idx[TT_LOSS_MAX_DIM], m = 0;
  for (int j = 0; j < t.ndim; ++j) {
    const long long ext = (t.shape[j] - 1) * st[j];
    (ext < 0 ? neg : pos) += ext;
    if (t.shape[j] > 1) idx[m++] = j;
  }
  for (int a = 1; a < m; ++a)                                    // dims of extent > 1 by |stride|
    for (int b = a; b > 0 && llabs(st[idx[b]]) < llabs(st[idx[b - 1]]); --b) { const int x = idx[b]; idx[b] = idx[b - 1]; idx[b - 1] = x; }
  long long span = 0;                                            // each |stride| must step past everything the smaller ones reach
  for (int a = 0; a < m; ++a) {
    const long long s = llabs(st[idx[a]]);
    if (s <= span) return false;
    span += (t.shape[idx[a]] - 1) * s;
  }
  lo = (uintptr_t)(p + neg);
  hi = (uintptr_t)(p + pos + 1);
  return true;
}

}  // namespace

extern "C" {

size_t tt_camera_loss_workspace_bytes(const tt_camera_loss_desc* d) {
  int gs = 0, gd = 0;
  if (d) camera_grid(*d, gs, gd);
  return (size_t)(gs + gd) * sizeof(CamPartial) + 256;
}

int tt_camera_loss(const tt_camera_loss_desc* d, float* out, void* ws, size_t ws_bytes, tt_stream_t stream) {
  TT_REQUIRE(d && out && ws && d->BN > 0 && (d->seg_logits || d->depth_logits), "tt_camera_loss", "bad arguments");
  TT_REQUIRE(!d->seg_logits || (d->seg_gt && d->seg_h > 0 && d->seg_w > 0 && d->seg_H > 0 && d->seg_W > 0 && d->seg_classes > 0 &&
                                d->seg_coff >= 0 && d->seg_coff + d->seg_classes <= d->seg_ld),
             "tt_camera_loss", "bad segmentation half");
  TT_REQUIRE(!d->depth_logits || (d->depth_gt && d->depth_h > 0 && d->depth_w > 0 && d->depth_factor > 0 && d->depth_bins > 0 &&
                                  d->depth_coff >= 0 && d->depth_coff + d->depth_bins <= d->depth_ld && d->depth_step > 0.f),
             "tt_camera_loss", "bad depth half");
  TT_REQUIRE(ws_bytes >= tt_camera_loss_workspace_bytes(d), "tt_camera_loss", "workspace too small");
  int gs, gd;
  camera_grid(*d, gs, gd);
  cudaStream_t s = (cudaStream_t)stream;
  CamPartial* part = (CamPartial*)ws;
  unsigned* counter = (unsigned*)((char*)ws + (size_t)(gs + gd) * sizeof(CamPartial));
  if (cudaMemsetAsync(counter, 0, sizeof(unsigned), s) != cudaSuccess) {
    tt_set_error("tt_camera_loss: clearing the arrival counter failed: %s", cudaGetErrorString(cudaGetLastError()));
    return TT_ERR_CUDA;
  }
  camera_loss_kernel<<<gs + gd, CAM_TPB, 0, s>>>(*d, gs, gd, part, counter, out);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_camera_loss");
  return TT_OK;
}

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

size_t tt_loss_backward_workspace_bytes(int n_terms) {
  return terms_bytes(n_terms) + grads_bytes(n_terms) + (size_t)(n_terms + 1) * sizeof(int) + 256;
}

int tt_loss_backward(const tt_loss_term* terms, int n_terms, const tt_loss_grad* grads, const float* grad_out, int n_slots, void* ws,
                     size_t ws_bytes, tt_stream_t stream) {
  const char* name = "tt_loss_backward";
  TT_REQUIRE(terms && grads && grad_out && ws && n_terms > 0 && n_terms <= 65535 && n_slots > 0, name, "bad arguments");
  TT_REQUIRE(ws_bytes >= tt_loss_backward_workspace_bytes(n_terms), name, "workspace too small");
  std::vector<uintptr_t> lo(2 * n_terms), hi(2 * n_terms);
  std::vector<int> owner(2 * n_terms), first(n_terms + 1);
  int n_ranges = 0;
  first[0] = 0;
  for (int k = 0; k < n_terms; ++k) {
    const tt_loss_term& t = terms[k];
    const tt_loss_grad& g = grads[k];
    bool ok = t.pred && t.ndim >= 1 && t.ndim <= TT_LOSS_MAX_DIM && t.kind >= TT_LOSS_SMOOTH_L1 && t.kind <= TT_LOSS_ACTION_L1;
    for (int d = 0; ok && d < t.ndim; ++d) ok = t.shape[d] >= 1;
    long long count = 1;
    for (int d = 0; ok && d < t.ndim; ++d) count *= t.shape[d];
    int ctas = 0;
    if (ok && g.grad_pred) {
      ok = g.up_slot >= 0 && g.up_count >= 1 && g.up_slot + (long long)g.up_count <= n_slots &&
           (t.kind != TT_LOSS_BETA_KL || (t.pred2 && t.gt && t.gt2));
      const long long want = (count + GRAD_PER_CTA - 1) / GRAD_PER_CTA;
      ctas = (int)(want < GRAD_MAX_CTAS ? want : GRAD_MAX_CTAS);
    }
    if (!ok) {
      tt_set_error("%s: bad term %d", name, k);
      return TT_ERR_INVALID;
    }
    const char* bad = nullptr;
    if (g.grad_pred && (t.kind == TT_LOSS_L1 || t.kind == TT_LOSS_ACTION_L1)) bad = "L1 / ACTION_L1 terms have no gradient";
    for (int w = 0; !bad && g.grad_pred && w < (t.kind == TT_LOSS_BETA_KL && g.grad_pred2 ? 2 : 1); ++w) {
      if (!grad_range(t, w ? g.grad_pred2 : g.grad_pred, g.grad_stride, lo[n_ranges], hi[n_ranges])) {
        bad = "grad_stride maps two elements to one address";
        break;
      }
      for (int r = 0; r < n_ranges; ++r)
        if (lo[n_ranges] < hi[r] && lo[r] < hi[n_ranges]) {
          tt_set_error("%s: unsupported gradient ranges: term %d overlaps term %d", name, k, owner[r]);
          return TT_ERR_UNSUPPORTED;
        }
      owner[n_ranges++] = k;
    }
    if (bad) {
      tt_set_error("%s: unsupported term %d: %s", name, k, bad);
      return TT_ERR_UNSUPPORTED;
    }
    first[k + 1] = first[k] + ctas;
  }
  const int total = first[n_terms];
  if (total == 0) return TT_OK;                                    // no term asks for a gradient
  cudaStream_t s = (cudaStream_t)stream;
  char* base = (char*)ws;
  tt_loss_term* dterms = (tt_loss_term*)base;
  tt_loss_grad* dgrads = (tt_loss_grad*)(base + terms_bytes(n_terms));
  int* dfirst = (int*)(base + terms_bytes(n_terms) + grads_bytes(n_terms));
  const bool staged = cudaMemcpyAsync(dterms, terms, (size_t)n_terms * sizeof(tt_loss_term), cudaMemcpyHostToDevice, s) == cudaSuccess &&
                      cudaMemcpyAsync(dgrads, grads, (size_t)n_terms * sizeof(tt_loss_grad), cudaMemcpyHostToDevice, s) == cudaSuccess &&
                      cudaMemcpyAsync(dfirst, first.data(), (size_t)(n_terms + 1) * sizeof(int), cudaMemcpyHostToDevice, s) == cudaSuccess;
  if (!staged) {
    tt_set_error("%s: staging the term table failed: %s", name, cudaGetErrorString(cudaGetLastError()));
    return TT_ERR_CUDA;
  }
  loss_grad_kernel<<<total, LOSS_TPB, 0, s>>>(dterms, dgrads, dfirst, n_terms, grad_out);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}

size_t tt_camera_loss_train_workspace_bytes(const tt_camera_loss_train_desc*) {
  return (size_t)CAMT_CTAS * sizeof(CamPartial) + 256;
}

int tt_camera_loss_train_forward(const tt_camera_loss_train_desc* d, float* out, tt_camera_loss_stats* stats, uint8_t* seg_target,
                                 uint8_t* depth_target, void* ws, size_t ws_bytes, tt_stream_t stream) {
  const char* name = "tt_camera_loss_train_forward";
  const int rc = check_camera_train(d, name);
  if (rc) return rc;
  if (ws_bytes < tt_camera_loss_train_workspace_bytes(d)) {
    tt_set_error("%s: unsupported ws_bytes: %zu, smaller than tt_camera_loss_train_workspace_bytes (%zu)", name, ws_bytes,
                 tt_camera_loss_train_workspace_bytes(d));
    return TT_ERR_UNSUPPORTED;
  }
  if (d->BN == 0) return TT_OK;
  TT_REQUIRE(out && stats && ws && (!d->seg_logits || d->seg_gt) && (!d->depth_logits || d->depth_gt), name, "null argument");
  int gs, gd;
  camera_train_grid(*d, gs, gd);
  const int f = d->depth_factor;
  const bool vec4 = d->depth_logits && f % 4 == 0 && ((long long)d->depth_w * f) % 4 == 0 && ((uintptr_t)d->depth_gt & 15) == 0;
  cudaStream_t s = (cudaStream_t)stream;
  CamPartial* part = (CamPartial*)ws;
  unsigned* counter = (unsigned*)((char*)ws + (size_t)CAMT_CTAS * sizeof(CamPartial));
  if (cudaMemsetAsync(counter, 0, sizeof(unsigned), s) != cudaSuccess) {
    tt_set_error("%s: clearing the arrival counter failed: %s", name, cudaGetErrorString(cudaGetLastError()));
    return TT_ERR_CUDA;
  }
  camera_loss_train_kernel<<<gs + gd, CAMT_TPB, 0, s>>>(*d, gs, gd, vec4, part, counter, out, stats, d->seg_logits ? seg_target : nullptr,
                                                        d->depth_logits ? depth_target : nullptr);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}

int tt_camera_loss_train_backward(const tt_camera_loss_train_desc* d, const tt_camera_loss_stats* stats, const uint8_t* seg_target,
                                  const uint8_t* depth_target, const float* grad_loss, float* grad_seg, float* grad_depth,
                                  tt_stream_t stream) {
  const char* name = "tt_camera_loss_train_backward";
  const int rc = check_camera_train(d, name);
  if (rc) return rc;
  if (!d->seg_logits) grad_seg = nullptr;
  if (!d->depth_logits) grad_depth = nullptr;
  if (d->BN == 0 || (!grad_seg && !grad_depth)) return TT_OK;
  TT_REQUIRE(stats && grad_loss && (!grad_seg || seg_target) && (!grad_depth || depth_target), name, "null argument");
  const int ts = (d->seg_h * d->seg_w + CAMT_TPB - 1) / CAMT_TPB, td = (d->depth_h * d->depth_w + CAMT_TPB - 1) / CAMT_TPB;
  const long long gs = grad_seg ? (long long)d->BN * ts : 0, gd = grad_depth ? (long long)d->BN * d->depth_bins * td : 0;
  TT_REQUIRE(gs + gd < (1ll << 31), name, "grid too large");
  camera_loss_grad_kernel<<<(unsigned)(gs + gd), CAMT_TPB, 0, (cudaStream_t)stream>>>(*d, (int)gs, stats, seg_target, depth_target, grad_loss,
                                                                                     grad_seg, grad_depth);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}

}  // extern "C"
