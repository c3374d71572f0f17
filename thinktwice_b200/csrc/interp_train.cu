// Training-side bilinear interpolation, align_corners = True (include/tt_b200.h section 17), on channels_last fp32 tensors, float4 over
// channels.
//   forward : ATen's CUDA arithmetic (area_pixel_compute_scale with align_corners, the same lerp order);
//   backward: a gather.  Along one dimension output index o reads input rows i0(o) = (int)(scale o) and i0(o) + (i0(o) < in - 1), and
//             i0 is non-decreasing in o, so the outputs reaching input row i are the contiguous range with i0 in {i - 1, i}.  Each input
//             pixel sums its rows x columns range in row-major order: no atomics, bitwise reproducible.  When the range is long (the
//             1 x 1 -> OH x OW broadcast sums every output pixel of its image) one CTA per input pixel splits it over 8 row lanes and
//             folds them in lane order, as the convolution's grad_bias column sums do.
#include "common.cuh"

extern long long g_tt_launches;

namespace {

constexpr int SPLIT_TERMS = 64;   // the backward splits an input pixel's sum over row lanes past this many output pixels

TT_DEVICE float4 f4_axpy(float a, float4 x, float4 y) { return make_float4(y.x + a * x.x, y.y + a * x.y, y.z + a * x.z, y.w + a * x.w); }

// ATen's area_pixel_compute_scale (align_corners): the source coordinate of output index o is scale * o
float axis_scale(int in, int out) { return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f; }

// the source coordinate scale * o is rounded to fp32 before anything uses it (never contracted into an FMA)
__host__ __device__ __forceinline__ float src_coord(float scale, int o) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(scale, (float)o);
#else
  return scale * (float)o;
#endif
}
__host__ __device__ __forceinline__ int src_row(float scale, int o) { return (int)src_coord(scale, o); }

// the first output index o in [0, out] with src_row(scale, o) >= t
__host__ __device__ __forceinline__ int first_reaching(float scale, int t, int out) {
  if (t <= 0) return 0;
  if (!(scale > 0.f)) return out;
  int o = (int)fminf(ceilf((float)t / scale), (float)out);
  while (o > 0 && src_row(scale, o - 1) >= t) --o;
  while (o < out && src_row(scale, o) < t) ++o;
  return o;
}

// the weight with which output index o reads input index i along one dimension of extent `in` (0 when it reads only the other row)
TT_DEVICE float axis_weight(float scale, int o, int i, int in) {
  const float r = src_coord(scale, o);
  const int i0 = (int)r, i1 = i0 + (i0 < in - 1 ? 1 : 0);
  const float l1 = r - (float)i0, l0 = 1.f - l1;
  return (i0 == i ? l0 : 0.f) + (i1 == i ? l1 : 0.f);
}

__global__ void interp_fwd_kernel(const float4* __restrict__ x, float4* __restrict__ y, int N, int H, int W, int OH, int OW, int C4, float sh,
                                  float sw) {
  const long long total = (long long)N * OH * OW * C4;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % C4);
    long long t = e / C4;
    const int ow = (int)(t % OW);
    t /= OW;
    const int oh = (int)(t % OH), n = (int)(t / OH);
    const float h1r = src_coord(sh, oh), w1r = src_coord(sw, ow);
    const int h1 = (int)h1r, w1 = (int)w1r;
    const int h1p = h1 < H - 1 ? 1 : 0, w1p = w1 < W - 1 ? 1 : 0;
    const float h1l = h1r - (float)h1, h0l = 1.f - h1l, w1l = w1r - (float)w1, w0l = 1.f - w1l;
    const float4* row0 = x + ((long long)n * H + h1) * W * C4 + c;
    const float4* row1 = row0 + (long long)h1p * W * C4;
    const float4 a = __ldg(row0 + (long long)w1 * C4), b = __ldg(row0 + (long long)(w1 + w1p) * C4);
    const float4 p = __ldg(row1 + (long long)w1 * C4), q = __ldg(row1 + (long long)(w1 + w1p) * C4);
    float4 r;
    r.x = h0l * (w0l * a.x + w1l * b.x) + h1l * (w0l * p.x + w1l * q.x);
    r.y = h0l * (w0l * a.y + w1l * b.y) + h1l * (w0l * p.y + w1l * q.y);
    r.z = h0l * (w0l * a.z + w1l * b.z) + h1l * (w0l * p.z + w1l * q.z);
    r.w = h0l * (w0l * a.w + w1l * b.w) + h1l * (w0l * p.w + w1l * q.w);
    y[e] = r;
  }
}

// one thread per input float4: the rows x columns range in row-major order
__global__ void interp_bwd_gather_kernel(const float4* __restrict__ gy, float4* __restrict__ gx, int N, int H, int W, int OH, int OW, int C4,
                                         float sh, float sw) {
  const long long total = (long long)N * H * W * C4;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % C4);
    long long t = e / C4;
    const int j = (int)(t % W);
    t /= W;
    const int i = (int)(t % H), n = (int)(t / H);
    const int h0 = first_reaching(sh, i - 1, OH), h1 = first_reaching(sh, i + 1, OH);
    const int w0 = first_reaching(sw, j - 1, OW), w1 = first_reaching(sw, j + 1, OW);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int oh = h0; oh < h1; ++oh) {
      const float a = axis_weight(sh, oh, i, H);
      const float4* row = gy + ((long long)n * OH + oh) * OW * C4 + c;
      for (int ow = w0; ow < w1; ++ow) acc = f4_axpy(a * axis_weight(sw, ow, j, W), __ldg(row + (long long)ow * C4), acc);
    }
    gx[e] = acc;
  }
}

// one CTA per (input pixel, 32 float4 columns): 8 row lanes take every 8th output pixel of the range, folded in lane order
__global__ void __launch_bounds__(256) interp_bwd_split_kernel(const float4* __restrict__ gy, float4* __restrict__ gx, int H, int W, int OH,
                                                                int OW, int C4, float sh, float sw) {
  __shared__ float4 red[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, c = blockIdx.y * 32 + tx;
  const long long pix = blockIdx.x;
  const int j = (int)(pix % W), i = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
  const int h0 = first_reaching(sh, i - 1, OH), h1 = first_reaching(sh, i + 1, OH);
  const int w0 = first_reaching(sw, j - 1, OW), w1 = first_reaching(sw, j + 1, OW);
  const int nw = w1 - w0, terms = (h1 - h0) * nw;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C4)
    for (int k = ty; k < terms; k += 8) {
      const int oh = h0 + k / nw, ow = w0 + k % nw;
      acc = f4_axpy(axis_weight(sh, oh, i, H) * axis_weight(sw, ow, j, W), __ldg(gy + (((long long)n * OH + oh) * OW + ow) * C4 + c), acc);
    }
  red[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && c < C4) {
    float4 s = red[0][tx];
    for (int q = 1; q < 8; ++q) { s.x += red[q][tx].x; s.y += red[q][tx].y; s.z += red[q][tx].z; s.w += red[q][tx].w; }
    gx[pix * C4 + c] = s;
  }
}

// the longest range of output indices reaching one input index along a dimension (host: the same float arithmetic as the device)
int max_reach(float scale, int in, int out) {
  int m = 0;
  for (int i = 0; i < in; ++i) {
    const int r = first_reaching(scale, i + 1, out) - first_reaching(scale, i - 1, out);
    m = r > m ? r : m;
  }
  return m;
}

int grid_for(long long total) {
  const long long nb = (total + 255) / 256, cap = (long long)tt_num_sms() * 32;
  return (int)(nb < 1 ? 1 : nb > cap ? cap : nb);
}

int check(const tt_interp_bilinear_train_desc* d, const char* name) {
  if (!d) {
    tt_set_error("%s: null descriptor", name);
    return TT_ERR_INVALID;
  }
  const char* bad = nullptr;
  const long long lim = 1LL << 31;
  if (d->align_corners != 1) bad = "align_corners: only 1 (True) is supported";
  else if (d->C <= 0 || d->C % 4) bad = "C: must be a positive multiple of 4";
  else if (d->N < 0 || d->H < 1 || d->W < 1) bad = "N / H / W: N must be >= 0, H and W >= 1";
  else if (d->OH < 1 || d->OW < 1) bad = "OH / OW: must be >= 1";
  else if ((long long)d->N * d->H * d->W * d->C >= lim || (long long)d->N * d->OH * d->OW * d->C >= lim)
    bad = "N: pixel x channel counts past 32-bit indexing";
  if (bad) {
    tt_set_error("%s: unsupported %s", name, bad);
    return TT_ERR_UNSUPPORTED;
  }
  return TT_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" int tt_interp_bilinear_train_forward(const tt_interp_bilinear_train_desc* d, const float* x, float* y, tt_stream_t stream) {
  static const char* name = "tt_interp_bilinear_train_forward";
  const int rc = check(d, name);
  if (rc != TT_OK) return rc;
  if (d->N == 0) return TT_OK;
  TT_REQUIRE(x && y && aligned16(x) && aligned16(y), name, "x and y must be non-NULL and 16-byte aligned");
  const long long total = (long long)d->N * d->OH * d->OW * (d->C / 4);
  interp_fwd_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), d->N,
                                                                        d->H, d->W, d->OH, d->OW, d->C / 4, axis_scale(d->H, d->OH),
                                                                        axis_scale(d->W, d->OW));
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}

extern "C" int tt_interp_bilinear_train_backward(const tt_interp_bilinear_train_desc* d, const float* grad_y, float* grad_x,
                                                 tt_stream_t stream) {
  static const char* name = "tt_interp_bilinear_train_backward";
  const int rc = check(d, name);
  if (rc != TT_OK) return rc;
  if (d->N == 0) return TT_OK;
  TT_REQUIRE(grad_y && grad_x && aligned16(grad_y) && aligned16(grad_x), name, "grad_y and grad_x must be non-NULL and 16-byte aligned");
  const float sh = axis_scale(d->H, d->OH), sw = axis_scale(d->W, d->OW);
  const int C4 = d->C / 4;
  const auto gy = reinterpret_cast<const float4*>(grad_y);
  const auto gx = reinterpret_cast<float4*>(grad_x);
  cudaStream_t st = (cudaStream_t)stream;
  if ((long long)max_reach(sh, d->H, d->OH) * max_reach(sw, d->W, d->OW) > SPLIT_TERMS)
    interp_bwd_split_kernel<<<dim3((unsigned)((long long)d->N * d->H * d->W), tt_cdiv(C4, 32)), 256, 0, st>>>(gy, gx, d->H, d->W, d->OH, d->OW,
                                                                                                            C4, sh, sw);
  else
    interp_bwd_gather_kernel<<<grid_for((long long)d->N * d->H * d->W * C4), 256, 0, st>>>(gy, gx, d->N, d->H, d->W, d->OH, d->OW, C4, sh, sw);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}
