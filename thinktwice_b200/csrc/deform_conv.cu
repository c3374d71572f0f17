// Training-side deformable convolution v1: mmcv's DeformConv2d forward and backward (lss.py:189-197 builds it as
// DeformConv2dPack: 3x3, padding 1, groups 4, deform_groups 1), on mmcv's NCHW tensors.
//
// Per chunk of at most im2col_step images (the columns of a whole batch would not fit: 925 MB at 32 x 512 x 28 x 56):
//   forward : x, offset -> channels-last copies; columns by the inference column builder (tt_dcn_im2col, unchanged);
//             per group, y = col . W^T on the 3xTF32 tensor-core conv (tt_conv2d impl 3 as a 1x1 conv, no split-K, so every
//             output pixel's sum has one fixed order whatever the chunking); y -> NCHW.
//   backward: columns again (for grad_weight), dY -> channels-last;
//             grad_weight += dY^T . col on the A-transposed GEMM (tt_gemm_at: split over pixels, fixed-order fold);
//             grad_col = dY . W per group on the same tensor-core conv (overwrites the columns);
//             grad_offset: a warp per (pixel, tap) reduces grad_col x the corner differences over the channels (no atomics);
//             grad_input: every column gradient is scattered to its four bilinear corners with red.add.v4.f32.
// The weight's hi / lo TF32 planes (and their per-group transpose for grad_col) are packed by a kernel inside every call:
// weights change every optimiser step.
#include "common.cuh"

extern long long g_tt_launches;

int tt_conv2d_tc(const tt_conv_desc* d, const float* x, const float* w, const float* bias, const float* res,
                 const float* res2, float* y, void* workspace, cudaStream_t st, bool allow_split_k);
bool tt_conv2d_tc_supported(const tt_conv_desc* d, const void* x, const void* w, const void* y);
size_t tt_gemm_at_workspace_bytes(int batch, int M, int N);
int tt_gemm_at(const float* A, int lda, long long a_batch, const float* B, int ldb, long long b_batch, float* Cm, int ldc, long long c_batch,
               int batch, int M, int N, int K, int accumulate, void* ws, size_t ws_bytes, cudaStream_t st);

namespace {

constexpr int OFF_LD = 18;   // channels-last offsets: (dy, dx) of the 9 taps

TT_DEVICE float rn_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// weight (Cout, Cg, 3, 3) -> wf [G][2][Cog][9 * Cg] (forward, k = tap * Cg + c) and wb [G][2][9 * Cg][Cog] (grad_col);
// plane 0 = RN_tf32(w), plane 1 = RN_tf32(w - hi), the tt_conv2d impl 3 weight format
__global__ void dcn_pack_weight_kernel(const float* __restrict__ w, float* __restrict__ wf, float* __restrict__ wb, int Cout, int Cg, int G) {
  const int Cog = Cout / G, K9 = 9 * Cg;
  const long long total = (long long)Cout * K9, plane = (long long)Cog * K9;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(e / K9), r = (int)(e - (long long)co * K9), c = r / 9, tap = r - c * 9;
    const float v = w[e], hi = rn_tf32(v), lo = rn_tf32(v - hi);
    const int g = co / Cog, o = co - g * Cog, k = tap * Cg + c;
    float* f = wf + 2 * plane * g;
    f[(long long)o * K9 + k] = hi;
    f[plane + (long long)o * K9 + k] = lo;
    float* b = wb + 2 * plane * g;
    b[(long long)k * Cog + o] = hi;
    b[plane + (long long)k * Cog + o] = lo;
  }
}

// grad_weight (Cout, Cg, 3, 3) <- dw [Cout][9 * Cg] (k = tap * Cg + c)
__global__ void dcn_unpack_grad_weight_kernel(const float* __restrict__ dw, float* __restrict__ gw, int Cout, int Cg) {
  const int K9 = 9 * Cg;
  const long long total = (long long)Cout * K9;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(e / K9), r = (int)(e - (long long)co * K9), c = r / 9, tap = r - c * 9;
    gw[e] = dw[(long long)co * K9 + tap * Cg + c];
  }
}

// the sampling point of (pixel m, tap) exactly as dcn_im2col_kernel computes it
struct Sample {
  bool in;
  int hl, wl;
  float lh, lw;
};
TT_DEVICE Sample sample_at(const float* off_cl, long long m, int tap, int H, int W) {
  const int wo = (int)(m % W), ho = (int)((m / W) % H);
  const float oh = __ldg(off_cl + m * OFF_LD + 2 * tap), ow = __ldg(off_cl + m * OFF_LD + 2 * tap + 1);
  const float h = (float)(ho - 1 + tap / 3) + oh;
  const float w = (float)(wo - 1 + tap % 3) + ow;
  Sample s;
  s.in = h > -1.f && w > -1.f && h < (float)H && w < (float)W;
  s.hl = s.in ? (int)floorf(h) : 0;
  s.wl = s.in ? (int)floorf(w) : 0;
  s.lh = h - s.hl;
  s.lw = w - s.wl;
  return s;
}

// grad_input (channels-last, zeroed) += bilinear scatter of grad_col: one thread = 4 channels of one (pixel, tap)
__global__ void dcn_col2im_kernel(const float* __restrict__ gcol, const float* __restrict__ off_cl, float* __restrict__ gx, int H, int W,
                                  int C, int G, long long total) {
  const int C4 = C / 4, Cg = C / G;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const long long t = i / C4;
    const int tap = (int)(t % 9);
    const long long m = t / 9;
    const Sample s = sample_at(off_cl, m, tap, H, W);
    if (!s.in) continue;
    const int c = c4 * 4, g = c / Cg, cg = c - g * Cg;
    const float4 v = *reinterpret_cast<const float4*>(gcol + ((m * G + g) * 9 + tap) * Cg + cg);
    const long long n = m / ((long long)H * W);
    float* base = gx + n * H * W * C + c;
    const int hh = s.hl + 1, wh = s.wl + 1;
    const float uh = 1.f - s.lh, uw = 1.f - s.lw;
    const float w1 = uh * uw, w2 = uh * s.lw, w3 = s.lh * uw, w4 = s.lh * s.lw;
    if (s.hl >= 0 && s.wl >= 0) tt_red_add_v4(base + ((long long)s.hl * W + s.wl) * C, w1 * v.x, w1 * v.y, w1 * v.z, w1 * v.w);
    if (s.hl >= 0 && wh <= W - 1) tt_red_add_v4(base + ((long long)s.hl * W + wh) * C, w2 * v.x, w2 * v.y, w2 * v.z, w2 * v.w);
    if (hh <= H - 1 && s.wl >= 0) tt_red_add_v4(base + ((long long)hh * W + s.wl) * C, w3 * v.x, w3 * v.y, w3 * v.z, w3 * v.w);
    if (hh <= H - 1 && wh <= W - 1) tt_red_add_v4(base + ((long long)hh * W + wh) * C, w4 * v.x, w4 * v.y, w4 * v.z, w4 * v.w);
  }
}

// grad_offset (NCHW, (N, 18, H, W)) of the chunk: a warp per (pixel, tap); lane l takes the float4 channel groups
// l, l + 32, ... and the warp adds the lanes with a fixed butterfly, so the result does not depend on launch or chunking.
//   d value / dh = (1 - lw) (v_hh,wl - v_hl,wl) + lw (v_hh,wh - v_hl,wh),  d value / dw = (1 - lh) (v_hl,wh - v_hl,wl) + lh (v_hh,wh - v_hh,wl)
// with out-of-image corners zero and both derivatives zero outside (-1, H) x (-1, W) (mmcv's get_coordinate_weight).
__global__ void dcn_col2im_coord_kernel(const float* __restrict__ gcol, const float* __restrict__ x_cl, const float* __restrict__ off_cl,
                                        float* __restrict__ goff, int H, int W, int C, int G, long long items) {
  const int C4 = C / 4, Cg = C / G, lane = threadIdx.x & 31;
  const long long HW = (long long)H * W;
  const long long wstep = (long long)gridDim.x * (blockDim.x / 32);
  for (long long it = blockIdx.x * (long long)(blockDim.x / 32) + (threadIdx.x >> 5); it < items; it += wstep) {
    const int tap = (int)(it % 9);
    const long long m = it / 9;
    const Sample s = sample_at(off_cl, m, tap, H, W);
    float dh = 0.f, dw = 0.f;
    if (s.in) {
      const long long n = m / HW;
      const float4* base = reinterpret_cast<const float4*>(x_cl + n * HW * C);
      const int hh = s.hl + 1, wh = s.wl + 1;
      const bool ok1 = s.hl >= 0 && s.wl >= 0, ok2 = s.hl >= 0 && wh <= W - 1, ok3 = hh <= H - 1 && s.wl >= 0, ok4 = hh <= H - 1 && wh <= W - 1;
      const float uh = 1.f - s.lh, uw = 1.f - s.lw;
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int c4 = lane; c4 < C4; c4 += 32) {
        const float4 v1 = ok1 ? __ldg(base + ((long long)s.hl * W + s.wl) * C4 + c4) : z;
        const float4 v2 = ok2 ? __ldg(base + ((long long)s.hl * W + wh) * C4 + c4) : z;
        const float4 v3 = ok3 ? __ldg(base + ((long long)hh * W + s.wl) * C4 + c4) : z;
        const float4 v4 = ok4 ? __ldg(base + ((long long)hh * W + wh) * C4 + c4) : z;
        const int c = c4 * 4, g = c / Cg, cg = c - g * Cg;
        const float4 gc = *reinterpret_cast<const float4*>(gcol + ((m * G + g) * 9 + tap) * Cg + cg);
        dh += gc.x * (uw * (v3.x - v1.x) + s.lw * (v4.x - v2.x)) + gc.y * (uw * (v3.y - v1.y) + s.lw * (v4.y - v2.y)) +
              gc.z * (uw * (v3.z - v1.z) + s.lw * (v4.z - v2.z)) + gc.w * (uw * (v3.w - v1.w) + s.lw * (v4.w - v2.w));
        dw += gc.x * (uh * (v2.x - v1.x) + s.lh * (v4.x - v3.x)) + gc.y * (uh * (v2.y - v1.y) + s.lh * (v4.y - v3.y)) +
              gc.z * (uh * (v2.z - v1.z) + s.lh * (v4.z - v3.z)) + gc.w * (uh * (v2.w - v1.w) + s.lh * (v4.w - v3.w));
      }
    }
    dh = warp_sum(dh);
    dw = warp_sum(dw);
    if (lane == 0) {
      const long long n = m / HW, pix = m - n * HW;
      goff[(n * 18 + 2 * tap) * HW + pix] = dh;
      goff[(n * 18 + 2 * tap + 1) * HW + pix] = dw;
    }
  }
}

int grid_for(long long total, int per_block) {
  const long long nb = (total + per_block - 1) / per_block, cap = (long long)tt_num_sms() * 32;
  return (int)(nb < 1 ? 1 : nb > cap ? cap : nb);
}

// the workspace of one call, carved in 256-byte aligned pieces
struct Ws {
  float *wf, *wb, *x, *off, *col, *y, *gx, *dw, *part;
  size_t part_bytes, bytes;
};
Ws carve(const tt_deform_conv_desc* d, void* base) {
  const int step = d->im2col_step < d->N ? d->im2col_step : d->N;
  const long long P = (long long)step * d->H * d->W, Cg = d->C / d->groups, Cog = d->Cout / d->groups;
  const size_t part = tt_gemm_at_workspace_bytes(d->groups, (int)Cog, (int)(9 * Cg));
  const size_t sizes[9] = {(size_t)2 * d->Cout * 9 * Cg * 4, (size_t)2 * d->Cout * 9 * Cg * 4, (size_t)P * d->C * 4,
                           (size_t)P * OFF_LD * 4,           (size_t)P * 9 * d->C * 4,        (size_t)P * d->Cout * 4,
                           (size_t)P * d->C * 4,             (size_t)d->Cout * 9 * Cg * 4,    part};
  Ws w;
  float** slots[9] = {&w.wf, &w.wb, &w.x, &w.off, &w.col, &w.y, &w.gx, &w.dw, &w.part};
  size_t o = 0;
  for (int i = 0; i < 9; ++i) {
    *slots[i] = base ? reinterpret_cast<float*>(static_cast<char*>(base) + o) : nullptr;
    o += (sizes[i] + 255) / 256 * 256;
  }
  w.part_bytes = part;
  w.bytes = o;
  return w;
}

// refuses what the reference does not build, naming the parameter
int check_desc(const tt_deform_conv_desc* d, const char* name) {
  TT_REQUIRE(d, name, "null descriptor");
  TT_REQUIRE(d->N > 0 && d->C > 0 && d->H > 0 && d->W > 0 && d->Cout > 0, name, "N, C, H, W and Cout must be positive");
  const char* bad = nullptr;
  if (d->kernel_h != 3 || d->kernel_w != 3) bad = "kernel_size: only 3x3 is supported";
  else if (d->stride != 1) bad = "stride: only 1 is supported";
  else if (d->padding != 1) bad = "padding: only 1 is supported";
  else if (d->dilation != 1) bad = "dilation: only 1 is supported";
  else if (d->deform_groups != 1) bad = "deform_groups: only 1 is supported";
  else if (d->groups < 1 || d->C % d->groups || d->Cout % d->groups) bad = "groups: must divide C and Cout";
  else if ((d->C / d->groups) % 4) bad = "groups: C / groups must be a multiple of 4";
  else if ((d->Cout / d->groups) % 4) bad = "groups: Cout / groups must be a multiple of 4";
  else if (d->im2col_step < 1) bad = "im2col_step: must be >= 1";
  if (bad) {
    tt_set_error("%s: unsupported %s", name, bad);
    return TT_ERR_UNSUPPORTED;
  }
  return TT_OK;
}

// per group g: y[m][y_coff_g + o] = sum_k x[m][x_coff_g + k] * w_g[o][k] on the 3xTF32 tensor-core conv (1x1, no split-K)
int group_gemm(const tt_deform_conv_desc* d, int pix_n, const float* x, int K, int x_ld, const float* w, int Nout, float* y, int y_ld,
               cudaStream_t st, const char* name) {
  for (int g = 0; g < d->groups; ++g) {
    tt_conv_desc c = {};
    c.N = pix_n; c.H = d->H; c.W = d->W; c.Cin = K; c.x_ld = x_ld; c.x_coff = g * K;
    c.Cout = Nout; c.KH = c.KW = 1; c.stride = 1; c.pad = 0; c.dil = 1; c.groups = 1;
    c.OH = d->H; c.OW = d->W; c.y_ld = y_ld; c.y_coff = g * Nout; c.yH = d->H; c.yW = d->W;
    c.oy_mul = c.ox_mul = 1; c.act = TT_ACT_NONE; c.impl = 3;
    const float* wg = w + (size_t)2 * K * Nout * g;
    if (!tt_conv2d_tc_supported(&c, x, wg, y)) {
      tt_set_error("%s: the tensor-core GEMM refused the group layout", name);
      return TT_ERR_UNSUPPORTED;
    }
    const int rc = tt_conv2d_tc(&c, x, wg, nullptr, nullptr, nullptr, y, nullptr, st, false);
    if (rc) return rc;
  }
  return TT_OK;
}

}  // namespace

extern "C" size_t tt_deform_conv_workspace_bytes(const tt_deform_conv_desc* d) {
  if (!d || check_desc(d, "tt_deform_conv_workspace_bytes") != TT_OK) return 0;
  return carve(d, nullptr).bytes;
}

#define DCN_CALL(expr)                   \
  do {                                   \
    const int rc__ = (expr);             \
    if (rc__ != TT_OK) return rc__;      \
  } while (0)

extern "C" int tt_deform_conv_forward(const tt_deform_conv_desc* d, const float* input, const float* offset, const float* weight,
                                      float* output, void* ws, size_t ws_bytes, tt_stream_t stream) {
  static const char* name = "tt_deform_conv_forward";
  DCN_CALL(check_desc(d, name));
  TT_REQUIRE(input && offset && weight && output, name, "null argument");
  const Ws w = carve(d, ws);
  TT_REQUIRE(ws && ws_bytes >= w.bytes, name, "workspace smaller than tt_deform_conv_workspace_bytes");
  cudaStream_t st = (cudaStream_t)stream;
  const int Cg = d->C / d->groups, Cog = d->Cout / d->groups, step = d->im2col_step < d->N ? d->im2col_step : d->N;
  const long long HW = (long long)d->H * d->W;
  dcn_pack_weight_kernel<<<grid_for((long long)d->Cout * 9 * Cg, 256), 256, 0, st>>>(weight, w.wf, w.wb, d->Cout, Cg, d->groups);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  for (int n0 = 0; n0 < d->N; n0 += step) {
    const int nc = d->N - n0 < step ? d->N - n0 : step;
    DCN_CALL(tt_nchw_to_nhwc(input + n0 * HW * d->C, w.x, nc, d->C, d->H, d->W, d->C, 0, d->C, stream));
    DCN_CALL(tt_nchw_to_nhwc(offset + n0 * HW * OFF_LD, w.off, nc, OFF_LD, d->H, d->W, OFF_LD, 0, OFF_LD, stream));
    DCN_CALL(tt_dcn_im2col(w.x, w.off, OFF_LD, w.col, nc, d->H, d->W, d->C, d->groups, stream));
    DCN_CALL(group_gemm(d, nc, w.col, 9 * Cg, 9 * d->C, w.wf, Cog, w.y, d->Cout, st, name));
    DCN_CALL(tt_nhwc_to_nchw(w.y, d->Cout, 0, output + n0 * HW * d->Cout, nc, d->Cout, d->H, d->W, stream));
  }
  return TT_OK;
}

extern "C" int tt_deform_conv_backward(const tt_deform_conv_desc* d, const float* input, const float* offset, const float* weight,
                                       const float* grad_output, float* grad_input, float* grad_offset, float* grad_weight, void* ws,
                                       size_t ws_bytes, tt_stream_t stream) {
  static const char* name = "tt_deform_conv_backward";
  DCN_CALL(check_desc(d, name));
  TT_REQUIRE(input && offset && weight && grad_output, name, "null argument");
  const Ws w = carve(d, ws);
  TT_REQUIRE(ws && ws_bytes >= w.bytes, name, "workspace smaller than tt_deform_conv_workspace_bytes");
  if (!grad_input && !grad_offset && !grad_weight) return TT_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int Cg = d->C / d->groups, Cog = d->Cout / d->groups, step = d->im2col_step < d->N ? d->im2col_step : d->N;
  const long long HW = (long long)d->H * d->W;
  dcn_pack_weight_kernel<<<grid_for((long long)d->Cout * 9 * Cg, 256), 256, 0, st>>>(weight, w.wf, w.wb, d->Cout, Cg, d->groups);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  for (int n0 = 0; n0 < d->N; n0 += step) {
    const int nc = d->N - n0 < step ? d->N - n0 : step;
    const long long P = nc * HW;
    DCN_CALL(tt_nchw_to_nhwc(input + n0 * HW * d->C, w.x, nc, d->C, d->H, d->W, d->C, 0, d->C, stream));
    DCN_CALL(tt_nchw_to_nhwc(offset + n0 * HW * OFF_LD, w.off, nc, OFF_LD, d->H, d->W, OFF_LD, 0, OFF_LD, stream));
    DCN_CALL(tt_nchw_to_nhwc(grad_output + n0 * HW * d->Cout, w.y, nc, d->Cout, d->H, d->W, d->Cout, 0, d->Cout, stream));
    if (grad_weight) {   // dw[g][o][k] (+)= sum_m dY[m][g * Cog + o] * col[m][g * 9 Cg + k]
      DCN_CALL(tt_dcn_im2col(w.x, w.off, OFF_LD, w.col, nc, d->H, d->W, d->C, d->groups, stream));
      DCN_CALL(tt_gemm_at(w.y, d->Cout, Cog, w.col, 9 * d->C, 9 * Cg, w.dw, 9 * Cg, (long long)Cog * 9 * Cg, d->groups, Cog, 9 * Cg,
                          (int)P, n0 > 0, w.part, w.part_bytes, st));
    }
    if (!grad_input && !grad_offset) continue;
    DCN_CALL(group_gemm(d, nc, w.y, Cog, d->Cout, w.wb, 9 * Cg, w.col, 9 * d->C, st, name));   // grad_col over the columns
    if (grad_offset) {
      const long long items = P * 9;
      dcn_col2im_coord_kernel<<<grid_for(items, 8), 256, 0, st>>>(w.col, w.x, w.off, grad_offset + n0 * HW * OFF_LD, d->H, d->W, d->C,
                                                                  d->groups, items);
      ++g_tt_launches;
      TT_CHECK_LAUNCH(name);
    }
    if (grad_input) {
      if (cudaMemsetAsync(w.gx, 0, (size_t)P * d->C * 4, st) != cudaSuccess) {
        tt_set_error("%s: memset failed", name);
        return TT_ERR_CUDA;
      }
      const long long total = P * 9 * (d->C / 4);
      dcn_col2im_kernel<<<grid_for(total, 256), 256, 0, st>>>(w.col, w.off, w.gx, d->H, d->W, d->C, d->groups, total);
      ++g_tt_launches;
      TT_CHECK_LAUNCH(name);
      DCN_CALL(tt_nhwc_to_nchw(w.gx, d->C, 0, grad_input + n0 * HW * d->C, nc, d->C, d->H, d->W, stream));
    }
  }
  if (grad_weight) {
    dcn_unpack_grad_weight_kernel<<<grid_for((long long)d->Cout * 9 * Cg, 256), 256, 0, st>>>(w.dw, grad_weight, d->Cout, Cg);
    ++g_tt_launches;
    TT_CHECK_LAUNCH(name);
  }
  return TT_OK;
}
