// Agent-side pre-processing on the GPU (SURVEY.md §8f row f1): what the reference does on the CPU between the CARLA sensors and
// forward_inference, as two HBM-bound kernels.
//   * images: uint8 HWC camera frames -> undistort (grid_sample through the rectification map) -> bilinear resize -> crop -> /255 ->
//     Normalize, written as the network's input tensor (fp32 NCHW) and / or straight into the row-packed stem's operand planes
//     (open_loop_training/code/datasets/pipelines/transform.py:275-341 IDAImageTransform.__call__, :346-378 img_transform,
//      :142-163 ImageTransformMulti);
//   * LiDAR: the previous half sweep moved into the current ego frame and concatenated with the current one
//     (leaderboard/team_code/thinktwice_agent.py:340-352).
// The arithmetic follows PyTorch's CPU kernels operation for operation (the fused-multiply-add placement was determined against
// torch: tests/test_preprocess_cpu.py pins the restatement in oracle/preprocess.py bit for bit), so the GPU result equals the
// reference pipeline's to the last bit wherever the compiler keeps the written operation order — hence the explicit intrinsics.
#include <cuda_fp16.h>

#include "common.cuh"

extern long long g_tt_launches;

namespace {

constexpr float H_MAX = 65504.f;
constexpr float LO_SCALE = 2048.f;

TT_DEVICE void split_h(float x, __half& hi, __half& lo) {
  const float c = fminf(fmaxf(x, -H_MAX), H_MAX);
  hi = __float2half_rn(c);
  lo = __float2half_rn((c - __half2float(hi)) * LO_SCALE);
}

// F.grid_sample(bilinear, zeros, align_corners=False) of one raw pixel position: all three channels of the HWC byte image.
// ATen's vectorised CPU kernel: ix = fma(gx + 1, W / 2, -0.5); weights e = 1 - w, s = 1 - n; out = fma chain nw, ne, sw, se.
TT_DEVICE void undistort3(const uint8_t* __restrict__ img, const float2* __restrict__ grid, int H, int W, int y, int x, float out[3]) {
  const float2 g = __ldg(grid + (long long)y * W + x);
  const float ix = __fmaf_rn(__fadd_rn(g.x, 1.f), 0.5f * (float)W, -0.5f);
  const float iy = __fmaf_rn(__fadd_rn(g.y, 1.f), 0.5f * (float)H, -0.5f);
  const float fx = floorf(ix), fy = floorf(iy);
  const float w = __fsub_rn(ix, fx), n = __fsub_rn(iy, fy);
  const float e = __fsub_rn(1.f, w), s = __fsub_rn(1.f, n);
  const float wt[4] = {__fmul_rn(s, e), __fmul_rn(s, w), __fmul_rn(n, e), __fmul_rn(n, w)};
  // |ix| beyond the int range (a map that points far outside the image) would overflow the conversion: such taps are out of bounds anyway
  const bool sane = fabsf(ix) < 1e9f && fabsf(iy) < 1e9f;
  const int x0 = sane ? (int)fx : -2, y0 = sane ? (int)fy : -2;
  out[0] = out[1] = out[2] = 0.f;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int xx = x0 + (t & 1), yy = y0 + (t >> 1);
    float v[3] = {0.f, 0.f, 0.f};
    if (xx >= 0 && xx < W && yy >= 0 && yy < H) {
      const uint8_t* p = img + ((long long)yy * W + xx) * 3;
      v[0] = (float)__ldg(p); v[1] = (float)__ldg(p + 1); v[2] = (float)__ldg(p + 2);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = t == 0 ? __fmul_rn(v[c], wt[0]) : __fmaf_rn(v[c], wt[t], out[c]);
  }
}

TT_DEVICE void raw3(const uint8_t* __restrict__ img, int W, int y, int x, float out[3]) {
  const uint8_t* p = img + ((long long)y * W + x) * 3;
  out[0] = (float)__ldg(p); out[1] = (float)__ldg(p + 1); out[2] = (float)__ldg(p + 2);
}

// one thread = one output pixel (3 channels): 4 resize taps x 4 undistort taps of the byte image.  Neighbouring threads walk
// neighbouring raw pixels (stride H / newH ~ 1.8 px), so the byte loads of a warp fall into a handful of 128-byte lines and the
// rectification map (8 B per raw pixel, shared by every image) stays in L2.
__global__ void preprocess_u8_kernel(const uint8_t* __restrict__ raw, const float2* __restrict__ grid, float* __restrict__ out_nchw,
                                     __half* __restrict__ ys, long long ys_plane, tt_preproc_desc d, long long total) {
  const float sch = (float)d.H / (float)d.newH, scw = (float)d.W / (float)d.newW;   // area_pixel_compute_scale (size given, not scale_factor)
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % d.outW);
    const long long t = i / d.outW;
    const int oy = (int)(t % d.outH), n = (int)(t / d.outH);
    // torch upsample_bilinear2d (align_corners=False, antialias=False) of resized pixel (oy + crop_y, ox + crop_x)
    const float fy = fmaxf(__fmaf_rn(sch, (float)(oy + d.crop_y) + 0.5f, -0.5f), 0.f);
    const float fx = fmaxf(__fmaf_rn(scw, (float)(ox + d.crop_x) + 0.5f, -0.5f), 0.f);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < d.H - 1), x1 = x0 + (x0 < d.W - 1);
    const float ly1 = __fsub_rn(fy, (float)y0), lx1 = __fsub_rn(fx, (float)x0);
    const float ly0 = __fsub_rn(1.f, ly1), lx0 = __fsub_rn(1.f, lx1);
    const uint8_t* img = raw + (long long)n * d.H * d.W * 3;
    float p00[3], p01[3], p10[3], p11[3];
    if (d.undistort) {
      undistort3(img, grid, d.H, d.W, y0, x0, p00); undistort3(img, grid, d.H, d.W, y0, x1, p01);
      undistort3(img, grid, d.H, d.W, y1, x0, p10); undistort3(img, grid, d.H, d.W, y1, x1, p11);
    } else {
      raw3(img, d.W, y0, x0, p00); raw3(img, d.W, y0, x1, p01); raw3(img, d.W, y1, x0, p10); raw3(img, d.W, y1, x1, p11);
    }
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float r0 = __fmaf_rn(p00[c], lx0, __fmul_rn(p01[c], lx1));
      const float r1 = __fmaf_rn(p10[c], lx0, __fmul_rn(p11[c], lx1));
      const float r = __fmaf_rn(ly0, r0, __fmul_rn(ly1, r1));
      // ImageTransformMulti: .div(255) then Normalize = sub(mean).div(std)
      v[c] = __fdiv_rn(__fsub_rn(__fdiv_rn(r, d.div), d.mean[c]), d.std[c]);
    }
    if (out_nchw) {
      const long long plane = (long long)d.outH * d.outW;
      float* o = out_nchw + (long long)n * 3 * plane + (long long)oy * d.outW + ox;
      o[0] = v[0]; o[plane] = v[1]; o[2 * plane] = v[2];
    }
    if (ys) {                                                   // the stem's operand layout: tt_image_to_split8
      __half hi[8], lo[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (c < 3) split_h(v[c], hi[c], lo[c]);
        else hi[c] = lo[c] = __float2half_rn(0.f);
      }
      const long long o = (((long long)n * d.pad_H + oy + d.pad_top) * d.pad_W + ox + d.pad_left) * 8;
      *reinterpret_cast<uint4*>(ys + o) = *reinterpret_cast<const uint4*>(hi);
      *reinterpret_cast<uint4*>(ys + ys_plane + o) = *reinterpret_cast<const uint4*>(lo);
    }
  }
}

// thinktwice_agent.py:340-352: numpy promotes everything to float64 (np.ones / np.dot), the result is cast to float32 at the end
__global__ void lidar_stitch_kernel(const float* __restrict__ prev, int n_prev, const float* __restrict__ now, int n_now,
                                    const double* __restrict__ rel, double z_add, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_prev + n_now) return;
  float4 o;
  if (i < n_prev) {
    const float4 p = __ldg(reinterpret_cast<const float4*>(prev) + i);
    double r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      // np.einsum('ij,kj->ki'): sum over j in index order, no fused multiply-add on the host
      double acc = __dmul_rn(rel[k * 4 + 0], (double)p.x);
      acc = __dadd_rn(acc, __dmul_rn(rel[k * 4 + 1], (double)p.y));
      acc = __dadd_rn(acc, __dmul_rn(rel[k * 4 + 2], (double)p.z));
      acc = __dadd_rn(acc, rel[k * 4 + 3]);                      // homogeneous 1
      r[k] = acc;
    }
    o = make_float4((float)r[0], (float)r[1], (float)__dadd_rn(r[2], z_add), p.w);
  } else {
    const float4 p = __ldg(reinterpret_cast<const float4*>(now) + (i - n_prev));
    o = make_float4(p.x, p.y, (float)__dadd_rn((double)p.z, z_add), p.w);
  }
  reinterpret_cast<float4*>(out)[i] = o;
}

// carla_dataset.py:314-328 (union2one, "dense-fusion"): a sweep's (x, y, z, intensity) rows multiplied by curr2key as 4-vectors (the
// reference uses the intensity as the homogeneous coordinate) plus a timestamp column; mat == NULL: the key frame (copied, timestamp 0)
__global__ void points_union_kernel(const float* __restrict__ src, int n, const float* __restrict__ mat, float ts, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = __ldg(reinterpret_cast<const float4*>(src) + i);
  float o[4] = {p.x, p.y, p.z, p.w};
  if (mat) {
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = fmaf(mat[k * 4 + 3], p.w, fmaf(mat[k * 4 + 2], p.z, fmaf(mat[k * 4 + 1], p.y, mat[k * 4] * p.x)));
  }
  float* d = dst + (long long)i * 5;
  d[0] = o[0]; d[1] = o[1]; d[2] = o[2]; d[3] = o[3]; d[4] = ts;
}

}  // namespace

extern "C" {

int tt_preprocess_u8(const tt_preproc_desc* d, const uint8_t* raw, const float* map_grid, float* out_nchw, void* out_split8,
                     long long split_plane, tt_stream_t stream) {
  TT_REQUIRE(d && raw && (out_nchw || out_split8), "tt_preprocess_u8", "null argument");
  TT_REQUIRE(d->n_img >= 0 && d->H > 0 && d->W > 0 && d->newH > 0 && d->newW > 0 && d->outH > 0 && d->outW > 0 && d->crop_x >= 0 && d->crop_y >= 0 &&
                 d->crop_y + d->outH <= d->newH && d->crop_x + d->outW <= d->newW,
             "tt_preprocess_u8", "the crop window must lie inside the resized image");
  TT_REQUIRE(!d->undistort || map_grid, "tt_preprocess_u8", "undistort needs the rectification map");
  TT_REQUIRE((reinterpret_cast<uintptr_t>(map_grid) & 7) == 0, "tt_preprocess_u8", "map_grid must be 8-byte aligned");
  if (out_split8)
    TT_REQUIRE(d->pad_top >= 0 && d->pad_left >= 0 && d->pad_top + d->outH <= d->pad_H && d->pad_left + d->outW <= d->pad_W && split_plane % 8 == 0 &&
                   (reinterpret_cast<uintptr_t>(out_split8) & 15) == 0,
               "tt_preprocess_u8", "bad stem-plane geometry");
  if (out_split8)                                               // n_img padded slots of 8 halves must fit each plane (lo' starts split_plane on)
    TT_REQUIRE((long long)d->n_img * d->pad_H * d->pad_W * 8 <= split_plane, "tt_preprocess_u8",
               "n_img stem slots (n_img * pad_H * pad_W * 8 halves) exceed the stem-plane capacity split_plane");
  const long long total = (long long)d->n_img * d->outH * d->outW;
  if (total == 0) return TT_OK;
  const long long want = (total + 255) / 256;
  const int nb = (int)(want > tt_num_sms() * 16 ? tt_num_sms() * 16 : want);
  preprocess_u8_kernel<<<nb, 256, 0, (cudaStream_t)stream>>>(raw, reinterpret_cast<const float2*>(map_grid), out_nchw, static_cast<__half*>(out_split8),
                                                             split_plane, *d, total);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_preprocess_u8");
  return TT_OK;
}

int tt_lidar_stitch(const float* prev, int n_prev, const float* now, int n_now, const double* rel_mat, double z_add, float* out,
                    tt_stream_t stream) {
  TT_REQUIRE(out && n_prev >= 0 && n_now >= 0 && (n_prev == 0 || (prev && rel_mat)) && (n_now == 0 || now), "tt_lidar_stitch", "null argument");
  TT_REQUIRE(((reinterpret_cast<uintptr_t>(prev) | reinterpret_cast<uintptr_t>(now) | reinterpret_cast<uintptr_t>(out)) & 15) == 0, "tt_lidar_stitch",
             "point arrays must be 16-byte aligned ([n][4] floats)");
  const int n = n_prev + n_now;
  if (n == 0) return TT_OK;
  lidar_stitch_kernel<<<tt_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(prev, n_prev, now, n_now, rel_mat, z_add, out);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_lidar_stitch");
  return TT_OK;
}

int tt_points_union(const float* src, int n, const float* curr2key, float timestamp, float* dst, tt_stream_t stream) {
  TT_REQUIRE(n >= 0 && (n == 0 || (src && dst)) && (reinterpret_cast<uintptr_t>(src) & 15) == 0, "tt_points_union", "bad arguments ([n][4] floats, 16-byte aligned)");
  if (n == 0) return TT_OK;
  points_union_kernel<<<tt_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(src, n, curr2key, timestamp, dst);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_points_union");
  return TT_OK;
}

}  // extern "C"
