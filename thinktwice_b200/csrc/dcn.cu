// Deformable convolution v1 column builder (mmcv DeformConv2dPack, lss.py:189-197).
// One thread = 4 channels of one (pixel, tap): the four bilinear corners are 128-bit channels-last
// loads, the column row is written grouped as [pixel][group][tap][C/groups] so the following grouped
// GEMM (tt_conv2d, KH=KW=1, Cin = 9*C, groups) sees one contiguous K range per group.
#include "common.cuh"

extern long long g_tt_launches;

namespace {

__global__ void dcn_im2col_kernel(const float* __restrict__ x, const float* __restrict__ off, int off_ld,
                                  float* __restrict__ col, int N, int H, int W, int C, int G, long long total) {
  const int C4 = C / 4, Cg = C / G;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    long long t = i / C4;
    const int tap = t % 9;
    const long long m = t / 9;
    const int wo = m % W;
    const int ho = (m / W) % H;
    const int n = m / ((long long)W * H);
    const float oh = __ldg(off + m * off_ld + 2 * tap), ow = __ldg(off + m * off_ld + 2 * tap + 1);
    const float h = (float)(ho - 1 + tap / 3) + oh;
    const float w = (float)(wo - 1 + tap % 3) + ow;
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    if (h > -1.f && w > -1.f && h < (float)H && w < (float)W) {
      const int hl = (int)floorf(h), wl = (int)floorf(w);
      const int hh = hl + 1, wh = wl + 1;
      const float lh = h - hl, lw = w - wl, uh = 1.f - lh, uw = 1.f - lw;
      const float4* base = reinterpret_cast<const float4*>(x) + (long long)n * H * W * C4 + c4;
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 v1 = (hl >= 0 && wl >= 0) ? __ldg(base + ((long long)hl * W + wl) * C4) : z;
      const float4 v2 = (hl >= 0 && wh <= W - 1) ? __ldg(base + ((long long)hl * W + wh) * C4) : z;
      const float4 v3 = (hh <= H - 1 && wl >= 0) ? __ldg(base + ((long long)hh * W + wl) * C4) : z;
      const float4 v4 = (hh <= H - 1 && wh <= W - 1) ? __ldg(base + ((long long)hh * W + wh) * C4) : z;
      const float w1 = uh * uw, w2 = uh * lw, w3 = lh * uw, w4 = lh * lw;
      r.x = w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x;
      r.y = w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y;
      r.z = w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z;
      r.w = w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w;
    }
    const int c = c4 * 4, g = c / Cg, cg = c - g * Cg;
    *reinterpret_cast<float4*>(col + ((m * G + g) * 9 + tap) * Cg + cg) = r;
  }
}

}  // namespace

extern "C" int tt_dcn_im2col(const float* x, const float* offset, int off_ld, float* col, int N, int H, int W, int C,
                             int groups, tt_stream_t stream) {
  TT_REQUIRE(x && offset && col, "tt_dcn_im2col", "null argument");
  TT_REQUIRE(C % 4 == 0 && groups >= 1 && C % groups == 0 && (C / groups) % 4 == 0, "tt_dcn_im2col", "bad channels");
  const long long total = (long long)N * H * W * 9 * (C / 4);
  if (total == 0) return TT_OK;
  const long long nb = (total + 255) / 256;
  dcn_im2col_kernel<<<(int)(nb > tt_num_sms() * 32 ? tt_num_sms() * 32 : nb), 256, 0, (cudaStream_t)stream>>>(x, offset, off_ld, col, N, H, W,
                                                                                         C, groups, total);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_dcn_im2col");
  return TT_OK;
}
