// Memory-bound helpers: layout changes, pooling, interpolation, SE gates, LayerNorm, small glue.
// All tensors fp32 channels-last; threads are mapped so the channel dimension is contiguous across a
// warp (coalesced, 128-bit where the channel count allows).
#include "common.cuh"

extern long long g_tt_launches;
#define TT_LAUNCHED(name) do { ++g_tt_launches; TT_CHECK_LAUNCH(name); } while (0)

namespace {

constexpr int TPB = 256;
inline int blocks_for(long long n, int cap = tt_num_sms() * 16) {
  long long b = (n + TPB - 1) / TPB;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// ---- NCHW <-> NHWC through a 32x32 shared-memory transpose tile (both sides coalesced)
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int HW, int y_ld,
                                    int y_coff, int cpad, int W, int out_W, long long out_HW, int top, int left) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, p = p0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && p < HW) ? x[((long long)n * C + c) * HW + p] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int p = p0 + i, c = c0 + threadIdx.x;
    if (p < HW && c < cpad) {
      const int h = p / W, w = p - h * W;                        // destination may be a larger (zero-bordered) image
      y[((long long)n * out_HW + (long long)(h + top) * out_W + w + left) * y_ld + y_coff + c] = tile[threadIdx.x][i];
    }
  }
}

__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, int x_ld, int x_coff, float* __restrict__ y, int C,
                                    int HW) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int p = p0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (p < HW && c < C) ? x[((long long)n * HW + p) * x_ld + x_coff + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, p = p0 + threadIdx.x;
    if (c < C && p < HW) y[((long long)n * C + c) * HW + p] = tile[threadIdx.x][i];
  }
}

__global__ void maxpool3x3s2_kernel(const float4* __restrict__ x, float4* __restrict__ y, int N, int H, int W, int C4,
                                    int OH, int OW) {
  const long long total = (long long)N * OH * OW * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % C4;
    long long t = i / C4;
    const int ow = t % OW; t /= OW;
    const int oh = t % OH;
    const int n = t / OH;
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
    for (int dh = 0; dh < 3; ++dh) {
      const int ih = oh * 2 - 1 + dh;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int dw = 0; dw < 3; ++dw) {
        const int iw = ow * 2 - 1 + dw;
        if (iw < 0 || iw >= W) continue;
        const float4 v = __ldg(&x[((long long)(n * H + ih) * W + iw) * C4 + c]);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
    y[i] = m;
  }
}

__global__ void upsample2x_ac_kernel(const float4* __restrict__ x, float4* __restrict__ y, int N, int H, int W, int C4) {
  const int OH = 2 * H, OW = 2 * W;
  const float sh = OH > 1 ? (float)(H - 1) / (float)(OH - 1) : 0.f;
  const float sw = OW > 1 ? (float)(W - 1) / (float)(OW - 1) : 0.f;
  const long long total = (long long)N * OH * OW * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % C4;
    long long t = i / C4;
    const int ow = t % OW; t /= OW;
    const int oh = t % OH;
    const int n = t / OH;
    const float fy = sh * oh, fx = sw * ow;                     // align_corners=True source index
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
    const float4 a = __ldg(&x[((long long)(n * H + y0) * W + x0) * C4 + c]);
    const float4 b = __ldg(&x[((long long)(n * H + y0) * W + x1) * C4 + c]);
    const float4 cc = __ldg(&x[((long long)(n * H + y1) * W + x0) * C4 + c]);
    const float4 dd = __ldg(&x[((long long)(n * H + y1) * W + x1) * C4 + c]);
    float4 r;
    r.x = hy * (hx * a.x + lx * b.x) + ly * (hx * cc.x + lx * dd.x);
    r.y = hy * (hx * a.y + lx * b.y) + ly * (hx * cc.y + lx * dd.y);
    r.z = hy * (hx * a.z + lx * b.z) + ly * (hx * cc.z + lx * dd.z);
    r.w = hy * (hx * a.w + lx * b.w) + ly * (hx * cc.w + lx * dd.w);
    y[i] = r;
  }
}

// one CTA per (n, 32-channel slab): threads = 32 channels x 8 pixel lanes
__global__ void pool_hw_kernel(const float* __restrict__ x, int x_ld, int x_coff, float* __restrict__ y, int HW, int C,
                               float wmean, float wmax) {
  __shared__ float ssum[8][33], smax[8][33];
  const int n = blockIdx.y;
  const int c = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f, m = -INFINITY;
  if (c < C)
    for (int p = threadIdx.y; p < HW; p += 8) {
      const float v = x[((long long)n * HW + p) * x_ld + x_coff + c];
      s += v;
      m = fmaxf(m, v);
    }
  ssum[threadIdx.y][threadIdx.x] = s;
  smax[threadIdx.y][threadIdx.x] = m;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
#pragma unroll
    for (int i = 1; i < 8; ++i) { s += ssum[i][threadIdx.x]; m = fmaxf(m, smax[i][threadIdx.x]); }
    y[(long long)n * C + c] = wmean * (s / (float)HW) + (wmax != 0.f ? wmax * m : 0.f);
  }
}

__global__ void broadcast_rows_kernel(const float* __restrict__ v, float* __restrict__ y, int HW, int C, int y_ld,
                                      int y_coff, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % C;
    const long long pix = i / C;
    const int n = pix / HW;
    y[pix * y_ld + y_coff + c] = v[(long long)n * C + c];
  }
}

__global__ void se_gate_kernel(const float4* __restrict__ x, const float4* __restrict__ g, float4* __restrict__ y, int HW,
                               int C4, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % C4;
    const int n = (i / C4) / HW;
    const float4 a = x[i];
    const float4 s = __ldg(&g[(long long)n * C4 + c]);
    y[i] = make_float4(a.x * tt_act(s.x, TT_ACT_SIGMOID), a.y * tt_act(s.y, TT_ACT_SIGMOID),
                       a.z * tt_act(s.z, TT_ACT_SIGMOID), a.w * tt_act(s.w, TT_ACT_SIGMOID));
  }
}

__global__ void se_apply_kernel(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ sc,
                                int sc_ld, int sc_coff, float* __restrict__ y, int y_ld, int y_coff, int HW, int C,
                                long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % C;
    const long long pix = i / C;
    const int n = pix / HW;
    const float v = x[i] * tt_act(g[(long long)n * C + c], TT_ACT_SIGMOID) + sc[pix * sc_ld + sc_coff + c];
    y[pix * y_ld + y_coff + c] = v > 0.f ? v : 0.f;
  }
}

__global__ void anti_transpose_kernel(const float* __restrict__ x, float* __restrict__ y, int S, int C, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % C;
    long long t = i / C;
    const int j = t % S; t /= S;
    const int ii = t % S;
    const int n = t / S;
    y[i] = x[(((long long)n * S + (S - 1 - j)) * S + (S - 1 - ii)) * C + c];
  }
}

__global__ void copy2d_kernel(const float* __restrict__ src, int src_ld, float* __restrict__ dst, int dst_ld, int cols,
                              int rdiv, int rmod, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % cols;
    const long long r = i / cols;
    const long long sr = (r / rdiv) % rmod;
    dst[r * dst_ld + c] = src[sr * src_ld + c];
  }
}

// one warp per row, two-pass (mean, then centred variance) like torch's LayerNorm
__global__ void layernorm_kernel(const float* __restrict__ x, int x_ld, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, float* __restrict__ y, int y_ld, int rows, int D,
                                 const int* __restrict__ row_count) {
  const int warps = blockDim.x / 32;
  const int row = blockIdx.x * warps + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  int R = rows;
  if (row_count) R = min(R, *row_count);
  if (row >= R) return;
  const float* xr = x + (long long)row * x_ld;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) s += xr[i];
  const float mean = warp_sum(s) / (float)D;
  float v = 0.f;
  for (int i = lane; i < D; i += 32) { const float t = xr[i] - mean; v += t * t; }
  const float rstd = rsqrtf(warp_sum(v) / (float)D + 1e-5f);
  float* yr = y + (long long)row * y_ld;
  for (int i = lane; i < D; i += 32) yr[i] = (xr[i] - mean) * rstd * gamma[i] + beta[i];
}

__global__ void eltwise_kernel(int op, int act, const float* __restrict__ a, int a_ld, const float* __restrict__ b,
                               int b_ld, const float* __restrict__ c, int c_ld, float* __restrict__ y, int y_ld, int cols,
                               long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int col = i % cols;
    const long long r = i / cols;
    const float av = a[r * a_ld + col];
    float v;
    switch (op) {
      case 0: v = av + b[r * b_ld + col]; break;
      case 1: v = (1.f - av) * b[r * b_ld + col]; break;
      case 2: v = (1.f - av) * b[r * b_ld + col] + av * c[r * c_ld + col]; break;
      case 4: v = av + logf(-expm1f(-av)); break;               // inverse softplus (thinktwice_decoder.py:22-23)
      default: v = av; break;
    }
    y[r * y_ld + col] = tt_act(v, act);
  }
}

__global__ void fill_kernel(float* __restrict__ y, float v, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) y[i] = v;
}

__global__ void gru_input_kernel(const float* __restrict__ wp, const float* __restrict__ ctrl, int t, int T, float* buf,
                                 int ld, int HW, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % 6;
    const long long pix = i / 6;
    const int b = pix / HW;
    const float v = c < 2 ? wp[((long long)b * T + t) * 2 + c] : ctrl[((long long)b * T + t) * 4 + (c - 2)];
    buf[pix * ld + c] = v;
  }
}

}  // namespace

extern "C" {

int tt_nchw_to_nhwc(const float* x, float* y, int N, int C, int H, int W, int y_ld, int y_coff, int cpad,
                    tt_stream_t stream) {
  TT_REQUIRE(x && y && cpad >= C, "tt_nchw_to_nhwc", "bad arguments");
  dim3 grid(tt_cdiv((long long)H * W, 32), tt_cdiv(cpad, 32), N), block(32, 8);
  nchw_to_nhwc_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, y, C, H * W, y_ld, y_coff, cpad, W, W, (long long)H * W, 0, 0);
  TT_LAUNCHED("tt_nchw_to_nhwc");
  return TT_OK;
}

int tt_nchw_to_nhwc_padded(const float* x, float* y, int N, int C, int H, int W, int y_ld, int cpad, int out_H, int out_W,
                           int top, int left, tt_stream_t stream) {
  TT_REQUIRE(x && y && cpad >= C && top >= 0 && left >= 0 && top + H <= out_H && left + W <= out_W, "tt_nchw_to_nhwc_padded",
             "bad arguments");
  dim3 grid(tt_cdiv((long long)H * W, 32), tt_cdiv(cpad, 32), N), block(32, 8);
  nchw_to_nhwc_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, y, C, H * W, y_ld, 0, cpad, W, out_W, (long long)out_H * out_W,
                                                                top, left);
  TT_LAUNCHED("tt_nchw_to_nhwc_padded");
  return TT_OK;
}

int tt_nhwc_to_nchw(const float* x, int x_ld, int x_coff, float* y, int N, int C, int H, int W, tt_stream_t stream) {
  TT_REQUIRE(x && y, "tt_nhwc_to_nchw", "null argument");
  dim3 grid(tt_cdiv((long long)H * W, 32), tt_cdiv(C, 32), N), block(32, 8);
  nhwc_to_nchw_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, x_ld, x_coff, y, C, H * W);
  TT_LAUNCHED("tt_nhwc_to_nchw");
  return TT_OK;
}

int tt_maxpool3x3s2(const float* x, float* y, int N, int H, int W, int C, tt_stream_t stream) {
  TT_REQUIRE(x && y && C % 4 == 0, "tt_maxpool3x3s2", "C must be a multiple of 4");
  const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1;
  const long long total = (long long)N * OH * OW * (C / 4);
  maxpool3x3s2_kernel<<<blocks_for(total), TPB, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), N, H, W, C / 4, OH, OW);
  TT_LAUNCHED("tt_maxpool3x3s2");
  return TT_OK;
}

int tt_upsample2x_bilinear_ac(const float* x, float* y, int N, int H, int W, int C, tt_stream_t stream) {
  TT_REQUIRE(x && y && C % 4 == 0, "tt_upsample2x_bilinear_ac", "C must be a multiple of 4");
  const long long total = (long long)N * 4 * H * W * (C / 4);
  upsample2x_ac_kernel<<<blocks_for(total), TPB, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), N, H, W, C / 4);
  TT_LAUNCHED("tt_upsample2x_bilinear_ac");
  return TT_OK;
}

int tt_global_avgpool(const float* x, int x_ld, int x_coff, float* y, int N, int HW, int C, tt_stream_t stream) {
  TT_REQUIRE(x && y, "tt_global_avgpool", "null argument");
  dim3 grid(tt_cdiv(C, 32), N), block(32, 8);
  pool_hw_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, x_ld, x_coff, y, HW, C, 1.f, 0.f);
  TT_LAUNCHED("tt_global_avgpool");
  return TT_OK;
}

int tt_se_pool(const float* x, float* s, int N, int HW, int C, tt_stream_t stream) {
  TT_REQUIRE(x && s, "tt_se_pool", "null argument");
  dim3 grid(tt_cdiv(C, 32), N), block(32, 8);
  pool_hw_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, C, 0, s, HW, C, 0.5f, 0.5f);
  TT_LAUNCHED("tt_se_pool");
  return TT_OK;
}

int tt_broadcast_rows(const float* v, float* y, int N, int HW, int C, int y_ld, int y_coff, tt_stream_t stream) {
  TT_REQUIRE(v && y, "tt_broadcast_rows", "null argument");
  const long long total = (long long)N * HW * C;
  broadcast_rows_kernel<<<blocks_for(total), TPB, 0, (cudaStream_t)stream>>>(v, y, HW, C, y_ld, y_coff, total);
  TT_LAUNCHED("tt_broadcast_rows");
  return TT_OK;
}

int tt_se_gate(const float* x, const float* g, float* y, int N, int HW, int C, tt_stream_t stream) {
  TT_REQUIRE(x && g && y && C % 4 == 0, "tt_se_gate", "C must be a multiple of 4");
  const long long total = (long long)N * HW * (C / 4);
  se_gate_kernel<<<blocks_for(total), TPB, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(g), reinterpret_cast<float4*>(y), HW, C / 4, total);
  TT_LAUNCHED("tt_se_gate");
  return TT_OK;
}

int tt_se_apply(const float* x, const float* g, const float* shortcut, int sc_ld, int sc_coff, float* y, int y_ld,
                int y_coff, int N, int HW, int C, tt_stream_t stream) {
  TT_REQUIRE(x && g && shortcut && y, "tt_se_apply", "null argument");
  const long long total = (long long)N * HW * C;
  se_apply_kernel<<<blocks_for(total), TPB, 0, (cudaStream_t)stream>>>(x, g, shortcut, sc_ld, sc_coff, y, y_ld, y_coff, HW, C, total);
  TT_LAUNCHED("tt_se_apply");
  return TT_OK;
}

int tt_anti_transpose(const float* x, float* y, int N, int S, int C, tt_stream_t stream) {
  TT_REQUIRE(x && y && x != y, "tt_anti_transpose", "needs distinct buffers");
  const long long total = (long long)N * S * S * C;
  anti_transpose_kernel<<<blocks_for(total), TPB, 0, (cudaStream_t)stream>>>(x, y, S, C, total);
  TT_LAUNCHED("tt_anti_transpose");
  return TT_OK;
}

int tt_copy2d(const float* src, int src_ld, float* dst, int dst_ld, int rows, int cols, int rdiv, int rmod,
              tt_stream_t stream) {
  TT_REQUIRE(src && dst && rdiv >= 1 && rmod >= 1, "tt_copy2d", "bad arguments");
  const long long total = (long long)rows * cols;
  if (total == 0) return TT_OK;
  copy2d_kernel<<<blocks_for(total), TPB, 0, (cudaStream_t)stream>>>(src, src_ld, dst, dst_ld, cols, rdiv, rmod, total);
  TT_LAUNCHED("tt_copy2d");
  return TT_OK;
}

int tt_layernorm(const float* x, int x_ld, const float* gamma, const float* beta, float* y, int y_ld, int rows, int D,
                 const int* row_count, tt_stream_t stream) {
  TT_REQUIRE(x && gamma && beta && y, "tt_layernorm", "null argument");
  if (rows == 0) return TT_OK;
  layernorm_kernel<<<tt_cdiv(rows, 8), 256, 0, (cudaStream_t)stream>>>(x, x_ld, gamma, beta, y, y_ld, rows, D, row_count);
  TT_LAUNCHED("tt_layernorm");
  return TT_OK;
}

int tt_eltwise(int op, int act, const float* a, int a_ld, const float* b, int b_ld, const float* c, int c_ld, float* y,
               int y_ld, int rows, int cols, tt_stream_t stream) {
  TT_REQUIRE(a && y && op >= 0 && op <= 4, "tt_eltwise", "bad arguments");
  TT_REQUIRE(op >= 3 || b, "tt_eltwise", "operand b missing");
  TT_REQUIRE(op != 2 || c, "tt_eltwise", "operand c missing");
  const long long total = (long long)rows * cols;
  if (total == 0) return TT_OK;
  eltwise_kernel<<<blocks_for(total), TPB, 0, (cudaStream_t)stream>>>(op, act, a, a_ld, b, b_ld, c, c_ld, y, y_ld, cols, total);
  TT_LAUNCHED("tt_eltwise");
  return TT_OK;
}

int tt_fill(float* y, float v, long long n, tt_stream_t stream) {
  TT_REQUIRE(y, "tt_fill", "null argument");
  if (n == 0) return TT_OK;
  fill_kernel<<<blocks_for(n), TPB, 0, (cudaStream_t)stream>>>(y, v, n);
  TT_LAUNCHED("tt_fill");
  return TT_OK;
}

int tt_gru_input(const float* wp, const float* ctrl_sp, int t, int T, float* buf, int ld, int B, int HW,
                 tt_stream_t stream) {
  TT_REQUIRE(wp && ctrl_sp && buf, "tt_gru_input", "null argument");
  const long long total = (long long)B * HW * 6;
  gru_input_kernel<<<blocks_for(total), TPB, 0, (cudaStream_t)stream>>>(wp, ctrl_sp, t, T, buf, ld, HW, total);
  TT_LAUNCHED("tt_gru_input");
  return TT_OK;
}

}  // extern "C"
