// Training-side dense convolution: torch.nn.Conv2d forward and backward (groups 1, stride 1 or 2) on channels_last fp32 tensors,
// every product on the 3xTF32 tensor cores.
//
//   forward    : weight -> [2][Cout][taps][Cin] hi / lo TF32 planes, then the implicit-GEMM conv (tt_conv2d_tc impl 3, no split-K), bias
//                in its epilogue;
//   grad_x     : grad_x[s q + p] = sum over the taps kh with (p + pad - kh dil) = 0 mod s of grad_y[(p + pad - kh dil) / s + q] w[kh]
//                (per dimension).  For each output phase (py, px) in [0, s)^2 the reaching taps are kh0, kh0 - step, ... (step =
//                s / gcd(s, dil)), so the phase is a stride-1 convolution of grad_y with the flipped, Cin / Cout-transposed sub-kernel,
//                dilation step dil / s, origin (p + pad - kh0 dil) / s, stored through the conv's pixel scatter (oy_mul = ox_mul = s,
//                oy_add = py, ox_add = px).  Stride 1 is the single phase (0, 0).  A phase no tap reaches is written as zeros; rows of
//                a phase whose taps all fall past grad_y read TMA's zero fill and come out zero;
//   grad_weight: per tap, grad_y^T x(tap-shifted) on the A-transposed GEMM's conv mode (tt_gemm_at_conv; a 1x1 stride-1 layer is
//                its plain mode), split over pixels and folded in a fixed order;
//   grad_bias  : per-channel column sums of grad_y over fixed row chunks, folded in chunk order.
// No floating-point atomics and no red.add split-K anywhere: every output is bitwise reproducible.
#include "common.cuh"

extern long long g_tt_launches;

int tt_conv2d_tc(const tt_conv_desc* d, const float* x, const float* w, const float* bias, const float* res,
                 const float* res2, float* y, void* workspace, cudaStream_t st, bool allow_split_k);
int tt_conv2d_tc_origin(const tt_conv_desc* d, int org_h, int org_w, const float* x, const float* w_tc, const float* bias, const float* res,
                        const float* res2, float* y, cudaStream_t st, bool allow_split_k);
size_t tt_gemm_at_workspace_bytes(int batch, int M, int N);
int tt_gemm_at(const float* A, int lda, long long a_batch, const float* B, int ldb, long long b_batch, float* Cm, int ldc, long long c_batch,
               int batch, int M, int N, int K, int accumulate, void* ws, size_t ws_bytes, cudaStream_t st);
int tt_gemm_at_conv(const float* gy, const float* x, float* gw, int n_img, int H, int W, int OH, int OW, int KH, int KW, int stride, int pad,
                    int dil, int M, int Cin, void* ws, size_t ws_bytes, cudaStream_t st);

namespace {

constexpr int BIAS_ROWS = 512, BIAS_CHUNKS = 1024;   // grad_bias: at least BIAS_ROWS rows per chunk, at most BIAS_CHUNKS chunks

TT_DEVICE float rn_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// one output phase of grad_x, per dimension: the first reaching tap k0, the tap count n, the origin and the phase's output extent
struct Dim {
  int k0, n, org, ext;
};
struct Phases {
  Dim h[2], w[2];
  long long off[4];   // floats from the start of the packed grad_x weights to phase (py, px) = ph / s, ph % s
  int s, step, dil;   // stride, tap step inside a phase, the phases' dilation
};

int gcd(int a, int b) { return b ? gcd(b, a % b) : a; }

Dim phase_dim(int p, int K, int s, int pad, int dil, int in_extent) {
  Dim r = {0, 0, 0, in_extent > p ? (in_extent - p + s - 1) / s : 0};
  for (int k = K - 1; k >= 0; --k)
    if ((((p + pad - k * dil) % s) + s) % s == 0) {
      if (r.n == 0) { r.k0 = k; r.org = (p + pad - k * dil) / s; }
      ++r.n;
    }
  return r;
}

Phases make_phases(const tt_conv2d_train_desc* d) {
  Phases P;
  P.s = d->stride;
  P.step = d->stride / gcd(d->stride, d->dil);
  P.dil = P.step * d->dil / d->stride;
  long long off = 0;
  for (int p = 0; p < P.s; ++p) {
    P.h[p] = phase_dim(p, d->KH, P.s, d->pad, d->dil, d->H);
    P.w[p] = phase_dim(p, d->KW, P.s, d->pad, d->dil, d->W);
  }
  for (int ph = 0; ph < P.s * P.s; ++ph) {
    P.off[ph] = off;
    off += 2LL * d->Cin * P.h[ph / P.s].n * P.w[ph % P.s].n * d->Cout;
  }
  return P;
}

// weight (Cout, Cin, KH, KW) -> forward planes wf [2][Cout][KH*KW][Cin] and, when wb, the grad_x planes of every phase:
// wb + off[ph] = [2][Cin][nh * nw][Cout], tap (jh, jw) of phase (py, px) = weight tap (kh0 - jh step, kw0 - jw step)
__global__ void c2t_pack_weight_kernel(const float* __restrict__ w, float* __restrict__ wf, float* __restrict__ wb, int Cout, int Cin, int KH,
                                       int KW, int pad, int dil, const Phases P) {
  const int taps = KH * KW;
  const long long total = (long long)Cout * Cin * taps, plane = total;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(e % taps), ci = (int)((e / taps) % Cin), co = (int)(e / ((long long)taps * Cin));
    const float v = w[e], hi = rn_tf32(v), lo = rn_tf32(v - hi);
    if (wf) {
      const long long i = ((long long)co * taps + t) * Cin + ci;
      wf[i] = hi;
      wf[plane + i] = lo;
    }
    if (wb) {
      const int kh = t / KW, kw = t - kh * KW;
      const int py = (((kh * dil - pad) % P.s) + P.s) % P.s, px = (((kw * dil - pad) % P.s) + P.s) % P.s;
      const Dim& dh = P.h[py];
      const Dim& dw = P.w[px];
      const int jh = (dh.k0 - kh) / P.step, jw = (dw.k0 - kw) / P.step, tp = dh.n * dw.n;
      float* b = wb + P.off[py * P.s + px];
      const long long i = ((long long)ci * tp + jh * dw.n + jw) * Cout + co;
      b[i] = hi;
      b[(long long)Cin * tp * Cout + i] = lo;
    }
  }
}

// grad_x pixels of the phases in `mask` (bit py * s + px) no tap reaches: zeros
__global__ void c2t_zero_phases_kernel(float* __restrict__ gx, int N, int H, int W, int C, int s, int mask) {
  const int C4 = C / 4;
  const long long total = (long long)N * H * W * C4;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long pix = e / C4;
    const int w = (int)(pix % W), h = (int)((pix / W) % H);
    if (mask >> ((h % s) * s + (w % s)) & 1) reinterpret_cast<float4*>(gx)[e] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// grad_bias, pass 1: part[g][c] = sum of gy[r][c] over chunk g's rows; 8 row lanes x 32 float4 columns, lanes added in lane order
__global__ void __launch_bounds__(256) c2t_bias_part_kernel(const float* __restrict__ gy, int P, int C, int rows_per, float* __restrict__ part) {
  __shared__ float4 red[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, c = (blockIdx.x * 32 + tx) * 4, g = blockIdx.y;
  const int r0 = g * rows_per, r1 = min(P, r0 + rows_per);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C)
    for (int r = r0 + ty; r < r1; r += 8) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(gy + (long long)r * C + c));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  red[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && c < C) {
    float4 s = red[0][tx];
    for (int q = 1; q < 8; ++q) { s.x += red[q][tx].x; s.y += red[q][tx].y; s.z += red[q][tx].z; s.w += red[q][tx].w; }
    *reinterpret_cast<float4*>(part + (long long)g * C + c) = s;
  }
}

// grad_bias, pass 2: gb[c] = part[0][c] + part[1][c] + ...  (in this order)
__global__ void c2t_bias_fold_kernel(const float* __restrict__ part, int chunks, int C, float* __restrict__ gb) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    float v = 0.f;
    for (int g = 0; g < chunks; ++g) v += part[(long long)g * C + c];
    gb[c] = v;
  }
}

int grid_for(long long total, int per_block) {
  const long long nb = (total + per_block - 1) / per_block, cap = (long long)tt_num_sms() * 32;
  return (int)(nb < 1 ? 1 : nb > cap ? cap : nb);
}

int bias_chunks(long long P) {
  const long long c = (P + BIAS_ROWS - 1) / BIAS_ROWS;
  return (int)(c < 1 ? 1 : c > BIAS_CHUNKS ? BIAS_CHUNKS : c);
}

// the workspace of one call, carved in 256-byte aligned pieces
struct Ws {
  float *wf, *wb, *part, *bpart;
  size_t part_bytes, bytes;
};
Ws carve(const tt_conv2d_train_desc* d, void* base) {
  const long long wsz = (long long)d->Cout * d->Cin * d->KH * d->KW;
  const size_t part = tt_gemm_at_workspace_bytes(d->KH * d->KW, d->Cout, d->Cin);
  const size_t sizes[4] = {(size_t)2 * wsz * 4, (size_t)2 * wsz * 4, part, (size_t)BIAS_CHUNKS * d->Cout * 4};
  Ws w;
  float** slots[4] = {&w.wf, &w.wb, &w.part, &w.bpart};
  size_t o = 0;
  for (int i = 0; i < 4; ++i) {
    *slots[i] = base ? reinterpret_cast<float*>(static_cast<char*>(base) + o) : nullptr;
    o += (sizes[i] + 255) / 256 * 256;
  }
  w.part_bytes = part;
  w.bytes = o;
  return w;
}

// refuses what the reference does not build, naming the parameter; touches no pointer and no device
int check_desc(const tt_conv2d_train_desc* d, const char* name) {
  if (!d) {
    tt_set_error("%s: null descriptor", name);
    return TT_ERR_INVALID;
  }
  const char* bad = nullptr;
  const long long oh = d->stride > 0 ? ((long long)d->H + 2LL * d->pad - (long long)d->dil * (d->KH - 1) - 1) / d->stride + 1 : 0;
  const long long ow = d->stride > 0 ? ((long long)d->W + 2LL * d->pad - (long long)d->dil * (d->KW - 1) - 1) / d->stride + 1 : 0;
  const long long lim = 1LL << 31;
  if (d->groups != 1) bad = "groups: only 1 is supported";
  else if (d->stride != 1 && d->stride != 2) bad = "stride: only 1 and 2 are supported";
  else if (d->Cin <= 0 || d->Cin % 4) bad = "Cin: must be a positive multiple of 4";
  else if (d->Cout <= 0 || d->Cout % 4) bad = "Cout: must be a positive multiple of 4";
  else if (d->KH < 1 || d->KW < 1) bad = "KH / KW: must be >= 1";
  else if (d->pad < 0) bad = "pad: must be >= 0";
  else if (d->dil < 1) bad = "dil: must be >= 1";
  else if (d->bias != 0 && d->bias != 1) bad = "bias: must be 0 or 1";
  else if (d->N < 0 || d->H < 1 || d->W < 1) bad = "N / H / W: N must be >= 0, H and W >= 1";
  else if (d->OH != oh || oh < 1) bad = "OH: does not match (H + 2 pad - dil (KH - 1) - 1) / stride + 1";
  else if (d->OW != ow || ow < 1) bad = "OW: does not match (W + 2 pad - dil (KW - 1) - 1) / stride + 1";
  else if ((long long)d->N * d->H * d->W * d->Cin >= lim || (long long)d->N * d->OH * d->OW * d->Cout >= lim)
    bad = "N: pixel x channel counts past 32-bit indexing";
  else if ((long long)d->Cout * d->Cin * d->KH * d->KW * 16 >= lim) bad = "KH / KW: weight element count past 32-bit indexing";
  if (bad) {
    tt_set_error("%s: unsupported %s", name, bad);
    return TT_ERR_UNSUPPORTED;
  }
  return TT_OK;
}

int check_ws(const tt_conv2d_train_desc* d, size_t ws_bytes, const char* name) {
  if (ws_bytes < carve(d, nullptr).bytes) {
    tt_set_error("%s: unsupported ws_bytes: smaller than tt_conv2d_train_workspace_bytes", name);
    return TT_ERR_UNSUPPORTED;
  }
  return TT_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

tt_conv_desc tc_desc(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, int OH, int OW) {
  tt_conv_desc c = {};
  c.N = N; c.H = H; c.W = W; c.Cin = Cin; c.x_ld = Cin;
  c.Cout = Cout; c.KH = KH; c.KW = KW; c.stride = stride; c.pad = pad; c.dil = dil; c.groups = 1;
  c.OH = OH; c.OW = OW; c.y_ld = Cout; c.yH = OH; c.yW = OW;
  c.oy_mul = c.ox_mul = 1; c.act = TT_ACT_NONE; c.impl = 3;
  return c;
}

#define C2T_CALL(expr)                   \
  do {                                   \
    const int rc__ = (expr);             \
    if (rc__ != TT_OK) return rc__;      \
  } while (0)

}  // namespace

extern "C" size_t tt_conv2d_train_workspace_bytes(const tt_conv2d_train_desc* d) {
  if (check_desc(d, "tt_conv2d_train_workspace_bytes") != TT_OK) return 0;
  return carve(d, nullptr).bytes;
}

extern "C" int tt_conv2d_train_forward(const tt_conv2d_train_desc* d, const float* x, const float* weight, const float* bias, float* y,
                                       void* ws, size_t ws_bytes, tt_stream_t stream) {
  static const char* name = "tt_conv2d_train_forward";
  C2T_CALL(check_desc(d, name));
  C2T_CALL(check_ws(d, ws_bytes, name));
  if (d->N == 0) return TT_OK;
  TT_REQUIRE(x && weight && y && ws && (bias || !d->bias), name, "null argument");
  TT_REQUIRE(aligned16(x) && aligned16(y) && aligned16(ws) && (!bias || aligned16(bias)), name, "x, y, bias and ws must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const Ws w = carve(d, ws);
  const Phases P = make_phases(d);
  c2t_pack_weight_kernel<<<grid_for((long long)d->Cout * d->Cin * d->KH * d->KW, 256), 256, 0, st>>>(weight, w.wf, nullptr, d->Cout, d->Cin,
                                                                                                       d->KH, d->KW, d->pad, d->dil, P);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  const tt_conv_desc c = tc_desc(d->N, d->H, d->W, d->Cin, d->Cout, d->KH, d->KW, d->stride, d->pad, d->dil, d->OH, d->OW);
  return tt_conv2d_tc(&c, x, w.wf, d->bias ? bias : nullptr, nullptr, nullptr, y, nullptr, st, false);
}

extern "C" int tt_conv2d_train_backward(const tt_conv2d_train_desc* d, const float* x, const float* weight, const float* grad_y,
                                        float* grad_x, float* grad_weight, float* grad_bias, void* ws, size_t ws_bytes, tt_stream_t stream) {
  static const char* name = "tt_conv2d_train_backward";
  C2T_CALL(check_desc(d, name));
  C2T_CALL(check_ws(d, ws_bytes, name));
  if (!d->bias) grad_bias = nullptr;
  if (!grad_x && !grad_weight && !grad_bias) return TT_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const long long wsz = (long long)d->Cout * d->Cin * d->KH * d->KW;
  if (d->N == 0) {   // an empty batch: zero gradients, no kernel
    if ((grad_weight && cudaMemsetAsync(grad_weight, 0, (size_t)wsz * 4, st) != cudaSuccess) ||
        (grad_bias && cudaMemsetAsync(grad_bias, 0, (size_t)d->Cout * 4, st) != cudaSuccess)) {
      tt_set_error("%s: memset failed", name);
      return TT_ERR_CUDA;
    }
    return TT_OK;
  }
  TT_REQUIRE(grad_y && ws && (!grad_x || weight) && (!grad_weight || x), name, "null argument");
  TT_REQUIRE(aligned16(grad_y) && aligned16(ws) && (!grad_x || aligned16(grad_x)) && (!grad_weight || aligned16(x)) &&
                 (!grad_bias || aligned16(grad_bias)),
             name, "x, grad_y, grad_x, grad_bias and ws must be 16-byte aligned");
  const Ws w = carve(d, ws);
  const long long P = (long long)d->N * d->OH * d->OW;
  if (grad_x) {
    const Phases ph = make_phases(d);
    c2t_pack_weight_kernel<<<grid_for(wsz, 256), 256, 0, st>>>(weight, nullptr, w.wb, d->Cout, d->Cin, d->KH, d->KW, d->pad, d->dil, ph);
    ++g_tt_launches;
    TT_CHECK_LAUNCH(name);
    int empty = 0;
    for (int q = 0; q < ph.s * ph.s; ++q) {
      const Dim& dh = ph.h[q / ph.s];
      const Dim& dw = ph.w[q % ph.s];
      if (dh.ext == 0 || dw.ext == 0) continue;                 // no grad_x pixel in this phase
      if (dh.n == 0 || dw.n == 0) { empty |= 1 << q; continue; }
      tt_conv_desc c = tc_desc(d->N, d->OH, d->OW, d->Cout, d->Cin, dh.n, dw.n, 1, 0, ph.dil, dh.ext, dw.ext);
      c.yH = d->H; c.yW = d->W;
      c.oy_mul = c.ox_mul = ph.s; c.oy_add = q / ph.s; c.ox_add = q % ph.s;
      C2T_CALL(tt_conv2d_tc_origin(&c, dh.org, dw.org, grad_y, w.wb + ph.off[q], nullptr, nullptr, nullptr, grad_x, st, false));
    }
    if (empty) {
      c2t_zero_phases_kernel<<<grid_for((long long)d->N * d->H * d->W * (d->Cin / 4), 256), 256, 0, st>>>(grad_x, d->N, d->H, d->W, d->Cin,
                                                                                                          ph.s, empty);
      ++g_tt_launches;
      TT_CHECK_LAUNCH(name);
    }
  }
  if (grad_weight) {
    if (d->KH == 1 && d->KW == 1 && d->stride == 1 && d->pad == 0) {   // pixel k of grad_y meets pixel k of x: the plain contraction
      C2T_CALL(tt_gemm_at(grad_y, d->Cout, 0, x, d->Cin, 0, grad_weight, d->Cin, 0, 1, d->Cout, d->Cin, (int)P, 0, w.part, w.part_bytes, st));
    } else {
      C2T_CALL(tt_gemm_at_conv(grad_y, x, grad_weight, d->N, d->H, d->W, d->OH, d->OW, d->KH, d->KW, d->stride, d->pad, d->dil, d->Cout,
                               d->Cin, w.part, w.part_bytes, st));
    }
  }
  if (grad_bias) {
    const int chunks = bias_chunks(P), rows_per = (int)((P + chunks - 1) / chunks);
    c2t_bias_part_kernel<<<dim3(tt_cdiv(d->Cout, 128), chunks), 256, 0, st>>>(grad_y, (int)P, d->Cout, rows_per, w.bpart);
    ++g_tt_launches;
    TT_CHECK_LAUNCH(name);
    c2t_bias_fold_kernel<<<tt_cdiv(d->Cout, 256), 256, 0, st>>>(w.bpart, chunks, d->Cout, grad_bias);
    ++g_tt_launches;
    TT_CHECK_LAUNCH(name);
  }
  return TT_OK;
}
