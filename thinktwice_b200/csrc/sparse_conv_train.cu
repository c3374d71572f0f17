// Training-side sparse convolution: spconv 2.x SubMConv3d / SparseConv3d forward and backward (mmdet3d SparseEncoder,
// lidarnet.py:24-58, cfg thinktwice.py:167-176) on fp32 rows and the rulebook's tap-major pair lists.
//
//   forward    : y = sum_t W_t x[pairs_in]   on tt_sparse_conv (3xTF32 gather-GEMM, or fp32 SIMT for thin layers), red.add over taps;
//   grad_input : the same kernel with pairs_in / pairs_out swapped and every W_t transposed: for one tap the map between input and
//                output rows is one-to-one both ways, so the rows of one tap stay distinct;
//   grad_weight: per tap, gy[pairs_out]^T x[pairs_in] on the gathered A-transposed GEMM (tt_gemm_at_gather, 3xTF32), or an fp32
//                SIMT kernel when rows are not float4-addressable (conv_input's 5 channels); both fold their K pieces in a fixed
//                order, so grad_weight is bitwise reproducible over the ordered pair lists of tt_sparse_pairs_ordered.
// The weight is repacked by a kernel inside every call (it changes every optimiser step), as in deform_conv.cu.
#include <cub/block/block_scan.cuh>

#include "common.cuh"

extern long long g_tt_launches;

bool tt_sparse_conv_tc_supported(const tt_sparse_conv_desc* d, const void* x, const void* w, const void* y);
size_t tt_gemm_at_workspace_bytes(int batch, int M, int N);
int tt_gemm_at_gather(const float* A, int lda, const int* rows_a, const float* B, int ldb, const int* rows_b, const int* count, int pair_cap,
                      float* Cm, int ldc, long long c_batch, int batch, int M, int N, void* ws, size_t ws_bytes, cudaStream_t st);

namespace {

constexpr int MAX_KVOL = 32, WG_SPLITS = 16, PCH = 256;   // PCH: output rows per chunk of the ordered compaction

TT_DEVICE float rn_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// weight (Cout, kvol, Cin) -> the operand layout of tt_sparse_conv for the forward (dir 0) or grad_input (dir 1):
//   tensor cores: [2][Cout][kvol][Cin] (dir 0) / [2][Cin][kvol][Cout] (dir 1) hi / lo TF32 planes;
//   SIMT:         [kvol][Cin][Cout]    (dir 0) / [kvol][Cout][Cin]    (dir 1) fp32.
__global__ void sc_pack_weight_kernel(const float* __restrict__ w, float* __restrict__ dst, int Cout, int kvol, int Cin, int tc, int dir) {
  const long long total = (long long)Cout * kvol * Cin;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % Cin), t = (int)((e / Cin) % kvol), co = (int)(e / ((long long)Cin * kvol));
    const float v = w[e];
    if (tc) {
      const float hi = rn_tf32(v), lo = rn_tf32(v - hi);
      const long long i = dir ? ((long long)c * kvol + t) * Cout + co : e;
      dst[i] = hi;
      dst[total + i] = lo;
    } else {
      dst[dir ? ((long long)t * Cout + co) * Cin + c : ((long long)t * Cin + c) * Cout + co] = v;
    }
  }
}

// fp32 weight gradient of one (K piece, tap): part[s][t][i][j] = sum over the piece's pairs k of gy[pout[k]][i] * x[pin[k]][j].
// Threads split the piece into G interleaved lanes per element and the lanes are added in lane order: a fixed order.
__global__ void __launch_bounds__(256) sc_wgrad_simt_kernel(const float* __restrict__ gy, int gy_ld, const float* __restrict__ x, int x_ld,
                                                            const int* __restrict__ pin, const int* __restrict__ pout,
                                                            const int* __restrict__ pcount, int pair_cap, int Cout, int Cin, int kvol,
                                                            float* __restrict__ part) {
  __shared__ float red[256];
  const int s = blockIdx.x, t = blockIdx.y, splits = gridDim.x, tid = threadIdx.x;
  const int K = min(pcount[t], pair_cap), per = (K + splits - 1) / splits, kb = s * per, ke = min(K, kb + per);
  const int MN = Cout * Cin, G = MN >= 256 ? 1 : 256 / MN, E = G > 1 ? MN : 256;
  const int* pi = pin + (long long)t * pair_cap;
  const int* po = pout + (long long)t * pair_cap;
  float* out = part + ((long long)s * kvol + t) * MN;
  for (int e0 = 0; e0 < MN; e0 += E) {
    const int g = tid / E, e = e0 + tid % E;
    float acc = 0.f;
    if (g < G && e < MN) {
      const int i = e / Cin, j = e - (e / Cin) * Cin;
      for (int k = kb + g; k < ke; k += G) acc += __ldg(gy + (long long)__ldg(po + k) * gy_ld + i) * __ldg(x + (long long)__ldg(pi + k) * x_ld + j);
    }
    red[tid] = acc;
    __syncthreads();
    if (tid < E && e0 + tid < MN) {
      float v = 0.f;
      for (int q = 0; q < G; ++q) v += red[q * E + tid];
      out[e0 + tid] = v;
    }
    __syncthreads();
  }
}

// grad_weight (Cout, kvol, Cin)[i][t][j] = part[0][t][i][j] + part[1][t][i][j] + ...  (in this order)
__global__ void sc_wgrad_fold_kernel(const float* __restrict__ part, int splits, int kvol, int Cout, int Cin, float* __restrict__ gw) {
  const long long MN = (long long)Cout * Cin, total = kvol * MN;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(e % Cin), t = (int)((e / Cin) % kvol), i = (int)(e / ((long long)Cin * kvol));
    const long long src = (long long)t * MN + (long long)i * Cin + j;
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += part[s * total + src];
    gw[e] = v;
  }
}

// ---------------------------------------------------------------- ordered pair lists from the neighbour table
// A block owns PCH output rows and stages their nbr rows (coalesced); per tap it scans the hit flags of its rows.
// pass 0 writes the per-(tap, chunk) hit counts; pass 1 (after sc_pairs_scan_kernel turned them into offsets) writes the pairs.
template <bool WRITE>
__global__ void __launch_bounds__(PCH) sc_pairs_chunk_kernel(const int* __restrict__ nbr, const int* __restrict__ out_count, int cap_out,
                                                             int kvol, int n_chunks, int* __restrict__ cnt, int pair_cap,
                                                             int* __restrict__ pairs_in, int* __restrict__ pairs_out) {
  typedef cub::BlockScan<int, PCH> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int tile[PCH * MAX_KVOL];
  const int c = blockIdx.x, tid = threadIdx.x;
  const int n = min(*out_count, cap_out), o0 = c * PCH, rows = max(0, min(PCH, n - o0));
  for (int e = tid; e < rows * kvol; e += PCH) tile[e] = nbr[(long long)o0 * kvol + e];
  __syncthreads();
  for (int t = 0; t < kvol; ++t) {
    const int r = tid < rows ? tile[tid * kvol + t] : -1;
    int pos, total;
    Scan(tmp).ExclusiveSum(r >= 0 ? 1 : 0, pos, total);
    if (!WRITE) {
      if (tid == 0) cnt[(long long)t * n_chunks + c] = total;
    } else if (r >= 0) {
      const int at = cnt[(long long)t * n_chunks + c] + pos;
      if (at < pair_cap) {
        pairs_in[(long long)t * pair_cap + at] = r;
        pairs_out[(long long)t * pair_cap + at] = o0 + tid;
      }
    }
    __syncthreads();                                     // tmp is reused by the next tap's scan
  }
}

// per tap (one block each): chunk counts -> exclusive offsets in place; pair_count[t] = min(total, pair_cap)
__global__ void __launch_bounds__(1024) sc_pairs_scan_kernel(int* __restrict__ cnt, int n_chunks, int pair_cap, int* __restrict__ pair_count) {
  typedef cub::BlockScan<int, 1024> Scan;
  __shared__ typename Scan::TempStorage tmp;
  int* row = cnt + (long long)blockIdx.x * n_chunks;
  int base = 0;
  for (int c0 = 0; c0 < n_chunks; c0 += 1024) {
    const int c = c0 + threadIdx.x;
    const int v = c < n_chunks ? row[c] : 0;
    int pos, total;
    Scan(tmp).ExclusiveSum(v, pos, total);
    if (c < n_chunks) row[c] = base + pos;
    base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) pair_count[blockIdx.x] = min(base, pair_cap);
}

int grid_for(long long total) {
  const long long nb = (total + 255) / 256, cap = (long long)tt_num_sms() * 8;
  return (int)(nb < 1 ? 1 : nb > cap ? cap : nb);
}

bool eq3(const int* v, int a, int b, int c) { return v[0] == a && v[1] == b && v[2] == c; }

// refuses what the reference does not build, naming the parameter
int check_desc(const tt_sparse_conv_train_desc* d, const char* name) {
  TT_REQUIRE(d, name, "null descriptor");
  const char* bad = nullptr;
  const int kprod = d->k[0] * d->k[1] * d->k[2];
  if (d->transposed) bad = "transposed: transposed sparse convolutions are not supported";
  else if (d->inverse) bad = "inverse: inverse sparse convolutions are not supported";
  else if (d->bias) bad = "bias: only bias-free convolutions are supported";
  else if (d->groups != 1) bad = "groups: only 1 is supported";
  else if (!eq3(d->dilation, 1, 1, 1)) bad = "dilation: only 1 is supported";
  else if (d->kvol < 1 || d->kvol > MAX_KVOL) bad = "kvol: at most 32 taps are supported";
  else if (d->kvol != kprod) bad = "kvol: must equal the kernel volume";
  else if (d->subm) {
    if (!eq3(d->k, 3, 3, 3)) bad = "kernel_size: SubM supports 3x3x3 only";
    else if (!eq3(d->stride, 1, 1, 1)) bad = "stride: SubM supports stride 1 only";
    else if (!eq3(d->padding, 1, 1, 1)) bad = "padding: SubM supports padding 1 only";
  } else if (eq3(d->k, 3, 3, 3)) {
    if (!eq3(d->stride, 2, 2, 2)) bad = "stride: a strided 3x3x3 conv supports stride 2 only";
    else if (!eq3(d->padding, 1, 1, 1) && !eq3(d->padding, 0, 1, 1)) bad = "padding: a strided 3x3x3 conv supports padding 1 or (0, 1, 1)";
  } else if (eq3(d->k, 3, 1, 1)) {
    if (!eq3(d->stride, 2, 1, 1)) bad = "stride: a (3, 1, 1) conv supports stride (2, 1, 1) only";
    else if (!eq3(d->padding, 0, 0, 0)) bad = "padding: a (3, 1, 1) conv supports padding 0 only";
  } else {
    bad = "kernel_size: only 3x3x3 and (3, 1, 1) are supported";
  }
  if (bad) {
    tt_set_error("%s: unsupported %s", name, bad);
    return TT_ERR_UNSUPPORTED;
  }
  TT_REQUIRE(d->Cin > 0 && d->Cout > 0 && d->cap_in >= 0 && d->cap_out >= 0 && d->pair_cap >= 1, name,
             "Cin, Cout and pair_cap must be positive, the row capacities non-negative");
  TT_REQUIRE(d->in_ld >= d->Cin && d->out_ld >= d->Cout, name, "row pitches must hold the channels");
  return TT_OK;
}

// the workspace: packed weight (two fp32 planes of the weight's size), then the grad_weight partials
struct Ws {
  float *w, *part;
  size_t part_bytes, bytes;
};
Ws carve(const tt_sparse_conv_train_desc* d, void* base) {
  const size_t wsz = (size_t)2 * d->Cout * d->kvol * d->Cin * 4;
  const size_t simt = (size_t)WG_SPLITS * d->kvol * d->Cout * d->Cin * 4;
  const size_t tc = tt_gemm_at_workspace_bytes(d->kvol, d->Cout, d->Cin);
  Ws w;
  w.part_bytes = simt > tc ? simt : tc;
  const size_t o = (wsz + 255) / 256 * 256;
  w.w = base ? reinterpret_cast<float*>(base) : nullptr;
  w.part = base ? reinterpret_cast<float*>(static_cast<char*>(base) + o) : nullptr;
  w.bytes = o + (w.part_bytes + 255) / 256 * 256;
  return w;
}

// y[o] (rows < *count, zeroed first) += sum over the pairs of W_t x[i] through tt_sparse_conv (no bias, residual or activation)
int gather_conv(int Cin, int Cout, int kvol, int in_ld, int out_ld, int cap_out, int pair_cap, const float* x, const float* wt_src,
                float* wpack, const int* pin, const int* pout, const int* pcount, const int* count, float* y, int dir, cudaStream_t st,
                const char* name) {
  tt_sparse_conv_desc sd;
  sd.Cin = Cin; sd.Cout = Cout; sd.kvol = kvol; sd.in_ld = in_ld; sd.out_ld = out_ld; sd.res_ld = 0;
  sd.cap_out = cap_out; sd.pair_cap = pair_cap; sd.act = TT_ACT_NONE; sd.impl = 3;
  const bool tc = tt_sparse_conv_tc_supported(&sd, x, wpack, y);
  sd.impl = tc ? 3 : 1;
  // wt_src is the (Cout_w, kvol, Cin_w) weight; dir 1 packs its transpose, so (Cin, Cout) here are (Cout_w, Cin_w)
  const int Cout_w = dir ? Cin : Cout, Cin_w = dir ? Cout : Cin;
  sc_pack_weight_kernel<<<grid_for((long long)Cout_w * kvol * Cin_w), 256, 0, st>>>(wt_src, wpack, Cout_w, kvol, Cin_w, tc, dir);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return tt_sparse_conv(&sd, x, wpack, nullptr, nullptr, pin, pout, pcount, count, y, (tt_stream_t)st);
}

}  // namespace

extern "C" {

size_t tt_sparse_conv_train_workspace_bytes(const tt_sparse_conv_train_desc* d) {
  if (!d || check_desc(d, "tt_sparse_conv_train_workspace_bytes") != TT_OK) return 0;
  return carve(d, nullptr).bytes;
}

int tt_sparse_conv_train_forward(const tt_sparse_conv_train_desc* d, const float* feats_in, const float* weight, const int* pairs_in,
                                 const int* pairs_out, const int* pair_count, const int* out_count, float* feats_out, void* ws,
                                 size_t ws_bytes, tt_stream_t stream) {
  static const char* name = "tt_sparse_conv_train_forward";
  const int rc = check_desc(d, name);
  if (rc != TT_OK) return rc;
  TT_REQUIRE(feats_in && weight && pairs_in && pairs_out && pair_count && out_count && feats_out, name, "null argument");
  const Ws w = carve(d, ws);
  TT_REQUIRE(ws && ws_bytes >= w.bytes, name, "workspace smaller than tt_sparse_conv_train_workspace_bytes");
  if (d->cap_out == 0) return TT_OK;
  return gather_conv(d->Cin, d->Cout, d->kvol, d->in_ld, d->out_ld, d->cap_out, d->pair_cap, feats_in, weight, w.w, pairs_in, pairs_out,
                     pair_count, out_count, feats_out, 0, (cudaStream_t)stream, name);
}

int tt_sparse_conv_train_backward(const tt_sparse_conv_train_desc* d, const float* feats_in, const float* weight, const float* grad_out,
                                  const int* pairs_in, const int* pairs_out, const int* pair_count, const int* in_count,
                                  const int* out_count, float* grad_in, float* grad_weight, void* ws, size_t ws_bytes,
                                  tt_stream_t stream) {
  static const char* name = "tt_sparse_conv_train_backward";
  const int rc = check_desc(d, name);
  if (rc != TT_OK) return rc;
  TT_REQUIRE(feats_in && weight && grad_out && pairs_in && pairs_out && pair_count && in_count && out_count, name, "null argument");
  const Ws w = carve(d, ws);
  TT_REQUIRE(ws && ws_bytes >= w.bytes, name, "workspace smaller than tt_sparse_conv_train_workspace_bytes");
  cudaStream_t st = (cudaStream_t)stream;
  if (grad_in && d->cap_in > 0) {            // grad_x[i] = sum W_t^T gy[o]: input and output roles swapped
    const int r = gather_conv(d->Cout, d->Cin, d->kvol, d->out_ld, d->in_ld, d->cap_in, d->pair_cap, grad_out, weight, w.w, pairs_out,
                              pairs_in, pair_count, in_count, grad_in, 1, st, name);
    if (r != TT_OK) return r;
  }
  if (!grad_weight) return TT_OK;
  const bool tc = d->Cin % 4 == 0 && d->Cout % 4 == 0 && d->in_ld % 4 == 0 && d->out_ld % 4 == 0 &&
                  ((reinterpret_cast<uintptr_t>(feats_in) | reinterpret_cast<uintptr_t>(grad_out)) & 15) == 0;
  if (tc)                                    // C[t][i][j] -> grad_weight[i][t][j]: ldc = kvol * Cin, c_batch = Cin
    return tt_gemm_at_gather(grad_out, d->out_ld, pairs_out, feats_in, d->in_ld, pairs_in, pair_count, d->pair_cap, grad_weight,
                             d->kvol * d->Cin, d->Cin, d->kvol, d->Cout, d->Cin, w.part, w.part_bytes, st);
  int splits = tt_cdiv(d->pair_cap, 4096);
  splits = splits < 1 ? 1 : splits > WG_SPLITS ? WG_SPLITS : splits;
  sc_wgrad_simt_kernel<<<dim3(splits, d->kvol), 256, 0, st>>>(grad_out, d->out_ld, feats_in, d->in_ld, pairs_in, pairs_out, pair_count,
                                                               d->pair_cap, d->Cout, d->Cin, d->kvol, w.part);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  sc_wgrad_fold_kernel<<<grid_for((long long)d->kvol * d->Cout * d->Cin), 256, 0, st>>>(w.part, splits, d->kvol, d->Cout, d->Cin, grad_weight);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}

size_t tt_sparse_pairs_ordered_workspace_bytes(int cap_out, int kvol) {
  if (cap_out < 0 || kvol < 1) return 0;
  return (size_t)kvol * tt_cdiv(cap_out > 0 ? cap_out : 1, PCH) * sizeof(int);
}

int tt_sparse_pairs_ordered(const int* nbr, const int* out_count, int cap_out, int kvol, int pair_cap, int* pairs_in, int* pairs_out,
                            int* pair_count, void* ws, size_t ws_bytes, tt_stream_t stream) {
  static const char* name = "tt_sparse_pairs_ordered";
  TT_REQUIRE(nbr && out_count && pairs_in && pairs_out && pair_count, name, "null argument");
  TT_REQUIRE(kvol >= 1 && kvol <= MAX_KVOL && cap_out >= 0 && pair_cap >= 0, name, "kvol must be in [1, 32], capacities non-negative");
  TT_REQUIRE(ws && ws_bytes >= tt_sparse_pairs_ordered_workspace_bytes(cap_out, kvol), name,
             "workspace smaller than tt_sparse_pairs_ordered_workspace_bytes");
  cudaStream_t st = (cudaStream_t)stream;
  const int n_chunks = tt_cdiv(cap_out > 0 ? cap_out : 1, PCH);
  int* cnt = static_cast<int*>(ws);
  sc_pairs_chunk_kernel<false><<<n_chunks, PCH, 0, st>>>(nbr, out_count, cap_out, kvol, n_chunks, cnt, pair_cap, pairs_in, pairs_out);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  sc_pairs_scan_kernel<<<kvol, 1024, 0, st>>>(cnt, n_chunks, pair_cap, pair_count);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  sc_pairs_chunk_kernel<true><<<n_chunks, PCH, 0, st>>>(nbr, out_count, cap_out, kvol, n_chunks, cnt, pair_cap, pairs_in, pairs_out);
  ++g_tt_launches;
  TT_CHECK_LAUNCH(name);
  return TT_OK;
}

}  // extern "C"
