// A-transposed contraction on the tensor cores (wgmma, 3xTF32): the weight-gradient GEMM of a convolution.
//
//   C[b][i][j] (+)= sum_k A[k][a_batch * b + i] * B[k][b_batch * b + j],   i < M, j < N, k < K
//
// Both operands arrive with the reduction index outermost (a pixel's row of output gradients, a pixel's column row), so
// this is a reduction over pixels, unlike every other contraction here (which reduces over taps x Cin of one pixel).
//   * wgmma .tf32 reads only K-major shared-memory operands: 16-byte cp.async copies bring the raw [32 k][BM i] and
//     [32 k][BN j] slabs into a 3-stage staging ring as they lie in memory; every thread then reads 4 k of one row
//     (conflict-free: a warp reads 32 consecutive floats of one k) and writes them transposed, split into hi / lo
//     TF32 planes, as one 16-byte chunk of a 128-byte-swizzled K-major row (conflict-free: 8 consecutive rows land in
//     8 distinct chunks);
//   * each K slab issues hi*hi + hi*lo + lo*hi (3xTF32, as tt_conv2d impl 3) into two register accumulators that are
//     restarted every CHUNK slabs and folded into fp32 sums with round-to-nearest adds;
//   * split-K: the K range is cut into `splits` contiguous pieces, one CTA per (tile, piece); each writes its partial
//     tile to the workspace and a fold kernel adds the pieces in piece order.  No floating-point atomics: the result
//     is bitwise reproducible from run to run on the same GPU.
// Gather mode (tt_gemm_at_gather, the weight gradient of a sparse convolution): batch b is a kernel tap, row k of A / B is
// row rows_a[b][k] / rows_b[b][k] of one shared matrix, and K = count[b] is read on the device.  The split count is fixed on
// the host from the pair capacity; each CTA derives its piece of K from the device count, so no host sync is needed and the
// fold order stays fixed.  The plain instance the deformable convolution uses is the MODE = AT_PLAIN template.
// Conv mode (tt_gemm_at_conv, the weight gradient of a dense convolution): batch b is tap (kh, kw), row k of A is pixel k of the
// output gradient [P][M] and row k of B is the input pixel (n, oh * stride - pad + kh * dil, ow * stride - pad + kw * dil) of the
// channels-last input [N][H][W][N cols], zero-filled (cp.async src-size 0) when it falls outside the image.  Its fold writes the
// torch weight layout (M, N, KH, KW) directly.
#include "common.cuh"
#include "tc_ptx.cuh"

extern long long g_tt_launches;

namespace {

constexpr int BM = 128, BN = 64, KS = 32, STAGES = 3, CHUNK = 2, NT = 256, MAX_SPLITS = 16;
constexpr int RAW_A = KS * BM * 4, RAW_B = KS * BN * 4;          // staging: [k][i], [k][j]
constexpr int OP_A = BM * 128, OP_B = BN * 128;                  // operands: [row][32 k] swizzled, one plane
constexpr int OP_BYTES = 2 * OP_A + 2 * OP_B;                    // hi + lo of both
constexpr int SMEM = 2 * OP_BYTES + STAGES * (RAW_A + RAW_B) + 1024;

struct AtArgs {
  const float* A; const float* B; float* part;
  int M, N, K, lda, ldb;
  long long a_batch, b_batch;
  int m_tiles, n_tiles, batch, splits, k_per;   // k_per: K slabs per split
  const int *rows_a, *rows_b, *count;           // gather mode: [batch][pair_cap] row lists, [batch] K
  int pair_cap;
};
// conv mode: input / output maps and the kernel geometry.  A separate kernel parameter, so that the plain and gather instances
// keep the AtArgs layout (and the code) they were built with
struct AtConv {
  int H, W, OH, OW, KW, stride, pad, dil;
};

enum { AT_PLAIN = 0, AT_GATHER = 1, AT_CONV = 2 };

TT_DEVICE void split_rn(float x, float& hi, float& lo) {
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
  lo = x - hi;
}
TT_DEVICE void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> TT_DEVICE void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int MODE>
__global__ void __launch_bounds__(NT, 1) gemm_at_kernel(const AtArgs p, const AtConv cv) {
  constexpr bool GATHER = MODE == AT_GATHER, CONV = MODE == AT_CONV;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ops = smem;                                     // [2][A hi | A lo | B hi | B lo]
  uint8_t* raw = smem + 2 * OP_BYTES;                      // [STAGES][A raw | B raw]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2;

  int t = blockIdx.x;
  const int ks = t % p.splits; t /= p.splits;
  const int nt = t % p.n_tiles; t /= p.n_tiles;
  const int mt = t % p.m_tiles;
  const int b = t / p.m_tiles;
  const int i0 = mt * BM, j0 = nt * BN;
  const int K = GATHER ? min(__ldg(p.count + b), p.pair_cap) : p.K;
  const int n_slabs_total = (K + KS - 1) / KS;
  const int k_per = GATHER ? (n_slabs_total + p.splits - 1) / p.splits : p.k_per;
  const int kb = ks * k_per, ke = min(n_slabs_total, kb + k_per);
  const int n_it = max(ke - kb, 0);
  const float* A = GATHER ? p.A : p.A + p.a_batch * b;
  const float* Bm = GATHER ? p.B : p.B + p.b_batch * b;
  const int* rows_a = GATHER ? p.rows_a + (long long)b * p.pair_cap : nullptr;
  const int* rows_b = GATHER ? p.rows_b + (long long)b * p.pair_cap : nullptr;

  auto load = [&](int it, int s) {                         // slab kb + it -> staging stage s (zero-fill outside K / M / N)
    const int k0 = (kb + it) * KS;
    const uint32_t ra = smem_u32(raw + s * (RAW_A + RAW_B)), rb = ra + RAW_A;
#pragma unroll
    for (int r = 0; r < RAW_A / 16 / NT; ++r) {            // 4 chunks per thread: row k = c / 32, float4 column c % 32
      const int c = tid + r * NT, kk = c >> 5, q = c & 31;
      const int k = k0 + kk, i = i0 + q * 4;
      const bool ok = k < K && i < p.M;
      const long long row = GATHER ? (ok ? (long long)__ldg(rows_a + k) : 0) : k;
      cp_async16(ra + c * 16, ok ? A + row * p.lda + i : p.A, ok ? 16 : 0);
    }
#pragma unroll
    for (int r = 0; r < RAW_B / 16 / NT; ++r) {            // 2 chunks per thread: row k = c / 16, float4 column c % 16
      const int c = tid + r * NT, kk = c >> 4, q = c & 15;
      const int k = k0 + kk, j = j0 + q * 4;
      const bool ok = k < K && j < p.N;
      if constexpr (CONV) {                                // output pixel k -> the input pixel this tap reads, or zeros
        const int kh = b / cv.KW, kw = b - kh * cv.KW;     // this batch's tap
        const int ow = k % cv.OW, t2 = k / cv.OW, oh = t2 % cv.OH, n = t2 / cv.OH;
        const int ih = oh * cv.stride - cv.pad + kh * cv.dil, iw = ow * cv.stride - cv.pad + kw * cv.dil;
        const bool in = ok && ih >= 0 && ih < cv.H && iw >= 0 && iw < cv.W;
        cp_async16(rb + c * 16, in ? p.B + (((long long)n * cv.H + ih) * cv.W + iw) * p.ldb + j : p.B, in ? 16 : 0);
      } else {
        const long long row = GATHER ? (ok ? (long long)__ldg(rows_b + k) : 0) : k;
        cp_async16(rb + c * 16, ok ? Bm + row * p.ldb + j : p.B, ok ? 16 : 0);
      }
    }
  };
  // staging stage s -> operand buffer o: transpose to K-major, split into hi / lo, 128-byte swizzle
  auto transform = [&](int s, int o) {
    const float* ra = reinterpret_cast<const float*>(raw + s * (RAW_A + RAW_B));
    const float* rb = ra + KS * BM;
    const uint32_t oa = smem_u32(ops + o * OP_BYTES), ob = oa + 2 * OP_A;
#pragma unroll
    for (int r = 0; r < BM * 8 / NT; ++r) {
      const int c = tid + r * NT, row = c % BM, kc = c / BM;
      float4 v, h, l;
      v.x = ra[(4 * kc + 0) * BM + row]; v.y = ra[(4 * kc + 1) * BM + row];
      v.z = ra[(4 * kc + 2) * BM + row]; v.w = ra[(4 * kc + 3) * BM + row];
      split_rn(v.x, h.x, l.x); split_rn(v.y, h.y, l.y); split_rn(v.z, h.z, l.z); split_rn(v.w, h.w, l.w);
      const uint32_t a = oa + row * 128 + ((kc ^ (row & 7)) << 4);
      sts128(a, h);
      sts128(a + OP_A, l);
    }
#pragma unroll
    for (int r = 0; r < BN * 8 / NT; ++r) {
      const int c = tid + r * NT, row = c % BN, kc = c / BN;
      float4 v, h, l;
      v.x = rb[(4 * kc + 0) * BN + row]; v.y = rb[(4 * kc + 1) * BN + row];
      v.z = rb[(4 * kc + 2) * BN + row]; v.w = rb[(4 * kc + 3) * BN + row];
      split_rn(v.x, h.x, l.x); split_rn(v.y, h.y, l.y); split_rn(v.z, h.z, l.z); split_rn(v.w, h.w, l.w);
      const uint32_t a = ob + row * 128 + ((kc ^ (row & 7)) << 4);
      sts128(a, h);
      sts128(a + OP_B, l);
    }
  };

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < n_it) load(s, s);
    cp_async_commit();
  }
  float sum[BN / 2], acc[BN / 2], cor[BN / 2];
#pragma unroll
  for (int j = 0; j < BN / 2; ++j) sum[j] = acc[j] = cor[j] = 0.f;
  for (int it = 0; it < n_it; ++it) {
    cp_async_wait<STAGES - 2>();                          // this thread's copies of slab `it` landed
    __syncthreads();                                       // everyone's did; operand buffer it % 2 is no longer read by wgmma
    if (it + STAGES - 1 < n_it) load(it + STAGES - 1, (it + STAGES - 1) % STAGES);
    cp_async_commit();
    transform(it % STAGES, it & 1);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
    __syncthreads();
    const uint32_t a_hi = smem_u32(ops + (it & 1) * OP_BYTES) + wg * (OP_A / 2), a_lo = a_hi + OP_A;
    const uint32_t b_hi = smem_u32(ops + (it & 1) * OP_BYTES) + 2 * OP_A, b_lo = b_hi + OP_B;
    const bool first = it % CHUNK == 0;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KS / 8; ++kk) {
      const uint32_t off = kk * 32, z = (first && kk == 0) ? 0u : 1u;
      wgmma_tf32<BN>(acc, make_smem_desc(a_hi + off), make_smem_desc(b_hi + off), z);
      wgmma_tf32<BN>(cor, make_smem_desc(a_hi + off), make_smem_desc(b_lo + off), z);
      wgmma_tf32<BN>(cor, make_smem_desc(a_lo + off), make_smem_desc(b_hi + off), 1u);
    }
    wgmma_commit();
    if (it % CHUNK == CHUNK - 1 || it == n_it - 1) {       // end of a register chunk: fold into the fp32 sums
      wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) sum[j] += acc[j] + cor[j];
    } else {
      wgmma_wait<1>();
    }
  }
  cp_async_wait<0>();
  // partial tile -> workspace [split][batch][M][N]; fragment: d[4 j + {0,1}] at row lane / 4, d[4 j + {2,3}] at row lane / 4 + 8,
  // columns 8 j + 2 (lane % 4) + {0, 1}, of this warp's 16 rows
  float* out = p.part + ((long long)ks * p.batch + b) * p.M * p.N;
  const int rbase = i0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = j0 + 8 * j + 2 * (lane & 3);
    if (col >= p.N) continue;
    if (rbase < p.M) *reinterpret_cast<float2*>(out + (long long)rbase * p.N + col) = make_float2(sum[4 * j], sum[4 * j + 1]);
    if (rbase + 8 < p.M) *reinterpret_cast<float2*>(out + (long long)(rbase + 8) * p.N + col) = make_float2(sum[4 * j + 2], sum[4 * j + 3]);
  }
}

// C[b][i][j] = (accumulate ? C[b][i][j] : 0) + part[0][b][i][j] + part[1][b][i][j] + ...  (in this order)
__global__ void gemm_at_fold_kernel(const float* __restrict__ part, int splits, int batch, int M, int N, float* __restrict__ Cm, int ldc,
                                    long long c_batch, int accumulate) {
  const long long per = (long long)M * N, total = batch * per;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(e / per);
    const long long r = e - b * per;
    const int i = (int)(r / N), j = (int)(r - (long long)i * N);
    float* dst = Cm + b * c_batch + (long long)i * ldc + j;
    float v = accumulate ? *dst : 0.f;
    for (int s = 0; s < splits; ++s) v += part[s * total + e];
    *dst = v;
  }
}

// K split: the count in [1, MAX_SPLITS] that fills whole waves of one-CTA-per-SM best, at least 4 slabs per piece
int at_splits(int batch, int M, int N, int K) {
  const long long tiles = (long long)batch * tt_cdiv(M, BM) * tt_cdiv(N, BN);
  const int slabs = tt_cdiv(K, KS), sms = tt_num_sms();
  int best = 1;
  double best_eff = -1;
  for (int s = 1; s <= MAX_SPLITS && (s == 1 || slabs / s >= 4); ++s) {
    const long long items = tiles * s, waves = (items + sms - 1) / sms;
    const double eff = (double)items / (double)(waves * sms);
    if (eff > best_eff + 1e-9) { best_eff = eff; best = s; }
  }
  return best;
}

}  // namespace

// partial tiles of the largest split count: the size does not depend on the device (or need one)
size_t tt_gemm_at_workspace_bytes(int batch, int M, int N) {
  if (batch <= 0 || M <= 0 || N <= 0) return 0;
  return (size_t)MAX_SPLITS * batch * M * N * sizeof(float);
}

int tt_gemm_at(const float* A, int lda, long long a_batch, const float* B, int ldb, long long b_batch, float* Cm, int ldc, long long c_batch,
               int batch, int M, int N, int K, int accumulate, void* ws, size_t ws_bytes, cudaStream_t st) {
  TT_REQUIRE(A && B && Cm, "tt_gemm_at", "null argument");
  TT_REQUIRE(M % 4 == 0 && N % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 && a_batch % 4 == 0 && b_batch % 4 == 0 &&
                 ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) & 15) == 0,
             "tt_gemm_at", "M, N, lda, ldb and the batch offsets must be multiples of 4 floats, A and B 16-byte aligned");
  if (batch <= 0 || M <= 0 || N <= 0) return TT_OK;
  if (K <= 0) {
    if (!accumulate)
      for (int b = 0; b < batch; ++b)
        if (cudaMemset2DAsync(Cm + b * c_batch, (size_t)ldc * 4, 0, (size_t)N * 4, M, st) != cudaSuccess) {
          tt_set_error("tt_gemm_at: memset failed"); return TT_ERR_CUDA;
        }
    return TT_OK;
  }
  const size_t need = (size_t)at_splits(batch, M, N, K) * batch * M * N * sizeof(float);
  TT_REQUIRE(ws && ws_bytes >= need, "tt_gemm_at", "workspace smaller than tt_gemm_at_workspace_bytes");
  AtArgs a;
  a.A = A; a.B = B; a.part = static_cast<float*>(ws);
  a.M = M; a.N = N; a.K = K; a.lda = lda; a.ldb = ldb; a.a_batch = a_batch; a.b_batch = b_batch;
  a.m_tiles = tt_cdiv(M, BM); a.n_tiles = tt_cdiv(N, BN); a.batch = batch;
  a.splits = at_splits(batch, M, N, K);
  a.k_per = tt_cdiv(tt_cdiv(K, KS), a.splits);
  a.rows_a = a.rows_b = a.count = nullptr; a.pair_cap = 0;
  static bool set = false;
  if (!set) { cudaFuncSetAttribute(gemm_at_kernel<AT_PLAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM); set = true; }
  const long long items = (long long)batch * a.m_tiles * a.n_tiles * a.splits;
  gemm_at_kernel<AT_PLAIN><<<(unsigned)items, NT, SMEM, st>>>(a, AtConv{});
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_gemm_at");
  const long long total = (long long)batch * M * N;
  const long long nb = (total + 255) / 256;
  gemm_at_fold_kernel<<<(int)(nb > tt_num_sms() * 8 ? tt_num_sms() * 8 : nb), 256, 0, st>>>(a.part, a.splits, batch, M, N, Cm, ldc,
                                                                                             c_batch, accumulate);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_gemm_at(fold)");
  return TT_OK;
}

// Gather form: C[b][i][j] = sum_{k < count[b]} A[rows_a[b][k]][i] * B[rows_b[b][k]][j] (i < M, j < N), every tap b written (an empty
// tap gives zeros).  Same tiles, 3xTF32 products and fixed-order fold as tt_gemm_at; ws: tt_gemm_at_workspace_bytes(batch, M, N).
int tt_gemm_at_gather(const float* A, int lda, const int* rows_a, const float* B, int ldb, const int* rows_b, const int* count, int pair_cap,
                      float* Cm, int ldc, long long c_batch, int batch, int M, int N, void* ws, size_t ws_bytes, cudaStream_t st) {
  TT_REQUIRE(A && B && Cm && rows_a && rows_b && count, "tt_gemm_at_gather", "null argument");
  TT_REQUIRE(M % 4 == 0 && N % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 &&
                 ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) & 15) == 0,
             "tt_gemm_at_gather", "M, N, lda and ldb must be multiples of 4 floats, A and B 16-byte aligned");
  if (batch <= 0 || M <= 0 || N <= 0) return TT_OK;
  AtArgs a;
  a.A = A; a.B = B; a.part = static_cast<float*>(ws);
  a.M = M; a.N = N; a.K = 0; a.lda = lda; a.ldb = ldb; a.a_batch = a.b_batch = 0;
  a.m_tiles = tt_cdiv(M, BM); a.n_tiles = tt_cdiv(N, BN); a.batch = batch;
  a.splits = at_splits(batch, M, N, pair_cap > 0 ? pair_cap : 1);   // from the capacity: the counts stay on the device
  a.k_per = 0;
  a.rows_a = rows_a; a.rows_b = rows_b; a.count = count; a.pair_cap = pair_cap;
  TT_REQUIRE(ws && ws_bytes >= (size_t)a.splits * batch * M * N * sizeof(float), "tt_gemm_at_gather",
             "workspace smaller than tt_gemm_at_workspace_bytes");
  static bool set = false;
  if (!set) { cudaFuncSetAttribute(gemm_at_kernel<AT_GATHER>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM); set = true; }
  const long long items = (long long)batch * a.m_tiles * a.n_tiles * a.splits;
  gemm_at_kernel<AT_GATHER><<<(unsigned)items, NT, SMEM, st>>>(a, AtConv{});
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_gemm_at_gather");
  const long long total = (long long)batch * M * N;
  const long long nb = (total + 255) / 256;
  gemm_at_fold_kernel<<<(int)(nb > tt_num_sms() * 8 ? tt_num_sms() * 8 : nb), 256, 0, st>>>(a.part, a.splits, batch, M, N, Cm, ldc,
                                                                                             c_batch, 0);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_gemm_at_gather(fold)");
  return TT_OK;
}

// grad_weight (M, N, taps)[i][j][t] = part[0][t][i][j] + part[1][t][i][j] + ...  (in this order): torch's (Cout, Cin, KH, KW)
static __global__ void gemm_at_fold_conv_kernel(const float* __restrict__ part, int splits, int taps, int M, int N, float* __restrict__ gw) {
  const long long MN = (long long)M * N, total = taps * MN;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(e % taps), j = (int)((e / taps) % N), i = (int)(e / ((long long)taps * N));
    const long long src = (long long)t * MN + (long long)i * N + j;
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += part[s * total + src];
    gw[e] = v;
  }
}

// Conv form: gw[i][j][kh][kw] = sum over output pixels k < N*OH*OW of gy[k][i] * x(pixel k, tap (kh, kw))[j], gy [P][M] (row pitch M),
// x [N][H][W][Cin = N cols] (row pitch Cin).  Same tiles, 3xTF32 products, fixed split count and fold order as tt_gemm_at (bitwise
// reproducible); ws: tt_gemm_at_workspace_bytes(KH * KW, M, Cin).
int tt_gemm_at_conv(const float* gy, const float* x, float* gw, int n_img, int H, int W, int OH, int OW, int KH, int KW, int stride, int pad,
                    int dil, int M, int Cin, void* ws, size_t ws_bytes, cudaStream_t st) {
  TT_REQUIRE(gy && x && gw, "tt_gemm_at_conv", "null argument");
  TT_REQUIRE(M % 4 == 0 && Cin % 4 == 0 && ((reinterpret_cast<uintptr_t>(gy) | reinterpret_cast<uintptr_t>(x)) & 15) == 0, "tt_gemm_at_conv",
             "M and Cin must be multiples of 4 floats, gy and x 16-byte aligned");
  const int taps = KH * KW, K = n_img * OH * OW;
  if (taps <= 0 || M <= 0 || Cin <= 0) return TT_OK;
  if (K <= 0) {
    if (cudaMemsetAsync(gw, 0, (size_t)taps * M * Cin * 4, st) != cudaSuccess) { tt_set_error("tt_gemm_at_conv: memset failed"); return TT_ERR_CUDA; }
    return TT_OK;
  }
  AtArgs a;
  a.A = gy; a.B = x; a.part = static_cast<float*>(ws);
  a.M = M; a.N = Cin; a.K = K; a.lda = M; a.ldb = Cin; a.a_batch = a.b_batch = 0;
  a.m_tiles = tt_cdiv(M, BM); a.n_tiles = tt_cdiv(Cin, BN); a.batch = taps;
  a.splits = at_splits(taps, M, Cin, K);
  a.k_per = tt_cdiv(tt_cdiv(K, KS), a.splits);
  a.rows_a = a.rows_b = a.count = nullptr; a.pair_cap = 0;
  const AtConv cv = {H, W, OH, OW, KW, stride, pad, dil};
  TT_REQUIRE(ws && ws_bytes >= (size_t)a.splits * taps * M * Cin * sizeof(float), "tt_gemm_at_conv",
             "workspace smaller than tt_gemm_at_workspace_bytes");
  static bool set = false;
  if (!set) { cudaFuncSetAttribute(gemm_at_kernel<AT_CONV>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM); set = true; }
  const long long items = (long long)taps * a.m_tiles * a.n_tiles * a.splits;
  gemm_at_kernel<AT_CONV><<<(unsigned)items, NT, SMEM, st>>>(a, cv);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_gemm_at_conv");
  const long long total = (long long)taps * M * Cin;
  const long long nb = (total + 255) / 256;
  gemm_at_fold_conv_kernel<<<(int)(nb > tt_num_sms() * 8 ? tt_num_sms() * 8 : nb), 256, 0, st>>>(a.part, a.splits, taps, M, Cin, gw);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_gemm_at_conv(fold)");
  return TT_OK;
}
