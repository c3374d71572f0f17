// SIMT fp32 implicit-GEMM convolution / linear / sparse-conv engine (exact fp32 FFMA path).
//
// One kernel family serves every contraction on the path: A rows are produced on the fly either from
// the conv geometry (dense NHWC input, zero padding, stride, dilation, groups) or from a rulebook
// (`gather`, the sparse-conv neighbour table).  B is the pre-packed [K][Cout] weight with BatchNorm
// folded in.  The epilogue fuses bias, up to two residuals (incl. nearest x2 up-sampled, PAFPN
// top-down), activation, channel-offset (concat) and pixel-scatter (k2s2 transposed conv) stores.
//
// Tiling: BMxBNx16 per CTA, 256 threads, TMxTN register tile split into 4x4 quadrants so that
// shared-memory reads are conflict-free 128-bit loads (A broadcast, B contiguous), global->register
// prefetch of the next K slab overlapped with the FFMA block, double-buffered shared memory.
#include <string.h>

#include "common.cuh"

extern long long g_tt_launches;

namespace {

struct ConvArgs {
  tt_conv_desc d;
  const float* x;
  const float* w;
  const float* bias;
  const float* res;
  const float* res2;
  const int* gather;
  const int* m_count;
  float* y;
  int M, Cin_g, Cout_g, Kg, taps;
  int splits, k_per_split;   // split-K (small-M / large-K layers): partial sums go to `partial`, reduced by a 2nd kernel
  float* partial;            // [splits][M][Cout]
  const int* out_index;      // gather mode: output row of GEMM row m (tap-major sparse conv pairs); NULL = m
  int accumulate;            // gather mode: 1: y[row] += result (rows of one launch are distinct); 2: atomic (red.add)
};

// what differs between the work items of one launch (the fused sparse conv walks (tap, row tile, column tile) items)
struct TileSel {
  const float* w;
  const int* gather;
  const int* out_index;
  int n_tile;
};

constexpr int BK = 16;

template <int BM, int BN, int TM, int TN, bool VECA, bool VECB>
__device__ __forceinline__ void conv_tile(const ConvArgs& p, const TileSel& ts, const int m0, const int M, float (*As)[BK][BM],
                                          float (*Bs)[BK][BN]) {
  constexpr int NA = BM * BK / 256;          // A floats per thread per slab (8 or 4)
  constexpr int NB = BK * BN / 256;          // B floats per thread per slab (8 or 4)
  constexpr int QM = TM / 4, QN = TN / 4;
  constexpr int TX = BN / TN;

  const tt_conv_desc& d = p.d;
  const int tid = threadIdx.x;
  const int g = blockIdx.z / p.splits;
  const int sp = blockIdx.z - g * p.splits;
  const int k_begin = sp * p.k_per_split;
  const int k_end = min(p.Kg, k_begin + p.k_per_split);
  const int n0 = ts.n_tile * BN;

  // ---- A loader state: one output row per thread, NA consecutive k
  const int a_row = tid % BM;
  const int a_k = (tid / BM) * NA;
  const int m = m0 + a_row;
  const bool a_valid = m < M;
  int an = 0, ih0 = 0, iw0 = 0;
  if (a_valid && !ts.gather) {
    int ow = m % d.OW;
    int t = m / d.OW;
    int oh = t % d.OH;
    an = t / d.OH;
    ih0 = oh * d.stride - d.pad;
    iw0 = ow * d.stride - d.pad;
  }
  const float* xg = p.x + d.x_coff + g * p.Cin_g;
  const long long xhs = d.x_hstride ? d.x_hstride : (long long)d.W * d.x_ld;
  const long long xns = d.x_nstride ? d.x_nstride : (long long)d.H * xhs;
  const long long yns = d.y_nstride ? d.y_nstride : (long long)d.yH * d.yW * d.y_ld;

  // ---- B loader state
  constexpr int BTPR = BN / 4;               // threads per B row
  const int b_col = (tid % BTPR) * 4;
  const int b_k = tid / BTPR;                // rows covered per pass: 256 / BTPR
  constexpr int BPASS = BK / (256 / BTPR);
  static_assert(BPASS * 4 == NB, "B tiling");
  const float* wg = ts.w + g * p.Cout_g;

  float ra[NA];
  float rb[NB];

  auto load_a = [&](int k0) {
#pragma unroll
    for (int j = 0; j < NA; j += 4) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      const int kg = k0 + a_k + j;
      if (VECA) {
        if (a_valid && kg < k_end) {
          const int tap = kg / p.Cin_g;
          const int c = kg - tap * p.Cin_g;
          const float* src = nullptr;
          if (ts.gather) {
            const int r = ts.gather[(long long)m * p.taps + tap];
            if (r >= 0) src = xg + (long long)r * d.x_ld + c;
          } else {
            const int kh = tap / d.KW, kw = tap - kh * d.KW;
            const int ih = ih0 + kh * d.dil, iw = iw0 + kw * d.dil;
            if (ih >= 0 && ih < d.H && iw >= 0 && iw < d.W)
              src = xg + an * xns + ih * xhs + (long long)iw * d.x_ld + c;
          }
          if (src) v = __ldg(reinterpret_cast<const float4*>(src));
        }
      } else {
        float e[4] = {0.f, 0.f, 0.f, 0.f};
        if (a_valid) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int k = kg + i;
            if (k < k_end) {
              const int tap = k / p.Cin_g;
              const int c = k - tap * p.Cin_g;
              if (ts.gather) {
                const int r = ts.gather[(long long)m * p.taps + tap];
                if (r >= 0) e[i] = __ldg(xg + (long long)r * d.x_ld + c);
              } else {
                const int kh = tap / d.KW, kw = tap - kh * d.KW;
                const int ih = ih0 + kh * d.dil, iw = iw0 + kw * d.dil;
                if (ih >= 0 && ih < d.H && iw >= 0 && iw < d.W)
                  e[i] = __ldg(xg + an * xns + ih * xhs + (long long)iw * d.x_ld + c);
              }
            }
          }
        }
        v = make_float4(e[0], e[1], e[2], e[3]);
      }
      ra[j] = v.x; ra[j + 1] = v.y; ra[j + 2] = v.z; ra[j + 3] = v.w;
    }
  };
  auto load_b = [&](int k0) {
#pragma unroll
    for (int ps = 0; ps < BPASS; ++ps) {
      const int k = k0 + b_k + ps * (256 / BTPR);
      const int n = n0 + b_col;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k < k_end) {
        const float* src = wg + (long long)k * d.Cout + n;
        if (VECB) {
          if (n < p.Cout_g) v = __ldg(reinterpret_cast<const float4*>(src));
        } else {
          if (n + 0 < p.Cout_g) v.x = __ldg(src + 0);
          if (n + 1 < p.Cout_g) v.y = __ldg(src + 1);
          if (n + 2 < p.Cout_g) v.z = __ldg(src + 2);
          if (n + 3 < p.Cout_g) v.w = __ldg(src + 3);
        }
      }
      rb[ps * 4 + 0] = v.x; rb[ps * 4 + 1] = v.y; rb[ps * 4 + 2] = v.z; rb[ps * 4 + 3] = v.w;
    }
  };
  auto store_smem = [&](int buf) {
#pragma unroll
    for (int j = 0; j < NA; ++j) As[buf][a_k + j][a_row] = ra[j];
#pragma unroll
    for (int ps = 0; ps < BPASS; ++ps)
      *reinterpret_cast<float4*>(&Bs[buf][b_k + ps * (256 / BTPR)][b_col]) =
          make_float4(rb[ps * 4], rb[ps * 4 + 1], rb[ps * 4 + 2], rb[ps * 4 + 3]);
  };

  const int tx = tid % TX, ty = tid / TX;
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nk = (k_end - k_begin + BK - 1) / BK;
  load_a(k_begin);
  load_b(k_begin);
  store_smem(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) {
      load_a(k_begin + (kt + 1) * BK);
      load_b(k_begin + (kt + 1) * BK);
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int q = 0; q < QM; ++q) {
        const float4 v = *reinterpret_cast<const float4*>(&As[buf][k][q * (BM / QM) + ty * 4]);
        a[q * 4] = v.x; a[q * 4 + 1] = v.y; a[q * 4 + 2] = v.z; a[q * 4 + 3] = v.w;
      }
#pragma unroll
      for (int q = 0; q < QN; ++q) {
        const float4 v = *reinterpret_cast<const float4*>(&Bs[buf][k][q * (BN / QN) + tx * 4]);
        b[q * 4] = v.x; b[q * 4 + 1] = v.y; b[q * 4 + 2] = v.z; b[q * 4 + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_smem(buf ^ 1);
      __syncthreads();
    }
  }

  // ---- split-K: raw partial sums, the reduce kernel applies the epilogue
  if (p.splits > 1) {
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int row = m0 + (i / 4) * (BM / QM) + ty * 4 + (i % 4);
      if (row >= M) continue;
      float* prow = p.partial + ((long long)sp * p.M + row) * d.Cout + g * p.Cout_g;
#pragma unroll
      for (int q = 0; q < QN; ++q)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = n0 + q * (BN / QN) + tx * 4 + j;
          if (col < p.Cout_g) prow[col] = acc[i][q * 4 + j];
        }
    }
    return;
  }
  // ---- epilogue
  const bool vec_out = VECB && (d.y_ld % 4 == 0) && (d.y_coff % 4 == 0) &&
                       (p.res == nullptr || (d.res_ld % 4 == 0 && d.res_coff % 4 == 0)) &&
                       (p.res2 == nullptr || (d.res2_ld % 4 == 0 && d.res2_coff % 4 == 0));
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int row = m0 + (i / 4) * (BM / QM) + ty * 4 + (i % 4);
    if (row >= M) continue;
    long long yoff, rpix = row, r1pix = row;
    int n = 0;
    if (ts.gather) {
      yoff = (long long)(ts.out_index ? ts.out_index[row] : row) * d.y_ld;
    } else {
      const int ow = row % d.OW;
      const int t = row / d.OW;
      const int oh = t % d.OH;
      n = t / d.OH;
      yoff = n * yns + ((long long)(oh * d.oy_mul + d.oy_add) * d.yW + ow * d.ox_mul + d.ox_add) * d.y_ld;
      if (d.res_mode == TT_RES_UP2_NEAREST) {
        const int rh = (oh * d.res_H) / d.OH, rw = (ow * d.res_W) / d.OW;
        r1pix = ((long long)n * d.res_H + rh) * d.res_W + rw;
      }
    }
    float* yrow = p.y + yoff + d.y_coff + g * p.Cout_g;
    const float* r1 = p.res ? p.res + r1pix * d.res_ld + d.res_coff + g * p.Cout_g : nullptr;
    const float* r2 = p.res2 ? p.res2 + rpix * d.res2_ld + d.res2_coff + g * p.Cout_g : nullptr;
    const float* bs = p.bias ? p.bias + (d.bias_n_mod ? (long long)(n % d.bias_n_mod) * d.Cout : 0) + g * p.Cout_g : nullptr;
#pragma unroll
    for (int q = 0; q < QN; ++q) {
      const int col = n0 + q * (BN / QN) + tx * 4;
      if (col >= p.Cout_g) continue;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = acc[i][q * 4 + j];
      if (p.accumulate == 2) {                              // fused tap-major sparse conv: taps race on a row -> red.add
        if (vec_out) tt_red_add_v4(yrow + col, v[0], v[1], v[2], v[3]);
        else {
#pragma unroll
          for (int j = 0; j < 4; ++j) if (col + j < p.Cout_g) atomicAdd(yrow + col + j, v[j]);
        }
        continue;
      }
      if (p.accumulate) {                                   // read-modify-write of a row this launch owns
        if (vec_out) { const float4 t = *reinterpret_cast<const float4*>(yrow + col); v[0] += t.x; v[1] += t.y; v[2] += t.z; v[3] += t.w; }
        else {
#pragma unroll
          for (int j = 0; j < 4; ++j) if (col + j < p.Cout_g) v[j] += yrow[col + j];
        }
      }
      if (vec_out) {
        if (bs) { const float4 t = __ldg(reinterpret_cast<const float4*>(bs + col)); v[0] += t.x; v[1] += t.y; v[2] += t.z; v[3] += t.w; }
        if (r1) { const float4 t = *reinterpret_cast<const float4*>(r1 + col); v[0] += t.x; v[1] += t.y; v[2] += t.z; v[3] += t.w; }
        if (r2) { const float4 t = *reinterpret_cast<const float4*>(r2 + col); v[0] += t.x; v[1] += t.y; v[2] += t.z; v[3] += t.w; }
        *reinterpret_cast<float4*>(yrow + col) =
            make_float4(tt_act(v[0], d.act), tt_act(v[1], d.act), tt_act(v[2], d.act), tt_act(v[3], d.act));
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (col + j < p.Cout_g) {
            float t = v[j];
            if (bs) t += __ldg(bs + col + j);
            if (r1) t += r1[col + j];
            if (r2) t += r2[col + j];
            yrow[col + j] = tt_act(t, d.act);
          }
        }
      }
    }
  }
}

// grid.x walks the M tiles with a grid stride, so a launch sized for a row CAPACITY (sparse rulebooks: the real row
// count is a device scalar) does not pay for thousands of empty CTAs.
template <int BM, int BN, int TM, int TN, bool VECA, bool VECB>
__global__ void __launch_bounds__(256) conv_igemm_simt(const ConvArgs p) {
  __shared__ __align__(16) float As[2][BK][BM];
  __shared__ __align__(16) float Bs[2][BK][BN];
  int M = p.M;
  if (p.m_count) M = min(M, *p.m_count);
  const TileSel ts = {p.w, p.gather, p.out_index, (int)blockIdx.y};
  for (int mt = blockIdx.x; mt * BM < M; mt += gridDim.x) {
    conv_tile<BM, BN, TM, TN, VECA, VECB>(p, ts, mt * BM, M, As, Bs);
    __syncthreads();                           // the next tile reuses the shared-memory slabs
  }
}

// Fused tap-major sparse convolution: ONE launch walks every (tap, 64-pair tile, 64-column tile) work item of a layer.
// The per-tap launches it replaces were latency-bound (a few 64-row tiles each, K <= 128) and serialised by the stream;
// here all taps' tiles are in flight together and accumulate into the bias-initialised output rows with red.add.
constexpr int MAX_KVOL = 32;
template <bool VECA, bool VECB>
__global__ void __launch_bounds__(256) sparse_conv_taps_kernel(const ConvArgs p, const int* __restrict__ pairs_in,
                                                               const int* __restrict__ pairs_out,
                                                               const int* __restrict__ pair_count, int kvol, int pair_cap) {
  __shared__ __align__(16) float As[2][BK][64];
  __shared__ __align__(16) float Bs[2][BK][64];
  __shared__ int first[MAX_KVOL + 1], cnt[MAX_KVOL];
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int t = 0; t < kvol; ++t) {
      const int c = min(pair_count[t], pair_cap);
      cnt[t] = c;
      first[t] = acc;
      acc += (c + 63) / 64;
    }
    first[kvol] = acc;
  }
  __syncthreads();
  const int n_tiles = (p.Cout_g + 63) / 64;
  const int total = first[kvol] * n_tiles;
  for (int item = blockIdx.x; item < total; item += gridDim.x) {
    const int mt_all = item / n_tiles;
    int tap = 0;
    while (first[tap + 1] <= mt_all) ++tap;
    const TileSel ts = {p.w + (long long)tap * p.Cin_g * p.d.Cout, pairs_in + (long long)tap * pair_cap,
                        pairs_out + (long long)tap * pair_cap, item - mt_all * n_tiles};
    conv_tile<64, 64, 4, 4, VECA, VECB>(p, ts, (mt_all - first[tap]) * 64, cnt[tap], As, Bs);
    __syncthreads();
  }
}

__global__ void splitk_reduce_kernel(const ConvArgs p) {
  const tt_conv_desc& d = p.d;
  int M = p.M;
  if (p.m_count) M = min(M, *p.m_count);
  const long long total = (long long)M * d.Cout;
  const long long yns = d.y_nstride ? d.y_nstride : (long long)d.yH * d.yW * d.y_ld;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int col = i % d.Cout;
    const int row = i / d.Cout;
    float v = 0.f;
    for (int s = 0; s < p.splits; ++s) v += p.partial[((long long)s * p.M + row) * d.Cout + col];   // fixed order
    long long yoff, r1pix = row;
    int n = 0;
    if (p.gather) {
      yoff = (long long)row * d.y_ld;
    } else {
      const int ow = row % d.OW;
      const int t = row / d.OW;
      const int oh = t % d.OH;
      n = t / d.OH;
      yoff = n * yns + ((long long)(oh * d.oy_mul + d.oy_add) * d.yW + ow * d.ox_mul + d.ox_add) * d.y_ld;
      if (d.res_mode == TT_RES_UP2_NEAREST) r1pix = ((long long)n * d.res_H + (oh * d.res_H) / d.OH) * d.res_W + (ow * d.res_W) / d.OW;
    }
    if (p.bias) v += __ldg(p.bias + (d.bias_n_mod ? (long long)(n % d.bias_n_mod) * d.Cout : 0) + col);
    if (p.res) v += p.res[r1pix * d.res_ld + d.res_coff + col];
    if (p.res2) v += p.res2[(long long)row * d.res2_ld + d.res2_coff + col];
    p.y[yoff + d.y_coff + col] = tt_act(v, d.act);
  }
}

template <int BM, int BN, int TM, int TN>
void launch_cfg(const ConvArgs& a, bool veca, bool vecb, cudaStream_t st) {
  int gx = tt_cdiv(a.M, BM);
  if (a.m_count && gx > tt_num_sms() * 8) gx = tt_num_sms() * 8;                  // capacity-sized launches: grid-stride over the tiles
  dim3 grid(gx, tt_cdiv(a.Cout_g, BN), a.d.groups * a.splits);
  if (veca && vecb) conv_igemm_simt<BM, BN, TM, TN, true, true><<<grid, 256, 0, st>>>(a);
  else if (veca) conv_igemm_simt<BM, BN, TM, TN, true, false><<<grid, 256, 0, st>>>(a);
  else if (vecb) conv_igemm_simt<BM, BN, TM, TN, false, true><<<grid, 256, 0, st>>>(a);
  else conv_igemm_simt<BM, BN, TM, TN, false, false><<<grid, 256, 0, st>>>(a);
}

}  // namespace

// split-K plan shared by the launcher and tt_conv2d_workspace_bytes
int tt_simt_splits(const tt_conv_desc* d, int has_gather) {
  const int taps = has_gather ? d->taps : d->KH * d->KW;
  const int M = has_gather ? d->M : d->N * d->OH * d->OW;
  const int Kg = taps * (d->Cin / d->groups);
  const long long tiles = (long long)tt_cdiv(M, 64) * tt_cdiv(d->Cout / d->groups, 64) * d->groups;
  if (has_gather || tiles >= 74 || Kg < 256) return 1;
  int s = tt_cdiv(296, tiles);
  if (s > Kg / 64) s = Kg / 64;
  if (s > 32) s = 32;
  return s < 2 ? 1 : s;
}

int tt_conv2d_simt(const tt_conv_desc* d, const float* x, const float* w, const float* bias, const float* res,
                   const float* res2, const int* gather, const int* m_count, float* y, void* workspace, cudaStream_t st) {
  ConvArgs a;
  a.d = *d;
  a.x = x; a.w = w; a.bias = bias; a.res = res; a.res2 = res2; a.gather = gather; a.m_count = m_count; a.y = y;
  a.Cin_g = d->Cin / d->groups;
  a.Cout_g = d->Cout / d->groups;
  if (gather) {
    a.taps = d->taps;
    a.M = d->M;
  } else {
    a.taps = d->KH * d->KW;
    a.M = d->N * d->OH * d->OW;
  }
  a.Kg = a.taps * a.Cin_g;
  if (a.M <= 0) return TT_OK;
  a.splits = workspace ? tt_simt_splits(d, gather != nullptr) : 1;
  a.k_per_split = a.splits > 1 ? tt_cdiv(tt_cdiv(a.Kg, a.splits), BK) * BK : a.Kg;
  a.partial = static_cast<float*>(workspace);
  a.out_index = nullptr;
  a.accumulate = 0;
  const bool veca = (a.Cin_g % 4 == 0) && (d->x_ld % 4 == 0) && (d->x_coff % 4 == 0) && (d->x_nstride % 4 == 0) && (d->x_hstride % 4 == 0) &&
                    ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  const bool vecb = (a.Cout_g % 4 == 0) && (d->Cout % 4 == 0) && (d->y_nstride % 4 == 0) && ((reinterpret_cast<uintptr_t>(w) & 15) == 0) &&
                    (bias == nullptr || (reinterpret_cast<uintptr_t>(bias) & 15) == 0) &&
                    ((reinterpret_cast<uintptr_t>(y) & 15) == 0) &&
                    (res == nullptr || (reinterpret_cast<uintptr_t>(res) & 15) == 0) &&
                    (res2 == nullptr || (reinterpret_cast<uintptr_t>(res2) & 15) == 0);
  // tile choice: big tiles when they still fill the SMs, otherwise smaller ones
  const long long big = (long long)tt_cdiv(a.M, 128) * tt_cdiv(a.Cout_g, 128) * d->groups;
  if (a.splits > 1) {
    launch_cfg<64, 64, 4, 4>(a, veca, vecb, st);
    ++g_tt_launches;
    TT_CHECK_LAUNCH("tt_conv2d(simt split-k)");
    const long long total = (long long)a.M * d->Cout;
    splitk_reduce_kernel<<<(int)((total + 255) / 256 > 1184 ? 1184 : (total + 255) / 256), 256, 0, st>>>(a);
    ++g_tt_launches;
    TT_CHECK_LAUNCH("tt_conv2d(simt split-k reduce)");
    return TT_OK;
  }
  if (a.Cout_g > 64 && big >= tt_num_sms()) launch_cfg<128, 128, 8, 8>(a, veca, vecb, st);
  else if (a.Cout_g <= 64 && (long long)tt_cdiv(a.M, 128) * d->groups >= tt_num_sms()) launch_cfg<128, 64, 8, 4>(a, veca, vecb, st);
  else launch_cfg<64, 64, 4, 4>(a, veca, vecb, st);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_conv2d(simt)");
  return TT_OK;
}


// ------------------------------------------------------------------------------------------------------------------
// Tap-major sparse convolution (spconv SubMConv3d / SparseConv3d): the rulebook lists, per kernel tap, the (input row,
// output row) pairs that exist.  One gather-GEMM launch per tap over just those pairs — instead of a 27-tap dense
// gather where ~3 taps are populated.  All taps of a layer run in one launch (sparse_conv_taps_kernel) and accumulate
// into the bias-initialised output rows with red.add.f32 (summation order across taps is not fixed: results repeat to
// fp32 rounding, not bitwise).  out = act(sum_taps W_tap . in[pair] + bias + res).
namespace {
__global__ void sparse_rows_init_kernel(float* __restrict__ y, int ld, const float* __restrict__ bias, int C,
                                        const int* __restrict__ count, int cap) {
  const int n = min(*count, cap);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)n * C; i += (long long)gridDim.x * blockDim.x)
    y[(i / C) * ld + (i % C)] = bias ? __ldg(bias + (i % C)) : 0.f;
}
__global__ void sparse_rows_finish_kernel(float* __restrict__ y, int ld, const float* __restrict__ res, int res_ld, int C,
                                          const int* __restrict__ count, int cap, int act) {
  const int n = min(*count, cap);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)n * C; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C;
    const int c = i % C;
    float v = y[r * ld + c];
    if (res) v += res[r * res_ld + c];
    y[r * ld + c] = tt_act(v, act);
  }
}
}  // namespace

bool tt_sparse_conv_tc_supported(const tt_sparse_conv_desc* d, const void* x, const void* w, const void* y);
int tt_sparse_conv_tc(const tt_sparse_conv_desc* d, const float* feats_in, const float* w_tc, const int* pairs_in,
                      const int* pairs_out, const int* pair_count, float* feats_out, cudaStream_t st);

extern "C" int tt_sparse_conv(const tt_sparse_conv_desc* d, const float* feats_in, const float* w, const float* bias,
                              const float* res, const int* pairs_in, const int* pairs_out, const int* pair_count,
                              const int* out_count, float* feats_out, tt_stream_t stream) {
  TT_REQUIRE(d && feats_in && w && pairs_in && pairs_out && pair_count && out_count && feats_out, "tt_sparse_conv", "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (d->cap_out <= 0) return TT_OK;
  const long long tot = (long long)d->cap_out * d->Cout;
  const int nb = (int)((tot + 255) / 256 > 1184 ? 1184 : (tot + 255) / 256);
  sparse_rows_init_kernel<<<nb, 256, 0, st>>>(feats_out, d->out_ld, bias, d->Cout, out_count, d->cap_out);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_sparse_conv(init)");
  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.d.N = a.d.H = a.d.W = a.d.OH = a.d.OW = a.d.yH = a.d.yW = 1;
  a.d.KH = a.d.KW = a.d.stride = a.d.dil = a.d.groups = 1;
  a.d.oy_mul = a.d.ox_mul = 1;
  a.d.Cin = d->Cin; a.d.x_ld = d->in_ld; a.d.Cout = d->Cout; a.d.y_ld = d->out_ld;
  a.d.act = TT_ACT_NONE;
  a.x = feats_in; a.y = feats_out;
  a.M = d->pair_cap; a.Cin_g = d->Cin; a.Cout_g = d->Cout; a.Kg = d->Cin; a.taps = 1;
  a.splits = 1; a.k_per_split = a.Kg; a.accumulate = 1;
  const bool veca = (d->Cin % 4 == 0) && (d->in_ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(feats_in) & 15) == 0);
  const bool vecb = (d->Cout % 4 == 0) && (d->out_ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(w) & 15) == 0) &&
                    ((reinterpret_cast<uintptr_t>(feats_out) & 15) == 0);
  TT_REQUIRE(d->kvol <= MAX_KVOL, "tt_sparse_conv", "kernel volume above 32 taps");
  if (d->impl >= 2) {                                          // tensor-core gather-GEMM; w = [2][Cout][kvol][Cin] hi / lo planes
    if (!tt_sparse_conv_tc_supported(d, feats_in, w, feats_out)) {
      tt_set_error("tt_sparse_conv: impl %d needs Cin, Cout >= 32 and multiples of 4, in_ld / out_ld multiples of 4, 16-byte aligned pointers", d->impl);
      return TT_ERR_UNSUPPORTED;
    }
    const int rc = tt_sparse_conv_tc(d, feats_in, w, pairs_in, pairs_out, pair_count, feats_out, st);
    if (rc != TT_OK) return rc;
    sparse_rows_finish_kernel<<<nb, 256, 0, st>>>(feats_out, d->out_ld, res, d->res_ld, d->Cout, out_count, d->cap_out, d->act);
    ++g_tt_launches;
    TT_CHECK_LAUNCH("tt_sparse_conv(finish)");
    return TT_OK;
  }
  a.w = w;
  a.accumulate = 2;
  {
    const long long cap_tiles = (long long)d->kvol * tt_cdiv(d->pair_cap, 64) * tt_cdiv(d->Cout, 64);
    const int grid = (int)(cap_tiles < tt_num_sms() * 6 ? cap_tiles : tt_num_sms() * 6);
    if (veca && vecb) sparse_conv_taps_kernel<true, true><<<grid, 256, 0, st>>>(a, pairs_in, pairs_out, pair_count, d->kvol, d->pair_cap);
    else if (veca) sparse_conv_taps_kernel<true, false><<<grid, 256, 0, st>>>(a, pairs_in, pairs_out, pair_count, d->kvol, d->pair_cap);
    else if (vecb) sparse_conv_taps_kernel<false, true><<<grid, 256, 0, st>>>(a, pairs_in, pairs_out, pair_count, d->kvol, d->pair_cap);
    else sparse_conv_taps_kernel<false, false><<<grid, 256, 0, st>>>(a, pairs_in, pairs_out, pair_count, d->kvol, d->pair_cap);
    ++g_tt_launches;
  }
  TT_CHECK_LAUNCH("tt_sparse_conv(taps)");
  sparse_rows_finish_kernel<<<nb, 256, 0, st>>>(feats_out, d->out_ld, res, d->res_ld, d->Cout, out_count, d->cap_out, d->act);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_sparse_conv(finish)");
  return TT_OK;
}
