// Camera-feature -> BEV voxel pooling.
//
//  (a) tt_voxel_pooling_forward: ABI-compatible replacement of the reference launcher
//      (ops/voxel_pooling/src/voxel_pooling_forward_cuda.cu).  The reference maps one THREAD to one
//      point and loops 256 scalar atomics with 1 KB-strided reads; here one thread owns 4 channels of
//      one point, so feature reads are coalesced 128-bit loads and the accumulation is one 128-bit
//      vector reduction (red.global.add.v4.f32) per thread.
//  (b) tt_lift_splat: the fused path the model uses.  depth softmax (x) context (x) geometry -> BEV
//      without ever materialising the (B,N,D,H,W,C) tensor (514 MB per sweep at thinktwice.py shapes).
//      K1 walks each pixel's ray, merges consecutive depth bins that land in the same cell into one
//      (cell, weight) run;  K2/K3 bucket the runs per cell (integer atomics only);  K4 is a small
//      SpMM: one CTA per cell sums weight * context_row with coalesced 128-bit loads (context stays
//      L2-resident) and stores the BEV row once — no floating-point atomics, no memset.
#include "common.cuh"

extern long long g_tt_launches;
#define TT_LAUNCHED(name) do { ++g_tt_launches; TT_CHECK_LAUNCH(name); } while (0)

namespace {

TT_DEVICE void red_add_v4(float* addr, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

__global__ void voxel_pool_memo_kernel(int total_points, int num_points, int X, int Y, int Z, const int* __restrict__ geom,
                                       int* __restrict__ pos_memo) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total_points) return;
  const int x = geom[p * 3], y = geom[p * 3 + 1], z = geom[p * 3 + 2];
  if (x < 0 || x >= X || y < 0 || y >= Y || z < 0 || z >= Z) return;
  pos_memo[p * 3] = p / num_points;
  pos_memo[p * 3 + 1] = y;
  pos_memo[p * 3 + 2] = x;
}

template <bool VEC>
__global__ void voxel_pool_kernel(long long total, int num_points, int C, int CV, int X, int Y, int Z,
                                  const int* __restrict__ geom, const float* __restrict__ feats, float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = i % CV;
    const long long p = i / CV;
    const int x = __ldg(geom + p * 3), y = __ldg(geom + p * 3 + 1), z = __ldg(geom + p * 3 + 2);
    if (x < 0 || x >= X || y < 0 || y >= Y || z < 0 || z >= Z) continue;
    const int b = p / num_points;
    float* dst = out + (((long long)b * Y + y) * X + x) * C;
    if (VEC) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(feats + p * C) + cv);
      red_add_v4(dst + cv * 4, v);
    } else {
      atomicAdd(dst + cv, __ldg(feats + p * C + cv));
    }
  }
}

// ------------------------------------------------------------------------------------------------
struct LiftArgs {
  tt_lift_splat_desc d;
  const float* depth;
  const float* ctx;
  const float* mats;
  const float* fu;
  const float* fv;
  const float* fd;
  int* ent_cell;    // [pixels][D]
  float* ent_w;     // [pixels][D]
  int* nrun;        // [pixels]
  int* cell_cnt;    // [B*cells]
  int* cell_start;  // [B*cells + 1]
  int* cell_fill;   // [B*cells]
  int* list_pix;    // [pixels*D]
  float* list_w;
  float* bev;
  int pixels, cells;
};

constexpr int MAXD = 128;

// K1: one thread per feature-map pixel.
__global__ void lift_runs_kernel(const LiftArgs a) {
  const tt_lift_splat_desc& d = a.d;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= a.pixels) return;
  const int w = pix % d.fW;
  const int h = (pix / d.fW) % d.fH;
  const int bn = pix / (d.fW * d.fH);
  const int b = bn / d.N;
  const float* lg = a.depth + (long long)pix * d.ld_d + d.d_coff;
  // softmax over the D depth logits (lss.py:583)
  float mx = -INFINITY;
  for (int i = 0; i < d.D; ++i) mx = fmaxf(mx, lg[i]);
  float sum = 0.f;
  for (int i = 0; i < d.D; ++i) sum += expf(lg[i] - mx);
  const float inv = 1.f / sum;
  const float* Mi = a.mats + (long long)bn * 32;       // ida^-1
  const float* Mc = Mi + 16;                           // sensor2ego @ intrin^-1
  const float u = a.fu[w], v = a.fv[h];
  int cur = -2;
  float acc = 0.f;
  int nr = 0;
  int* ec = a.ent_cell + (long long)pix * d.D;
  float* ew = a.ent_w + (long long)pix * d.D;
  for (int i = 0; i < d.D; ++i) {
    const float dd = a.fd[i];
    // lss.py:496-505: p = ida^-1 (u, v, d, 1); (x*z, y*z, z, 1); combine @ p
    float q[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) q[r] = Mi[r * 4 + 0] * u + Mi[r * 4 + 1] * v + Mi[r * 4 + 2] * dd + Mi[r * 4 + 3] * 1.f;
    const float px = q[0] * q[2], py = q[1] * q[2], pz = q[2], pw = q[3];
    float e[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) e[r] = Mc[r * 4 + 0] * px + Mc[r * 4 + 1] * py + Mc[r * 4 + 2] * pz + Mc[r * 4 + 3] * pw;
    // lss.py:630-631: ((geom - lower) / size).int()  — truncation toward zero
    const int ix = (int)((e[0] - d.lower[0]) / d.size[0]);
    const int iy = (int)((e[1] - d.lower[1]) / d.size[1]);
    const int iz = (int)((e[2] - d.lower[2]) / d.size[2]);
    int cell = -1;
    if (ix >= 0 && ix < d.X && iy >= 0 && iy < d.Y && iz >= 0 && iz < d.Z) cell = iy * d.X + ix;
    const float pr = expf(lg[i] - mx) * inv;
    if (cell != cur) {
      if (cur >= 0) { ec[nr] = cur; ew[nr] = acc; ++nr; atomicAdd(&a.cell_cnt[b * a.cells + cur], 1); }
      cur = cell;
      acc = 0.f;
    }
    acc += pr;
  }
  if (cur >= 0) { ec[nr] = cur; ew[nr] = acc; ++nr; atomicAdd(&a.cell_cnt[b * a.cells + cur], 1); }
  a.nrun[pix] = nr;
}

// K2: exclusive scan of the per-cell counts (one CTA; the array is B*cells long, i.e. small).
__global__ void cell_scan_kernel(const int* __restrict__ cnt, int* __restrict__ start, int* __restrict__ fill, int n) {
  __shared__ int warp_tot[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int v = i < n ? cnt[i] : 0;
    int s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, s, o); if ((threadIdx.x & 31) >= o) s += t; }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
      int t = threadIdx.x < (blockDim.x >> 5) ? warp_tot[threadIdx.x] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int r = __shfl_up_sync(0xffffffffu, t, o); if (threadIdx.x >= o) t += r; }
      warp_tot[threadIdx.x] = t;
    }
    __syncthreads();
    const int wbase = (threadIdx.x >> 5) ? warp_tot[(threadIdx.x >> 5) - 1] : 0;
    if (i < n) { start[i] = carry + wbase + s - v; fill[i] = 0; }
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry += wbase + s;
    __syncthreads();
  }
  if (threadIdx.x == 0) start[n] = carry;
}

// K3: drop each run into its cell's segment.
__global__ void lift_place_kernel(const LiftArgs a) {
  const tt_lift_splat_desc& d = a.d;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= a.pixels) return;
  const int b = pix / (d.fW * d.fH * d.N);
  const int nr = a.nrun[pix];
  for (int r = 0; r < nr; ++r) {
    const int cell = b * a.cells + a.ent_cell[(long long)pix * d.D + r];
    const int pos = a.cell_start[cell] + atomicAdd(&a.cell_fill[cell], 1);
    a.list_pix[pos] = pix;
    a.list_w[pos] = a.ent_w[(long long)pix * d.D + r];
  }
}

// K4: one CTA (8 warps) per (frame, cell); lane owns float4 channel groups, warps split the entries.
__global__ void __launch_bounds__(256) lift_spmm_kernel(const LiftArgs a) {
  extern __shared__ float4 red[];                     // [8][C/4]
  const tt_lift_splat_desc& d = a.d;
  const int cellg = blockIdx.x;                       // b * cells + cell
  const int b = cellg / a.cells, cell = cellg % a.cells;
  const int beg = a.cell_start[cellg], end = a.cell_start[cellg + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int C4 = d.C / 4;
  for (int c0 = 0; c0 < C4; c0 += 64) {               // 64 float4 groups per pass: 2 per lane
    float4 s0 = make_float4(0.f, 0.f, 0.f, 0.f), s1 = s0;
    const int g0 = c0 + lane, g1 = c0 + lane + 32;
    for (int e = beg + warp; e < end; e += 8) {
      const int pix = a.list_pix[e];
      const float w = a.list_w[e];
      const float4* row = reinterpret_cast<const float4*>(a.ctx + (long long)pix * d.ld_c + d.c_coff);
      if (g0 < C4) { const float4 v = __ldg(row + g0); s0.x = fmaf(w, v.x, s0.x); s0.y = fmaf(w, v.y, s0.y); s0.z = fmaf(w, v.z, s0.z); s0.w = fmaf(w, v.w, s0.w); }
      if (g1 < C4) { const float4 v = __ldg(row + g1); s1.x = fmaf(w, v.x, s1.x); s1.y = fmaf(w, v.y, s1.y); s1.z = fmaf(w, v.z, s1.z); s1.w = fmaf(w, v.w, s1.w); }
    }
    red[warp * 64 + lane] = s0;
    red[warp * 64 + lane + 32] = s1;
    __syncthreads();
    if (threadIdx.x < 64 && c0 + threadIdx.x < C4) {
      float4 t = red[threadIdx.x];
#pragma unroll
      for (int wv = 1; wv < 8; ++wv) { const float4 o = red[wv * 64 + threadIdx.x]; t.x += o.x; t.y += o.y; t.z += o.z; t.w += o.w; }
      int oc = cell;
      if (d.anti_transpose) { const int y = cell / d.X, x = cell % d.X; oc = (d.X - 1 - x) * d.X + (d.Y - 1 - y); }
      float* dst = a.bev + ((long long)b * a.cells + oc) * d.bev_ld + d.bev_coff;
      reinterpret_cast<float4*>(dst)[c0 + threadIdx.x] = t;
    }
    __syncthreads();
  }
}

struct LiftWs { size_t ent_cell, ent_w, nrun, cell_cnt, cell_start, cell_fill, list_pix, list_w, total; };
inline size_t al(size_t v) { return (v + 255) & ~(size_t)255; }
LiftWs lift_layout(const tt_lift_splat_desc* d) {
  LiftWs w;
  const size_t pixels = (size_t)d->B * d->N * d->fH * d->fW, cells = (size_t)d->B * d->X * d->Y;
  size_t o = 0;
  w.ent_cell = o; o += al(pixels * d->D * 4);
  w.ent_w = o; o += al(pixels * d->D * 4);
  w.nrun = o; o += al(pixels * 4);
  w.cell_cnt = o; o += al(cells * 4);
  w.cell_start = o; o += al((cells + 1) * 4);
  w.cell_fill = o; o += al(cells * 4);
  w.list_pix = o; o += al(pixels * d->D * 4);
  w.list_w = o; o += al(pixels * d->D * 4);
  w.total = o;
  return w;
}

}  // namespace

extern "C" {

size_t tt_voxel_pooling_workspace_bytes(int, int, int, int) { return 0; }

int tt_voxel_pooling_forward(int batch_size, int num_points, int num_channels, int num_voxel_x, int num_voxel_y,
                             int num_voxel_z, const int* geom_xyz, const float* input_features,
                             float* output_features, int* pos_memo, void* /*workspace*/, tt_stream_t stream) {
  TT_REQUIRE(batch_size >= 0 && num_points >= 0 && num_channels > 0, "tt_voxel_pooling_forward", "bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  const long long tp = (long long)batch_size * num_points;
  if (tp == 0) return TT_OK;                                   // empty input: nothing to add (pointers may be NULL)
  TT_REQUIRE(geom_xyz && input_features && output_features, "tt_voxel_pooling_forward", "null argument");
  TT_REQUIRE(tp < (1ll << 31) / 3, "tt_voxel_pooling_forward", "too many points for int32 indexing");
  if (pos_memo) {
    voxel_pool_memo_kernel<<<tt_cdiv(tp, 256), 256, 0, st>>>((int)tp, num_points, num_voxel_x, num_voxel_y, num_voxel_z,
                                                              geom_xyz, pos_memo);
    TT_LAUNCHED("tt_voxel_pooling_forward(memo)");
  }
  const bool vec = (num_channels % 4 == 0) && ((reinterpret_cast<uintptr_t>(input_features) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(output_features) & 15) == 0);
  const int CV = vec ? num_channels / 4 : num_channels;
  const long long total = tp * CV;
  const int blocks = (int)((total + 255) / 256 > tt_num_sms() * 32 ? tt_num_sms() * 32 : (total + 255) / 256);
  if (vec)
    voxel_pool_kernel<true><<<blocks, 256, 0, st>>>(total, num_points, num_channels, CV, num_voxel_x, num_voxel_y,
                                                     num_voxel_z, geom_xyz, input_features, output_features);
  else
    voxel_pool_kernel<false><<<blocks, 256, 0, st>>>(total, num_points, num_channels, CV, num_voxel_x, num_voxel_y,
                                                      num_voxel_z, geom_xyz, input_features, output_features);
  TT_LAUNCHED("tt_voxel_pooling_forward");
  return TT_OK;
}

size_t tt_lift_splat_workspace_bytes(const tt_lift_splat_desc* d) { return d ? lift_layout(d).total : 0; }

int tt_lift_splat(const tt_lift_splat_desc* d, const float* depth_logits, const float* context, const float* mats,
                  const float* frustum_u, const float* frustum_v, const float* frustum_d, float* bev, void* workspace,
                  tt_stream_t stream) {
  TT_REQUIRE(d && depth_logits && context && mats && frustum_u && frustum_v && frustum_d && bev && workspace,
             "tt_lift_splat", "null argument");
  TT_REQUIRE(d->D <= MAXD && d->C % 4 == 0 && d->ld_c % 4 == 0 && d->c_coff % 4 == 0 && d->bev_ld % 4 == 0 &&
                 d->bev_coff % 4 == 0,
             "tt_lift_splat", "unsupported channel layout");
  TT_REQUIRE(!d->anti_transpose || d->X == d->Y, "tt_lift_splat", "anti_transpose needs a square grid");
  cudaStream_t st = (cudaStream_t)stream;
  const LiftWs L = lift_layout(d);
  char* ws = static_cast<char*>(workspace);
  LiftArgs a;
  a.d = *d;
  a.depth = depth_logits; a.ctx = context; a.mats = mats; a.fu = frustum_u; a.fv = frustum_v; a.fd = frustum_d;
  a.ent_cell = (int*)(ws + L.ent_cell); a.ent_w = (float*)(ws + L.ent_w); a.nrun = (int*)(ws + L.nrun);
  a.cell_cnt = (int*)(ws + L.cell_cnt); a.cell_start = (int*)(ws + L.cell_start); a.cell_fill = (int*)(ws + L.cell_fill);
  a.list_pix = (int*)(ws + L.list_pix); a.list_w = (float*)(ws + L.list_w);
  a.bev = bev;
  a.pixels = d->B * d->N * d->fH * d->fW;
  a.cells = d->X * d->Y;
  const int ncell = d->B * a.cells;
  if (cudaMemsetAsync(a.cell_cnt, 0, (size_t)ncell * 4, st) != cudaSuccess) { tt_set_error("tt_lift_splat: memset failed"); return TT_ERR_CUDA; }
  lift_runs_kernel<<<tt_cdiv(a.pixels, 128), 128, 0, st>>>(a);
  TT_LAUNCHED("tt_lift_splat(runs)");
  cell_scan_kernel<<<1, 1024, 0, st>>>(a.cell_cnt, a.cell_start, a.cell_fill, ncell);
  TT_LAUNCHED("tt_lift_splat(scan)");
  lift_place_kernel<<<tt_cdiv(a.pixels, 128), 128, 0, st>>>(a);
  TT_LAUNCHED("tt_lift_splat(place)");
  lift_spmm_kernel<<<ncell, 256, 8 * 64 * sizeof(float4), st>>>(a);
  TT_LAUNCHED("tt_lift_splat(spmm)");
  return TT_OK;
}

}  // extern "C"

// Link-level drop-in for the reference's launcher: ops/voxel_pooling/src/voxel_pooling_forward.cpp:21-22 declares exactly
// this C++ symbol and calls it from voxel_pooling_forward_wrapper (:36); the reference defines it in
// src/voxel_pooling_forward_cuda.cu:38-56.  Building the reference's .cpp against libtt_b200.so instead of its own .cu
// resolves here.  Same argument list, `void`; unlike the reference (which exit(-1)s on a launch error, :51-54) a failure is
// reported on stderr and through tt_last_error().
void voxel_pooling_forward_kernel_launcher(int batch_size, int num_points, int num_channels, int num_voxel_x, int num_voxel_y,
                                           int num_voxel_z, const int* geom_xyz, const float* input_features,
                                           float* output_features, int* pos_memo, cudaStream_t stream) {
  if (tt_voxel_pooling_forward(batch_size, num_points, num_channels, num_voxel_x, num_voxel_y, num_voxel_z, geom_xyz,
                               input_features, output_features, pos_memo, nullptr, (tt_stream_t)stream) != TT_OK)
    fprintf(stderr, "voxel_pooling_forward_kernel_launcher: %s\n", tt_last_error());
}
