// Hopper (sm_90a) implicit-GEMM convolution on SCALED-SPLIT FP16 operands ("f16s") — the successor of the 3xTF32 kernel in
// gemm_conv_tc.cu (same tiling, same epilogue contract, same fp32-class accuracy, half the operand bytes and twice the
// tensor-core rate).
//
// Operand format.  An fp32 value x is carried as two halves:  hi = RN_f16(x),  lo = RN_f16((x - hi) * 2^11).
//   x - hi is exact in fp32 and |x - hi| <= 2^-11 |x|, so lo is O(|x|) again (no fp16 underflow of the correction) and
//   x = hi + lo * 2^-11 to 2^-22 relative (fp16 has the same 11 significant bits as TF32): the same representation error as
//   the TF32 hi / lo split, at 4 bytes per element instead of 8.  Activations live in HBM in this form next to (or instead
//   of) their fp32 copy: a "split" tensor is two half planes [2][N][H][W][ld] written by the PRODUCING kernel's epilogue, so
//   the consumer's TMA loads deliver tensor-core-ready operands — no split pass, no shared-memory rewrite.
//   Range: |x| must stay below 65504 (hi saturates; counted in g_f16s_saturated, read with tt_f16s_saturation_count).
// Products.  Per K step (16 halves) three m64nBNk16 wgmma per warpgroup, the 3-product scheme of the TF32 kernel:
//   main  +=  A_hi x B_hi,   corr  +=  A_hi x B_lo',   corr  +=  A_lo' x B_hi
//   result = main + 2^-11 corr  (the dropped lo x lo term is 2^-22 relative).  main and corr are separate register arrays and every
//   instruction has the same shape: wgmma of different shapes on overlapping accumulators would be serialised by the compiler.  The register accumulator is restarted every
//   `chunk` stages and folded into fp32 sums with round-to-nearest FMAs, so the tensor core's own accumulation only ever
//   spans 2 x 64 K elements.
// Tiling follows gemm_conv_tc.cu: TMA box loads per tap (zero fill = padding, element strides = stride 2), persistent CTAs
// (one per SM), split-K and GATHER (sparse convolution).
// Warp roles: warpgroup 0 = producer (dense: one TMA thread; tap-major sparse: warp 0 gathers; output-stationary sparse: all four
// warps gather, one tile row per thread); warpgroups 1 and 2 = wgmma + epilogue for rows 0..63 / 64..127 of the tile.  The producer
// keeps 40 registers per thread (88 for the tap-major gather) and the MMA warpgroups take the rest (setmaxnreg), which lets a
// 128-column tile keep its 192 accumulators in registers.
#include <cuda.h>
#include <cuda_fp16.h>
#include <string.h>

#include "common.cuh"
#include "tc_ptx.cuh"

extern long long g_tt_launches;
extern int g_tt_debug;

__device__ unsigned int g_f16s_saturated = 0;     // number of values an epilogue had to clamp to the fp16 range

namespace {

constexpr int BM = 128;           // M tile: two warpgroups x 64 rows
constexpr int KE = 64;            // K elements per stage (one 128-byte swizzle row of halves)
constexpr int NTHREADS = 384;     // warpgroup 0 producer, warpgroups 1..2 MMA + epilogue
// registers per thread after setmaxnreg (a 384-thread CTA starts with 168): the TMA producer is one thread with a handful of
// values, and so is each thread of the output-stationary gather (one row, its indices in shared memory); the tap-major gather
// (GM 1) keeps the row indices of its pair tile in registers and needs more
template <int GM> constexpr int reg_producer() { return GM == 1 ? 88 : 40; }
template <int GM> constexpr int reg_mma() { return GM == 1 ? 208 : 232; }
static_assert(128 * reg_producer<0>() + 256 * reg_mma<0>() <= 168 * NTHREADS &&
              128 * reg_producer<1>() + 256 * reg_mma<1>() <= 168 * NTHREADS, "setmaxnreg must not ask for more than the CTA holds");
constexpr float LO_SCALE = 2048.f, LO_INV = 1.f / 2048.f;
constexpr int MAX_KVOL = 32;
// shared memory beyond the stage ring: 8 warp-private transposition slabs, barriers, the tap prefix (GM 1) and the per-stage tile
// length and tap masks (GM 2); then, output-stationary only, the neighbour block of the current 128-row tile
constexpr int EPI_BYTES = 8 * 16 * 20 * 4 + 512;
constexpr int NB_BYTES = 128 * MAX_KVOL * 4;
constexpr float H_MAX = 65504.f;

TT_DEVICE void tma_load_5d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// x -> (hi, lo') with saturation to the fp16 range; returns true when x had to be clamped (or is NaN).  A NaN stays NaN in both
// halves, as RN_f16 gives it (fmaxf / fminf would turn it into -65504; the .NaN forms cost the same): tt_split_f16 also sweeps arena
// rows no kernel has written
TT_DEVICE bool split_h(float x, __half& hi, __half& lo) {
  float c;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(c) : "f"(x), "f"(-H_MAX));
  asm("min.NaN.f32 %0, %0, %1;" : "+f"(c) : "f"(H_MAX));
  hi = __float2half_rn(c);
  lo = __float2half_rn((c - __half2float(hi)) * LO_SCALE);
  return c != x;
}
TT_DEVICE void split4(const float4& o, uint2& hi, uint2& lo, bool& sat) {
  __half h[4], l[4];
  sat |= split_h(o.x, h[0], l[0]);
  sat |= split_h(o.y, h[1], l[1]);
  sat |= split_h(o.z, h[2], l[2]);
  sat |= split_h(o.w, h[3], l[3]);
  hi.x = (uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16);
  hi.y = (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16);
  lo.x = (uint32_t)__half_as_ushort(l[0]) | ((uint32_t)__half_as_ushort(l[1]) << 16);
  lo.y = (uint32_t)__half_as_ushort(l[2]) | ((uint32_t)__half_as_ushort(l[3]) << 16);
}

// four hi / lo' pairs -> fp32 (hi + lo' 2^-11)
TT_DEVICE float4 merge_split4(const uint2& h, const uint2& l) {
  const __half2 h0 = *reinterpret_cast<const __half2*>(&h.x), h1 = *reinterpret_cast<const __half2*>(&h.y);
  const __half2 l0 = *reinterpret_cast<const __half2*>(&l.x), l1 = *reinterpret_cast<const __half2*>(&l.y);
  const float2 a = __half22float2(h0), b = __half22float2(h1), c = __half22float2(l0), e = __half22float2(l1);
  return make_float4(fmaf(c.x, LO_INV, a.x), fmaf(c.y, LO_INV, a.y), fmaf(e.x, LO_INV, b.x), fmaf(e.y, LO_INV, b.y));
}
TT_DEVICE float4 load_split4(const __half* hi_ptr, long long plane) {
  return merge_split4(*reinterpret_cast<const uint2*>(hi_ptr), *reinterpret_cast<const uint2*>(hi_ptr + plane));
}

// tt_act over four values with one test of the (kernel-uniform) activation for the inline cases: tested per element, the out-of-line
// call of the rare activations put two compares and three branches around every value of the epilogue
TT_DEVICE float4 act4(const float4& o, int act) {
  if (act == TT_ACT_NONE) return o;
  if (act == TT_ACT_RELU) return make_float4(fmaxf(o.x, 0.f), fmaxf(o.y, 0.f), fmaxf(o.z, 0.f), fmaxf(o.w, 0.f));
  return make_float4(tt_act(o.x, act), tt_act(o.y, act), tt_act(o.z, act), tt_act(o.w, act));
}

struct HArgs {
  tt_conv_desc d;
  const float* bias;
  const float* res;
  const float* res2;
  const __half* res_s;   // residuals given as split planes instead of fp32 (same element offsets; lo' plane res*_plane further)
  const __half* res2_s;
  long long res_plane, res2_plane;
  float* y;              // fp32 output (may be NULL when only the split planes are wanted)
  __half* ys;            // split output: hi plane at the same element offsets as y; lo' plane ys_plane halves further (or NULL)
  long long ys_plane;
  int TH, TW;            // tile rectangle (TH * TW <= 128); flat mode: TH = 1, TW = 128 over N*H*W pixels
  int tiles_w, tiles_h;
  int flat;
  int n_slabs;           // ceil(Cin / 64)
  int chunk;             // stages accumulated by the tensor core before the epilogue warpgroups fold them into fp32 sums
  int total_pix;
  int m_tiles, n_tiles;
  // GATHER (tap-major sparse convolution)
  const __half* gx;      // split feature rows: hi plane [.][gx_ld], lo' plane gx_plane halves further
  long long gx_plane;
  int gx_ld;
  const int* pairs_in;
  const int* pairs_out;
  const int* pair_count;
  int kvol, pair_cap;
  const int* nbr;        // output-stationary: [cap_rows][kvol] input row under each tap of an output row, -1 = none
  const int* out_count;  // output-stationary: number of output rows (device scalar)
  int cap_rows;
  int tps;               // output-stationary: taps per 64-half K slab (2 when Cin == 32, else 1)
  int splits, k_per;     // split-K: K stages per split
};

// GM (gather mode): 0 = dense convolution (TMA box loads); 1 = tap-major sparse convolution (work item = one tap's pair tile,
// red.add epilogue); 2 = output-stationary sparse convolution (work item = an output-row tile, K runs over the taps that some row
// of the tile uses, through the neighbour table; plain fused epilogue — no atomics, no init / finish passes).
template <int BN, int STAGES, int GM>
__global__ void __launch_bounds__(NTHREADS, 1)
conv_f16s_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const HArgs p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr int A_BYTES = BM * KE * 2;                    // 16 KB per plane
  constexpr int B_BYTES = BN * KE * 2;                    // per plane
  constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
  constexpr int SLAB = 16;                                // epilogue column slab
  constexpr int PITCH = SLAB + 4;                         // +4 floats: conflict-free transposition
  // rounded up to 1 KB as an offset from smem_raw, not through an integer: the compiler then keeps the shared address space, and the
  // epilogue's transposition compiles to shared-memory loads and stores instead of generic ones
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* tile_all = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);              // [8 MMA warps][16 rows][PITCH]
  uint64_t* bars = reinterpret_cast<uint64_t*>(tile_all + 8 * 16 * PITCH);
  uint64_t* full = bars;                                  // [STAGES]  producer -> MMA (operands landed)
  uint64_t* empty = bars + STAGES;                        // [STAGES]  MMA warps -> producer
  int* sp_first = reinterpret_cast<int*>(bars + 2 * STAGES);
  int* sp_cnt = sp_first + MAX_KVOL + 1;
  int* tile_k = sp_cnt + MAX_KVOL;                        // [STAGES] output-stationary: K stages of the tile a stage belongs to
  uint32_t* wmask = reinterpret_cast<uint32_t*>(tile_k + STAGES);                    // [4] per producer warp: taps its rows use
  int* nb_s = reinterpret_cast<int*>(smem + STAGES * STAGE_BYTES + EPI_BYTES);       // [BM][kvol] (GM == 2)

  const tt_conv_desc& d = p.d;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr bool GATHER = GM != 0;
  const int taps = d.KH * d.KW;
  const int k_iters = taps * p.n_slabs;
  const int os_rows = GM == 2 ? min(*p.out_count, p.cap_rows) : 0;     // output-stationary: rows that exist (device count)

  if (threadIdx.x == 0) {
    // full: one arrival with the expected bytes + one cp.async arrival per gathering thread (GM 1: warp 0; GM 2: warps 0..3)
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], GM == 2 ? 129 : GM == 1 ? 33 : 1); mbar_init(&empty[s], 8); }   // 8 MMA warps release a stage
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (GM == 1 && threadIdx.x == 64) {
    int acc = 0;
    for (int t = 0; t < p.kvol; ++t) {
      const int c = min(p.pair_count[t], p.pair_cap);
      sp_cnt[t] = c;
      sp_first[t] = acc;
      acc += (c + BM - 1) / BM;
    }
    sp_first[p.kvol] = acc;
  }
  __syncthreads();
  const int os_tiles = (os_rows + BM - 1) / BM;
  const int total_items = (GM == 1 ? sp_first[p.kvol] : GM == 2 ? os_tiles : p.m_tiles) * p.n_tiles * p.splits;
  auto decode = [&](int pt, int& nt, int& mt, int& tap, int& count, int& kb, int& ke) {
    const int ks = pt % p.splits;
    pt /= p.splits;
    kb = ks * p.k_per;
    ke = min(k_iters, kb + p.k_per);
    nt = pt % p.n_tiles;
    const int pm = pt / p.n_tiles;
    tap = 0; count = 0;
    if (GM == 2) {
      mt = pm;
      count = os_rows;
    } else if (GM == 1) {
      while (sp_first[tap + 1] <= pm) ++tap;
      mt = pm - sp_first[tap];
      count = sp_cnt[tap];
    } else {
      mt = pm;
    }
  };

  // weight slab of one stage: hi plane then lo' plane, BN rows each, loaded as two BN / 2-row boxes per plane
  auto load_weights = [&](uint8_t* st, uint64_t* bar, int k0, int tap, int n0) {
    uint8_t* bh = st + 2 * A_BYTES;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      tma_load_4d(bh + h * (B_BYTES / 2), &map_b, bar, k0, tap, n0 + h * (BN / 2), 0);
      tma_load_4d(bh + B_BYTES + h * (B_BYTES / 2), &map_b, bar, k0, tap, n0 + h * (BN / 2), 1);
    }
  };

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(reg_producer<GM>()));
    if (GM == 2) {
      // ===================================================================== output-stationary gather (4 warps) + weight TMA
      // Per tile: the tile's neighbour block [128 rows][kvol] goes to shared memory (rows at or past the device count read as -1:
      // the table may hold stale rows of a larger cloud there), each of the 128 producer threads gathers one row, and the K walk
      // visits only the K units that some row of the tile uses: taps, or tap pairs when two taps share a slab (Cin = 32).  The
      // tile's stage count reaches the MMA warps through tile_k[stage], written before the stage's full barrier arrival.  A tile
      // that uses no tap at all still runs one stage of zero rows, so that its epilogue writes bias + activation (+ residual).
      // Shared-memory budget: one 16 KB neighbour block next to the 4-stage ring (BN 64) / 3-stage ring (BN 128), about 220 KB;
      // a second block to prefetch the next tile's indices would cost a ring stage.  The block's loads are issued while the MMA
      // warps still consume the previous tile's stages in flight.  They are coalesced plain loads rather than one bulk copy: the
      // live part of the block ends at the device count, on any 4-byte boundary, and a bulk copy moves multiples of 16 bytes.
      const int t = threadIdx.x, kv = p.kvol;
      const int upb = p.tps == 2 ? 1 : 0;                    // K unit of tap k: k >> upb
      const int spu = p.tps == 2 ? 1 : p.n_slabs;             // stages per K unit
      const uint32_t txb = 2 * B_BYTES;
      int ig = 0;
      for (int pt = blockIdx.x; pt < total_items; pt += gridDim.x) {
        int nt, mt, tap, count, kb, ke;
        decode(pt, nt, mt, tap, count, kb, ke);
        const int n0 = nt * BN;
        asm volatile("bar.sync 1, 128;" ::: "memory");        // every producer thread is done with the previous block
        const int lim = min(count - mt * BM, BM) * kv;
        const int* nsrc = p.nbr + (long long)mt * BM * kv;
        for (int i = t; i < BM * kv; i += 128) nb_s[i] = i < lim ? __ldg(nsrc + i) : -1;
        asm volatile("bar.sync 1, 128;" ::: "memory");
        const int* my = nb_s + t * kv;                        // stride kvol (odd for 3^3 / 3 taps): conflict-free
        uint32_t bits = 0;
        for (int k = 0; k < kv; ++k) bits |= (my[k] >= 0 ? 1u : 0u) << (k >> upb);
        bits = __reduce_or_sync(0xffffffffu, bits);
        if (lane == 0) wmask[warp] = bits;
        asm volatile("bar.sync 1, 128;" ::: "memory");
        uint32_t mask = wmask[0] | wmask[1] | wmask[2] | wmask[3];
        const bool none = mask == 0;
        const int nst = none ? 1 : __popc(mask) * spu;
        if (none) mask = 1;
        for (int j = 0, slab = 0; j < nst; ++j, ++ig) {
          const int u = __ffs(mask) - 1;
          const int s = ig % STAGES;
          mbar_wait(&empty[s], ((ig / STAGES) & 1) ^ 1);
          uint8_t* st = smem + s * STAGE_BYTES;
          if (t == 0) {
            tile_k[s] = nst;
            mbar_expect_tx(&full[s], txb);                   // (release: orders the tile_k store before the MMA warps' acquire)
            // two taps per slab: weights viewed as [Cout][kvol * 32], K runs across the taps; else one tap's Cin per slab walk
            if (upb) load_weights(st, &full[s], u * KE, 0, n0);
            else load_weights(st, &full[s], slab * KE, u, n0);
          }
          const uint32_t dst = smem_u32(st) + t * 128;
          if (upb) {
            // chunks 0..3 of the row come from the neighbour under tap 2 u, chunks 4..7 from tap 2 u + 1
            const int ra = none ? -1 : my[2 * u], rb = (none || 2 * u + 1 >= kv) ? -1 : my[2 * u + 1];
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int row = jj < 4 ? ra : rb;
              const bool ok = row >= 0;
              const __half* src = p.gx + (long long)max(row, 0) * p.gx_ld + (jj & 3) * 8;
              const uint32_t o = (uint32_t)((jj ^ (t & 7)) << 4);          // 16-byte chunk jj of row t lives at chunk jj ^ (t & 7)
              cp_async16(dst + o, ok ? (const void*)src : (const void*)p.gx, ok ? 16 : 0);
              cp_async16(dst + A_BYTES + o, ok ? (const void*)(src + p.gx_plane) : (const void*)p.gx, ok ? 16 : 0);
            }
          } else {
            const int row = none ? -1 : my[u];
            const int c0 = slab * KE;
            const __half* src = p.gx + (long long)max(row, 0) * p.gx_ld + c0;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const bool ok = row >= 0 && c0 + jj * 8 < d.Cin;
              const uint32_t o = (uint32_t)((jj ^ (t & 7)) << 4);
              cp_async16(dst + o, ok ? (const void*)(src + jj * 8) : (const void*)p.gx, ok ? 16 : 0);
              cp_async16(dst + A_BYTES + o, ok ? (const void*)(src + p.gx_plane + jj * 8) : (const void*)p.gx, ok ? 16 : 0);
            }
          }
          cp_async_arrive_noinc(&full[s]);
          if (++slab == spu) { slab = 0; mask &= mask - 1; }
        }
      }
    } else if (warp == 0 && GM == 1) {
      // ===================================================================== tap-major gather producer (whole warp) + weight TMA
      const uint32_t txb = 2 * B_BYTES;
      int ig = 0;
      for (int pt = blockIdx.x; pt < total_items; pt += gridDim.x) {
        int nt, mt, tap, count, kb, ke;
        decode(pt, nt, mt, tap, count, kb, ke);
        const int n0 = nt * BN;
        const int* pin = p.pairs_in + (long long)tap * p.pair_cap;
        int rows[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int m = mt * BM + lane + 32 * i;
          rows[i] = m < count ? __ldg(pin + m) : -1;
        }
        for (int it = kb; it < ke; ++it, ++ig) {
          const int s = ig % STAGES;
          mbar_wait(&empty[s], ((ig / STAGES) & 1) ^ 1);
          uint8_t* st = smem + s * STAGE_BYTES;
          if (lane == 0) {
            mbar_expect_tx(&full[s], txb);
            load_weights(st, &full[s], it * KE, tap, n0);
          }
          const int c0 = it * KE;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int r = lane + 32 * i;
            const __half* src = p.gx + (long long)max(rows[i], 0) * p.gx_ld + c0;
            const uint32_t dst = smem_u32(st) + r * 128;
#pragma unroll
            for (int j = 0; j < 8; ++j) {                       // 16-byte chunk j (8 halves) of row r lives at chunk j ^ (r & 7)
              const bool ok = rows[i] >= 0 && c0 + j * 8 < d.Cin;
              const uint32_t o = (uint32_t)((j ^ (r & 7)) << 4);
              cp_async16(dst + o, ok ? (const void*)(src + j * 8) : (const void*)p.gx, ok ? 16 : 0);
              cp_async16(dst + A_BYTES + o, ok ? (const void*)(src + p.gx_plane + j * 8) : (const void*)p.gx, ok ? 16 : 0);
            }
          }
          cp_async_arrive_noinc(&full[s]);
        }
      }
    } else if (warp == 0 && lane == 0) {
      // ===================================================================== TMA producer
      const uint32_t a_box = (uint32_t)(p.flat ? BM : p.TH * p.TW) * KE * 2;   // bytes one activation box (one plane) delivers
      const uint32_t tx = 2 * a_box + 2 * B_BYTES;
      int ig = 0;
      for (int pt = blockIdx.x; pt < total_items; pt += gridDim.x) {
        int nt, mt, tap0, count, kb, ke;
        decode(pt, nt, mt, tap0, count, kb, ke);
        const int n0 = nt * BN;
        int cw0, ch0, cn;
        if (p.flat) { cw0 = mt * BM; ch0 = 0; cn = 0; }
        else {
          const int tw = mt % p.tiles_w, th = (mt / p.tiles_w) % p.tiles_h;
          cn = mt / (p.tiles_w * p.tiles_h);
          cw0 = tw * p.TW * d.stride - d.pad; ch0 = th * p.TH * d.stride - d.pad;
        }
        for (int it = kb; it < ke; ++it, ++ig) {
          const int s = ig % STAGES;
          mbar_wait(&empty[s], ((ig / STAGES) & 1) ^ 1);
          uint8_t* st = smem + s * STAGE_BYTES;
          const int tap = it / p.n_slabs, slab = it - tap * p.n_slabs;
          const int kh = tap / d.KW, kw = tap - kh * d.KW;
          mbar_expect_tx(&full[s], tx);
          if (p.flat) {
            tma_load_3d(st, &map_a, &full[s], slab * KE, cw0, 0);
            tma_load_3d(st + A_BYTES, &map_a, &full[s], slab * KE, cw0, 1);
          } else {
            const int cw = cw0 + kw * d.dil, ch = ch0 + kh * d.dil;
            tma_load_5d(st, &map_a, &full[s], slab * KE, cw, ch, cn, 0);
            tma_load_5d(st + A_BYTES, &map_a, &full[s], slab * KE, cw, ch, cn, 1);
          }
          load_weights(st, &full[s], slab * KE, tap, n0);
        }
      }
    }
  } else {
    // ===================================================================== MMA + epilogue (warpgroups 1, 2)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(reg_mma<GM>()));
    const int cw = warp - 4;                                // MMA warp 0..7
    const int wg = cw >> 2;                                 // warpgroup: tile rows [64 wg, 64 wg + 64)
    const int row0 = wg * 64 + (cw & 3) * 16;               // this warp's 16 accumulator rows
    const long long yns = d.y_nstride ? d.y_nstride : (long long)d.yH * d.yW * d.y_ld;
    const int HWo = d.OH * d.OW;
    float* tile = tile_all + cw * 16 * PITCH;               // warp-private transposition buffer [16 rows][PITCH]
    const int sub = lane >> 2, cl = (lane & 3) * 4;         // store phase: 4 lanes per row, 8 rows per warp instruction
    bool sat = false;
    int ig = 0;
    for (int pt = blockIdx.x; pt < total_items; pt += gridDim.x) {
      int nt, mt, tap, count, kb, ke;
      decode(pt, nt, mt, tap, count, kb, ke);
      if (GM == 2) {                                         // the producer chose the tile's K walk: its length rides with stage 0
        const int s = ig % STAGES;
        mbar_wait(&full[s], (ig / STAGES) & 1);
        ke = kb + tile_k[s];
      }
      const int nch = (ke - kb + p.chunk - 1) / p.chunk;
      // ---- K walk: chunks of `chunk` stages accumulated by the tensor core, folded into fp32 sums with RN FMAs
      float sum[BN / 2];
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) sum[j] = 0.f;
      auto release = [&](int s) {                            // this warp's wgmmas no longer read stage s
        __syncwarp();
        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty[s])) : "memory");
      };
      int it = kb;
      for (int c = 0; c < nch; ++c) {
        // main and correction accumulators.  The first wgmma of a chunk overwrites them (scale-d 0), but the asm operands are
        // read-write: without a definition here they would count as live around the work-item loop, through the epilogue.
        float acc[BN / 2], cor[BN / 2];
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) acc[j] = cor[j] = 0.f;
        const int it_end = min(it + p.chunk, ke);
        int held = -1;                                       // the stage whose wgmmas may still be in flight
        for (bool first = true; it < it_end; ++it, ++ig, first = false) {
          const int s = ig % STAGES;
          mbar_wait(&full[s], (ig / STAGES) & 1);
          if (GATHER) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // cp.async rows -> visible to wgmma
          const uint32_t a_hi = smem_u32(smem + s * STAGE_BYTES) + wg * (A_BYTES / 2), a_lo = a_hi + A_BYTES;
          const uint32_t b_hi = smem_u32(smem + s * STAGE_BYTES) + 2 * A_BYTES, b_lo = b_hi + B_BYTES;
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < KE / 16; ++kk) {             // K = 16 halves = 32 bytes inside the 128-byte swizzle row
            const uint32_t off = kk * 32, z = (first && kk == 0) ? 0u : 1u;
            wgmma_f16<BN>(acc, make_smem_desc(a_hi + off), make_smem_desc(b_hi + off), z);    // hi*hi
            wgmma_f16<BN>(cor, make_smem_desc(a_hi + off), make_smem_desc(b_lo + off), z);    // hi*lo'
            wgmma_f16<BN>(cor, make_smem_desc(a_lo + off), make_smem_desc(b_hi + off), 1u);   // lo'*hi
          }
          wgmma_commit();
          if (held >= 0) {                                   // one stage stays in flight: the previous one is complete now
            wgmma_wait<1>();
            release(held);
          }
          held = s;
        }
        wgmma_wait<0>();
        release(held);
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) sum[j] += fmaf(cor[j], LO_INV, acc[j]);
      }
      // ---- output / residual addresses of the two rows this lane stores (rows row0 + sub, row0 + 8 + sub); computed after the
      // K walk so that they do not hold registers across it
      const bool real_tile = GATHER ? mt * BM < count : mt < p.m_tiles;
      const int n0 = nt * BN;
      int fl[2];
      long long yo[2], o1[2], o2[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = row0 + i * 8 + sub;
        const int m = mt * BM + r;
        o2[i] = 0;
        if (GM == 2) {
          fl[i] = m < count ? 1 : 0;
          yo[i] = (long long)m * d.y_ld + d.y_coff;
          o1[i] = (long long)m * d.res_ld + d.res_coff;
        } else if (GM == 1) {
          const bool valid = m < count;
          const int orow = valid ? __ldg(p.pairs_out + (long long)tap * p.pair_cap + m) : 0;
          fl[i] = valid ? 1 : 0;
          yo[i] = (long long)orow * d.y_ld + d.y_coff;
          o1[i] = 0;
        } else {
          bool valid;
          int nimg, oh, ow;
          long long rrow;
          if (p.flat) {
            const int pix = m;                                 // (the host checked N * OH * OW < 2^31: 32-bit index math)
            valid = real_tile && pix < p.total_pix;
            nimg = pix / HWo;
            const int rem = pix - nimg * HWo;
            oh = rem / d.OW; ow = rem - oh * d.OW;
            rrow = pix;
          } else {
            const int tw = mt % p.tiles_w, th = (mt / p.tiles_w) % p.tiles_h;
            nimg = mt / (p.tiles_w * p.tiles_h);
            const int rh = r / p.TW, rw = r - rh * p.TW;
            oh = th * p.TH + rh; ow = tw * p.TW + rw;
            valid = real_tile && (r < p.TH * p.TW) && oh < d.OH && ow < d.OW;
            rrow = ((long long)nimg * d.OH + oh) * d.OW + ow;
          }
          o1[i] = (d.res_mode == TT_RES_UP2_NEAREST
                       ? ((long long)nimg * d.res_H + (oh * d.res_H) / d.OH) * d.res_W + (ow * d.res_W) / d.OW
                       : rrow) * d.res_ld + d.res_coff;
          o2[i] = rrow * d.res2_ld + d.res2_coff;
          yo[i] = nimg * yns + ((long long)(oh * d.oy_mul + d.oy_add) * d.yW + ow * d.ox_mul + d.ox_add) * d.y_ld + d.y_coff;
          fl[i] = (valid ? 1 : 0) | (nimg << 1);
        }
      }
      // ---- residual and bias strip: the loads for all BN / 16 slabs are issued before the first slab is stored, so that a thread
      // has its whole strip in flight at once instead of paying one memory round trip per 16 columns (acc[] / cor[] are dead here,
      // which leaves the registers).  A split residual stays as its raw hi / lo' halves until it is used.
      constexpr int NSL = BN / SLAB;
      const bool res_split = !p.res && p.res_s;
      uint4 rv[NSL][2];                                       // fp32 residual bits, or split (hi.x, hi.y, lo.x, lo.y); 0 = none
      float4 bv[NSL];                                         // bias vector; per-image rows (bias_n_mod) are loaded per slab below
#pragma unroll
      for (int sl = 0; sl < NSL; ++sl) {
        const int col = n0 + sl * SLAB + cl;
        const bool live = col < d.Cout;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          rv[sl][i] = make_uint4(0u, 0u, 0u, 0u);
          if (live && (fl[i] & 1)) {
            if (p.res) {
              rv[sl][i] = *reinterpret_cast<const uint4*>(p.res + o1[i] + col);
            } else if (p.res_s) {
              const uint2 h = *reinterpret_cast<const uint2*>(p.res_s + o1[i] + col);
              const uint2 l = *reinterpret_cast<const uint2*>(p.res_s + p.res_plane + o1[i] + col);
              rv[sl][i] = make_uint4(h.x, h.y, l.x, l.y);
            }
          }
        }
        bv[sl] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live && p.bias && !d.bias_n_mod) bv[sl] = __ldg(reinterpret_cast<const float4*>(p.bias + col));
      }
      // ---- coalesced store in 16-column slabs: registers -> warp-private smem (transpose) -> 64-byte row segments
#pragma unroll
      for (int sl = 0; sl < NSL; ++sl) {
        const int col = n0 + sl * SLAB + cl;
        const bool live = col < d.Cout;
        // second residual and bias_n_mod rows: per slab (a second strip spills at BN = 128); issued before the transposition to overlap it
        float4 rb[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (live && (fl[i] & 1)) {
            if (p.res2) rb[i] = *reinterpret_cast<const float4*>(p.res2 + o2[i] + col);
            else if (p.res2_s) rb[i] = load_split4(p.res2_s + o2[i] + col, p.res2_plane);
          }
        }
        __syncwarp();
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {                     // fragment column group j = 2 sl + jj: columns 8 jj + 2 (lane % 4) + {0, 1}
          const int j = 2 * sl + jj, cc = 8 * jj + 2 * (lane & 3);
          *reinterpret_cast<float2*>(&tile[sub * PITCH + cc]) = make_float2(sum[4 * j], sum[4 * j + 1]);
          *reinterpret_cast<float2*>(&tile[(sub + 8) * PITCH + cc]) = make_float2(sum[4 * j + 2], sum[4 * j + 3]);
        }
        __syncwarp();
        if (live) {
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            if (!(fl[i] & 1)) continue;
            const float4 acc4 = *reinterpret_cast<const float4*>(&tile[(i * 8 + sub) * PITCH + cl]);
            float4 b = bv[sl];
            if (p.bias && d.bias_n_mod) b = __ldg(reinterpret_cast<const float4*>(p.bias + (long long)((fl[i] >> 1) % d.bias_n_mod) * d.Cout + col));
            const uint4 r = rv[sl][i];
            const float4 ra = res_split ? merge_split4(make_uint2(r.x, r.y), make_uint2(r.z, r.w))
                                        : make_float4(__uint_as_float(r.x), __uint_as_float(r.y), __uint_as_float(r.z), __uint_as_float(r.w));
            float4 o = make_float4(acc4.x + b.x + ra.x + rb[i].x, acc4.y + b.y + ra.y + rb[i].y,
                                   acc4.z + b.z + ra.z + rb[i].z, acc4.w + b.w + ra.w + rb[i].w);
            const long long eo = yo[i] + col;
            if (GM == 1 || p.splits > 1) {                     // taps / K splits race on an output row: red.add (fp32 only)
              tt_red_add_v4(p.y + eo, o.x, o.y, o.z, o.w);
            } else {
              o = act4(o, d.act);
              if (p.y) *reinterpret_cast<float4*>(p.y + eo) = o;
              if (p.ys) {
                uint2 hi, lo;
                split4(o, hi, lo, sat);
                *reinterpret_cast<uint2*>(p.ys + eo) = hi;
                *reinterpret_cast<uint2*>(p.ys + p.ys_plane + eo) = lo;
              }
            }
          }
        }
      }
    }
    if (sat) atomicAdd(&g_f16s_saturated, 1u);
  }
}

// split-K / sparse companions.  init: y = bias + res + res2 before the tensor-core kernel red.adds its partial sums;
// finish: y = act(y) and, when asked, the split planes of the finished rows.
__global__ void f16s_splitk_init_kernel(const tt_conv_desc d, const float* __restrict__ bias, const float* __restrict__ res,
                                        const float* __restrict__ res2, const __half* __restrict__ res_s, long long res_plane,
                                        const __half* __restrict__ res2_s, long long res2_plane, float* __restrict__ y) {
  const int HWo = d.OH * d.OW, C4 = d.Cout / 4;
  const long long total = (long long)d.N * HWo * C4;
  const long long yns = d.y_nstride ? d.y_nstride : (long long)d.yH * d.yW * d.y_ld;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const long long pix = i / C4;
    const int n = (int)(pix / HWo);
    float4 v = bias ? __ldg(reinterpret_cast<const float4*>(bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (res) { const float4 t = *reinterpret_cast<const float4*>(res + pix * d.res_ld + d.res_coff + c); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
    if (res2) { const float4 t = *reinterpret_cast<const float4*>(res2 + pix * d.res2_ld + d.res2_coff + c); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
    if (res_s) { const float4 t = load_split4(res_s + pix * d.res_ld + d.res_coff + c, res_plane); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
    if (res2_s) { const float4 t = load_split4(res2_s + pix * d.res2_ld + d.res2_coff + c, res2_plane); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
    *reinterpret_cast<float4*>(y + n * yns + (pix - (long long)n * HWo) * d.y_ld + d.y_coff + c) = v;
  }
}
__global__ void f16s_splitk_finish_kernel(const tt_conv_desc d, float* __restrict__ y, __half* __restrict__ ys, long long ys_plane) {
  const int HWo = d.OH * d.OW, C4 = d.Cout / 4;
  const long long total = (long long)d.N * HWo * C4;
  const long long yns = d.y_nstride ? d.y_nstride : (long long)d.yH * d.yW * d.y_ld;
  bool sat = false;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const long long pix = i / C4;
    const int n = (int)(pix / HWo);
    const long long eo = n * yns + (pix - (long long)n * HWo) * d.y_ld + d.y_coff + c;
    float4 v = *reinterpret_cast<const float4*>(y + eo);
    v = make_float4(tt_act(v.x, d.act), tt_act(v.y, d.act), tt_act(v.z, d.act), tt_act(v.w, d.act));
    if (d.act != TT_ACT_NONE) *reinterpret_cast<float4*>(y + eo) = v;
    if (ys) {
      uint2 hi, lo;
      split4(v, hi, lo, sat);
      *reinterpret_cast<uint2*>(ys + eo) = hi;
      *reinterpret_cast<uint2*>(ys + ys_plane + eo) = lo;
    }
  }
  if (sat) atomicAdd(&g_f16s_saturated, 1u);
}

// generic fp32 rows -> split planes (producers that are not convolutions: pooling, resampling, gating, staging of inputs)
__global__ void split_rows_kernel(const float* __restrict__ x, long long x_ld, __half* __restrict__ ys, long long ys_plane,
                                  long long ys_ld, long long rows, int cols4, const int* __restrict__ row_count) {
  const long long total = (row_count ? min((long long)*row_count, rows) : rows) * cols4;
  bool sat = false;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols4;
    const int c = (int)(i - r * cols4) * 4;
    const float4 v = *reinterpret_cast<const float4*>(x + r * x_ld + c);
    uint2 hi, lo;
    split4(v, hi, lo, sat);
    *reinterpret_cast<uint2*>(ys + r * ys_ld + c) = hi;
    *reinterpret_cast<uint2*>(ys + ys_plane + r * ys_ld + c) = lo;
  }
  // not counted in g_f16s_saturated: this converter also sweeps arena regions no kernel has written yet (whole-buffer refreshes),
  // whose bit patterns are arbitrary; values that matter were produced — and counted — by a convolution epilogue
}

// split planes -> fp32 rows (a non-convolution kernel needs the fp32 value of a tensor that is stored as planes only)
__global__ void merge_rows_kernel(const __half* __restrict__ xs, long long xs_plane, long long xs_ld, float* __restrict__ y, long long y_ld,
                                  long long rows, int cols4) {
  const long long total = rows * cols4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols4;
    const int c = (int)(i - r * cols4) * 4;
    *reinterpret_cast<float4*>(y + r * y_ld + c) = load_split4(xs + r * xs_ld + c, xs_plane);
  }
}

// camera images NCHW fp32 (C <= 8) -> zero-bordered channels-last split planes with 8 halves per pixel: the layout the row-packed
// stem convolution reads (one 7-pixel tap row = 56 halves of a 64-half K slab).  One thread per pixel: coalesced plane reads,
// one 16-byte store per plane.
__global__ void image_to_split8_kernel(const float* __restrict__ x, __half* __restrict__ ys, long long ys_plane, int C, int H, int W,
                                       int out_H, int out_W, int top, int left, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(i % W);
    const long long t = i / W;
    const int h = (int)(t % H), n = (int)(t / H);
    __half hi[8], lo[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float v = c < C ? __ldg(x + (((long long)n * C + c) * H + h) * W + w) : 0.f;
      split_h(v, hi[c], lo[c]);
    }
    const long long o = (((long long)n * out_H + h + top) * out_W + w + left) * 8;
    *reinterpret_cast<uint4*>(ys + o) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(ys + ys_plane + o) = *reinterpret_cast<const uint4*>(lo);
  }
}

// nn.Upsample(scale_factor=2, bilinear, align_corners=True) (lss.py:267) from fp32 straight into split planes: the same arithmetic
// as upsample2x_ac_kernel (elementwise.cu), no fp32 copy of the 4x larger map
__global__ void upsample2x_split_kernel(const float4* __restrict__ x, __half* __restrict__ ys, long long ys_plane, int N, int H, int W, int C4) {
  const int OH = 2 * H, OW = 2 * W;
  const float sh = OH > 1 ? (float)(H - 1) / (float)(OH - 1) : 0.f;
  const float sw = OW > 1 ? (float)(W - 1) / (float)(OW - 1) : 0.f;
  const long long total = (long long)N * OH * OW * C4;
  bool sat = false;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % C4;
    long long t = i / C4;
    const int ow = t % OW; t /= OW;
    const int oh = t % OH;
    const int n = t / OH;
    const float fy = sh * oh, fx = sw * ow;
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
    uint2 hi, lo;
    split4(r, hi, lo, sat);
    *reinterpret_cast<uint2*>(ys + i * 4) = hi;
    *reinterpret_cast<uint2*>(ys + ys_plane + i * 4) = lo;
  }
  if (sat) atomicAdd(&g_f16s_saturated, 1u);
}

// Thin 1x1 convolutions (Cin <= 64, Cout <= 64) over large maps: 128 x 64 tensor-core tiles spend their time in per-tile overheads
// there (one K stage per tile; seg / seg->feature heads at 224 x 448: ~10 % of the HBM roof), while the arithmetic is a per-pixel
// 64 x 64 mat-vec at most.  One thread = one pixel: it streams its channel row from the split planes (full 128-byte lines), keeps
// the COUT accumulators in registers (fp32 FFMA against fp32 weights broadcast from shared memory: exact products, no operand
// split needed) and stores its output row (fp32 and / or planes).
// TAIL: Cin % 8 != 0, so the last 8-channel load also reads channels in [Cin, K8), which are not the tensor's (their weights are zero,
// but the halves there may be NaN: NaN * 0 = NaN) and are zeroed.  YS16: every plane row starts 16-byte aligned (y_ld, y_coff and the
// plane stride % 8), so a lane stores its 8 halves in one 16-byte store, else in two 8-byte ones.  Both are template parameters: as
// runtime tests they cost the common case (Cin % 8 == 0, aligned rows) 17-24 % at Cin 64 over 16 x 224 x 448 pixels (H100, 700 W).
template <int COUT, bool TAIL, bool YS16>
__global__ void __launch_bounds__(256) pointwise_f16s_kernel(const __half* __restrict__ xs, long long xs_plane, int x_ld, int Cin,
                                                              const float* __restrict__ w, const float* __restrict__ bias, int Cout,
                                                              float* __restrict__ y, __half* __restrict__ ys, long long ys_plane, int y_ld,
                                                              int act, long long npix, int co0) {
  constexpr int RP = COUT * 2 + 16;                                  // staging row pitch in bytes (+16: conflict-free 16-byte accesses)
  __shared__ __align__(16) float ws[64 * COUT];                      // [k][co0 + co], rows beyond Cin / columns beyond Cout are zero
  __shared__ float bs[COUT];
  __shared__ __align__(16) uint8_t stage[8][32 * RP];                // per warp: 32 pixels x COUT halves (one plane at a time)
  const int K8 = (Cin + 7) / 8 * 8;
  for (int i = threadIdx.x; i < 64 * COUT; i += blockDim.x) {
    const int k = i / COUT, co = i - k * COUT;
    ws[i] = (k < Cin && co0 + co < Cout) ? w[(long long)k * Cout + co0 + co] : 0.f;
  }
  for (int i = threadIdx.x; i < COUT; i += blockDim.x) bs[i] = (bias && co0 + i < Cout) ? bias[co0 + i] : 0.f;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  bool sat = false;
  // whole warps walk 32 consecutive pixels at a time (the tail warp clamps its loads and predicates its stores)
  for (long long base = (blockIdx.x * (long long)(blockDim.x >> 5) + warp) * 32; base < npix; base += (long long)gridDim.x * blockDim.x) {
    const long long pix = base + lane;
    const bool live = pix < npix;
    float acc[COUT];
#pragma unroll
    for (int co = 0; co < COUT; ++co) acc[co] = bs[co];
    const __half* xr = xs + (live ? pix : npix - 1) * x_ld;
    for (int k0 = 0; k0 < K8; k0 += 8) {
      const uint4 h = *reinterpret_cast<const uint4*>(xr + k0);
      const uint4 l = *reinterpret_cast<const uint4*>(xr + xs_plane + k0);
      const __half2* hp = reinterpret_cast<const __half2*>(&h);
      const __half2* lp = reinterpret_cast<const __half2*>(&l);
      float xv[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a = __half22float2(hp[j]), b = __half22float2(lp[j]);
        xv[2 * j] = fmaf(b.x, LO_INV, a.x);
        xv[2 * j + 1] = fmaf(b.y, LO_INV, a.y);
      }
      if (TAIL && k0 + 8 > Cin) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (k0 + j >= Cin) xv[j] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4* wr = reinterpret_cast<const float4*>(&ws[(k0 + j) * COUT]);
#pragma unroll
        for (int c4 = 0; c4 < COUT / 4; ++c4) {
          const float4 wv = wr[c4];                                    // same address in every lane: shared-memory broadcast
          acc[4 * c4] = fmaf(xv[j], wv.x, acc[4 * c4]);
          acc[4 * c4 + 1] = fmaf(xv[j], wv.y, acc[4 * c4 + 1]);
          acc[4 * c4 + 2] = fmaf(xv[j], wv.z, acc[4 * c4 + 2]);
          acc[4 * c4 + 3] = fmaf(xv[j], wv.w, acc[4 * c4 + 3]);
        }
      }
    }
    // ---- outputs.  fp32 rows: direct 16-byte stores.  Planes: this lane's COUT halves go through a per-warp staging buffer so that the
    // global stores are 16 bytes per lane with 4 (COUT 32) / 2 (COUT 16) lanes on one pixel row: full 32-byte sectors instead of 8-byte shards
    uint2 hv[COUT / 4], lv[COUT / 4];
#pragma unroll
    for (int c4 = 0; c4 < COUT / 4; ++c4) {
      const float4 o = make_float4(tt_act(acc[4 * c4], act), tt_act(acc[4 * c4 + 1], act), tt_act(acc[4 * c4 + 2], act), tt_act(acc[4 * c4 + 3], act));
      if (y && live && co0 + 4 * c4 < Cout) *reinterpret_cast<float4*>(y + pix * y_ld + co0 + 4 * c4) = o;
      split4(o, hv[c4], lv[c4], sat);
    }
    if (ys) {
      constexpr int LPR = COUT / 8;                                    // lanes per pixel row (16-byte chunks of COUT halves)
      constexpr int RPI = 32 / LPR;                                    // pixel rows per store instruction
      const int chunk = lane % LPR, rsub = lane / LPR;
#pragma unroll
      for (int pl = 0; pl < 2; ++pl) {
        __syncwarp();
#pragma unroll
        for (int c4 = 0; c4 < COUT / 4; ++c4) *reinterpret_cast<uint2*>(&stage[warp][lane * RP + c4 * 8]) = pl ? lv[c4] : hv[c4];
        __syncwarp();
#pragma unroll
        for (int it = 0; it < 32 / RPI; ++it) {
          const int prow = it * RPI + rsub;
          const long long gp = base + prow;
          if (gp < npix && co0 + chunk * 8 < Cout) {
            __half* dst = ys + (pl ? ys_plane : 0) + gp * y_ld + co0 + chunk * 8;
            const uint4 v = *reinterpret_cast<const uint4*>(&stage[warp][prow * RP + chunk * 16]);
            if (YS16) {
              *reinterpret_cast<uint4*>(dst) = v;
            } else {
              reinterpret_cast<uint2*>(dst)[0] = make_uint2(v.x, v.y);
              reinterpret_cast<uint2*>(dst)[1] = make_uint2(v.z, v.w);
            }
          }
        }
      }
    }
  }
  if (sat) atomicAdd(&g_f16s_saturated, 1u);
}

// sparse rows: y = act(y + res) for the first *count rows, plus their split planes
__global__ void f16s_sparse_finish_kernel(float* __restrict__ y, int y_ld, const float* __restrict__ res, int res_ld, int C,
                                          const int* __restrict__ count, int cap, int act, __half* __restrict__ ys, long long ys_plane) {
  const int C4 = C / 4;
  const long long total = (long long)min(*count, cap) * C4;
  bool sat = false;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C4;
    const int c = (int)(i - r * C4) * 4;
    float4 v = *reinterpret_cast<const float4*>(y + r * y_ld + c);
    if (res) { const float4 t = *reinterpret_cast<const float4*>(res + r * res_ld + c); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
    v = make_float4(tt_act(v.x, act), tt_act(v.y, act), tt_act(v.z, act), tt_act(v.w, act));
    *reinterpret_cast<float4*>(y + r * y_ld + c) = v;
    if (ys) {
      uint2 hi, lo;
      split4(v, hi, lo, sat);
      *reinterpret_cast<uint2*>(ys + r * y_ld + c) = hi;
      *reinterpret_cast<uint2*>(ys + ys_plane + r * y_ld + c) = lo;
    }
  }
  if (sat) atomicAdd(&g_f16s_saturated, 1u);
}
__global__ void f16s_sparse_init_kernel(float* __restrict__ y, int y_ld, const float* __restrict__ bias, int C,
                                        const int* __restrict__ count, int cap) {
  const int C4 = C / 4;
  const long long total = (long long)min(*count, cap) * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C4;
    const int c = (int)(i - r * C4) * 4;
    *reinterpret_cast<float4*>(y + r * y_ld + c) = bias ? __ldg(reinterpret_cast<const float4*>(bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// N tiles: each MMA thread holds BN / 2 main + BN / 2 correction accumulators plus BN / 2 fp32 sums, 96 registers at BN = 64 and
// 192 at BN = 128 (within the 232 setmaxnreg gives the MMA warpgroups).  A BN = 128 stage is 64 KB, so its ring is 3 stages deep;
// BN = 64 keeps 4 stages of 48 KB.  The tap-major sparse mode (GM 1) always uses BN = 64.
constexpr int BN_NARROW = 64, BN_WIDE = 128;

// persistent grid: one CTA per SM walks the (M unit, N tile, K split) work items; debug bits 8..15: SMs left to a concurrent branch
template <int BN, int GM>
cudaError_t launch_f16s(const CUtensorMap& ma, const CUtensorMap& mb, const HArgs& a, long long m_units, cudaStream_t st) {
  constexpr int STAGES = BN == BN_WIDE ? 3 : 4;
  constexpr int smem = STAGES * (2 * BM * KE * 2 + 2 * BN * KE * 2) + 1024 + EPI_BYTES + (GM == 2 ? NB_BYTES : 0);
  static_assert(smem <= 227 * 1024, "shared memory per block");
  static bool set = false;
  if (!set) { cudaFuncSetAttribute(conv_f16s_kernel<BN, STAGES, GM>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); set = true; }
  const long long num_sms = tt_num_sms() - ((g_tt_debug >> 8) & 0xFF);
  const long long items = m_units * a.n_tiles * a.splits;
  const long long grid = items < num_sms ? items : num_sms;
  conv_f16s_kernel<BN, STAGES, GM><<<(unsigned)(grid > 1 ? grid : 1), NTHREADS, smem, st>>>(ma, mb, a);
  return cudaGetLastError();
}

bool encode_weights(CUtensorMap* mb, const void* w_split, int Cin, int taps, int Cout, int BN, bool flat_k = false) {
  int cin_pad = (Cin + 7) & ~7;
  if (flat_k) { cin_pad *= taps; taps = 1; }                     // K = tap * Cin + c as ONE dimension (taps are contiguous per Cout row)
  cuuint64_t dims[4] = {(cuuint64_t)cin_pad, (cuuint64_t)taps, (cuuint64_t)Cout, 2};
  cuuint64_t str[3] = {(cuuint64_t)cin_pad * 2, (cuuint64_t)taps * cin_pad * 2, (cuuint64_t)Cout * taps * cin_pad * 2};
  cuuint32_t box[4] = {KE, 1, (cuuint32_t)(BN / 2), 1};          // a plane's BN-row slab is loaded as two half boxes
  return encode_map(mb, w_split, 4, dims, str, box, 1, CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
}

}  // namespace

extern "C" {

/* number of epilogue threads that clamped a value to +-65504 since the last call (synchronises `stream`) */
int tt_f16s_saturation_count(unsigned int* out_host, int reset, tt_stream_t stream) {
  TT_REQUIRE(out_host, "tt_f16s_saturation_count", "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemcpyFromSymbolAsync(out_host, g_f16s_saturated, sizeof(unsigned int), 0, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess) {
    tt_set_error("tt_f16s_saturation_count: %s", cudaGetErrorString(cudaGetLastError()));
    return TT_ERR_CUDA;
  }
  if (reset) {
    const unsigned int z = 0;
    if (cudaMemcpyToSymbolAsync(g_f16s_saturated, &z, sizeof(z), 0, cudaMemcpyHostToDevice, st) != cudaSuccess) return TT_ERR_CUDA;
    cudaStreamSynchronize(st);
  }
  return TT_OK;
}

int tt_split_f16(const float* x, long long x_ld, void* y_split, long long y_plane, long long y_ld, long long rows, int cols,
                 const int* row_count, tt_stream_t stream) {
  TT_REQUIRE(x && y_split && rows >= 0 && cols > 0, "tt_split_f16", "bad argument");
  TT_REQUIRE(cols % 4 == 0 && x_ld % 4 == 0 && y_ld % 4 == 0 && y_plane % 4 == 0 &&
                 ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && ((reinterpret_cast<uintptr_t>(y_split) & 7) == 0),
             "tt_split_f16", "needs 4-element alignment");
  if (rows == 0) return TT_OK;
  const long long total = rows * (cols / 4);
  const int nb = (int)((total + 255) / 256 > tt_num_sms() * 16 ? tt_num_sms() * 16 : (total + 255) / 256);
  split_rows_kernel<<<nb, 256, 0, (cudaStream_t)stream>>>(x, x_ld, static_cast<__half*>(y_split), y_plane, y_ld, rows, cols / 4, row_count);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_split_f16");
  return TT_OK;
}

int tt_image_to_split8(const float* x, void* y_split, long long y_plane, int N, int C, int H, int W, int out_H, int out_W, int top,
                       int left, tt_stream_t stream) {
  TT_REQUIRE(x && y_split && C >= 1 && C <= 8 && top >= 0 && left >= 0 && top + H <= out_H && left + W <= out_W && y_plane % 8 == 0 &&
                 (reinterpret_cast<uintptr_t>(y_split) & 15) == 0,
             "tt_image_to_split8", "bad arguments");
  const long long total = (long long)N * H * W;
  if (total == 0) return TT_OK;
  const int nb = (int)((total + 255) / 256 > tt_num_sms() * 32 ? tt_num_sms() * 32 : (total + 255) / 256);
  image_to_split8_kernel<<<nb, 256, 0, (cudaStream_t)stream>>>(x, static_cast<__half*>(y_split), y_plane, C, H, W, out_H, out_W, top, left, total);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_image_to_split8");
  return TT_OK;
}

int tt_upsample2x_bilinear_ac_split(const float* x, void* y_split, long long y_plane, int N, int H, int W, int C, tt_stream_t stream) {
  TT_REQUIRE(x && y_split && C % 4 == 0 && y_plane % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y_split) & 7) == 0,
             "tt_upsample2x_bilinear_ac_split", "C must be a multiple of 4, aligned pointers");
  const long long total = (long long)N * 4 * H * W * (C / 4);
  if (total == 0) return TT_OK;
  const int nb = (int)((total + 255) / 256 > tt_num_sms() * 32 ? tt_num_sms() * 32 : (total + 255) / 256);
  upsample2x_split_kernel<<<nb, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(x), static_cast<__half*>(y_split), y_plane, N, H, W, C / 4);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_upsample2x_bilinear_ac_split");
  return TT_OK;
}

int tt_pointwise_f16s(const tt_conv_desc* d, const tt_f16s_io* io, const float* w_kmajor, tt_stream_t stream) {
  TT_REQUIRE(d && io && io->x_split && w_kmajor && (io->y || io->y_split), "tt_pointwise_f16s", "null argument");
  const long long xhs = d->x_hstride ? d->x_hstride : (long long)d->W * d->x_ld;
  const long long xns = d->x_nstride ? d->x_nstride : (long long)d->H * xhs;
  const bool ok = d->KH == 1 && d->KW == 1 && d->stride == 1 && d->pad == 0 && d->groups == 1 && d->Cin <= 64 && d->Cout <= 64 && d->Cout % 4 == 0 &&
                  d->x_ld % 8 == 0 && (d->Cin + 7) / 8 * 8 <= d->x_ld && d->y_ld % 4 == 0 && d->y_coff % 4 == 0 && io->x_plane % 8 == 0 && io->y_plane % 4 == 0 &&
                  xhs == (long long)d->W * d->x_ld && xns == (long long)d->H * xhs && d->y_nstride == 0 && d->oy_mul == 1 && d->ox_mul == 1 &&
                  d->oy_add == 0 && d->ox_add == 0 && d->yH == d->OH && d->yW == d->OW && d->OH == d->H && d->OW == d->W &&
                  d->res_mode == TT_RES_NONE && !io->res && !io->res_split && !io->res2 && !io->res2_split && d->bias_n_mod == 0 &&
                  ((reinterpret_cast<uintptr_t>(io->x_split) | reinterpret_cast<uintptr_t>(io->y)) & 15) == 0 && (reinterpret_cast<uintptr_t>(io->y_split) & 7) == 0;
  if (!ok) {
    tt_set_error("tt_pointwise_f16s: needs a dense 1x1 stride-1 conv with Cin, Cout <= 64 (Cout %% 4), no residual, contiguous pixels");
    return TT_ERR_UNSUPPORTED;
  }
  const long long npix = (long long)d->N * d->H * d->W;
  if (npix == 0) return TT_OK;
  const int nb = (int)((npix + 255) / 256 > tt_num_sms() * 8 ? tt_num_sms() * 8 : (npix + 255) / 256);
  TT_REQUIRE(d->Cout % 8 == 0 || !io->y_split, "tt_pointwise_f16s", "plane output needs Cout % 8 == 0");
  const __half* xs = static_cast<const __half*>(io->x_split);
  __half* ys = static_cast<__half*>(io->y_split);
  float* y = io->y ? io->y + d->y_coff : nullptr;
  if (ys) ys += d->y_coff;
  cudaStream_t st = (cudaStream_t)stream;
  const bool tail = d->Cin % 8 != 0;
  const bool ys16 = !ys || (((reinterpret_cast<uintptr_t>(ys) & 15) == 0) && d->y_ld % 8 == 0 && io->y_plane % 8 == 0);
  auto launch = [&](auto kern, int co0) {
    kern<<<nb, 256, 0, st>>>(xs, io->x_plane, d->x_ld, d->Cin, w_kmajor, io->bias, d->Cout, y, ys, io->y_plane, d->y_ld, d->act, npix, co0);
  };
  // 32 output channels per pass (register budget: 2 CTAs per SM); wider layers take two passes over the (small) input rows
  for (int co0 = 0; co0 < d->Cout; co0 += 32) {
    if (d->Cout <= 16) {
      if (tail) ys16 ? launch(pointwise_f16s_kernel<16, true, true>, co0) : launch(pointwise_f16s_kernel<16, true, false>, co0);
      else ys16 ? launch(pointwise_f16s_kernel<16, false, true>, co0) : launch(pointwise_f16s_kernel<16, false, false>, co0);
    } else {
      if (tail) ys16 ? launch(pointwise_f16s_kernel<32, true, true>, co0) : launch(pointwise_f16s_kernel<32, true, false>, co0);
      else ys16 ? launch(pointwise_f16s_kernel<32, false, true>, co0) : launch(pointwise_f16s_kernel<32, false, false>, co0);
    }
    if (co0) ++g_tt_launches;
  }
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_pointwise_f16s");
  return TT_OK;
}

int tt_merge_f16(const void* x_split, long long x_plane, long long x_ld, float* y, long long y_ld, long long rows, int cols,
                 tt_stream_t stream) {
  TT_REQUIRE(x_split && y && rows >= 0 && cols > 0, "tt_merge_f16", "bad argument");
  TT_REQUIRE(cols % 4 == 0 && x_ld % 4 == 0 && y_ld % 4 == 0 && x_plane % 4 == 0 && ((reinterpret_cast<uintptr_t>(y) & 15) == 0) &&
                 ((reinterpret_cast<uintptr_t>(x_split) & 7) == 0),
             "tt_merge_f16", "needs 4-element alignment");
  if (rows == 0) return TT_OK;
  const long long total = rows * (cols / 4);
  const int nb = (int)((total + 255) / 256 > tt_num_sms() * 16 ? tt_num_sms() * 16 : (total + 255) / 256);
  merge_rows_kernel<<<nb, 256, 0, (cudaStream_t)stream>>>(static_cast<const __half*>(x_split), x_plane, x_ld, y, y_ld, rows, cols / 4);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_merge_f16");
  return TT_OK;
}

int tt_conv2d_f16s(const tt_conv_desc* d, const tt_f16s_io* io, tt_stream_t stream) {
  TT_REQUIRE(d && io && io->x_split && io->w_split && (io->y || io->y_split), "tt_conv2d_f16s", "null argument");
  const void* x_split = io->x_split; const long long x_plane = io->x_plane;
  const void* w_split = io->w_split; const float* bias = io->bias;
  const float* res = io->res; const float* res2 = io->res2;
  float* y = io->y; void* y_split = io->y_split; const long long y_plane = io->y_plane;
  TT_REQUIRE(d->res_mode == TT_RES_NONE || res != nullptr || io->res_split != nullptr, "tt_conv2d_f16s", "res_mode set without a residual");
  TT_REQUIRE(!(res && io->res_split) && !(res2 && io->res2_split), "tt_conv2d_f16s", "a residual is given either as fp32 or as split planes");
  const long long xhs = d->x_hstride ? d->x_hstride : (long long)d->W * d->x_ld;
  const long long xns = d->x_nstride ? d->x_nstride : (long long)d->H * xhs;
  const bool ok = d->groups == 1 && (d->stride == 1 || d->stride == 2) && d->Cout % 4 == 0 && d->x_ld % 8 == 0 && xhs % 8 == 0 &&
                  xns % 8 == 0 && x_plane % 8 == 0 && d->y_ld % 4 == 0 && d->y_coff % 4 == 0 && d->y_nstride % 4 == 0 && y_plane % 4 == 0 &&
                  (d->res_mode == TT_RES_NONE || (d->res_ld % 4 == 0 && d->res_coff % 4 == 0)) && d->res2_ld % 4 == 0 && d->res2_coff % 4 == 0 &&
                  io->res_plane % 4 == 0 && io->res2_plane % 4 == 0 &&
                  ((reinterpret_cast<uintptr_t>(x_split) | reinterpret_cast<uintptr_t>(w_split) | reinterpret_cast<uintptr_t>(y) |
                    reinterpret_cast<uintptr_t>(res) | reinterpret_cast<uintptr_t>(res2) | reinterpret_cast<uintptr_t>(bias)) & 15) == 0 &&
                  ((reinterpret_cast<uintptr_t>(y_split) | reinterpret_cast<uintptr_t>(io->res_split) | reinterpret_cast<uintptr_t>(io->res2_split)) & 7) == 0 &&
                  d->OH == (d->H + 2 * d->pad - d->dil * (d->KH - 1) - 1) / d->stride + 1 &&
                  d->OW == (d->W + 2 * d->pad - d->dil * (d->KW - 1) - 1) / d->stride + 1;
  if (!ok) {
    tt_set_error("tt_conv2d_f16s: unsupported shape / alignment (groups 1, stride 1|2, x_ld %% 8, y_ld %% 4, 16-byte aligned pointers)");
    return TT_ERR_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int taps = d->KH * d->KW;
  const long long npix_in = (long long)d->N * d->H * d->W;
  HArgs a;
  memset(&a, 0, sizeof(a));
  a.d = *d;
  a.bias = bias; a.res = res; a.res2 = res2; a.y = y;
  a.res_s = static_cast<const __half*>(io->res_split); a.res_plane = io->res_plane;
  a.res2_s = static_cast<const __half*>(io->res2_split); a.res2_plane = io->res2_plane;
  a.ys = static_cast<__half*>(y_split); a.ys_plane = y_plane;
  a.chunk = (g_tt_debug & 0x40000) ? 1 : (g_tt_debug & 0x20000) ? 4 : 2;
  a.n_slabs = (d->Cin + KE - 1) / KE;
  if ((long long)d->N * d->OH * d->OW >= (1ll << 31) - BM || npix_in >= (1ll << 31) - BM) {
    tt_set_error("tt_conv2d_f16s: more than 2^31 pixels");
    return TT_ERR_UNSUPPORTED;
  }
  a.total_pix = d->N * d->OH * d->OW;
  a.flat = (taps == 1 && d->pad == 0 && d->stride == 1 && xhs == (long long)d->W * d->x_ld && xns == (long long)d->H * xhs) ? 1 : 0;
  CUtensorMap ma, mb;
  int grid_x;
  if (a.flat) {
    a.TH = 1; a.TW = BM; a.tiles_w = a.tiles_h = 1;
    cuuint64_t dims[3] = {(cuuint64_t)d->Cin, (cuuint64_t)npix_in, 2};
    cuuint64_t str[2] = {(cuuint64_t)d->x_ld * 2, (cuuint64_t)x_plane * 2};
    cuuint32_t box[3] = {KE, BM, 1};
    if (!encode_map(&ma, x_split, 3, dims, str, box, 1, CU_TENSOR_MAP_DATA_TYPE_FLOAT16)) return TT_ERR_CUDA;
    grid_x = tt_cdiv(npix_in, BM);
  } else {
    int best_th = 1, best_tw = 1;
    double best = -1;
    for (int tw = 1; tw <= 128 && tw * d->stride <= 256; ++tw) {
      const int th = 128 / tw;
      if (th < 1) break;
      const double cover = (double)d->OW * d->OH / ((double)tt_cdiv(d->OW, tw) * tw * tt_cdiv(d->OH, th) * th);
      const double eff = cover * (tw * th) / 128.0;
      if (eff > best + 1e-9) { best = eff; best_th = th; best_tw = tw; }
    }
    a.TH = best_th; a.TW = best_tw;
    a.tiles_w = tt_cdiv(d->OW, a.TW); a.tiles_h = tt_cdiv(d->OH, a.TH);
    cuuint64_t dims[5] = {(cuuint64_t)d->Cin, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->N, 2};
    cuuint64_t str[4] = {(cuuint64_t)d->x_ld * 2, (cuuint64_t)xhs * 2, (cuuint64_t)xns * 2, (cuuint64_t)x_plane * 2};
    cuuint32_t box[5] = {KE, (cuuint32_t)(a.TW * d->stride), (cuuint32_t)(a.TH * d->stride), 1, 1};
    if (!encode_map(&ma, x_split, 5, dims, str, box, d->stride, CU_TENSOR_MAP_DATA_TYPE_FLOAT16)) return TT_ERR_CUDA;
    grid_x = a.tiles_w * a.tiles_h * d->N;
  }
  a.m_tiles = grid_x;
  const int num_sms = tt_num_sms();
  // 128-column tiles read each A slab once per 128 output channels instead of 64 and need less shared-memory bandwidth per MMA.
  // They are used when Cout > 64 and the 128-column tiles alone give every SM one, so they never run split-K.  tools/conv_bench.py
  // on an H100 SXM: with N = 64 every shape with Cout >= 128 was 3-17 % faster on 128-column tiles (400 W card), while N = 4 layer4
  // convs that needed split-K to fill the SMs with 128-column tiles were 1.5-1.6x slower (700 W card: 77 vs 51 us for 3x3
  // 512 -> 512 at 14 x 28, 49 vs 31 us for 1x1 2048 -> 512).
  // Debug bit 0x400000 forces BN = 64 (A/B of the two tiles in one build).
  const bool wide = d->Cout > BN_NARROW && !(g_tt_debug & 0x400000) && (long long)a.m_tiles * tt_cdiv(d->Cout, BN_WIDE) >= num_sms;
  const int bn = wide ? BN_WIDE : BN_NARROW;
  if (!encode_weights(&mb, w_split, d->Cin, taps, d->Cout, bn)) return TT_ERR_CUDA;
  a.n_tiles = tt_cdiv(d->Cout, bn);
  const int k_iters = taps * a.n_slabs;
  a.splits = 1;
  a.k_per = k_iters;
  {
    const long long tiles = (long long)a.m_tiles * a.n_tiles;
    const bool plain = y != nullptr && d->oy_mul == 1 && d->ox_mul == 1 && d->oy_add == 0 && d->ox_add == 0 && d->yH == d->OH && d->yW == d->OW &&
                       d->res_mode != TT_RES_UP2_NEAREST && d->bias_n_mod == 0 && !(g_tt_debug & 128);
    if (plain && tiles <= num_sms / 2 && k_iters >= 8) {
      int sp = (int)((num_sms + tiles - 1) / tiles);
      if (sp > k_iters / 4) sp = k_iters / 4;
      if (sp > 32) sp = 32;
      if (sp >= 2) {
        a.k_per = tt_cdiv(k_iters, sp);
        a.splits = tt_cdiv(k_iters, a.k_per);
      }
    }
  }
  const long long total4 = (long long)d->N * d->OH * d->OW * (d->Cout / 4);
  const int nb_ew = (int)((total4 + 255) / 256 > tt_num_sms() * 8 ? tt_num_sms() * 8 : (total4 + 255) / 256);
  if (a.splits > 1) {
    f16s_splitk_init_kernel<<<nb_ew, 256, 0, st>>>(*d, bias, d->res_mode != TT_RES_NONE ? res : nullptr, res2,
                                                   d->res_mode != TT_RES_NONE ? a.res_s : nullptr, a.res_plane, a.res2_s, a.res2_plane, y);
    ++g_tt_launches;
    TT_CHECK_LAUNCH("tt_conv2d_f16s(split-k init)");
    a.bias = nullptr; a.res = nullptr; a.res2 = nullptr; a.res_s = nullptr; a.res2_s = nullptr;
    a.d.act = TT_ACT_NONE;
    a.d.res_mode = TT_RES_NONE;
  }
  const cudaError_t lerr = bn == BN_WIDE ? launch_f16s<BN_WIDE, 0>(ma, mb, a, a.m_tiles, st) : launch_f16s<BN_NARROW, 0>(ma, mb, a, a.m_tiles, st);
  if (lerr != cudaSuccess) { tt_set_error("tt_conv2d_f16s: launch failed: %s", cudaGetErrorString(lerr)); return TT_ERR_CUDA; }
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_conv2d_f16s");
  if (a.splits > 1 && (d->act != TT_ACT_NONE || y_split)) {
    f16s_splitk_finish_kernel<<<nb_ew, 256, 0, st>>>(*d, y, static_cast<__half*>(y_split), y_plane);
    ++g_tt_launches;
    TT_CHECK_LAUNCH("tt_conv2d_f16s(split-k finish)");
  }
  return TT_OK;
}

int tt_sparse_conv_f16s(const tt_sparse_conv_desc* d, const void* feats_in_split, long long in_plane, const void* w_split,
                        const float* bias, const float* res, const int* pairs_in, const int* pairs_out, const int* pair_count,
                        const int* out_count, float* feats_out, void* out_split, long long out_plane, tt_stream_t stream) {
  TT_REQUIRE(d && feats_in_split && w_split && pairs_in && pairs_out && pair_count && out_count && feats_out, "tt_sparse_conv_f16s", "null argument");
  if (d->Cin % 8 || d->Cout % 4 || d->in_ld % 8 || d->out_ld % 4 || d->Cin < 32 || d->Cout < 32 || d->kvol > MAX_KVOL || in_plane % 8 || out_plane % 4 ||
      (d->res_ld % 4) ||
      ((reinterpret_cast<uintptr_t>(feats_in_split) | reinterpret_cast<uintptr_t>(w_split) | reinterpret_cast<uintptr_t>(feats_out) |
        reinterpret_cast<uintptr_t>(res) | reinterpret_cast<uintptr_t>(bias)) & 15) || (reinterpret_cast<uintptr_t>(out_split) & 7)) {
    tt_set_error("tt_sparse_conv_f16s: needs Cin %% 8, Cout %% 4, Cin / Cout >= 32, in_ld %% 8, out_ld %% 4, 16-byte aligned pointers");
    return TT_ERR_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (d->cap_out <= 0) return TT_OK;
  const long long tot4 = (long long)d->cap_out * (d->Cout / 4);
  const int nb = (int)((tot4 + 255) / 256 > tt_num_sms() * 8 ? tt_num_sms() * 8 : (tot4 + 255) / 256);
  f16s_sparse_init_kernel<<<nb, 256, 0, st>>>(feats_out, d->out_ld, bias, d->Cout, out_count, d->cap_out);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_sparse_conv_f16s(init)");
  HArgs a;
  memset(&a, 0, sizeof(a));
  a.d.N = a.d.H = a.d.W = a.d.OH = a.d.OW = a.d.yH = a.d.yW = 1;
  a.d.KH = a.d.KW = a.d.stride = a.d.dil = a.d.groups = 1;
  a.d.oy_mul = a.d.ox_mul = 1;
  a.d.Cin = d->Cin; a.d.x_ld = d->in_ld; a.d.Cout = d->Cout; a.d.y_ld = d->out_ld;
  a.d.act = TT_ACT_NONE;
  a.y = feats_out;
  a.chunk = (g_tt_debug & 0x40000) ? 1 : (g_tt_debug & 0x20000) ? 4 : 2;
  a.n_slabs = (d->Cin + KE - 1) / KE;
  a.gx = static_cast<const __half*>(feats_in_split); a.gx_plane = in_plane; a.gx_ld = d->in_ld;
  a.pairs_in = pairs_in; a.pairs_out = pairs_out; a.pair_count = pair_count;
  a.kvol = d->kvol; a.pair_cap = d->pair_cap;
  a.splits = 1; a.k_per = a.n_slabs;
  a.n_tiles = tt_cdiv(d->Cout, BN_NARROW);
  CUtensorMap mb;
  if (!encode_weights(&mb, w_split, d->Cin, d->kvol, d->Cout, BN_NARROW)) return TT_ERR_CUDA;
  const long long cap_units = (long long)d->kvol * tt_cdiv(d->pair_cap, BM);      // upper bound of gathered M tiles over all taps
  const cudaError_t lerr = launch_f16s<BN_NARROW, 1>(mb, mb, a, cap_units, st);
  if (lerr != cudaSuccess) { tt_set_error("tt_sparse_conv_f16s: launch failed: %s", cudaGetErrorString(lerr)); return TT_ERR_CUDA; }
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_sparse_conv_f16s");
  f16s_sparse_finish_kernel<<<nb, 256, 0, st>>>(feats_out, d->out_ld, res, d->res_ld, d->Cout, out_count, d->cap_out, d->act,
                                                 static_cast<__half*>(out_split), out_plane);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_sparse_conv_f16s(finish)");
  return TT_OK;
}

int tt_sparse_conv_os_f16s(const tt_sparse_conv_desc* d, const tt_f16s_io* io, const int* nbr, const int* out_count, tt_stream_t stream) {
  TT_REQUIRE(d && io && io->x_split && io->w_split && (io->y || io->y_split) && nbr && out_count, "tt_sparse_conv_os_f16s", "null argument");
  TT_REQUIRE(!(io->res && io->res_split) && !io->res2 && !io->res2_split, "tt_sparse_conv_os_f16s", "one residual, fp32 or split planes");
  if (d->Cin % 8 || d->Cout % 4 || d->in_ld % 8 || d->out_ld % 4 || d->Cin < 32 || d->Cout < 32 || d->kvol < 1 || d->kvol > MAX_KVOL || io->x_plane % 8 || io->y_plane % 4 ||
      (d->res_ld % 4) || io->res_plane % 4 ||
      ((reinterpret_cast<uintptr_t>(io->x_split) | reinterpret_cast<uintptr_t>(io->w_split) | reinterpret_cast<uintptr_t>(io->y) |
        reinterpret_cast<uintptr_t>(io->res) | reinterpret_cast<uintptr_t>(io->bias)) & 15) ||
      ((reinterpret_cast<uintptr_t>(io->y_split) | reinterpret_cast<uintptr_t>(io->res_split)) & 7)) {
    tt_set_error("tt_sparse_conv_os_f16s: needs Cin %% 8, Cout %% 4, Cin / Cout >= 32, 1 <= kvol <= 32, in_ld %% 8, out_ld %% 4, 16-byte aligned pointers");
    return TT_ERR_UNSUPPORTED;
  }
  if (d->cap_out <= 0) return TT_OK;
  HArgs a;
  memset(&a, 0, sizeof(a));
  a.d.N = a.d.H = a.d.W = a.d.OH = a.d.OW = a.d.yH = a.d.yW = 1;
  a.d.KH = a.d.KW = a.d.stride = a.d.dil = a.d.groups = 1;
  a.d.oy_mul = a.d.ox_mul = 1;
  a.d.Cin = d->Cin; a.d.x_ld = d->in_ld; a.d.Cout = d->Cout; a.d.y_ld = d->out_ld;
  a.d.act = d->act;
  a.d.res_mode = (io->res || io->res_split) ? TT_RES_SAME : TT_RES_NONE;
  a.d.res_ld = d->res_ld;
  a.bias = io->bias; a.res = io->res;
  a.res_s = static_cast<const __half*>(io->res_split); a.res_plane = io->res_plane;
  a.y = io->y; a.ys = static_cast<__half*>(io->y_split); a.ys_plane = io->y_plane;
  a.chunk = (g_tt_debug & 0x40000) ? 1 : (g_tt_debug & 0x20000) ? 4 : 2;
  a.n_slabs = (d->Cin + KE - 1) / KE;
  a.gx = static_cast<const __half*>(io->x_split); a.gx_plane = io->x_plane; a.gx_ld = d->in_ld;
  a.kvol = d->kvol; a.nbr = nbr; a.out_count = out_count; a.cap_rows = d->cap_out;
  a.tps = (d->Cin == 32 && !(g_tt_debug & 0x200000)) ? 2 : 1;
  a.splits = 1; a.k_per = 1;                                      // (the kernel sizes each tile's K walk from its taps)
  // 128-column tiles for Cout >= 128: one gather of the tile's rows feeds all 128 output columns instead of being repeated by a
  // second 64-column work item.  Debug bit 0x400000 forces BN = 64 here too.
  const bool wide = d->Cout >= BN_WIDE && !(g_tt_debug & 0x400000);
  const int bn = wide ? BN_WIDE : BN_NARROW;
  a.n_tiles = tt_cdiv(d->Cout, bn);
  CUtensorMap mb;
  if (!encode_weights(&mb, io->w_split, d->Cin, d->kvol, d->Cout, bn, a.tps == 2)) return TT_ERR_CUDA;
  const long long cap_units = tt_cdiv(d->cap_out, BM);
  const cudaError_t lerr = wide ? launch_f16s<BN_WIDE, 2>(mb, mb, a, cap_units, (cudaStream_t)stream)
                                : launch_f16s<BN_NARROW, 2>(mb, mb, a, cap_units, (cudaStream_t)stream);
  if (lerr != cudaSuccess) { tt_set_error("tt_sparse_conv_os_f16s: launch failed: %s", cudaGetErrorString(lerr)); return TT_ERR_CUDA; }
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_sparse_conv_os_f16s");
  return TT_OK;
}

}  // extern "C"
