// Hopper (sm_90a) implicit-GEMM convolution on the tensor cores (wgmma, TF32 operands).
//
// GEMM view: M = output pixels (one 128-row tile = a TH x TW rectangle of one image, or 128 consecutive
// pixels for 1x1 convs), N = Cout (BN-wide tile), K = taps x Cin walked in 32-float (128-byte) slabs.
//   * operands are staged by TMA (cp.async.bulk.tensor, SWIZZLE_128B) into a 4-stage shared-memory ring:
//     the activation slab of tap (kh, kw) is ONE 4-D box load at a shifted origin — out-of-image pixels and
//     channels are zero-filled by the TMA unit, so padding / dilation cost nothing;
//   * two MMA warpgroups (rows 0..63 / 64..127 of the tile) issue wgmma.m64nNk8.f32.tf32.tf32 with the fp32
//     accumulator tile in registers;
//   * the raw fp32 activation slab is what TMA delivers; two "split" warps rewrite it in shared memory as hi (in place)
//     and lo (second buffer) before the MMA warpgroups may touch it — no pre-pass over the activations, no lo plane
//     streamed from L2;
//   * precision: fp32 operands are split x = hi + lo (activations: hi = RN_tf32(x), lo = x - hi, split in shared
//     memory; weights: hi / lo planes prepared once on the host) and every K slab issues hi*hi + hi*lo + lo*hi
//     ("3xTF32": ~21 mantissa bits per operand) as three m64nBNk8 instructions into two register arrays: main += A_hi x B_hi,
//     corr += A_hi x B_lo + A_lo x B_hi (one shape for all of them: wgmma of different shapes on overlapping accumulators
//     would be serialised by the compiler).  The tensor core adds into its fp32 accumulator with truncation, an error that grows
//     linearly with the number of accumulations, so every CHUNK K-slabs the register accumulator is restarted and folded
//     into fp32 sums with round-to-nearest FADDs.  impl == TF32x1: hi*hi only;
//   * epilogue: each MMA warp transposes its 16 accumulator rows through a warp-private shared-memory slab and stores
//     coalesced channels-last rows with bias + residual(s) + activation fused (concat offset / pixel scatter for
//     transposed convs handled in the store address);
//   * persistent CTAs (one per SM) walk the (M tile, N tile, K split) list;
//   * split-K for under-filled layers (few tiles, long K) and GATHER mode (tap-major sparse convolution: cp.async row
//     gather) both end in a red.add.v4.f32 epilogue into a pre-initialised output.
// Warp roles: warp 0 = TMA / gather producer, warp 1 idle, warps 2..3 = operand split, warps 4..11 = MMA + epilogue.
#include <cuda.h>
#include <string.h>

#include "common.cuh"
#include "tc_ptx.cuh"

extern long long g_tt_launches;
extern int g_tt_debug;

namespace {

constexpr int BM = 128;           // M tile: two warpgroups x 64 rows
constexpr int KS = 32;            // floats per K slab (one 128-byte swizzle row)
constexpr int NTHREADS = 384;     // warpgroup 0: producer + split warps; warpgroups 1..2: MMA + epilogue
// N tile: 3xTF32 holds BN fp32 accumulators (main | corr) plus BN / 2 fp32 sums per MMA thread, within the compiler's
// 168-register budget at 384 threads only for BN = 64
constexpr int BN = 64, STAGES = 4;

struct TcArgs {
  tt_conv_desc d;
  const float* bias;
  const float* res;
  const float* res2;
  float* y;
  int TH, TW;            // tile rectangle (TH * TW <= 128); flat mode: TH = 1, TW = 128 over N*H*W pixels
  int tiles_w, tiles_h;  // tiles per image along W and H
  int flat;              // 1: 1x1 conv on the flattened pixel axis
  int n_slabs;           // ceil(Cin / 32)
  int chunk;             // K slabs accumulated by the tensor core before the MMA warps fold them into fp32 sums
  int total_pix;         // N * OH * OW
  int m_tiles, n_tiles;  // persistent tile walk: tile t -> (m tile t / n_tiles, n tile t % n_tiles)
  // GATHER (tap-major sparse convolution): GEMM rows are the (input row, output row) pairs of one kernel tap
  const float* gx;       // feature rows [.][gx_ld]
  int gx_ld;
  const int* pairs_in;   // [kvol][pair_cap]
  const int* pairs_out;  // [kvol][pair_cap]
  const int* pair_count; // [kvol]
  int kvol, pair_cap;
  // split-K (under-filled layers: few tiles, long K): work item = (tile, N tile, K split); partial sums are
  // red.add-ed into an output the host pre-initialised with bias + residuals, activation applied by a finish kernel
  int splits, k_per;     // K slabs per split (k_per * splits >= taps * n_slabs)
  // input pixel of output (oh, ow) and tap (kh, kw): (oh * stride + org_h + kh * dil, ow * stride + org_w + kw * dil); -pad for a
  // plain convolution, per dimension and of either sign for the stride phases of a transposed (input-gradient) convolution
  int org_h, org_w;
};
constexpr int MAX_KVOL = 32;

// operand split used by the in-kernel split warps: hi = x rounded to nearest TF32 (ties away: one IADD + one LOP3 on
// the alu pipe), lo = x - hi (exact in fp32, one FADD on the fma pipe).  |lo| <= 2^-11 |x| with either sign, so the
// tensor core's own fp32 -> tf32 truncation of lo is an unbiased 2^-21-relative perturbation.
TT_DEVICE void split_rn(float x, float& hi, float& lo) {
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
  lo = x - hi;
}

// Persistent, warp-specialised kernel: each CTA walks work items pt = blockIdx.x, += gridDim.x.  The smem ring and all
// phase counters run ACROSS tiles, so while the MMA warps store tile i the TMA warp is already loading tile i + 1.
// GATHER = true turns the kernel into the tap-major sparse convolution (spconv SubMConv3d / SparseConv3d): work items
// are (tap, pair tile, N tile); warp 0 gathers the activation rows of a tile with 16-byte cp.async (zero-fill for
// the tile tail / channel tail) straight into the 128-byte-swizzled stage buffer, signalling the same `full` barrier
// the weight TMA uses; the epilogue accumulates into the bias-initialised output rows with red.add.v4.f32.
// TERMS: 3 = 3xTF32 (hi*hi + hi*lo + lo*hi), 1 = single-pass TF32 (hi*hi only); a template parameter so that the MMA loop has no
// run-time branch between wgmma instructions.
template <int TERMS, bool GATHER>
__global__ void __launch_bounds__(NTHREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b_hi,
               const __grid_constant__ CUtensorMap map_b_lo, const TcArgs p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr int A_BYTES = BM * KS * 4;                    // 16 KB
  constexpr int B_BYTES = BN * KS * 4;
  constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
  constexpr int SLAB = 16;                                // epilogue column slab
  constexpr int PITCH = SLAB + 4;                         // +4 floats: conflict-free transposition
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* tile_all = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);              // [8 MMA warps][16 rows][PITCH]
  uint64_t* bars = reinterpret_cast<uint64_t*>(tile_all + 8 * 16 * PITCH);
  uint64_t* full = bars;                                  // [STAGES]  TMA -> split warps (raw operands landed)
  uint64_t* empty = bars + STAGES;                        // [STAGES]  MMA warps -> TMA
  uint64_t* conv = bars + 2 * STAGES;                     // [STAGES]  split warps -> MMA (hi / lo written)
  int* sp_first = reinterpret_cast<int*>(bars + 3 * STAGES);   // GATHER: [kvol + 1] first tile of each tap
  int* sp_cnt = sp_first + MAX_KVOL + 1;                  // GATHER: [kvol] pairs of each tap

  const tt_conv_desc& d = p.d;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int taps = d.KH * d.KW;
  const int k_iters = taps * p.n_slabs;

  if (threadIdx.x == 0) {
    // full: the producer's expect_tx arrival (+ 32 cp.async arrivals in GATHER mode); empty: the 8 MMA warps; conv: 2 split warps
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], GATHER ? 33 : 1); mbar_init(&empty[s], 8); mbar_init(&conv[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (GATHER && threadIdx.x == 64) {                        // tile prefix over the taps
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
  const int total_items = (GATHER ? sp_first[p.kvol] : p.m_tiles) * p.n_tiles * p.splits;
  // work item -> (N tile, M tile, tap, rows of that tap)
  auto decode = [&](int pt, int& nt, int& mt, int& tap, int& count, int& kb, int& ke) {
    const int ks = pt % p.splits;
    pt /= p.splits;
    kb = ks * p.k_per;
    ke = min(k_iters, kb + p.k_per);
    nt = pt % p.n_tiles;
    const int pm = pt / p.n_tiles;
    tap = 0; count = 0;
    if (GATHER) {
      while (sp_first[tap + 1] <= pm) ++tap;
      mt = pm - sp_first[tap];
      count = sp_cnt[tap];
    } else {
      mt = pm;
    }
  };
  // weight slab of one stage: hi plane (+ lo plane), BN rows each, loaded as two BN / 2-row boxes per plane
  auto load_weights = [&](uint8_t* st, uint64_t* bar, int k0, int tap, int n0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      tma_load_3d(st + 2 * A_BYTES + h * (B_BYTES / 2), &map_b_hi, bar, k0, tap, n0 + h * (BN / 2));
      if (TERMS == 3) tma_load_3d(st + 2 * A_BYTES + B_BYTES + h * (B_BYTES / 2), &map_b_lo, bar, k0, tap, n0 + h * (BN / 2));
    }
  };

  if (warp < 4) {
    if (warp == 0 && GATHER) {
      // ===================================================================== gather producer (whole warp) + weight TMA
      const uint32_t txb = (TERMS == 3 ? 2 : 1) * B_BYTES;
      int ig = 0;
      for (int pt = blockIdx.x; pt < total_items; pt += gridDim.x) {
        int nt, mt, tap, count, kb, ke;
        decode(pt, nt, mt, tap, count, kb, ke);
        const int n0 = nt * BN;
        const int* pin = p.pairs_in + (long long)tap * p.pair_cap;
        int rows[4];                                            // this lane's rows: lane, lane + 32, lane + 64, lane + 96
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
            load_weights(st, &full[s], it * KS, tap, n0);
          }
          const int c0 = it * KS;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int r = lane + 32 * i;
            const float* src = p.gx + (long long)max(rows[i], 0) * p.gx_ld + c0;
            const uint32_t dst = smem_u32(st) + r * 128;
#pragma unroll
            for (int j = 0; j < 8; ++j) {                       // 16-byte chunk j of row r lives at chunk j ^ (r & 7)
              const bool ok = rows[i] >= 0 && c0 + j * 4 < d.Cin;
              cp_async16(dst + ((j ^ (r & 7)) << 4), ok ? src + j * 4 : p.gx, ok ? 16 : 0);
            }
          }
          cp_async_arrive_noinc(&full[s]);
        }
      }
    } else if (warp == 0 && lane == 0) {
      // ===================================================================== TMA producer
      const uint32_t a_box = (uint32_t)(p.flat ? BM : p.TH * p.TW) * KS * 4;   // bytes one activation box delivers
      const uint32_t tx = a_box + (TERMS == 3 ? 2 : 1) * B_BYTES;
      int ig = 0;                                                               // ring position, continues across tiles
      for (int pt = blockIdx.x; pt < total_items; pt += gridDim.x) {
        int nt, mt, tap0, count, kb, ke;
        decode(pt, nt, mt, tap0, count, kb, ke);
        const int n0 = nt * BN;
        int cw0, ch0, cn;
        if (p.flat) { cw0 = mt * BM; ch0 = 0; cn = 0; }
        else {
          const int tw = mt % p.tiles_w, th = (mt / p.tiles_w) % p.tiles_h;
          cn = mt / (p.tiles_w * p.tiles_h);
          cw0 = tw * p.TW * d.stride + p.org_w; ch0 = th * p.TH * d.stride + p.org_h;
        }
        for (int it = kb; it < ke; ++it, ++ig) {
          const int s = ig % STAGES;
          mbar_wait(&empty[s], ((ig / STAGES) & 1) ^ 1);
          uint8_t* st = smem + s * STAGE_BYTES;
          const int tap = it / p.n_slabs, slab = it - tap * p.n_slabs;
          const int kh = tap / d.KW, kw = tap - kh * d.KW;
          mbar_expect_tx(&full[s], tx);
          const int cw = p.flat ? cw0 : cw0 + kw * d.dil, ch = p.flat ? 0 : ch0 + kh * d.dil;
          tma_load_4d(st, &map_a, &full[s], slab * KS, cw, ch, cn);      // raw fp32 activations
          load_weights(st, &full[s], slab * KS, tap, n0);
        }
      }
    } else if (warp >= 2) {
      // ===================================================================== operand split (warps 2, 3)
      // Each warp owns 64 rows of the 128 x 32-float activation slab: raw -> hi in place, lo into the second buffer.
      // Element-wise at identical offsets, so the 128-byte swizzle TMA applied is irrelevant here.
      const int w2 = warp - 2;
      int ig = 0;
      for (int pt = blockIdx.x; pt < total_items; pt += gridDim.x) {
        int nt, mt, tap0, count, kb, ke;
        decode(pt, nt, mt, tap0, count, kb, ke);
        for (int it = kb; it < ke; ++it, ++ig) {
          const int s = ig % STAGES;
          mbar_wait(&full[s], (ig / STAGES) & 1);
          const uint32_t raw = smem_u32(smem + s * STAGE_BYTES) + w2 * (A_BYTES / 2) + lane * 16;   // lo at + A_BYTES
          // all loads of a batch are issued before any store: the loop is latency-bound otherwise
#pragma unroll
          for (int b0 = 0; b0 < A_BYTES / 32 / 32; b0 += 8) {    // 16 float4 per lane, two batches of 8
            float4 v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = lds128(raw + (b0 + u) * 512);
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              float4 h, l;
              split_rn(v[u].x, h.x, l.x); split_rn(v[u].y, h.y, l.y); split_rn(v[u].z, h.z, l.z); split_rn(v[u].w, h.w, l.w);
              sts128(raw + (b0 + u) * 512, h);
              if (TERMS == 3) sts128(raw + A_BYTES + (b0 + u) * 512, l);
            }
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
          __syncwarp();
          if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&conv[s])) : "memory");
        }
      }
    }
  } else {
    // ===================================================================== MMA + epilogue (warpgroups 1, 2)
    const int cw = warp - 4;                                // MMA warp 0..7
    const int wg = cw >> 2;                                 // warpgroup: tile rows [64 wg, 64 wg + 64)
    const int row0 = wg * 64 + (cw & 3) * 16;               // this warp's 16 accumulator rows
    const long long yns = d.y_nstride ? d.y_nstride : (long long)d.yH * d.yW * d.y_ld;
    const int HWo = d.OH * d.OW;
    float* tile = tile_all + cw * 16 * PITCH;               // warp-private transposition buffer [16 rows][PITCH]
    const int sub = lane >> 2, cl = (lane & 3) * 4;         // store phase: 4 lanes per row, 8 rows per warp instruction
    int ig = 0;
    for (int pt = blockIdx.x; pt < total_items; pt += gridDim.x) {
      int nt, mt, tap, count, kb, ke;
      decode(pt, nt, mt, tap, count, kb, ke);
      const int nch = (ke - kb + p.chunk - 1) / p.chunk;
      const bool real_tile = GATHER ? mt * BM < count : mt < p.m_tiles;
      const int n0 = nt * BN;
      // ---- output / residual addresses of the two rows this lane stores (rows row0 + sub, row0 + 8 + sub)
      int fl[2];
      long long yo[2], o1[2], o2[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = row0 + i * 8 + sub;
        if (GATHER) {
          const int m = mt * BM + r;
          const bool valid = m < count;
          const int orow = valid ? __ldg(p.pairs_out + (long long)tap * p.pair_cap + m) : 0;
          yo[i] = (long long)orow * d.y_ld + d.y_coff;
          o1[i] = 0; o2[i] = 0;
          fl[i] = valid ? 1 : 0;
        } else {
          bool valid;
          int nimg, oh, ow;
          long long rrow;
          if (p.flat) {
            const long long pix = (long long)mt * BM + r;
            valid = real_tile && pix < p.total_pix;
            nimg = (int)(pix / HWo);
            const int rem = (int)(pix - (long long)nimg * HWo);
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
      // ---- K walk: chunks of `chunk` slabs accumulated by the tensor core, folded into fp32 sums with RN adds
      float sum[BN / 2];
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) sum[j] = 0.f;
      auto release = [&](int s) {                            // this warp's wgmmas no longer read stage s
        __syncwarp();
        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty[s])) : "memory");
      };
      int it = kb;
      for (int c = 0; c < nch; ++c) {
        float acc[BN / 2], cor[BN / 2];                      // main and correction accumulators
        const int it_end = min(it + p.chunk, ke);
        int held = -1;                                       // the stage whose wgmmas may still be in flight
        for (bool first = true; it < it_end; ++it, ++ig, first = false) {
          const int s = ig % STAGES;
          mbar_wait(&conv[s], (ig / STAGES) & 1);           // operands landed AND split into hi / lo
          const uint32_t a_hi = smem_u32(smem + s * STAGE_BYTES) + wg * (A_BYTES / 2), a_lo = a_hi + A_BYTES;
          const uint32_t b_hi = smem_u32(smem + s * STAGE_BYTES) + 2 * A_BYTES, b_lo = b_hi + B_BYTES;
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < KS / 8; ++kk) {              // K = 8 tf32 = 32 bytes inside the 128-byte swizzle row
            const uint32_t off = kk * 32, z = (first && kk == 0) ? 0u : 1u;
            wgmma_tf32<BN>(acc, make_smem_desc(a_hi + off), make_smem_desc(b_hi + off), z);          // hi*hi
            if constexpr (TERMS == 3) {
              wgmma_tf32<BN>(cor, make_smem_desc(a_hi + off), make_smem_desc(b_lo + off), z);        // hi*lo
              wgmma_tf32<BN>(cor, make_smem_desc(a_lo + off), make_smem_desc(b_hi + off), 1u);       // lo*hi
            }
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
        if constexpr (TERMS == 3) {
#pragma unroll
          for (int j = 0; j < BN / 2; ++j) sum[j] += acc[j] + cor[j];   // fp32 RN adds
        } else {
#pragma unroll
          for (int j = 0; j < BN / 2; ++j) sum[j] += acc[j];
        }
      }
      // ---- coalesced store in 16-column slabs: registers -> warp-private smem (transpose) -> 64-byte row segments
#pragma unroll
      for (int sl = 0; sl < BN / SLAB; ++sl) {
        __syncwarp();                                          // the previous slab has been read back by this warp
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {                     // fragment column group j = 2 sl + jj: columns 8 jj + 2 (lane % 4) + {0, 1}
          const int j = 2 * sl + jj, cc = 8 * jj + 2 * (lane & 3);
          *reinterpret_cast<float2*>(&tile[sub * PITCH + cc]) = make_float2(sum[4 * j], sum[4 * j + 1]);
          *reinterpret_cast<float2*>(&tile[(sub + 8) * PITCH + cc]) = make_float2(sum[4 * j + 2], sum[4 * j + 3]);
        }
        __syncwarp();
        const int col = n0 + sl * SLAB + cl;
        if (col < d.Cout) {
          float4 acc4[2], ra[2], rb[2];
#pragma unroll
          for (int i = 0; i < 2; ++i) {                       // batch the loads of both rows (memory-level parallelism)
            acc4[i] = *reinterpret_cast<const float4*>(&tile[(i * 8 + sub) * PITCH + cl]);
            ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            rb[i] = ra[i];
            if (fl[i] & 1) {
              if (p.res) ra[i] = *reinterpret_cast<const float4*>(p.res + o1[i] + col);
              if (p.res2) rb[i] = *reinterpret_cast<const float4*>(p.res2 + o2[i] + col);
            }
          }
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            if (!(fl[i] & 1)) continue;
            float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.bias) bv = __ldg(reinterpret_cast<const float4*>(p.bias + (d.bias_n_mod ? (long long)((fl[i] >> 1) % d.bias_n_mod) * d.Cout : 0) + col));
            const float4 o = make_float4(acc4[i].x + bv.x + ra[i].x + rb[i].x, acc4[i].y + bv.y + ra[i].y + rb[i].y,
                                         acc4[i].z + bv.z + ra[i].z + rb[i].z, acc4[i].w + bv.w + ra[i].w + rb[i].w);
            float* dst = p.y + yo[i] + col;
            if (GATHER || p.splits > 1) {                      // taps / K splits race on an output row: red.add
              tt_red_add_v4(dst, o.x, o.y, o.z, o.w);
            } else {
              *reinterpret_cast<float4*>(dst) =
                  make_float4(tt_act(o.x, d.act), tt_act(o.y, d.act), tt_act(o.z, d.act), tt_act(o.w, d.act));
            }
          }
        }
      }
    }
  }
}

// split-K companions: y = bias + res + res2 before the tensor-core kernel red.adds its partial sums; y = act(y) after
__global__ void splitk_init_kernel(const tt_conv_desc d, const float* __restrict__ bias, const float* __restrict__ res,
                                   const float* __restrict__ res2, float* __restrict__ y) {
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
    *reinterpret_cast<float4*>(y + n * yns + (pix - (long long)n * HWo) * d.y_ld + d.y_coff + c) = v;
  }
}
__global__ void splitk_finish_kernel(const tt_conv_desc d, float* __restrict__ y) {
  const int HWo = d.OH * d.OW, C4 = d.Cout / 4;
  const long long total = (long long)d.N * HWo * C4;
  const long long yns = d.y_nstride ? d.y_nstride : (long long)d.yH * d.yW * d.y_ld;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const long long pix = i / C4;
    const int n = (int)(pix / HWo);
    float4* q = reinterpret_cast<float4*>(y + n * yns + (pix - (long long)n * HWo) * d.y_ld + d.y_coff + c);
    const float4 v = *q;
    *q = make_float4(tt_act(v.x, d.act), tt_act(v.y, d.act), tt_act(v.z, d.act), tt_act(v.w, d.act));
  }
}

// persistent grid: one CTA per SM (at most `max_ctas`) walks the `items` work items
template <int TERMS, bool GATHER>
cudaError_t launch_tc(const CUtensorMap& ma, const CUtensorMap& mb_hi, const CUtensorMap& mb_lo, const TcArgs& a, long long items,
                      long long max_ctas, cudaStream_t st) {
  // stage ring + 8 warp-private transposition slabs + barriers and the tap prefix
  constexpr int smem = STAGES * (2 * BM * KS * 4 + 2 * BN * KS * 4) + 1024 + 8 * 16 * 20 * 4 + 512;
  static_assert(smem <= 227 * 1024, "shared memory per block");
  static bool set = false;
  if (!set) { cudaFuncSetAttribute(conv_tc_kernel<TERMS, GATHER>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); set = true; }
  const long long grid = items < max_ctas ? items : max_ctas;
  conv_tc_kernel<TERMS, GATHER><<<(unsigned)(grid > 1 ? grid : 1), NTHREADS, smem, st>>>(ma, mb_hi, mb_lo, a);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ host side
}  // namespace

bool tt_conv2d_tc_supported(const tt_conv_desc* d, const void* x, const void* w, const void* y) {
  if (d->groups != 1 || (d->stride != 1 && d->stride != 2)) return false;
  if (d->Cin % 4 || d->Cout % 4 || d->x_ld % 4 || d->x_coff % 4 || d->y_ld % 4 || d->x_nstride % 4 || d->y_nstride % 4 || d->x_hstride % 4) return false;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(y)) & 15) return false;
  // the epilogue moves float4 vectors: output and residual channel offsets must keep them 16-byte aligned
  if (d->y_coff % 4) return false;
  if (d->res_mode != TT_RES_NONE && (d->res_ld % 4 || d->res_coff % 4)) return false;
  if (d->res2_ld % 4 || d->res2_coff % 4) return false;
  if (d->OH != (d->H + 2 * d->pad - d->dil * (d->KH - 1) - 1) / d->stride + 1 ||
      d->OW != (d->W + 2 * d->pad - d->dil * (d->KW - 1) - 1) / d->stride + 1) return false;
  return true;
}

int tt_simt_splits(const tt_conv_desc* d, int has_gather);

extern "C" size_t tt_conv2d_workspace_bytes(const tt_conv_desc* d) {
  if (!d) return 0;
  if (d->impl < 2) {                                          // SIMT: split-K partial sums for small-M / large-K layers
    const int s = tt_simt_splits(d, 0);
    return s > 1 ? (size_t)s * d->N * d->OH * d->OW * d->Cout * 4 : 0;
  }
  return 0;                                                   // tensor cores: operands are split inside the kernel
}

// w_tc: [2][Cout][taps][Cin] fp32 = TF32-exact hi plane then lo plane (prepared once per layer by the host).
// allow_split_k = false keeps every output row's sum in one fixed order (no red.add across K splits): the deformable
// convolution's outputs must not depend on how many images one call covers.
// tt_conv2d_tc_origin: the same with the input origin given per dimension (org_h, org_w) instead of -pad (d->pad is not read),
// and no shape predicate: OH / OW are whatever output extent the caller wants covered (input rows past the map read as zeros).
int tt_conv2d_tc_origin(const tt_conv_desc* d, int org_h, int org_w, const float* x, const float* w_tc, const float* bias, const float* res,
                        const float* res2, float* y, cudaStream_t st, bool allow_split_k) {
  const int terms = d->impl == 3 ? 3 : 1;
  const int taps = d->KH * d->KW;
  const long long npix_in = (long long)d->N * d->H * d->W;
  const long long xhs = d->x_hstride ? d->x_hstride : (long long)d->W * d->x_ld;   // input row pitch
  const long long xns = d->x_nstride ? d->x_nstride : (long long)d->H * xhs;
  const float* xa = x + d->x_coff;                            // TMA reads the activation tensor in place (ld / coff / image stride)
  TcArgs a;
  a.d = *d;
  a.bias = bias; a.res = res; a.res2 = res2; a.y = y;
  a.chunk = terms == 3 ? ((g_tt_debug & 0x40000) ? 1 : (g_tt_debug & 0x20000) ? 4 : 2) : 16;   // 2 slabs = K 64: 8 truncating accumulations per chunk
  a.n_slabs = (d->Cin + KS - 1) / KS;
  a.total_pix = d->N * d->OH * d->OW;
  a.org_h = org_h; a.org_w = org_w;
  a.flat = (taps == 1 && org_h == 0 && org_w == 0 && d->stride == 1 && d->OH == d->H && d->OW == d->W && xhs == (long long)d->W * d->x_ld &&
            xns == (long long)d->H * xhs) ? 1 : 0;
  CUtensorMap ma, mb_hi, mb_lo;
  int grid_x;
  if (a.flat) {
    a.TH = 1; a.TW = BM; a.tiles_w = a.tiles_h = 1;
    cuuint64_t dims[4] = {(cuuint64_t)d->Cin, (cuuint64_t)npix_in, 1, 1};       // dim 0 = logical channels: beyond Cin is zero-filled
    cuuint64_t str[3] = {(cuuint64_t)d->x_ld * 4, (cuuint64_t)npix_in * d->x_ld * 4, (cuuint64_t)npix_in * d->x_ld * 4};
    cuuint32_t box[4] = {KS, BM, 1, 1};
    if (!encode_map(&ma, xa, 4, dims, str, box)) return TT_ERR_CUDA;
    grid_x = tt_cdiv(npix_in, BM);
  } else {
    // rectangle with TH * TW <= 128 that wastes the fewest rows
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
    cuuint64_t dims[4] = {(cuuint64_t)d->Cin, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->N};
    cuuint64_t str[3] = {(cuuint64_t)d->x_ld * 4, (cuuint64_t)xhs * 4, (cuuint64_t)xns * 4};
    cuuint32_t box[4] = {KS, (cuuint32_t)(a.TW * d->stride), (cuuint32_t)(a.TH * d->stride), 1};
    if (!encode_map(&ma, xa, 4, dims, str, box, d->stride)) return TT_ERR_CUDA;
    grid_x = a.tiles_w * a.tiles_h * d->N;
  }
  {
    const size_t wplane = (size_t)d->Cout * taps * d->Cin;
    cuuint64_t dims[3] = {(cuuint64_t)d->Cin, (cuuint64_t)taps, (cuuint64_t)d->Cout};
    cuuint64_t str[2] = {(cuuint64_t)d->Cin * 4, (cuuint64_t)taps * d->Cin * 4};
    cuuint32_t box[3] = {KS, 1, (cuuint32_t)(BN / 2)};               // a plane's BN-row slab is loaded as two half boxes
    if (!encode_map(&mb_hi, w_tc, 3, dims, str, box)) return TT_ERR_CUDA;
    if (!encode_map(&mb_lo, w_tc + wplane, 3, dims, str, box)) return TT_ERR_CUDA;
  }
  a.m_tiles = grid_x;
  a.n_tiles = tt_cdiv(d->Cout, BN);
  const int num_sms = tt_num_sms();
  // split-K: a layer with few tiles and a long K (14x28 / 21x21 / 84x84 maps) leaves most SMs idle; spread K over
  // the idle SMs.  Needs a plain output layout (no pixel scatter, SAME residuals, one bias vector).
  const int k_iters = taps * a.n_slabs;
  a.splits = 1;
  a.k_per = k_iters;
  {
    const long long tiles = (long long)a.m_tiles * a.n_tiles;
    const bool plain = d->oy_mul == 1 && d->ox_mul == 1 && d->oy_add == 0 && d->ox_add == 0 && d->yH == d->OH && d->yW == d->OW &&
                       d->res_mode != TT_RES_UP2_NEAREST && d->bias_n_mod == 0 && !(g_tt_debug & 128);
    if (allow_split_k && plain && tiles <= num_sms / 2 && k_iters >= 16) {
      int sp = (int)((num_sms + tiles - 1) / tiles);
      if (sp > k_iters / 8) sp = k_iters / 8;
      if (sp > 32) sp = 32;
      if (sp >= 2) {
        a.k_per = tt_cdiv(k_iters, sp);
        a.splits = tt_cdiv(k_iters, a.k_per);
      }
    }
  }
  if (a.splits > 1) {
    const long long total4 = (long long)d->N * d->OH * d->OW * (d->Cout / 4);
    const int nb = (int)((total4 + 255) / 256 > num_sms * 8 ? num_sms * 8 : (total4 + 255) / 256);
    splitk_init_kernel<<<nb, 256, 0, st>>>(*d, bias, d->res_mode != TT_RES_NONE ? res : nullptr, res2, y);
    ++g_tt_launches;
    TT_CHECK_LAUNCH("tt_conv2d(tc split-k init)");
    a.bias = nullptr; a.res = nullptr; a.res2 = nullptr;
    a.d.act = TT_ACT_NONE;
    a.d.res_mode = TT_RES_NONE;
  }
  const long long items = (long long)a.m_tiles * a.n_tiles * a.splits;
  const long long ctas = num_sms - ((g_tt_debug >> 8) & 0xFF);
  const cudaError_t lerr = terms == 3 ? launch_tc<3, false>(ma, mb_hi, mb_lo, a, items, ctas, st) : launch_tc<1, false>(ma, mb_hi, mb_lo, a, items, ctas, st);   // debug bits 8..15: SMs left to a concurrent branch
  if (lerr != cudaSuccess) { tt_set_error("tt_conv2d(tc): launch failed: %s", cudaGetErrorString(lerr)); return TT_ERR_CUDA; }
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_conv2d(tc)");
  if (a.splits > 1 && d->act != TT_ACT_NONE) {
    const long long total4 = (long long)d->N * d->OH * d->OW * (d->Cout / 4);
    const int nb = (int)((total4 + 255) / 256 > num_sms * 8 ? num_sms * 8 : (total4 + 255) / 256);
    splitk_finish_kernel<<<nb, 256, 0, st>>>(*d, y);
    ++g_tt_launches;
    TT_CHECK_LAUNCH("tt_conv2d(tc split-k finish)");
  }
  return TT_OK;
}

int tt_conv2d_tc(const tt_conv_desc* d, const float* x, const float* w_tc, const float* bias, const float* res,
                 const float* res2, float* y, void* /*workspace*/, cudaStream_t st, bool allow_split_k) {
  return tt_conv2d_tc_origin(d, -d->pad, -d->pad, x, w_tc, bias, res, res2, y, st, allow_split_k);
}

// ------------------------------------------------------------------------------------------------------------------
// Tap-major sparse convolution on the tensor cores (GATHER mode of the kernel above).  The caller (tt_sparse_conv) has
// initialised the output rows with the bias and applies residual + activation afterwards.
bool tt_sparse_conv_tc_supported(const tt_sparse_conv_desc* d, const void* x, const void* w, const void* y) {
  if (d->Cin % 4 || d->Cout % 4 || d->in_ld % 4 || d->out_ld % 4 || d->Cin < 32 || d->Cout < 32 || d->kvol > MAX_KVOL) return false;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(y)) & 15) return false;
  return true;
}

int tt_sparse_conv_tc(const tt_sparse_conv_desc* d, const float* feats_in, const float* w_tc, const int* pairs_in,
                      const int* pairs_out, const int* pair_count, float* feats_out, cudaStream_t st) {
  TcArgs a;
  memset(&a, 0, sizeof(a));
  a.d.N = a.d.H = a.d.W = a.d.OH = a.d.OW = a.d.yH = a.d.yW = 1;
  a.d.KH = a.d.KW = a.d.stride = a.d.dil = a.d.groups = 1;
  a.d.oy_mul = a.d.ox_mul = 1;
  a.d.Cin = d->Cin; a.d.x_ld = d->in_ld; a.d.Cout = d->Cout; a.d.y_ld = d->out_ld;
  a.d.act = TT_ACT_NONE;
  a.y = feats_out;
  const int terms = d->impl == 3 ? 3 : 1;
  a.chunk = terms == 3 ? ((g_tt_debug & 0x40000) ? 1 : (g_tt_debug & 0x20000) ? 4 : 2) : 16;
  a.n_slabs = (d->Cin + KS - 1) / KS;
  a.gx = feats_in; a.gx_ld = d->in_ld;
  a.pairs_in = pairs_in; a.pairs_out = pairs_out; a.pair_count = pair_count;
  a.kvol = d->kvol; a.pair_cap = d->pair_cap;
  a.splits = 1; a.k_per = a.n_slabs;
  a.n_tiles = tt_cdiv(d->Cout, BN);
  CUtensorMap mb_hi, mb_lo;
  {
    const size_t wplane = (size_t)d->Cout * d->kvol * d->Cin;
    cuuint64_t dims[3] = {(cuuint64_t)d->Cin, (cuuint64_t)d->kvol, (cuuint64_t)d->Cout};
    cuuint64_t str[2] = {(cuuint64_t)d->Cin * 4, (cuuint64_t)d->kvol * d->Cin * 4};
    cuuint32_t box[3] = {KS, 1, (cuuint32_t)(BN / 2)};
    if (!encode_map(&mb_hi, w_tc, 3, dims, str, box)) return TT_ERR_CUDA;
    if (!encode_map(&mb_lo, w_tc + wplane, 3, dims, str, box)) return TT_ERR_CUDA;
  }
  const int num_sms = tt_num_sms();
  const long long cap_items = (long long)d->kvol * tt_cdiv(d->pair_cap, BM) * a.n_tiles;   // upper bound of gathered tiles over all taps
  const cudaError_t lerr = terms == 3 ? launch_tc<3, true>(mb_hi, mb_hi, mb_lo, a, cap_items, num_sms, st)
                                        : launch_tc<1, true>(mb_hi, mb_hi, mb_lo, a, cap_items, num_sms, st);
  if (lerr != cudaSuccess) { tt_set_error("tt_sparse_conv(tc): launch failed: %s", cudaGetErrorString(lerr)); return TT_ERR_CUDA; }
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_sparse_conv(tc)");
  return TT_OK;
}
