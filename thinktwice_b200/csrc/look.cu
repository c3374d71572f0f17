// Look module (thinktwice_decoder.py:88-187) and multi-scale deformable attention
// (multi_scale_deformable_attn_function.py:468-526 + mmcv ms_deform_attn_forward).
// The reference builds the rebatched queries with Python loops, `.nonzero()` and 4*B host syncs per
// layer; here projection, ordered compaction, query assembly and the 4-level bilinear FPN gather run
// on the device with the batch-wide max_len kept in a device scalar (no host round trip), and every
// feature gather is a channel-contiguous (coalesced) read of a channels-last map.  The *_frames entries bound and reduce
// the rows of each frame by that frame's own max_len (independent frames: B = 1 semantics per frame).
#include "common.cuh"

extern long long g_tt_launches;
#define TT_LAUNCHED(name) do { ++g_tt_launches; TT_CHECK_LAUNCH(name); } while (0)

namespace {

constexpr int ZL = 15;   // z levels: linspace(-4, 10, 15) = -4, -3, ..., 10 (thinktwice_decoder.py:160)

TT_DEVICE void look_point(const float* wp, int b, int T, int q, float* xyz) {
  const int t = q / ZL, zi = q % ZL;
  if (t < T) { xyz[0] = wp[(b * T + t) * 2]; xyz[1] = wp[(b * T + t) * 2 + 1]; }
  else {
    // static points (5,0), (0,-5), (0,5), (-5,0): thinktwice_decoder.py:157
    const int s = t - T;
    xyz[0] = s == 0 ? 5.f : (s == 3 ? -5.f : 0.f);
    xyz[1] = s == 1 ? -5.f : (s == 2 ? 5.f : 0.f);
  }
  xyz[2] = -4.f + (float)zi;
}

// one warp per (b, cam)
__global__ void look_project_kernel(const tt_look_desc d, const float* __restrict__ wp, const float* __restrict__ l2i,
                                    const float* __restrict__ ida, float* __restrict__ ref_cam, int* __restrict__ order,
                                    int* __restrict__ counts, int* max_len) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  if (wid >= d.B * d.num_cams) return;
  const int b = wid / d.num_cams;
  const float* M = l2i + (long long)wid * 16;
  const float* A = ida + (long long)wid * 16;
  const float eps = 1e-5f;
  int base = 0;
  for (int q0 = 0; q0 < d.num_query; q0 += 32) {
    const int q = q0 + lane;
    bool valid = false;
    if (q < d.num_query) {
      float p[3];
      look_point(wp, b, d.T, q, p);
      float c[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) c[r] = M[r * 4] * p[0] + M[r * 4 + 1] * p[1] + M[r * 4 + 2] * p[2] + M[r * 4 + 3] * 1.f;
      const float dz = fmaxf(c[2], eps);
      c[0] = c[0] / dz;
      c[1] = c[1] / dz;
      float e[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) e[r] = A[r * 4] * c[0] + A[r * 4 + 1] * c[1] + A[r * 4 + 2] * c[2] + A[r * 4 + 3] * c[3];
      const float x = e[0] / d.img_w, y = e[1] / d.img_h;
      valid = (e[2] > eps) && (y > 0.f) && (y < 1.f) && (x < 1.f) && (x > 0.f);
      ref_cam[((long long)wid * d.num_query + q) * 2] = x;
      ref_cam[((long long)wid * d.num_query + q) * 2 + 1] = y;
    }
    const unsigned m = __ballot_sync(0xffffffffu, valid);
    if (valid) order[(long long)wid * d.num_query + base + __popc(m & ((1u << lane) - 1))] = q;
    base += __popc(m);
  }
  if (lane == 0) { counts[wid] = base; atomicMax(max_len, base); }
}

// one CTA per rebatched row (bn, r)
__global__ void __launch_bounds__(256) look_rebatch_kernel(
    const tt_look_desc d, const float* __restrict__ wp, const float* __restrict__ ctrl_sp, const float* __restrict__ temb,
    const float* __restrict__ semb, const float* __restrict__ meas, const float* __restrict__ flat,
    const float* __restrict__ l0, const float* __restrict__ l1, const float* __restrict__ l2, const float* __restrict__ l3,
    const float* __restrict__ ref_cam, const int* __restrict__ order, const int* __restrict__ counts,
    float* __restrict__ rows, int rows_ld, float* __restrict__ ref_rebatch) {
  const int r = blockIdx.x % d.max_len_cap;
  const int bn = blockIdx.x / d.max_len_cap;
  const int b = bn / d.num_cams;
  float* row = rows + ((long long)bn * d.max_len_cap + r) * rows_ld;
  const int width = d.q_dim + d.levels * d.C;
  if (r >= counts[bn]) {
    for (int i = threadIdx.x; i < width; i += blockDim.x) row[i] = 0.f;
    if (threadIdx.x < 2) ref_rebatch[((long long)bn * d.max_len_cap + r) * 2 + threadIdx.x] = 0.f;
    return;
  }
  const int q = order[(long long)bn * d.num_query + r];
  const int t = q / ZL;
  const float rx = ref_cam[((long long)bn * d.num_query + q) * 2], ry = ref_cam[((long long)bn * d.num_query + q) * 2 + 1];
  if (threadIdx.x < 2) ref_rebatch[((long long)bn * d.max_len_cap + r) * 2 + threadIdx.x] = threadIdx.x ? ry : rx;
  // query = [ctrl 4 | xyz 3 | temporal/static emb E | meas Mm | flat Fl]  (thinktwice_decoder.py:164-171)
  const int E = d.emb_dim, Mm = d.meas_dim, Fl = d.flat_dim;
  for (int i = threadIdx.x; i < d.q_dim; i += blockDim.x) {
    float v;
    if (i < 4) v = t < d.T ? ctrl_sp[(b * d.T + t) * 4 + i] : 0.f;
    else if (i < 7) { float p[3]; look_point(wp, b, d.T, q, p); v = p[i - 4]; }
    else if (i < 7 + E) v = t < d.T ? temb[t * E + (i - 7)] : semb[(t - d.T) * E + (i - 7)];
    else if (i < 7 + E + Mm) v = meas[(long long)b * Mm + (i - 7 - E)];
    else v = flat[(long long)b * Fl + (i - 7 - E - Mm)];
    row[i] = v;
  }
  // F.grid_sample(feat, 2*ref-1, bilinear, zeros, align_corners=False) on every level; feature index c*L + l
  const float* lv[4] = {l0, l1, l2, l3};
  for (int c = threadIdx.x; c < d.C; c += blockDim.x) {
    for (int l = 0; l < d.levels; ++l) {
      const int H = d.lvl_h[l], W = d.lvl_w[l];
      const float x = rx * W - 0.5f, y = ry * H - 0.5f;
      const int x0 = (int)floorf(x), y0 = (int)floorf(y);
      const float lx = x - x0, ly = y - y0;
      const float* f = lv[l] + (long long)bn * H * W * d.C + c;
      float acc = 0.f;
      if (y0 >= 0 && y0 < H) {
        if (x0 >= 0 && x0 < W) acc += (1.f - ly) * (1.f - lx) * __ldg(f + ((long long)y0 * W + x0) * d.C);
        if (x0 + 1 >= 0 && x0 + 1 < W) acc += (1.f - ly) * lx * __ldg(f + ((long long)y0 * W + x0 + 1) * d.C);
      }
      if (y0 + 1 >= 0 && y0 + 1 < H) {
        if (x0 >= 0 && x0 < W) acc += ly * (1.f - lx) * __ldg(f + ((long long)(y0 + 1) * W + x0) * d.C);
        if (x0 + 1 >= 0 && x0 + 1 < W) acc += ly * lx * __ldg(f + ((long long)(y0 + 1) * W + x0 + 1) * d.C);
      }
      row[d.q_dim + c * d.levels + l] = acc;
    }
  }
}

// Row bound of one (frame, camera) image bn = b * cams + cam.  Batch-coupled (the reference's semantics at any B,
// thinktwice_decoder.py:137): the batch-wide max_len, one device scalar.  Per frame (the reference run on frame b alone, B = 1):
// the largest count over that frame's cameras, read from the counts tt_look_project wrote.
enum RowBound { kBatchMaxLen, kFrameMaxLen };

template <RowBound RB>
TT_DEVICE int look_row_bound(const int* bound, int bn, int cams) {
  if (RB == kBatchMaxLen) return *bound;
  const int* c = bound + (bn / cams) * cams;
  int ml = 0;
  for (int i = 0; i < cams; ++i) ml = max(ml, c[i]);
  return ml;
}

// one warp per (row, head); lane = channel of the head (dh == 32) and, for the softmax, sample index.  Rows at or past the
// row bound of their image are not computed (bound NULL: every row).
template <RowBound RB>
__global__ void __launch_bounds__(256) msda_kernel(const tt_msda_desc d, const float* __restrict__ value,
                                                   const float* __restrict__ off, const float* __restrict__ logits,
                                                   const float* __restrict__ ref, const int* __restrict__ bound, int cams,
                                                   float* __restrict__ out) {
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  const int head = wid % d.heads;
  const long long row = wid / d.heads;                      // bn * rows_cap + r
  if (row >= (long long)d.BN * d.rows_cap) return;
  const int r = row % d.rows_cap;
  const int bn = row / d.rows_cap;
  if (bound && r >= look_row_bound<RB>(bound, bn, cams)) return;
  const int S = d.levels * d.points;                        // 32 samples per head
  const int E = d.heads * d.dh;
  // softmax over the S logits of this head (msda:480-483)
  float lg = lane < S ? logits[row * (d.heads * S) + head * S + lane] : -INFINITY;
  const float mx = warp_max(lg);
  float ex = lane < S ? expf(lg - mx) : 0.f;
  const float aw = ex / warp_sum(ex);
  const float ox = lane < S ? off[(row * d.heads + head) * S * 2 + lane * 2] : 0.f;
  const float oy = lane < S ? off[(row * d.heads + head) * S * 2 + lane * 2 + 1] : 0.f;
  const float rx = ref[row * 2], ry = ref[row * 2 + 1];
  const int VL = d.value_ld ? d.value_ld : E;               // key-row pitch of the value buffer
  const float* vb = value + (long long)bn * d.num_keys * VL + d.value_coff + head * d.dh + lane;
  float acc = 0.f;
  for (int s = 0; s < S; ++s) {
    const int l = s / d.points;
    const int H = d.lvl_h[l], W = d.lvl_w[l];
    const float w_s = __shfl_sync(0xffffffffu, aw, s);
    const float dx = __shfl_sync(0xffffffffu, ox, s), dy = __shfl_sync(0xffffffffu, oy, s);
    // loc = ref + off / (W, H)  (msda:497-504);  pixel = loc * size - 0.5 (grid_sample, align_corners=False)
    const float x = (rx + dx / (float)W) * W - 0.5f, y = (ry + dy / (float)H) * H - 0.5f;
    if (!(x > -1.f && y > -1.f && x < (float)W && y < (float)H)) continue;
    const int x0 = (int)floorf(x), y0 = (int)floorf(y);
    const float lx = x - x0, ly = y - y0;
    const float* v = vb + (long long)d.lvl_start[l] * VL;
    float sv = 0.f;
    if (y0 >= 0) {
      if (x0 >= 0) sv += (1.f - ly) * (1.f - lx) * __ldg(v + ((long long)y0 * W + x0) * VL);
      if (x0 + 1 < W) sv += (1.f - ly) * lx * __ldg(v + ((long long)y0 * W + x0 + 1) * VL);
    }
    if (y0 + 1 < H) {
      if (x0 >= 0) sv += ly * (1.f - lx) * __ldg(v + ((long long)(y0 + 1) * W + x0) * VL);
      if (x0 + 1 < W) sv += ly * lx * __ldg(v + ((long long)(y0 + 1) * W + x0 + 1) * VL);
    }
    acc = fmaf(w_s, sv, acc);
  }
  if (lane < d.dh) out[row * E + head * d.dh + lane] = acc;
}

// msda:338-342 zeroes the first len(indexes[cam]) rows of every image and divides by it; that length is the number of frames
// in the forward call (B when coupled, 1 for a frame on its own), and the sum runs up to the row bound.
template <RowBound RB>
__global__ void look_reduce_kernel(const float* __restrict__ rows, int B, int cams, int cap, int C,
                                   const int* __restrict__ bound, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * cams * C) return;
  const int c = i % C, bn = i / C;
  const int ml = min(look_row_bound<RB>(bound, bn, cams), cap);
  const int first = RB == kBatchMaxLen ? B : 1;
  const float div = (float)(first > 1 ? first : 1);
  float s = 0.f;
  for (int r = first; r < ml; ++r) s += rows[((long long)bn * cap + r) * C + c] / div;
  out[i] = s;
}

}  // namespace

extern "C" {

int tt_look_project(const tt_look_desc* d, const float* wp, const float* lidar2img, const float* ida, float* ref_cam,
                    int* order, int* counts, int* max_len, tt_stream_t stream) {
  TT_REQUIRE(d && wp && lidar2img && ida && ref_cam && order && counts && max_len, "tt_look_project", "null argument");
  TT_REQUIRE(d->num_query == 2 * d->T * ZL && d->num_query <= d->max_len_cap, "tt_look_project", "num_query must be 2*T*15");
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemsetAsync(max_len, 0, 4, st) != cudaSuccess) { tt_set_error("tt_look_project: memset failed"); return TT_ERR_CUDA; }
  const int warps = d->B * d->num_cams;
  look_project_kernel<<<tt_cdiv(warps * 32, 128), 128, 0, st>>>(*d, wp, lidar2img, ida, ref_cam, order, counts, max_len);
  TT_LAUNCHED("tt_look_project");
  return TT_OK;
}

int tt_look_rebatch(const tt_look_desc* d, const float* wp, const float* ctrl_sp, const float* temporal_emb,
                    const float* static_emb, const float* meas, const float* flat, const float* const* mlvl,
                    const float* ref_cam, const int* order, const int* counts, float* rows, int rows_ld,
                    float* ref_rebatch, tt_stream_t stream) {
  TT_REQUIRE(d && wp && ctrl_sp && temporal_emb && static_emb && meas && flat && mlvl && ref_cam && order && counts && rows &&
                 ref_rebatch, "tt_look_rebatch", "null argument");
  TT_REQUIRE(d->levels == 4 && d->q_dim == 7 + d->emb_dim + d->meas_dim + d->flat_dim, "tt_look_rebatch", "bad layout");
  TT_REQUIRE(rows_ld >= d->q_dim + d->levels * d->C, "tt_look_rebatch", "rows_ld too small");
  look_rebatch_kernel<<<d->B * d->num_cams * d->max_len_cap, 256, 0, (cudaStream_t)stream>>>(
      *d, wp, ctrl_sp, temporal_emb, static_emb, meas, flat, mlvl[0], mlvl[1], mlvl[2], mlvl[3], ref_cam, order, counts, rows,
      rows_ld, ref_rebatch);
  TT_LAUNCHED("tt_look_rebatch");
  return TT_OK;
}

int tt_msda_forward(const tt_msda_desc* d, const float* value, const float* off, const float* logits, const float* ref,
                    const int* max_len, float* out, tt_stream_t stream) {
  TT_REQUIRE(d && value && off && logits && ref && out, "tt_msda_forward", "null argument");
  TT_REQUIRE(d->dh == 32 && d->levels * d->points <= 32 && d->levels <= 4, "tt_msda_forward", "needs dh == 32, <= 32 samples");
  const long long warps = (long long)d->BN * d->rows_cap * d->heads;
  if (warps == 0) return TT_OK;
  msda_kernel<kBatchMaxLen><<<tt_cdiv(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(*d, value, off, logits, ref, max_len, 1, out);
  TT_LAUNCHED("tt_msda_forward");
  return TT_OK;
}

int tt_msda_forward_frames(const tt_msda_desc* d, const float* value, const float* off, const float* logits, const float* ref,
                           const int* counts, int cams, float* out, tt_stream_t stream) {
  TT_REQUIRE(d && value && off && logits && ref && counts && out, "tt_msda_forward_frames", "null argument");
  TT_REQUIRE(d->dh == 32 && d->levels * d->points <= 32 && d->levels <= 4, "tt_msda_forward_frames", "needs dh == 32, <= 32 samples");
  TT_REQUIRE(cams > 0 && d->BN % cams == 0, "tt_msda_forward_frames", "BN must be a multiple of cams > 0");
  const long long warps = (long long)d->BN * d->rows_cap * d->heads;
  if (warps == 0) return TT_OK;
  msda_kernel<kFrameMaxLen><<<tt_cdiv(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(*d, value, off, logits, ref, counts, cams, out);
  TT_LAUNCHED("tt_msda_forward_frames");
  return TT_OK;
}

int tt_look_reduce(const float* rows, int B, int cams, int cap, int C, const int* max_len, float* out, tt_stream_t stream) {
  TT_REQUIRE(rows && max_len && out, "tt_look_reduce", "null argument");
  look_reduce_kernel<kBatchMaxLen><<<tt_cdiv((long long)B * cams * C, 256), 256, 0, (cudaStream_t)stream>>>(rows, B, cams, cap, C,
                                                                                                            max_len, out);
  TT_LAUNCHED("tt_look_reduce");
  return TT_OK;
}

int tt_look_reduce_frames(const float* rows, int B, int cams, int cap, int C, const int* counts, float* out, tt_stream_t stream) {
  TT_REQUIRE(rows && counts && out, "tt_look_reduce_frames", "null argument");
  TT_REQUIRE(B >= 0 && cams > 0 && cap > 0 && C > 0, "tt_look_reduce_frames", "bad sizes");
  if (B == 0) return TT_OK;
  look_reduce_kernel<kFrameMaxLen><<<tt_cdiv((long long)B * cams * C, 256), 256, 0, (cudaStream_t)stream>>>(rows, B, cams, cap, C,
                                                                                                            counts, out);
  TT_LAUNCHED("tt_look_reduce_frames");
  return TT_OK;
}

}  // extern "C"
