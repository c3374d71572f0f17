// Training-side native ops (SURVEY.md §8f row f4): what open_loop_training/train.py needs from the op library besides the forward.
//   * voxel pooling backward — the gather of open_loop_training/ops/voxel_pooling/voxel_pooling.py:57-69 as a kernel;
//   * multi-scale deformable attention forward / backward with the argument contract of mmcv's
//     ext_module.ms_deform_attn_forward / ms_deform_attn_backward, which the reference calls at
//     code/model_code/dense_heads/multi_scale_deformable_attn_function.py:64-70, 95-106 (fp16 class) and :141-147, 172-183 (fp32 class).
// Both are gather / scatter kernels on the HBM roof: one warp per (batch, query, head), lane = channel, so every corner read and every
// grad_value reduction is one 128-byte line; the per-sample scalars (grad of a sampling location / attention weight) are warp-shuffle
// reductions written without atomics.
#include "common.cuh"

extern long long g_tt_launches;

namespace {

// grad_in[b][p][:] = grad_out[memo_b][:][memo_y][memo_x] for kept points, 0 otherwise (voxel_pooling.py:60-66).
// grad_out is addressed through element strides (the autograd engine hands over (B, C, Y, X) views of either memory order).
__global__ void voxel_pool_bwd_kernel(const float* __restrict__ grad_out, long long sb, long long sc, long long sy, long long sx,
                                      const int* __restrict__ pos_memo, float* __restrict__ grad_in, long long total, int C) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long bp = i / C;
    const int mb = __ldg(pos_memo + bp * 3), my = __ldg(pos_memo + bp * 3 + 1), mx = __ldg(pos_memo + bp * 3 + 2);
    grad_in[i] = mb != -1 ? __ldg(grad_out + mb * sb + c * sc + my * sy + mx * sx) : 0.f;
  }
}
// C % 4 == 0: one thread = 4 channels of a point — the memo is read once per 16 bytes written, the store is one 128-bit transaction
// (the op is a pure write stream: B * P * C floats out, the (B, C, Y, X) gradient it gathers from is cache resident)
__global__ void voxel_pool_bwd4_kernel(const float* __restrict__ grad_out, long long sb, long long sc, long long sy, long long sx,
                                       const int* __restrict__ pos_memo, float4* __restrict__ grad_in, long long total4, int C4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const long long bp = i / C4;
    const int mb = __ldg(pos_memo + bp * 3), my = __ldg(pos_memo + bp * 3 + 1), mx = __ldg(pos_memo + bp * 3 + 2);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (mb != -1) {
      const float* g = grad_out + mb * sb + c * sc + my * sy + mx * sx;
      if (sc == 1) v = __ldg(reinterpret_cast<const float4*>(g));     // channels-last gradient (16-byte aligned: checked by the host)
      else v = make_float4(__ldg(g), __ldg(g + sc), __ldg(g + 2 * sc), __ldg(g + 3 * sc));
    }
    grad_in[i] = v;
  }
}

struct Tap {
  bool in;            // the sampling point touches the map at all (ms_deform_attn: h_im > -1 && w_im > -1 && h_im < H && w_im < W)
  int y0, x0, H, W;
  float lh, lw;
};

TT_DEVICE Tap make_tap(float lx, float ly, int H, int W) {
  Tap t;
  const float w_im = lx * W - 0.5f, h_im = ly * H - 0.5f;      // grid_sample(align_corners=False) pixel coordinates
  t.in = h_im > -1.f && w_im > -1.f && h_im < (float)H && w_im < (float)W;
  t.H = H; t.W = W;
  const float fy = floorf(h_im), fx = floorf(w_im);
  t.y0 = (int)fy; t.x0 = (int)fx;
  t.lh = h_im - fy; t.lw = w_im - fx;
  return t;
}

// out[b][q][h*dh + c] = sum_{l,p} attn * bilinear(value_l, loc)      (mmcv ms_deform_attn_forward)
__global__ void __launch_bounds__(256) msda_fwd_kernel(const tt_msda_desc d, const float* __restrict__ value, const float* __restrict__ loc,
                                                       const float* __restrict__ attn, float* __restrict__ out) {
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  const long long n_warps = (long long)d.BN * d.rows_cap * d.heads;
  if (wid >= n_warps) return;
  const int head = (int)(wid % d.heads);
  const long long bq = wid / d.heads;
  const int b = (int)(bq / d.rows_cap);
  const int S = d.levels * d.points, E = d.heads * d.dh;
  const int VL = d.value_ld ? d.value_ld : E;
  const float* vb = value + (long long)b * d.num_keys * VL + d.value_coff + head * d.dh;
  const float* lp = loc + (bq * d.heads + head) * (long long)S * 2;
  const float* ap = attn + (bq * d.heads + head) * (long long)S;
  for (int c = lane; c < d.dh; c += 32) {
    float acc = 0.f;
    for (int s = 0; s < S; ++s) {
      const int l = s / d.points;
      const Tap t = make_tap(__ldg(lp + 2 * s), __ldg(lp + 2 * s + 1), d.lvl_h[l], d.lvl_w[l]);
      if (!t.in) continue;
      const float* v = vb + (long long)d.lvl_start[l] * VL + c;
      const float hh = 1.f - t.lh, hw = 1.f - t.lw;
      float sv = 0.f;
      if (t.y0 >= 0) {
        if (t.x0 >= 0) sv += hh * hw * __ldg(v + ((long long)t.y0 * t.W + t.x0) * VL);
        if (t.x0 + 1 < t.W) sv += hh * t.lw * __ldg(v + ((long long)t.y0 * t.W + t.x0 + 1) * VL);
      }
      if (t.y0 + 1 < t.H) {
        if (t.x0 >= 0) sv += t.lh * hw * __ldg(v + ((long long)(t.y0 + 1) * t.W + t.x0) * VL);
        if (t.x0 + 1 < t.W) sv += t.lh * t.lw * __ldg(v + ((long long)(t.y0 + 1) * t.W + t.x0 + 1) * VL);
      }
      acc = fmaf(__ldg(ap + s), sv, acc);
    }
    out[bq * E + head * d.dh + c] = acc;
  }
}

// mmcv ms_deform_attn_backward: grad_value accumulates (red.add, 128-byte lines), grad_loc / grad_attn are owned by this warp.
__global__ void __launch_bounds__(256) msda_bwd_kernel(const tt_msda_desc d, const float* __restrict__ value, const float* __restrict__ loc,
                                                       const float* __restrict__ attn, const float* __restrict__ grad_out,
                                                       float* __restrict__ grad_value, float* __restrict__ grad_loc,
                                                       float* __restrict__ grad_attn) {
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  const long long n_warps = (long long)d.BN * d.rows_cap * d.heads;
  if (wid >= n_warps) return;
  const int head = (int)(wid % d.heads);
  const long long bq = wid / d.heads;
  const int b = (int)(bq / d.rows_cap);
  const int S = d.levels * d.points, E = d.heads * d.dh;
  const int VL = d.value_ld ? d.value_ld : E;
  const float* vb = value + (long long)b * d.num_keys * VL + d.value_coff + head * d.dh;
  float* gvb = grad_value + (long long)b * d.num_keys * E + head * d.dh;
  const long long sbase = (bq * d.heads + head) * (long long)S;
  const float* go = grad_out + bq * E + head * d.dh;
  for (int s = 0; s < S; ++s) {
    const int l = s / d.points;
    const Tap t = make_tap(__ldg(loc + (sbase + s) * 2), __ldg(loc + (sbase + s) * 2 + 1), d.lvl_h[l], d.lvl_w[l]);
    const float a = __ldg(attn + sbase + s);
    float g_a = 0.f, g_x = 0.f, g_y = 0.f;
    if (t.in) {
      const float hh = 1.f - t.lh, hw = 1.f - t.lw;
      const bool top = t.y0 >= 0, bot = t.y0 + 1 < t.H, lft = t.x0 >= 0, rgt = t.x0 + 1 < t.W;
      const long long k00 = (long long)d.lvl_start[l] + (long long)t.y0 * t.W + t.x0;
      for (int c = lane; c < d.dh; c += 32) {
        const float g = __ldg(go + c);
        const float v1 = top && lft ? __ldg(vb + k00 * VL + c) : 0.f;
        const float v2 = top && rgt ? __ldg(vb + (k00 + 1) * VL + c) : 0.f;
        const float v3 = bot && lft ? __ldg(vb + (k00 + t.W) * VL + c) : 0.f;
        const float v4 = bot && rgt ? __ldg(vb + (k00 + t.W + 1) * VL + c) : 0.f;
        const float ga = g * a;
        if (top && lft) atomicAdd(gvb + k00 * E + c, hh * hw * ga);
        if (top && rgt) atomicAdd(gvb + (k00 + 1) * E + c, hh * t.lw * ga);
        if (bot && lft) atomicAdd(gvb + (k00 + t.W) * E + c, t.lh * hw * ga);
        if (bot && rgt) atomicAdd(gvb + (k00 + t.W + 1) * E + c, t.lh * t.lw * ga);
        g_a += g * (hh * hw * v1 + hh * t.lw * v2 + t.lh * hw * v3 + t.lh * t.lw * v4);
        g_x += ga * (hh * (v2 - v1) + t.lh * (v4 - v3));        // d bilinear / d w_im
        g_y += ga * (hw * (v3 - v1) + t.lw * (v4 - v2));        // d bilinear / d h_im
      }
    }
    g_a = warp_sum(g_a); g_x = warp_sum(g_x); g_y = warp_sum(g_y);
    if (lane == 0) {
      grad_attn[sbase + s] = g_a;
      grad_loc[(sbase + s) * 2] = g_x * (float)t.W;             // w_im = loc_x * W - 0.5
      grad_loc[(sbase + s) * 2 + 1] = g_y * (float)t.H;
    }
  }
}

}  // namespace

extern "C" {

int tt_voxel_pooling_backward(int batch_size, int num_points, int num_channels, const float* grad_output, long long stride_b,
                              long long stride_c, long long stride_y, long long stride_x, const int* pos_memo, float* grad_input,
                              tt_stream_t stream) {
  TT_REQUIRE(grad_output && pos_memo && grad_input && batch_size >= 0 && num_points >= 0 && num_channels > 0, "tt_voxel_pooling_backward",
             "bad arguments");
  const long long total = (long long)batch_size * num_points * num_channels;
  if (total == 0) return TT_OK;
  const bool vec4 = num_channels % 4 == 0 && (reinterpret_cast<uintptr_t>(grad_input) & 15) == 0 &&
                    (stride_c != 1 || ((reinterpret_cast<uintptr_t>(grad_output) & 15) == 0 && ((stride_b | stride_y | stride_x) & 3) == 0));
  if (vec4) {
    const long long total4 = total / 4, want4 = (total4 + 255) / 256;
    voxel_pool_bwd4_kernel<<<(int)(want4 > tt_num_sms() * 32 ? tt_num_sms() * 32 : want4), 256, 0, (cudaStream_t)stream>>>(
        grad_output, stride_b, stride_c, stride_y, stride_x, pos_memo, reinterpret_cast<float4*>(grad_input), total4, num_channels / 4);
  } else {
    const long long want = (total + 255) / 256;
    voxel_pool_bwd_kernel<<<(int)(want > tt_num_sms() * 32 ? tt_num_sms() * 32 : want), 256, 0, (cudaStream_t)stream>>>(grad_output, stride_b, stride_c, stride_y, stride_x,
                                                                                                      pos_memo, grad_input, total, num_channels);
  }
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_voxel_pooling_backward");
  return TT_OK;
}

static int msda_generic_check(const tt_msda_desc* d, const char* name) {
  TT_REQUIRE(d->BN >= 0 && d->rows_cap >= 0 && d->heads > 0 && d->dh > 0 && d->levels >= 1 && d->levels <= 4 && d->points >= 1, name,
             "needs 1..4 levels");
  long long keys = 0;
  for (int l = 0; l < d->levels; ++l) {
    TT_REQUIRE(d->lvl_h[l] > 0 && d->lvl_w[l] > 0 && d->lvl_start[l] == keys, name, "level_start_index must be the running sum of h * w");
    keys += (long long)d->lvl_h[l] * d->lvl_w[l];
  }
  TT_REQUIRE(keys == d->num_keys, name, "num_keys != sum of the level sizes");
  return TT_OK;
}

int tt_ms_deform_attn_forward(const tt_msda_desc* d, const float* value, const float* sampling_loc, const float* attn_weight, float* output,
                              tt_stream_t stream) {
  TT_REQUIRE(d && value && sampling_loc && attn_weight && output, "tt_ms_deform_attn_forward", "null argument");
  if (int rc = msda_generic_check(d, "tt_ms_deform_attn_forward")) return rc;
  const long long warps = (long long)d->BN * d->rows_cap * d->heads;
  if (warps == 0) return TT_OK;
  msda_fwd_kernel<<<tt_cdiv(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(*d, value, sampling_loc, attn_weight, output);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_ms_deform_attn_forward");
  return TT_OK;
}

int tt_ms_deform_attn_backward(const tt_msda_desc* d, const float* value, const float* sampling_loc, const float* attn_weight,
                               const float* grad_output, float* grad_value, float* grad_sampling_loc, float* grad_attn_weight,
                               tt_stream_t stream) {
  TT_REQUIRE(d && value && sampling_loc && attn_weight && grad_output && grad_value && grad_sampling_loc && grad_attn_weight,
             "tt_ms_deform_attn_backward", "null argument");
  if (int rc = msda_generic_check(d, "tt_ms_deform_attn_backward")) return rc;
  const long long warps = (long long)d->BN * d->rows_cap * d->heads;
  if (warps == 0) return TT_OK;
  msda_bwd_kernel<<<tt_cdiv(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(*d, value, sampling_loc, attn_weight, grad_output, grad_value,
                                                                              grad_sampling_loc, grad_attn_weight);
  ++g_tt_launches;
  TT_CHECK_LAUNCH("tt_ms_deform_attn_backward");
  return TT_OK;
}

}  // extern "C"
