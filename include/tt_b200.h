/*
 * tt_b200.h — C ABI of libtt_b200.so: the H100-native (sm_90a) operator library for the
 * ThinkTwice per-frame forward path.  It replaces `open_loop_training/ops` of the reference
 * (OpenDriveLab/ThinkTwice) and the third-party native ops the path crosses (mmcv._ext
 * ms_deform_attn / deform_conv / hard_voxelize, spconv, cuDNN/cuBLAS through torch.nn), and the training-side
 * gradients of the native ops, losses and dense convolutions on the reference's training step (sections 9, 10b and 12 to 16).
 *
 * Conventions (SURVEY.md §8b "External native ABIs"):
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless it says "host";
 *   - activations are fp32 channels-last: a feature map is [N][H][W][ld] floats, the logical
 *     channels of a tensor live at [coff, coff + C) inside the pixel's `ld` floats, so a concat
 *     is just several producers writing into one buffer;
 *   - every call is asynchronous on `stream` (a cudaStream_t), takes no locks, keeps no global
 *     state except the last-error string, and NEVER calls exit(): 0 = ok, negative = tt_status;
 *   - the caller owns and allocates all buffers.
 *
 * Each entry cites the reference interface it replaces (paths relative to
 * /root/reference/open_loop_training).
 */
#ifndef TT_B200_H_
#define TT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* tt_stream_t; /* cudaStream_t */

typedef enum { TT_OK = 0, TT_ERR_INVALID = -1, TT_ERR_CUDA = -2, TT_ERR_UNSUPPORTED = -3 } tt_status;
enum { TT_ACT_NONE = 0, TT_ACT_RELU = 1, TT_ACT_GELU = 2, TT_ACT_SIGMOID = 3, TT_ACT_SOFTPLUS = 4,
       TT_ACT_SOFTPLUS_CLAMP = 5 /* clamp(softplus(x), min=1e-3): thinktwice_decoder.py:484 */ };
enum { TT_RES_NONE = 0, TT_RES_SAME = 1, TT_RES_UP2_NEAREST = 2 };

int tt_version(void);
const char* tt_last_error(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
long long tt_launch_count(void);
/* diagnosis knobs for kernel micro-benchmarks (tools/conv_bench.py); 0 in normal operation.  128: no split-K in the tensor-core
 * convs; bits 8..15: SMs the persistent tensor-core kernels leave free; 0x20000 / 0x40000: register accumulator folded every 4 / 1
 * stages instead of 2 (in the output-stationary sparse conv: every 4 / 1 executed stages, the taps a tile skips not counted);
 * 0x200000: one tap per K slab in the output-stationary sparse conv; 0x400000: 64-column tiles for every dense f16s conv and every
 * output-stationary sparse conv (no 128-column tiles).  Unknown bits: TT_ERR_INVALID, nothing set. */
int tt_debug_set(int flags);

/* ------------------------------------------------------------------------------------------
 * (1) voxel pooling — drop-in for the reference's only in-tree native op.
 * Replaces: ops/voxel_pooling/src/voxel_pooling_forward.cpp:21-22 and
 *           src/voxel_pooling_forward_cuda.cu:38-42 `voxel_pooling_forward_kernel_launcher`.
 * Same argument list and ownership rules (caller zero-fills output_features [B][Y][X][C] and
 * fills pos_memo [B][P][3] with -1; the op accumulates in place) but returns a status instead
 * of exiting.  geom_xyz int32 [B][P][3] (x, y, z); input_features fp32 [B][P][C].
 * Like the reference it accumulates with fp32 atomics (sum order unspecified), but with coalesced
 * 128-bit feature loads and one 128-bit vector reduction per 4 channels.  The model itself uses
 * tt_lift_splat below, which has no floating-point atomics.
 * `workspace` must hold tt_voxel_pooling_workspace_bytes(...) bytes (may be NULL when that is 0).
 */
size_t tt_voxel_pooling_workspace_bytes(int batch_size, int num_points, int num_voxel_x, int num_voxel_y);
int tt_voxel_pooling_forward(int batch_size, int num_points, int num_channels, int num_voxel_x, int num_voxel_y,
                             int num_voxel_z, const int* geom_xyz, const float* input_features,
                             float* output_features, int* pos_memo, void* workspace, tt_stream_t stream);

/* Fused lift-splat: lss.py:582-632 (depth softmax, outer product with the context features,
 * frustum geometry, voxel index, scatter-add) without the (B,N,D,H,W,C) intermediate.
 *   depth_logits : [BN][fH][fW][ld_d] channels-last, D logits at [d_coff, d_coff + D)
 *   context      : [BN][fH][fW][ld_c] channels-last, C features at [c_coff, c_coff + C)
 *   mats         : [BN][2][16] fp32 row-major 4x4: ida^-1 and sensor2ego*intrin^-1 (lss.py:496,502)
 *   frustum_u [fW], frustum_v [fH], frustum_d [D]: the image-plane / depth coordinates of the
 *                  reference's `frustum` buffer (lss.py:454-471), passed in so both sides use the same floats
 *   bev          : [B][Y][X][bev_ld] (+bev_coff), OVERWRITTEN (not accumulated); if `anti_transpose`
 *                  the rot90(flip) of encoder_decoder_framework.py:241 is folded into the store.
 * voxel index = trunc((p - lower) / size) exactly as lss.py:630-631 (`.int()` truncates toward 0).
 */
typedef struct {
  int B, N, D, fH, fW, C;
  int ld_d, d_coff, ld_c, c_coff;
  float lower[3], size[3];       /* lower = (voxel_coord - voxel_size/2) as computed in fp32 by lss.py:630 */
  int X, Y, Z;
  int bev_ld, bev_coff;
  int anti_transpose;
} tt_lift_splat_desc;
size_t tt_lift_splat_workspace_bytes(const tt_lift_splat_desc* d);
int tt_lift_splat(const tt_lift_splat_desc* d, const float* depth_logits, const float* context, const float* mats,
                  const float* frustum_u, const float* frustum_v, const float* frustum_d, float* bev, void* workspace,
                  tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (2) implicit-GEMM convolution / linear layer.
 * Replaces every torch.nn.Conv2d / ConvTranspose2d(k2s2) / Linear on the path (cuDNN/cuBLAS via
 * torch, SURVEY §2.2 N6) and, with `gather`, spconv SubMConv3d / SparseConv3d (N5).
 *   y[pix(m)][y_coff + n] = act( sum_k A[m][k] * w[k][n] + bias[n] + res[...] + res2[...] )
 *   A[m][k], k = tap * Cin_g + c : the input pixel of output row m under tap (kh, kw), channel
 *   g*Cin_g + c, zero outside the image; or, when gather != NULL, row gather[m*taps + tap] of x
 *   (-1 = zero row) — the sparse-conv rulebook.
 *   w: impl 0/1: packed [taps * Cin_g][Cout] fp32 (BatchNorm already folded in); impl 2/3 (tensor cores): packed
 *      [2][Cout][taps][Cin] = `hi = RN_tf32(w)` plane followed by the `lo = RN_tf32(w - hi)` plane.  bias [Cout] or NULL.
 * Output row m = (n, oh, ow) is stored at pixel (n, oh*oy_mul + oy_add, ow*ox_mul + ox_add) of a
 * [N][yH][yW][y_ld] buffer (a k2s2 transposed conv is four such calls).
 * If m_count != NULL only the first *m_count rows (a device int) are computed.
 * `impl`: 0/1 = SIMT fp32 FFMA (exact), 2 = tensor-core single-pass TF32 (operands rounded to nearest TF32),
 *         3 = tensor-core 3xTF32 (hi*hi + hi*lo + lo*hi, fp32-class); 4 = scaled-split fp16 through tt_conv2d_f16s.  impl 2/3 need stride 1 or 2, groups 1, channels,
 *         x_ld, x_coff, y_ld, y_coff, res_coff, res2_coff and the strides % 4 == 0, 16-byte aligned x / w / y / bias / res / res2 (TMA reads the activations in place and splits them in
 *         shared memory; no workspace); else TT_ERR_UNSUPPORTED.
 *         For impl 0/1 the workspace is optional: when given (size from tt_conv2d_workspace_bytes) small-M / large-K
 *         layers run split-K with a deterministic fixed-order reduction.
 */
typedef struct {
  int N, H, W, Cin, x_ld, x_coff;
  long long x_nstride, y_nstride;  /* floats between consecutive images; 0 = dense (H*W*x_ld, yH*yW*y_ld) */
  long long x_hstride;             /* floats between consecutive input rows; 0 = dense (W*x_ld).  With x_ld < Cin the
                                    * "channels" of a pixel run on into the next pixels of the row: a KW-wide tap row
                                    * of a thin-channel conv becomes ONE K slab (row-packed stem conv, see lss.py) */
  int Cout, KH, KW, stride, pad, dil, groups;
  int OH, OW;
  int y_ld, y_coff, yH, yW, oy_mul, oy_add, ox_mul, ox_add;
  int act;
  int bias_n_mod;                 /* 0: bias[Cout]; k > 0: per-image bias table, row (n % k) of bias[k][Cout] */
  int res_mode, res_ld, res_coff; /* res: same pixel grid as the output rows (SAME) or coarser (UP2_NEAREST) */
  int res_H, res_W;               /* UP2_NEAREST: residual map size; source pixel = floor(o * res / O) */
  int res2_ld, res2_coff;         /* optional second SAME residual */
  int taps;                       /* gather mode: taps per row (KH=KW=1 then); else ignored */
  int M;                          /* gather mode: row capacity; else ignored (N*OH*OW) */
  int impl;
} tt_conv_desc;
size_t tt_conv2d_workspace_bytes(const tt_conv_desc* d);
int tt_conv2d(const tt_conv_desc* d, const float* x, const float* w, const float* bias, const float* res,
              const float* res2, const int* gather, const int* m_count, float* y, void* workspace, tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (2b) the same contraction on SCALED-SPLIT FP16 operands (impl 4, csrc/gemm_conv_f16s.cu) — the default tensor-core
 * engine.  Replaces the same reference calls as (2): every torch.nn.Conv2d / ConvTranspose2d / Linear on the path
 * (lss.py, encoder_decoder_framework.py:81-138, thinktwice_decoder.py) and spconv's convolutions (lidarnet.py:42-52).
 * A "split" tensor is two __half planes over the SAME [N][H][W][ld] element grid as its fp32 twin:
 *   hi = RN_f16(x),  lo' = RN_f16((x - hi) * 2048)   =>   x = hi + lo' / 2048 to 2^-22 relative (|x| < 65504).
 * `x_split` / `y_split` point at the hi plane (already advanced to the tensor's channel offset); the lo' plane lies
 * `*_plane` halves further.  Split activations are written by the producing kernel's epilogue (`y_split` here), so a
 * consumer's TMA loads are tensor-core ready; tt_split_f16 converts fp32 rows produced by other kernels.
 *   w_split: [2][Cout][taps][Cin8] halves, Cin8 = Cin rounded up to 8 (zero padded), plane 0 = hi, plane 1 = lo'.
 *   products: hi*hi + (hi*lo' + lo'*hi) / 2048, fp32 accumulation drained into registers every 128 K elements.
 *   y (fp32) and y_split are both optional outputs (at least one) — a tensor only convolutions read needs no fp32 copy;
 *   each residual is given EITHER as fp32 (res / res2) or as split planes (res_split / res2_split, same element offsets).
 * Needs groups 1, stride 1|2, x_ld % 8 == 0 (halves), y_ld % 4 == 0, 16-byte aligned pointers, else TT_ERR_UNSUPPORTED.
 */
typedef struct {
  const void* x_split; long long x_plane;     /* input: hi plane pointer (at the channel offset), halves to the lo' plane */
  const void* w_split;                        /* [2][Cout][taps][Cin8] */
  const float* bias;                          /* fp32 [Cout] (or table, bias_n_mod) or NULL */
  const float* res;  const void* res_split;  long long res_plane;
  const float* res2; const void* res2_split; long long res2_plane;
  float* y; void* y_split; long long y_plane; /* outputs */
} tt_f16s_io;
int tt_conv2d_f16s(const tt_conv_desc* d, const tt_f16s_io* io, tt_stream_t stream);
/* Thin 1x1 stride-1 convolution (Cin <= 64, Cout <= 64, no residual, contiguous pixels) as a per-pixel fp32 mat-vec: one thread per
 * pixel reads its channel row from the split planes `io->x_split`, multiplies with the fp32 K-major weights `w_kmajor` [Cin][Cout] (the
 * tt_conv2d impl 0/1 layout) and writes fp32 rows and / or planes.  For maps so large and channels so few that 128 x 64 tensor-core tiles
 * are all overhead (the segmentation head at 224 x 448). */
int tt_pointwise_f16s(const tt_conv_desc* d, const tt_f16s_io* io, const float* w_kmajor, tt_stream_t stream);
/* fp32 rows [rows][x_ld] (first `cols` columns) -> split planes [2][rows][y_ld]; only the first *row_count rows when given.  Values are
 * clamped to +-65504 first (infinities too); a NaN stays NaN in both planes. */
int tt_split_f16(const float* x, long long x_ld, void* y_split, long long y_plane, long long y_ld, long long rows, int cols,
                 const int* row_count, tt_stream_t stream);
/* NCHW fp32 images (C <= 8) -> zero-bordered channels-last split planes [2][N][out_H][out_W][8 halves] at pixel offset (top, left): the
 * input layout of the row-packed stem convolution on the f16s engine (replaces tt_nchw_to_nhwc_padded + tt_split_f16; the border
 * is never written: zero the buffer once). */
int tt_image_to_split8(const float* x, void* y_split, long long y_plane, int N, int C, int H, int W, int out_H, int out_W, int top,
                       int left, tt_stream_t stream);
/* tt_upsample2x_bilinear_ac (lss.py:267) with the result written as split planes [2][N][2H][2W][C] only */
int tt_upsample2x_bilinear_ac_split(const float* x, void* y_split, long long y_plane, int N, int H, int W, int C, tt_stream_t stream);
/* split planes -> fp32 rows (hi + lo' / 2048): for a non-convolution kernel that must read a tensor stored as planes only */
int tt_merge_f16(const void* x_split, long long x_plane, long long x_ld, float* y, long long y_ld, long long rows, int cols,
                 tt_stream_t stream);
/* epilogue threads that had to clamp a value to +-65504 since the last reset (host int; synchronises `stream`) */
int tt_f16s_saturation_count(unsigned int* out_host, int reset, tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (3) memory-bound helpers (torch elementwise / pooling / interpolation ops, SURVEY N8)
 */
/* NCHW fp32 -> channels-last with `ld` floats per pixel (channels >= C are zero-filled up to cpad) */
/* same, into a larger [N][out_H][out_W][y_ld] buffer at pixel offset (top, left): physical zero padding for
 * row-packed convolutions (the border is never written: zero it once). */
int tt_nchw_to_nhwc_padded(const float* x, float* y, int N, int C, int H, int W, int y_ld, int cpad, int out_H,
                           int out_W, int top, int left, tt_stream_t stream);
int tt_nchw_to_nhwc(const float* x, float* y, int N, int C, int H, int W, int y_ld, int y_coff, int cpad,
                    tt_stream_t stream);
int tt_nhwc_to_nchw(const float* x, int x_ld, int x_coff, float* y, int N, int C, int H, int W, tt_stream_t stream);
/* F.max_pool2d(x, 3, stride 2, padding 1) — mmdet ResNet stem */
int tt_maxpool3x3s2(const float* x, float* y, int N, int H, int W, int C, tt_stream_t stream);
/* nn.Upsample(scale_factor=2, bilinear, align_corners=True) — lss.py:267 */
int tt_upsample2x_bilinear_ac(const float* x, float* y, int N, int H, int W, int C, tt_stream_t stream);
/* mean over H*W -> [N][C] — lss.py:80 AdaptiveAvgPool2d */
int tt_global_avgpool(const float* x, int x_ld, int x_coff, float* y, int N, int HW, int C, tt_stream_t stream);
/* y[n][p][y_coff + c] = v[n][c] (bilinear resize of a 1x1 map == broadcast, lss.py:100-103) */
int tt_broadcast_rows(const float* v, float* y, int N, int HW, int C, int y_ld, int y_coff, tt_stream_t stream);
/* y = x * sigmoid(g[n][c]) — SELayer, lss.py:158 (g holds conv_expand output, pre-sigmoid) */
int tt_se_gate(const float* x, const float* g, float* y, int N, int HW, int C, tt_stream_t stream);
/* s[n][c] = 0.5*mean_hw + 0.5*max_hw — code/utils.py:90-91 */
int tt_se_pool(const float* x, float* s, int N, int HW, int C, tt_stream_t stream);
/* y = relu(x * sigmoid(g[n][c]) + shortcut) — code/utils.py:96,118-120 */
int tt_se_apply(const float* x, const float* g, const float* shortcut, int sc_ld, int sc_coff, float* y, int y_ld,
                int y_coff, int N, int HW, int C, tt_stream_t stream);
/* out[i][j] = x[H-1-j][W-1-i] per image/channel: rot90(flip(x,[2]),1,[2,3]) — framework:241,246 */
int tt_anti_transpose(const float* x, float* y, int N, int S, int C, tt_stream_t stream);
/* dst[r][c] = src[src_row(r)][c], src_row = (r / rdiv) % rmod; strides in floats */
int tt_copy2d(const float* src, int src_ld, float* dst, int dst_ld, int rows, int cols, int rdiv, int rmod,
              tt_stream_t stream);
/* LayerNorm over the last dim (eps 1e-5), rows x D, output stride y_ld */
int tt_layernorm(const float* x, int x_ld, const float* gamma, const float* beta, float* y, int y_ld, int rows,
                 int D, const int* row_count, tt_stream_t stream);
/* elementwise: op 0: y = a + b; 1: y = (1 - a) * b; 2: y = (1 - a) * b + a * c; 3: y = act(a);
 * 4: y = act(a + log(-expm1(-a))), the inverse of softplus (thinktwice_decoder.py:22-23; a > 0) */
int tt_eltwise(int op, int act, const float* a, int a_ld, const float* b, int b_ld, const float* c, int c_ld, float* y,
               int y_ld, int rows, int cols, tt_stream_t stream);
int tt_fill(float* y, float v, long long n, tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (4) deformable convolution v1 — mmcv DeformConv2dPack (lss.py:189-197), 3x3, pad 1, stride 1,
 * deform_groups 1.  Produces the sampled columns [N*H*W][groups][9][C/groups]; the grouped GEMM is
 * tt_conv2d(KH=KW=1, Cin = 9*C, groups).  `offset`: [N][H][W][off_ld], 18 channels (dy, dx per tap).
 */
int tt_dcn_im2col(const float* x, const float* offset, int off_ld, float* col, int N, int H, int W, int C, int groups,
                  tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (5) LiDAR branch: mmcv hard Voxelization + mmdet3d HardSimpleVFE + spconv rulebooks
 * (lidarnet.py:87-96, cfg thinktwice.py:161-176).
 */
typedef struct {
  int B, P, F;                   /* frames, points per frame, floats per point (5) */
  float lower[3], vsize[3];
  int grid[3];                   /* x, y, z voxel counts (672, 672, 70) */
  int zmax;                      /* voxels with z index >= zmax are dropped (sparse_shape z = 41) */
  int max_points, max_voxels;    /* 10, 160000 (eval) */
  int cap;                       /* capacity of the site arrays */
} tt_voxelize_desc;
size_t tt_voxelize_workspace_bytes(const tt_voxelize_desc* d);
/* feats [cap][F] = mean of the first max_points points (input order) of each voxel; coords [cap][4]
 * (b, z, y, x); *count = number of voxels.  Site order is unspecified (results do not depend on it). */
int tt_voxelize_mean(const tt_voxelize_desc* d, const float* points, float* feats, int* coords, int* count,
                     void* workspace, tt_stream_t stream);

typedef struct {
  int B;
  int in_shape[3], out_shape[3]; /* z, y, x */
  int k[3], s[3], p[3];
  int subm;                      /* 1: output sites = input sites */
  int cap_in, cap_out;
  int table_size;                /* power of two >= 2 * max(cap_in, cap_out) */
} tt_rulebook_desc;
size_t tt_rulebook_workspace_bytes(const tt_rulebook_desc* d);
/* Builds out_coords/out_count (copied from the input for subm) and, whichever is non-NULL:
 *   nbr [cap_out][kvol]                      : input row per (output row, tap) or -1 (output-stationary gather), and/or
 *   pairs_in / pairs_out [kvol][cap_out], pair_count [kvol] : tap-major (input row, output row) lists. */
int tt_sparse_rulebook(const tt_rulebook_desc* d, const int* in_coords, const int* in_count, int* out_coords,
                       int* out_count, int* nbr, int* pairs_in, int* pairs_out, int* pair_count, void* workspace,
                       tt_stream_t stream);
/* Tap-major sparse convolution: out[o] = act(sum_tap w[tap] . in[i] + bias + res[o]) over the rulebook's pairs; one
 * launch walks every (tap, pair tile) and accumulates into the bias-initialised output rows with red.add.f32 (the
 * summation order across taps is not fixed: results repeat to fp32 rounding, not bitwise).
 * impl 0/1: SIMT fp32, w = [kvol][Cin][Cout] fp32 (BatchNorm folded).
 * impl 2/3: tensor-core TF32 / 3xTF32 gather-GEMM, w = [2][Cout][kvol][Cin] hi / lo planes (as tt_conv2d); needs
 *           Cin, Cout >= 32 and % 4 == 0, in_ld / out_ld % 4 == 0, 16-byte aligned pointers, else TT_ERR_UNSUPPORTED.
 * res: optional [cap_out][res_ld] (SparseBasicBlock identity). */
typedef struct {
  int Cin, Cout, kvol;
  int in_ld, out_ld, res_ld;
  int cap_out, pair_cap;         /* pair lists are [kvol][pair_cap] */
  int act;
  int impl;
} tt_sparse_conv_desc;
int tt_sparse_conv(const tt_sparse_conv_desc* d, const float* feats_in, const float* w, const float* bias,
                   const float* res, const int* pairs_in, const int* pairs_out, const int* pair_count,
                   const int* out_count, float* feats_out, tt_stream_t stream);
/* tt_sparse_conv on scaled-split fp16 operands (see 2b): feats_in_split [2][cap_in][in_ld] halves; writes the fp32 rows
 * and, when out_split != NULL, their split planes [2][cap_out][out_ld].  w_split = [2][Cout][kvol][Cin8]. */
int tt_sparse_conv_f16s(const tt_sparse_conv_desc* d, const void* feats_in_split, long long in_plane, const void* w_split,
                        const float* bias, const float* res, const int* pairs_in, const int* pairs_out, const int* pair_count,
                        const int* out_count, float* feats_out, void* out_split, long long out_plane, tt_stream_t stream);
/* Output-stationary sparse convolution on scaled-split fp16 operands: ONE launch, no atomics.  A work item is a tile of 128 output
 * rows; K runs over all kvol taps through the neighbour table `nbr` [cap_out][kvol] (input row under each tap, -1 = none: a zero
 * row), so the sum of an output row is formed on the tensor cores in a fixed order and stored once with bias + residual + activation fused
 * (fp32 rows `io->y` and / or split planes `io->y_split`; residual as fp32 `io->res` or planes `io->res_split`).  Pays for empty
 * (row, tap) slots with zero rows — the better form once a fair share of the taps is populated (dilated / dense-ish clouds);
 * tt_sparse_conv_f16s (tap-major pair lists, red.add) is the form for very sparse neighbourhoods.  io->x_split = input planes
 * [2][cap_in][in_ld]; w_split = [2][Cout][kvol][Cin8]; d->cap_out = row capacity, *out_count = rows that exist. */
int tt_sparse_conv_os_f16s(const tt_sparse_conv_desc* d, const tt_f16s_io* io, const int* nbr, const int* out_count,
                           tt_stream_t stream);
/* dense()[N][C][D][H][W].view(N, C*D, H, W) (lidarnet.py:53-56) written channels-last, channel = c*D + z,
 * with the framework's anti-transpose (framework:246) folded in when asked; `dense` must be zero-filled. */
int tt_sparse_to_bev(const float* feats, const int* coords, const int* count, int cap, int C, int D, int H, int W,
                     int anti_transpose, float* dense, tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (6) Look module (thinktwice_decoder.py:88-187) and multi-scale deformable attention
 * (mmcv._ext.ms_deform_attn_forward, multi_scale_deformable_attn_function.py:72-78, 468-526).
 */
typedef struct {
  int B, num_cams, num_query;    /* 4 cams, 120 look points = (T waypoints + T static points) x 15 z levels */
  int T;                         /* pred_len (4) */
  float img_w, img_h;
  int levels;
  int lvl_h[4], lvl_w[4];
  int C;                         /* 256 channels per FPN level */
  int q_dim;                     /* 4 + 3 + emb_dim + meas_dim + flat_dim = 519 */
  int emb_dim, meas_dim, flat_dim;
  int max_len_cap;               /* rows per (b, cam) in the rebatched buffers (>= num_query) */
} tt_look_desc;
/* thinktwice_decoder.py:155-160 + :88-114,129-137: build the look points from the current waypoints
 * wp [B][T][2], project them into every camera (lidar2img [B][cams][16], clamp depth to 1e-5, ida
 * [B][cams][16], normalise by the image size), validity mask, ordered compaction.
 * Outputs: ref_cam [B][cams][Q][2], order [B][cams][Q] (compacted query ids), counts [B][cams], *max_len. */
int tt_look_project(const tt_look_desc* d, const float* wp, const float* lidar2img, const float* ida, float* ref_cam,
                    int* order, int* counts, int* max_len, tt_stream_t stream);
/* thinktwice_decoder.py:117-127,140-150,161-171: rows [B*cams][cap][rows_ld] = [query | bilinear samples of the 4
 * FPN levels at the ref point (feature index c*levels + l)], zero rows past counts; ref_rebatch [B*cams][cap][2].
 * query = [softplus ctrl 4 | xyz 3 | temporal / static embedding | measurement feat | flattened BEV feat].
 * mlvl: host array of 4 device pointers, each [B*cams][h][w][C] channels-last. */
int tt_look_rebatch(const tt_look_desc* d, const float* wp, const float* ctrl_sp, const float* temporal_emb,
                    const float* static_emb, const float* meas, const float* flat, const float* const* mlvl,
                    const float* ref_cam, const int* order, const int* counts, float* rows, int rows_ld,
                    float* ref_rebatch, tt_stream_t stream);
typedef struct {
  int BN, rows_cap, heads, levels, points, dh; /* 8 heads, 4 levels, 8 points, 32 */
  int lvl_h[4], lvl_w[4], lvl_start[4];
  int num_keys;
  int value_ld, value_coff;      /* floats per key row of `value` (0 = heads*dh) and first channel: several layers' value projections
                                  * computed by ONE convolution share a buffer */
} tt_msda_desc;
/* value [BN][num_keys][value_ld] (channels value_coff .. value_coff + heads*dh); off [BN*cap][heads*levels*points*2]; logits [BN*cap][heads*levels*points];
 * ref [BN*cap][2]; out [BN*cap][heads*dh].  Softmax over levels*points is fused. */
int tt_msda_forward(const tt_msda_desc* d, const float* value, const float* off, const float* logits, const float* ref,
                    const int* max_len, float* out, tt_stream_t stream);
/* msda:338-342: zero the first B rows of every (b, cam), divide by B, sum rows < max_len -> [B][cams*C] */
int tt_look_reduce(const float* rows, int B, int cams, int cap, int C, const int* max_len, float* out,
                   tt_stream_t stream);
/* Independent frames: every frame of the batch computed as the reference computes it alone, at B = 1 (the closed-loop agent's
 * batch, leaderboard/team_code/thinktwice_agent.py:446-454).  The reference's row bound is the max_len of thinktwice_decoder.py:137,
 * a maximum over every (frame, camera) of the call; here each frame b has its own
 *   max_len_b = max over cams of counts[b][cam]   (counts [B][cams] as tt_look_project writes them; device memory, no host sync).
 * tt_msda_forward_frames: tt_msda_forward computing only rows r < max_len_b of the images bn = b * cams + cam (d->BN = B * cams);
 * the other rows of `out` are not written.  Never more rows than tt_msda_forward with the batch-wide max_len. */
int tt_msda_forward_frames(const tt_msda_desc* d, const float* value, const float* off, const float* logits, const float* ref,
                           const int* counts, int cams, float* out, tt_stream_t stream);
/* msda:338-342 at B = 1 per frame: out[b][cam*C + c] = sum over 1 <= r < min(max_len_b, cap) of rows[b][cam][r][c] (row 0 zeroed,
 * divisor 1).  Rows in [counts[b][cam], max_len_b) are the zero-query rows tt_look_rebatch wrote; they count, as in the reference. */
int tt_look_reduce_frames(const float* rows, int B, int cams, int cap, int C, const int* counts, float* out,
                          tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (7) decoder glue
 */
/* GRU input plane (dense_heads/utils.py:93-104): buf[b][p][0:6] = (wp_t, softplus ctrl_t) of step t */
int tt_gru_input(const float* wp, const float* ctrl_sp, int t, int T, float* buf, int ld, int B, int HW,
                 tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (8) agent-side pre-processing (SURVEY.md 8f row f1): the CPU work between the CARLA sensors and forward_inference.
 */
typedef struct {
  int n_img;            /* images in `raw` (T * N per tick, or B * T * N) */
  int H, W;             /* raw camera frame (900 x 1600: thinktwice_agent.py:237) */
  int newH, newW;       /* resize_dims of sample_ida_augmentation (transform.py:264-267): int(H * resize), int(W * resize) */
  int outH, outW;       /* final_dim = the crop window's size (448 x 896) */
  int crop_x, crop_y;   /* crop[:2] (transform.py:268-271) */
  int undistort;        /* cfg["undistort"]: sample the raw frame through map_grid first (transform.py:281-282) */
  float div;            /* 255 (transform.py:162) */
  float mean[3], std[3];/* T.Normalize constants (transform.py:144) */
  int pad_H, pad_W, pad_top, pad_left; /* geometry of the stem-plane output (see tt_image_to_split8); ignored without out_split8 */
} tt_preproc_desc;
/* Replaces IDAImageTransform.__call__ + img_transform + ImageTransformMulti(aug=False) for the test-time branch
 * (code/datasets/pipelines/transform.py:275-341, 346-378, 149-163): raw uint8 [n_img][H][W][3] (RGB, as the agent holds it:
 * thinktwice_agent.py:297-300) -> grid_sample(map_grid, bilinear, zeros, align_corners=False) -> T.Resize((newH, newW)) [bilinear,
 * no antialias: torchvision 0.13.1 of docs/INSTALL.md] -> crop -> /div -> (x - mean) / std.
 * map_grid: fp32 [H][W][2] normalised (x, y) exactly as transform.py:237-240 builds it (one map for every image; may be NULL without
 * undistort).  out_nchw: fp32 [n_img][3][outH][outW] (the `img` tensor of the batch dict) and / or out_split8: the row-packed stem's
 * operand planes [2][n_img][pad_H][pad_W][8 halves] (plane stride split_plane halves; border never written).  Either may be NULL.
 * With out_split8, n_img * pad_H * pad_W * 8 > split_plane (the slots would run past a plane) is refused with TT_ERR_INVALID. */
int tt_preprocess_u8(const tt_preproc_desc* d, const uint8_t* raw, const float* map_grid, float* out_nchw, void* out_split8,
                     long long split_plane, tt_stream_t stream);
/* thinktwice_agent.py:340-352: out [n_prev + n_now][4] = [rel_mat (4x4 fp64, row-major, DEVICE) applied to prev's xyz | now], z += z_add (2.5);
 * float64 arithmetic like the numpy original, intensity untouched. */
int tt_lidar_stitch(const float* prev, int n_prev, const float* now, int n_now, const double* rel_mat, double z_add, float* out,
                    tt_stream_t stream);
/* code/datasets/carla_dataset.py:314-328 (union2one): dst [n][5] = [curr2key (4x4 fp32, row-major, DEVICE; NULL = key frame: copy) applied to the
 * (x, y, z, intensity) 4-vector of src [n][4] | timestamp]; the caller places the sweeps back to back (key frame first). */
int tt_points_union(const float* src, int n, const float* curr2key, float timestamp, float* dst, tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (9) training-side ops (SURVEY.md 8f row f4): what open_loop_training/train.py needs from the op library besides the forward.
 */
/* Replaces the indexing backward of ops/voxel_pooling/voxel_pooling.py:57-69: grad_input [B][P][C] (fully written) =
 * grad_output[pos_memo b][:][pos_memo y][pos_memo x] where pos_memo [B][P][3] != -1, else 0.  grad_output is the (B, C, Y, X)
 * tensor autograd hands over, addressed by ELEMENT strides (either memory order, no copy). */
int tt_voxel_pooling_backward(int batch_size, int num_points, int num_channels, const float* grad_output, long long stride_b,
                              long long stride_c, long long stride_y, long long stride_x, const int* pos_memo, float* grad_input,
                              tt_stream_t stream);
/* Replace mmcv's ext_module.ms_deform_attn_forward / ms_deform_attn_backward as the reference calls them
 * (code/model_code/dense_heads/multi_scale_deformable_attn_function.py:141-147, 172-183; im2col_step has no meaning here).
 * d: BN = bs, rows_cap = num_queries, heads, levels (<= 4), points, dh, lvl_h / lvl_w / lvl_start = value_spatial_shapes /
 * value_level_start_index, num_keys; value_ld / value_coff as in tt_msda_forward (0 = dense).
 * value [bs][num_keys][heads][dh]; sampling_loc [bs][q][heads][levels][points][2] (x, y) in [0, 1]; attn_weight [bs][q][heads][levels][points];
 * output / grad_output [bs][q][heads*dh].  Backward: grad_value [bs][num_keys][heads][dh] must be ZERO-filled by the caller (as the
 * reference does: msda:168) and is accumulated with fp32 atomics; grad_sampling_loc / grad_attn_weight are fully written. */
int tt_ms_deform_attn_forward(const tt_msda_desc* d, const float* value, const float* sampling_loc, const float* attn_weight, float* output,
                              tt_stream_t stream);
int tt_ms_deform_attn_backward(const tt_msda_desc* d, const float* value, const float* sampling_loc, const float* attn_weight,
                               const float* grad_output, float* grad_value, float* grad_sampling_loc, float* grad_attn_weight,
                               tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (10) open-loop validation losses (thinktwice_decoder.py:536-620): every term of ThinkTwiceDecoder.loss in ONE launch.
 * A term reduces an element-wise function of (pred, gt) over a logical tensor of up to 6 dims, each operand addressed by ELEMENT
 * strides (0 = broadcast along that dim), so channels-last arena maps are read against NCHW ground truth without a copy.
 */
#define TT_LOSS_MAX_DIM 6
enum {
  TT_LOSS_SMOOTH_L1 = 0,        /* F.smooth_l1_loss, beta 1 */
  TT_LOSS_SMOOTH_L1_CLAMP = 1,  /* clamp(smooth_l1(.), -5, 5) element-wise, then the mean (NaN stays NaN, as torch.clamp) */
  TT_LOSS_L1 = 2,               /* |pred - gt| */
  TT_LOSS_BETA_KL = 3,          /* kl_divergence(Beta(gt, gt2), Beta(pred, pred2)) in fp64; NaN unless all four are finite and > 0 */
  TT_LOSS_ACTION_L1 = 4         /* |_get_action_beta(pred, pred2) - _get_action_beta(gt, gt2)| of component `aux` (framework:623-636) */
};
typedef struct {
  const float* pred;            /* BETA_KL / ACTION_L1: alpha of the prediction */
  const float* pred2;           /* BETA_KL / ACTION_L1: beta of the prediction (strides of pred); otherwise unused */
  const float* gt;              /* NULL: a zero target */
  const float* gt2;             /* BETA_KL / ACTION_L1: beta of the target (strides of gt) */
  long long shape[TT_LOSS_MAX_DIM];
  long long pred_stride[TT_LOSS_MAX_DIM];
  long long gt_stride[TT_LOSS_MAX_DIM];
  int ndim;                     /* 1 .. TT_LOSS_MAX_DIM */
  int kind;                     /* TT_LOSS_* */
  int slot;                     /* output slot: terms sharing a slot are added in term order */
  int aux;                      /* ACTION_L1: the action component (0 throttle / brake, 1 steer) */
  double scale;                 /* weight / element count: the term contributes scale * sum of its elements */
} tt_loss_term;
/* out[s] (fp32) = sum over the terms t with slot s, in term order, of terms[t].scale * (fp64 sum of t's elements).  Each term is
 * split into a fixed number of element ranges, each range reduced in a fixed order by one CTA, and the last CTA to finish adds the
 * range sums in a fixed order: two calls on the same inputs give bitwise equal results.  `terms` is HOST memory (copied into ws
 * on `stream`); ws: tt_loss_workspace_bytes(n_terms) bytes of device memory, not shared with a concurrent call. */
size_t tt_loss_workspace_bytes(int n_terms);
int tt_loss_reduce(const tt_loss_term* terms, int n_terms, float* out, int n_slots, void* ws, size_t ws_bytes, tt_stream_t stream);
/* (10b) the decoder terms' gradient (training side, SURVEY.md 8f row f4).  grads[k] goes with terms[k] (the same table tt_loss_reduce
 * reads).  Term k's upstream gradient is u_k = sum of grad_out[up_slot .. up_slot + up_count) in slot order (fp64), so a (B, 1) loss
 * whose slots all feed one term (value_loss's pred_value_traj mean) needs one term, and a term fed by one frame's slot needs count 1.
 * With d = pred - gt and s(d) = clamp(d, -1, 1) (torch's smooth_l1 backward, beta 1; NaN stays NaN), every element of the term gets
 *   SMOOTH_L1       : grad_pred = u * scale * s(d)
 *   SMOOTH_L1_CLAMP : grad_pred = (-5 <= smooth_l1(d) <= 5 ? u : 0) * scale * s(d)   (torch.clamp's backward passes the bounds)
 *   BETA_KL         : grad_pred  = u * scale * (psi(a2) - psi(a2 + b2) - psi(a1) + psi(a1 + b1)),
 *                     grad_pred2 = u * scale * (psi(b2) - psi(a2 + b2) - psi(b1) + psi(a1 + b1)),  a1, b1 = gt, gt2; a2, b2 = pred, pred2
 * in fp64, rounded once.  A term with grad_pred NULL is skipped; L1 and ACTION_L1 terms (computed under no_grad by the reference) with
 * a gradient pointer are refused.  Refused with TT_ERR_UNSUPPORTED (the reason in tt_last_error) before anything is staged: a gradient
 * view that maps two elements to one address, and two terms (or grad_pred / grad_pred2 of one term) whose gradient address ranges
 * [lowest, highest element] intersect.  So every gradient element is written by exactly one thread, once, without atomics: bitwise
 * reproducible.  Elements no term covers are not written.  `terms` / `grads` are HOST memory (copied into ws on `stream`); grad_out
 * [n_slots] is device memory; ws: tt_loss_backward_workspace_bytes(n_terms) bytes, not shared with a concurrent call. */
typedef struct {
  float* grad_pred;             /* dL/dpred over the term's shape at grad_stride; NULL: no gradient for this term */
  float* grad_pred2;            /* BETA_KL: dL/dpred2 at the same strides (may be NULL); otherwise unused */
  long long grad_stride[TT_LOSS_MAX_DIM];
  int up_slot, up_count;        /* upstream gradient = sum of grad_out[up_slot .. up_slot + up_count) */
} tt_loss_grad;
size_t tt_loss_backward_workspace_bytes(int n_terms);
int tt_loss_backward(const tt_loss_term* terms, int n_terms, const tt_loss_grad* grads, const float* grad_out, int n_slots, void* ws,
                     size_t ws_bytes, tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (11) the camera branch's supervision of the key frame (encoder_decoder_framework.py:171-190, 442-491; utils.py:31-47):
 *   seg_loss   = weight * FocalLoss(alpha, gamma, ignore_index)(seg logits, nearest-resized labels .long()), the focal transform applied
 *                to the MEAN cross entropy over the non-ignored pixels (NaN when every pixel is ignored, as torch);
 *   depth_loss = sum over the foreground cells of BCE-with-logits(depth logits, one-hot bin) / max(1, foreground cells), the bins from
 *                the min over each factor x factor block of the depth map (0 -> 1e5 first, a NaN pixel makes the block NaN).
 * Either half is off when its logits pointer is NULL.  Logits are read in place from channels-last maps (class c of pixel p at
 * logits[p * ld + coff + c]; channels past `classes` / `bins` are never read); the ground truth is the full-resolution fp32 maps.
 */
typedef struct {
  const float* seg_logits;      /* (BN, seg_h, seg_w) pixels of seg_ld floats; NULL: no seg_loss */
  const float* seg_gt;          /* (BN, seg_H, seg_W) labels as floats; pixel (y, x) reads label (src(y), src(x)), ATen's nearest index */
  const float* depth_logits;    /* (BN, depth_h, depth_w) pixels of depth_ld floats; NULL: no depth_loss */
  const float* depth_gt;        /* (BN, depth_h * depth_factor, depth_w * depth_factor) depths */
  int BN;
  int seg_h, seg_w, seg_H, seg_W, seg_ld, seg_coff, seg_classes, seg_ignore;
  float seg_alpha, seg_gamma, seg_weight;
  int depth_h, depth_w, depth_factor, depth_ld, depth_coff, depth_bins;
  float depth_offset;           /* fp32 (d_bound[0] - d_bound[2]): bin value v = (min depth - depth_offset) / depth_step in fp32 */
  float depth_step;             /* fp32 d_bound[2] */
} tt_camera_loss_desc;
/* out[0] = seg_loss, out[1] = depth_loss (fp32; a half that is off leaves its slot untouched).  Per-CTA fp64 sums and integer counts,
 * folded in a fixed order by the last CTA: two calls on the same inputs give bitwise equal results.  A label whose truncation lies
 * outside [0, seg_classes) and is not seg_ignore (torch raises) makes seg_loss NaN.  ws: tt_camera_loss_workspace_bytes(d) bytes of
 * device memory, not shared with a concurrent call. */
size_t tt_camera_loss_workspace_bytes(const tt_camera_loss_desc* d);
int tt_camera_loss(const tt_camera_loss_desc* d, float* out, void* ws, size_t ws_bytes, tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (12) training-side deformable convolution (SURVEY.md 8f row f4): mmcv's DeformConv2d forward / backward
 * (mmcv/ops/deform_conv.py, DeformConv2dFunction; the reference builds it at lss.py:189-197) on mmcv's tensors, all contiguous
 * fp32: input (N, C, H, W), offset (N, 18, H, W) with (dy, dx) interleaved per tap, weight (Cout, C / groups, 3, 3),
 * output / grad_output (N, Cout, H, W).  Sampling as tt_dcn_im2col: zero unless -1 < h < H and -1 < w < W, out-of-image
 * corners zero.  Products in 3xTF32 on the tensor cores, fp32 accumulation.
 * Supported is what the reference builds: 3x3, stride 1, padding 1, dilation 1, deform_groups 1, no bias, C % groups ==
 * Cout % groups == 0, (C / groups) % 4 == (Cout / groups) % 4 == 0; anything else returns TT_ERR_UNSUPPORTED with the
 * parameter named in tt_last_error.  Images are processed in chunks of at most im2col_step (the workspace holds one chunk's
 * columns); output, grad_input and grad_offset do not depend on the chunking.
 * Backward: grad_input / grad_offset / grad_weight are fully written; any of them may be NULL and is then not computed.
 * grad_weight and grad_offset are bitwise reproducible (fixed-order reductions); grad_input is accumulated with fp32 atomics.
 * ws: tt_deform_conv_workspace_bytes(d) bytes of device memory, not shared with a concurrent call.
 */
typedef struct {
  int N, C, H, W, Cout, groups, im2col_step;
  int kernel_h, kernel_w, stride, padding, dilation, deform_groups;
} tt_deform_conv_desc;
size_t tt_deform_conv_workspace_bytes(const tt_deform_conv_desc* d);
int tt_deform_conv_forward(const tt_deform_conv_desc* d, const float* input, const float* offset, const float* weight, float* output,
                           void* ws, size_t ws_bytes, tt_stream_t stream);
int tt_deform_conv_backward(const tt_deform_conv_desc* d, const float* input, const float* offset, const float* weight,
                            const float* grad_output, float* grad_input, float* grad_offset, float* grad_weight, void* ws,
                            size_t ws_bytes, tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (13) training-side sparse convolution (SURVEY.md 8f row f4): spconv 2.x SubMConv3d / SparseConv3d forward and backward, as
 * mmdet3d's SparseEncoder builds them (lidarnet.py:24-58, cfg thinktwice.py:167-176).  Features are fp32 rows (row pitch in_ld /
 * out_ld floats), weight (Cout, kvol, Cin) is spconv 2.x's (Cout, kd, kh, kw, Cin) with tap t the row-major flattening of (kd, kh, kw).
 * For the rulebook's pairs P_t = {(i, o)} of tap t, W_t = weight[:, t, :]:
 *   y[o] = sum_t sum_{(i,o) in P_t} W_t x[i];  grad_x[i] = sum_t sum_{(i,o) in P_t} W_t^T gy[o];  grad_W_t = sum_{(i,o) in P_t} gy[o] x[i]^T.
 * Supported is what the reference builds: SubM 3x3x3 (stride 1, padding 1); strided 3x3x3, stride 2, padding 1 or (0, 1, 1);
 * (3, 1, 1), stride (2, 1, 1), padding 0; dilation 1, groups 1, no bias, not transposed or inverse, kvol <= 32.  Anything else
 * returns TT_ERR_UNSUPPORTED with the parameter named in tt_last_error.
 * Forward and grad_input run on the tap-major gather-GEMM of tt_sparse_conv: 3xTF32 tensor cores when Cin, Cout >= 32 (multiples
 * of 4, pitches multiples of 4, 16-byte aligned rows), fp32 SIMT otherwise; they accumulate over taps with red.add.f32, so they
 * repeat to fp32 rounding, not bitwise.  grad_weight is a per-tap gathered A-transposed contraction (3xTF32 tensor cores when
 * Cin, Cout, in_ld, out_ld are multiples of 4, an fp32 SIMT kernel otherwise) folded in a fixed order: bitwise reproducible when
 * the pair lists are (tt_sparse_pairs_ordered).  The weight is repacked by a kernel in every call (it changes every step).
 * Row counts stay on the device: rows < *out_count (*in_count) of feats_out (grad_in) are written, the others untouched.
 */
typedef struct {
  int Cin, Cout, kvol;
  int cap_in, cap_out;           /* row capacities of feats_in / grad_in and feats_out / grad_out */
  int pair_cap;                  /* pair lists are [kvol][pair_cap]; pair_cap >= the largest tap's pair count */
  int in_ld, out_ld;             /* row pitches (floats) of the input-side and output-side rows */
  int k[3], stride[3], padding[3], dilation[3];   /* z, y, x */
  int subm, groups, bias, transposed, inverse;
} tt_sparse_conv_train_desc;
/* 0 when the descriptor is refused (tt_last_error names why); every supported convolution needs a workspace. */
size_t tt_sparse_conv_train_workspace_bytes(const tt_sparse_conv_train_desc* d);
int tt_sparse_conv_train_forward(const tt_sparse_conv_train_desc* d, const float* feats_in, const float* weight, const int* pairs_in,
                                 const int* pairs_out, const int* pair_count, const int* out_count, float* feats_out, void* ws,
                                 size_t ws_bytes, tt_stream_t stream);
/* grad_in (rows < *in_count) and grad_weight (Cout, kvol, Cin) are fully written; either may be NULL and is then not computed. */
int tt_sparse_conv_train_backward(const tt_sparse_conv_train_desc* d, const float* feats_in, const float* weight, const float* grad_out,
                                  const int* pairs_in, const int* pairs_out, const int* pair_count, const int* in_count,
                                  const int* out_count, float* grad_in, float* grad_weight, void* ws, size_t ws_bytes,
                                  tt_stream_t stream);
/* Pair lists in a fixed order from the neighbour table nbr [cap_out][kvol] of tt_sparse_rulebook (rows >= *out_count are not read):
 * per tap, the pairs in ascending output row, pairs_in / pairs_out [kvol][pair_cap], pair_count [kvol].  pair_cap must be at least
 * the largest tap's count (min(input rows, output rows) always is); ws: tt_sparse_pairs_ordered_workspace_bytes(cap_out, kvol). */
size_t tt_sparse_pairs_ordered_workspace_bytes(int cap_out, int kvol);
int tt_sparse_pairs_ordered(const int* nbr, const int* out_count, int cap_out, int kvol, int pair_cap, int* pairs_in, int* pairs_out,
                            int* pair_count, void* ws, size_t ws_bytes, tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (14) training-side lift-splat (SURVEY.md 8f row f4): lss.py:583-615 (depth softmax, outer product with the context, frustum
 * geometry, voxel pooling) with a gradient, on torch's NCHW fp32 tensors and without the (BN, C, D, fH, fW) frustum tensor.
 * Pixel p of frame b has logits l[p][:], softmax pi[p][:], context f[p][:] and, for bin d, cell(p, d) = y * X + x computed as
 * tt_lift_splat computes it (bda absent), or -1 outside the grid.  G = dL/dbev.
 *   forward : bev[b][cell][:] = sum over (p, d) with cell(p, d) = cell of pi[p][d] f[p][:]          (exactly tt_lift_splat)
 *   backward: g[p][d] = f[p][:] . G[b][:][cell(p, d)] (0 outside the grid);
 *             grad_logits[p][d] = pi[p][d] (g[p][d] - sum_j pi[p][j] g[p][j]);
 *             grad_context[p][:] = sum_d pi[p][d] G[b][:][cell(p, d)].
 *   depth_logits [BN][D][fH][fW] at batch stride depth_bstride floats (so the view depth_feature[:, :D] needs no copy);
 *   context [BN][C][fH][fW] contiguous; mats / frustum_u / frustum_v / frustum_d as tt_lift_splat.
 * Forward: bev [B][Y][X][C] is fully overwritten; when bin_cell != NULL it also gets bin_cell [BN*fH*fW][D], the cell the kernel
 * assigned to every bin or -1: the only state the backward needs besides the inputs.  As tt_lift_splat, the integer-atomic
 * placement orders each cell's sum differently from run to run (repeatable to fp32 rounding, not bitwise).
 * Backward: grad_bev (B, C, Y, X) is addressed by ELEMENT strides (any memory order, a channel slice of a concat); the cells are
 * the recorded bin_cell, never recomputed.  grad_logits [BN][D][fH][fW] and grad_context [BN][C][fH][fW] (contiguous) are fully
 * written; either may be NULL and is then not computed.  Gathers only, in a fixed order: bitwise reproducible.
 * Refused with TT_ERR_UNSUPPORTED, the parameter named in tt_last_error, before any pointer or device is touched: D > 128,
 * C % 4 != 0, C > 512, B*X*Y cells or B*N*fH*fW*D bins past 32-bit indexing, a row tile (C + D) * fW past shared memory, and
 * ws_bytes < tt_lift_splat_train_workspace_bytes(d).  B = 0 launches nothing.
 * ws: tt_lift_splat_train_workspace_bytes(d) bytes of device memory (0 when d is refused), not shared with a concurrent call.
 */
typedef struct {
  int B, N, D, fH, fW, C;
  long long depth_bstride;       /* floats between consecutive images of depth_logits (>= D*fH*fW) */
  float lower[3], size[3];       /* as tt_lift_splat_desc */
  int X, Y, Z;
} tt_lift_splat_train_desc;
size_t tt_lift_splat_train_workspace_bytes(const tt_lift_splat_train_desc* d);
int tt_lift_splat_train_forward(const tt_lift_splat_train_desc* d, const float* depth_logits, const float* context, const float* mats,
                                const float* frustum_u, const float* frustum_v, const float* frustum_d, float* bev, int* bin_cell,
                                void* ws, size_t ws_bytes, tt_stream_t stream);
int tt_lift_splat_train_backward(const tt_lift_splat_train_desc* d, const float* depth_logits, const float* context, const int* bin_cell,
                                 const float* grad_bev, long long stride_b, long long stride_c, long long stride_y, long long stride_x,
                                 float* grad_logits, float* grad_context, void* ws, size_t ws_bytes, tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (15) training-side camera supervision (SURVEY.md 8f row f4): section 11's seg_loss / depth_loss with a gradient, on torch's NCHW fp32
 * logits (encoder_decoder_framework.py:171-190).  Ground truth, quirks and sums are tt_camera_loss's: labels read at ATen's nearest
 * index and truncated by .long(); depth 0 -> 1e5 before the min-pool; a NaN pixel makes its block background; the focal transform of
 * the batch-MEAN cross entropy; fixed-order fp64 sums folded by the last CTA, bitwise reproducible.
 * Logits: class / bin c of pixel (n, y, x) at logits[n * stride[0] + c * stride[1] + y * stride[2] + x * stride[3]]; the h x w plane
 * must be dense (stride[3] = 1, stride[2] = w), so the seg head's output and the view depth_feature[:, :D] pass without a copy.
 * Forward: out[0] = seg_loss, out[1] = depth_loss (a half that is off leaves its slot untouched), and *stats (device memory).  When
 * seg_target / depth_target are non-NULL it also records the target of every logit pixel: seg_target [BN][seg_h][seg_w] = the class,
 * or 255 for an ignored pixel (or a label torch rejects); depth_target [BN][depth_h][depth_w] = the bin 1..depth_bins, or 0 for a
 * background cell.  The backward reads these records and *stats, never the ground truth.
 * Backward: grad_loss = (dL/dseg_loss, dL/ddepth_loss), 2 device floats.  With k0 = grad_loss[0] * stats->seg_factor and
 * k1 = grad_loss[1] / max(1, nfg):
 *   grad_seg  [BN][C][seg_h][seg_w]   = k0 * (softmax_c(p) - [c = label(p)]) on counted pixels, 0 on ignored pixels;
 *   grad_depth[BN][D][depth_h][depth_w] = k1 * (sigmoid(x_pd) - [d = bin(p) - 1]) on foreground cells, 0 on background cells;
 * both contiguous NCHW and fully written; either may be NULL and is then skipped.  Element-wise, no atomics: bitwise reproducible.
 * Refused with TT_ERR_UNSUPPORTED, the parameter named in tt_last_error, before any pointer is touched: seg_classes > 32 (the
 * backward's register tile), depth_bins > 255 (a byte target), a plane that is not dense, pixel / cell / ground-truth counts past
 * 32-bit indexing, and (forward) ws_bytes < tt_camera_loss_train_workspace_bytes(d).  BN = 0 launches nothing and writes nothing.
 */
typedef struct {
  const float* seg_logits;      /* (BN, seg_classes, seg_h, seg_w) at seg_stride; NULL: no seg_loss */
  const float* seg_gt;          /* (BN, seg_H, seg_W) labels as floats, as tt_camera_loss_desc */
  const float* depth_logits;    /* (BN, depth_bins, depth_h, depth_w) at depth_stride; NULL: no depth_loss */
  const float* depth_gt;        /* (BN, depth_h * depth_factor, depth_w * depth_factor) depths */
  long long seg_stride[4];      /* element strides of (n, c, y, x) */
  long long depth_stride[4];
  int BN;
  int seg_h, seg_w, seg_H, seg_W, seg_classes, seg_ignore;
  float seg_alpha, seg_gamma, seg_weight;
  int depth_h, depth_w, depth_factor, depth_bins;
  float depth_offset, depth_step;  /* as tt_camera_loss_desc */
} tt_camera_loss_train_desc;
typedef struct {
  double ce;                    /* mean cross entropy over the counted pixels (NaN: none counted, or a rejected label) */
  double seg_factor;            /* seg_weight * f'(ce) / nseg, f(ce) = alpha * ce * (1 - e^-ce)^gamma: d seg_loss / d CE sum */
  long long nseg, nfg, bad;     /* counted pixels / foreground cells / labels torch rejects */
} tt_camera_loss_stats;
size_t tt_camera_loss_train_workspace_bytes(const tt_camera_loss_train_desc* d);
int tt_camera_loss_train_forward(const tt_camera_loss_train_desc* d, float* out, tt_camera_loss_stats* stats, uint8_t* seg_target,
                                 uint8_t* depth_target, void* ws, size_t ws_bytes, tt_stream_t stream);
int tt_camera_loss_train_backward(const tt_camera_loss_train_desc* d, const tt_camera_loss_stats* stats, const uint8_t* seg_target,
                                  const uint8_t* depth_target, const float* grad_loss, float* grad_seg, float* grad_depth,
                                  tt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (16) training-side dense convolution (SURVEY.md 2.2 N6): torch.nn.Conv2d forward and backward, for the layers a training step
 * puts through forward and backward (the camera trunk with frozen_stages=-1, the DepthNet, the seg head, the BEV fusion, SECOND).
 *   y[n][oh][ow][o] = bias[o] + sum_{i, kh, kw} weight[o][i][kh][kw] x[n][oh * stride - pad + kh * dil][ow * stride - pad + kw * dil][i]
 * with out-of-image input pixels zero.  Activations and their gradients in torch's channels_last storage: x, grad_x [N][H][W][Cin],
 * y, grad_y [N][OH][OW][Cout]; weight, grad_weight torch's contiguous (Cout, Cin, KH, KW); bias, grad_bias [Cout].  Products in
 * 3xTF32 on the tensor cores (fp32-class over fp32's whole exponent range), fp32 accumulation.  The weight is repacked by a kernel
 * in every call (it changes every optimiser step).
 *   forward : the implicit-GEMM tensor-core convolution, bias in its epilogue;
 *   grad_x  : stride 1, one convolution of grad_y with the flipped, transposed kernel; stride 2, one stride-1 convolution per output
 *             phase (y mod 2, x mod 2) with the sub-kernel of the taps that reach it, stored through a pixel scatter; pixels no tap
 *             reaches are written as zeros.  No im2col, no zero-inserted copy of grad_y;
 *   grad_weight: per tap, grad_y^T x(shifted) as a contraction over the output pixels (A-transposed tensor-core GEMM), split over
 *             pixels and folded in a fixed order;
 *   grad_bias: per-channel sum of grad_y over the pixels in fixed chunks, folded in a fixed order.
 * Determinism: y, grad_x, grad_weight and grad_bias are each bitwise reproducible from run to run on the same GPU (no split-K with
 * red.add, no floating-point atomics).
 * Supported: groups 1, stride 1 or 2, Cin and Cout multiples of 4, any kernel size, padding >= 0 and dilation >= 1, OH / OW equal
 * to (H + 2 pad - dil (KH - 1) - 1) / stride + 1 (resp. W, KW) and at least 1, pixel and element counts within 32-bit indexing.
 * Anything else, and ws_bytes < tt_conv2d_train_workspace_bytes(d), returns TT_ERR_UNSUPPORTED with the parameter named in
 * tt_last_error, before any pointer or device is touched.  N = 0 launches no kernel (grad_weight / grad_bias are zeroed by memset).
 * Forward: y is fully written; bias is read when d->bias (NULL otherwise).  Backward: grad_x, grad_weight and grad_bias (when
 * d->bias) are fully written; any of them may be NULL and is then not computed.
 * ws: tt_conv2d_train_workspace_bytes(d) bytes of device memory, not shared with a concurrent call.
 */
typedef struct {
  int N, H, W, Cin, Cout, KH, KW, stride, pad, dil, groups, bias;
  int OH, OW;
} tt_conv2d_train_desc;
size_t tt_conv2d_train_workspace_bytes(const tt_conv2d_train_desc* d);   /* 0 when refused */
int tt_conv2d_train_forward(const tt_conv2d_train_desc* d, const float* x, const float* weight, const float* bias, float* y,
                            void* ws, size_t ws_bytes, tt_stream_t stream);
int tt_conv2d_train_backward(const tt_conv2d_train_desc* d, const float* x, const float* weight, const float* grad_y,
                             float* grad_x, float* grad_weight, float* grad_bias, void* ws, size_t ws_bytes, tt_stream_t stream);

#ifdef __cplusplus
}
/* C++ linkage, mangled exactly like the reference's own definition (ops/voxel_pooling/src/voxel_pooling_forward_cuda.cu:38,
 * declared at src/voxel_pooling_forward.cpp:21-22): the reference's pybind wrapper links against libtt_b200.so unchanged.
 * `cudaStream_t` is `struct CUstream_st*`. */
struct CUstream_st;
void voxel_pooling_forward_kernel_launcher(int batch_size, int num_points, int num_channels, int num_voxel_x, int num_voxel_y,
                                           int num_voxel_z, const int* geom_xyz, const float* input_features,
                                           float* output_features, int* pos_memo, struct CUstream_st* stream);
#endif
#endif /* TT_B200_H_ */
