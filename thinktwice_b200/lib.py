"""ctypes binding of libtt_b200.so (include/tt_b200.h).

PyTorch is used only as the owner of device memory and streams: every wrapper takes tensors, passes
`data_ptr()` / the current CUDA stream to the C ABI and raises on a non-zero status.  There is no CPU
or eager fallback: if the library is missing or a tensor is not on a CUDA device this fails loudly.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libtt_b200.so')

ACT_NONE, ACT_RELU, ACT_GELU, ACT_SIGMOID, ACT_SOFTPLUS, ACT_SOFTPLUS_CLAMP = 0, 1, 2, 3, 4, 5
RES_NONE, RES_SAME, RES_UP2 = 0, 1, 2
IMPL_AUTO, IMPL_SIMT, IMPL_TF32, IMPL_3XTF32, IMPL_F16S = 0, 1, 2, 3, 4
ELT_INV_SOFTPLUS = 4            # tt_eltwise op: y = act(a + log(-expm1(-a)))
LOSS_SMOOTH_L1, LOSS_SMOOTH_L1_CLAMP, LOSS_L1, LOSS_BETA_KL, LOSS_ACTION_L1 = 0, 1, 2, 3, 4
LOSS_MAX_DIM = 6


class TTError(RuntimeError):
    pass


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('N', 'H', 'W', 'Cin', 'x_ld', 'x_coff')] + \
               [('x_nstride', C.c_longlong), ('y_nstride', C.c_longlong), ('x_hstride', C.c_longlong)] + \
               [(n, C.c_int) for n in ('Cout', 'KH', 'KW', 'stride', 'pad', 'dil', 'groups', 'OH', 'OW',
                                        'y_ld', 'y_coff', 'yH', 'yW', 'oy_mul', 'oy_add', 'ox_mul', 'ox_add',
                                        'act', 'bias_n_mod', 'res_mode', 'res_ld', 'res_coff', 'res_H', 'res_W',
                                        'res2_ld', 'res2_coff', 'taps', 'M', 'impl')]


class F16sIO(C.Structure):
    """tt_f16s_io (include/tt_b200.h): the pointers of one tt_conv2d_f16s call."""
    _fields_ = [('x_split', C.c_void_p), ('x_plane', C.c_longlong), ('w_split', C.c_void_p), ('bias', C.c_void_p),
                ('res', C.c_void_p), ('res_split', C.c_void_p), ('res_plane', C.c_longlong),
                ('res2', C.c_void_p), ('res2_split', C.c_void_p), ('res2_plane', C.c_longlong),
                ('y', C.c_void_p), ('y_split', C.c_void_p), ('y_plane', C.c_longlong)]


class LiftSplatDesc(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('B', 'N', 'D', 'fH', 'fW', 'C', 'ld_d', 'd_coff', 'ld_c', 'c_coff')] + \
               [('lower', C.c_float * 3), ('size', C.c_float * 3)] + \
               [(n, C.c_int) for n in ('X', 'Y', 'Z', 'bev_ld', 'bev_coff', 'anti_transpose')]


class VoxelizeDesc(C.Structure):
    _fields_ = [('B', C.c_int), ('P', C.c_int), ('F', C.c_int), ('lower', C.c_float * 3), ('vsize', C.c_float * 3),
                ('grid', C.c_int * 3), ('zmax', C.c_int), ('max_points', C.c_int), ('max_voxels', C.c_int),
                ('cap', C.c_int)]


class RulebookDesc(C.Structure):
    _fields_ = [('B', C.c_int), ('in_shape', C.c_int * 3), ('out_shape', C.c_int * 3), ('k', C.c_int * 3),
                ('s', C.c_int * 3), ('p', C.c_int * 3), ('subm', C.c_int), ('cap_in', C.c_int), ('cap_out', C.c_int),
                ('table_size', C.c_int)]


class SparseConvDesc(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('Cin', 'Cout', 'kvol', 'in_ld', 'out_ld', 'res_ld', 'cap_out', 'pair_cap', 'act', 'impl')]


class LookDesc(C.Structure):
    _fields_ = [('B', C.c_int), ('num_cams', C.c_int), ('num_query', C.c_int), ('T', C.c_int),
                ('img_w', C.c_float), ('img_h', C.c_float), ('levels', C.c_int),
                ('lvl_h', C.c_int * 4), ('lvl_w', C.c_int * 4), ('C', C.c_int), ('q_dim', C.c_int),
                ('emb_dim', C.c_int), ('meas_dim', C.c_int), ('flat_dim', C.c_int), ('max_len_cap', C.c_int)]


class MsdaDesc(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('BN', 'rows_cap', 'heads', 'levels', 'points', 'dh')] + \
               [('lvl_h', C.c_int * 4), ('lvl_w', C.c_int * 4), ('lvl_start', C.c_int * 4), ('num_keys', C.c_int), ('value_ld', C.c_int),
                ('value_coff', C.c_int)]


class PreprocDesc(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('n_img', 'H', 'W', 'newH', 'newW', 'outH', 'outW', 'crop_x', 'crop_y', 'undistort')] + \
               [('div', C.c_float), ('mean', C.c_float * 3), ('std', C.c_float * 3)] + \
               [(n, C.c_int) for n in ('pad_H', 'pad_W', 'pad_top', 'pad_left')]


class LossTerm(C.Structure):
    """tt_loss_term (include/tt_b200.h section 10): one term of tt_loss_reduce."""
    _fields_ = [('pred', C.c_void_p), ('pred2', C.c_void_p), ('gt', C.c_void_p), ('gt2', C.c_void_p),
                ('shape', C.c_longlong * LOSS_MAX_DIM), ('pred_stride', C.c_longlong * LOSS_MAX_DIM), ('gt_stride', C.c_longlong * LOSS_MAX_DIM),
                ('ndim', C.c_int), ('kind', C.c_int), ('slot', C.c_int), ('aux', C.c_int), ('scale', C.c_double)]


class LossGrad(C.Structure):
    """tt_loss_grad (include/tt_b200.h section 10b): the gradient outputs and upstream slots of one term of tt_loss_backward."""
    _fields_ = [('grad_pred', C.c_void_p), ('grad_pred2', C.c_void_p), ('grad_stride', C.c_longlong * LOSS_MAX_DIM),
                ('up_slot', C.c_int), ('up_count', C.c_int)]


class CameraLossDesc(C.Structure):
    """tt_camera_loss_desc (include/tt_b200.h section 11): the segmentation and depth halves of tt_camera_loss."""
    _fields_ = [('seg_logits', C.c_void_p), ('seg_gt', C.c_void_p), ('depth_logits', C.c_void_p), ('depth_gt', C.c_void_p), ('BN', C.c_int)] + \
               [(n, C.c_int) for n in ('seg_h', 'seg_w', 'seg_H', 'seg_W', 'seg_ld', 'seg_coff', 'seg_classes', 'seg_ignore')] + \
               [(n, C.c_float) for n in ('seg_alpha', 'seg_gamma', 'seg_weight')] + \
               [(n, C.c_int) for n in ('depth_h', 'depth_w', 'depth_factor', 'depth_ld', 'depth_coff', 'depth_bins')] + \
               [('depth_offset', C.c_float), ('depth_step', C.c_float)]


class DeformConvDesc(C.Structure):
    """tt_deform_conv_desc (include/tt_b200.h section 12): shape and parameters of one deformable convolution."""
    _fields_ = [(n, C.c_int) for n in ('N', 'C', 'H', 'W', 'Cout', 'groups', 'im2col_step', 'kernel_h', 'kernel_w', 'stride',
                                        'padding', 'dilation', 'deform_groups')]


class SparseConvTrainDesc(C.Structure):
    """tt_sparse_conv_train_desc (include/tt_b200.h section 13): shape, capacities and parameters of one training-side sparse conv."""
    _fields_ = [(n, C.c_int) for n in ('Cin', 'Cout', 'kvol', 'cap_in', 'cap_out', 'pair_cap', 'in_ld', 'out_ld')] + \
               [(n, C.c_int * 3) for n in ('k', 'stride', 'padding', 'dilation')] + \
               [(n, C.c_int) for n in ('subm', 'groups', 'bias', 'transposed', 'inverse')]


class LiftSplatTrainDesc(C.Structure):
    """tt_lift_splat_train_desc (include/tt_b200.h section 14): shapes, logits batch stride and voxel grid of the training lift-splat."""
    _fields_ = [(n, C.c_int) for n in ('B', 'N', 'D', 'fH', 'fW', 'C')] + [('depth_bstride', C.c_longlong)] + \
               [('lower', C.c_float * 3), ('size', C.c_float * 3)] + [(n, C.c_int) for n in ('X', 'Y', 'Z')]


class CameraLossTrainDesc(C.Structure):
    """tt_camera_loss_train_desc (include/tt_b200.h section 15): the two halves of the training camera supervision on NCHW logits."""
    _fields_ = [('seg_logits', C.c_void_p), ('seg_gt', C.c_void_p), ('depth_logits', C.c_void_p), ('depth_gt', C.c_void_p),
                ('seg_stride', C.c_longlong * 4), ('depth_stride', C.c_longlong * 4), ('BN', C.c_int)] + \
               [(n, C.c_int) for n in ('seg_h', 'seg_w', 'seg_H', 'seg_W', 'seg_classes', 'seg_ignore')] + \
               [(n, C.c_float) for n in ('seg_alpha', 'seg_gamma', 'seg_weight')] + \
               [(n, C.c_int) for n in ('depth_h', 'depth_w', 'depth_factor', 'depth_bins')] + \
               [('depth_offset', C.c_float), ('depth_step', C.c_float)]


class CameraLossStats(C.Structure):
    """tt_camera_loss_stats (include/tt_b200.h section 15): what the training camera forward leaves on the device for its backward."""
    _fields_ = [('ce', C.c_double), ('seg_factor', C.c_double), ('nseg', C.c_longlong), ('nfg', C.c_longlong), ('bad', C.c_longlong)]


class Conv2dTrainDesc(C.Structure):
    """tt_conv2d_train_desc (include/tt_b200.h section 16): shape and parameters of one training-side dense convolution."""
    _fields_ = [(n, C.c_int) for n in ('N', 'H', 'W', 'Cin', 'Cout', 'KH', 'KW', 'stride', 'pad', 'dil', 'groups', 'bias', 'OH', 'OW')]


class ConvTranspose2dTrainDesc(C.Structure):
    """tt_conv_transpose2d_train_desc (include/tt_b200.h section 17): shape and parameters of one training-side transposed convolution."""
    _fields_ = [(n, C.c_int) for n in ('N', 'H', 'W', 'Cin', 'Cout', 'KH', 'KW', 'stride', 'pad', 'output_padding', 'dil', 'groups', 'bias',
                                        'OH', 'OW')]


class InterpBilinearTrainDesc(C.Structure):
    """tt_interp_bilinear_train_desc (include/tt_b200.h section 17): shapes of one align_corners bilinear interpolation."""
    _fields_ = [(n, C.c_int) for n in ('N', 'C', 'H', 'W', 'OH', 'OW', 'align_corners')]


class BatchNormTrainDesc(C.Structure):
    """tt_batch_norm_train_desc (include/tt_b200.h section 18): rows, channels, ranks and options of one training-side batch norm."""
    _fields_ = [('M', C.c_longlong), ('count', C.c_longlong)] + \
               [(n, C.c_int) for n in ('C', 'R', 'affine', 'track_running_stats', 'training', 'residual', 'act')] + \
               [('eps', C.c_double), ('factor', C.c_double)]


_lib = None


def load():
    """dlopen the in-tree library; raises TTError when it is absent (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise TTError(f'{LIB_PATH} is missing: run `python -c "import __graft_entry__ as g; g.build()"` '
                      '(nvcc, sm_90a).  thinktwice_b200 has no CPU / eager fallback.')
    lib = C.CDLL(LIB_PATH)
    lib.tt_last_error.restype = C.c_char_p
    lib.tt_launch_count.restype = C.c_longlong
    for n in ('tt_voxel_pooling_workspace_bytes', 'tt_lift_splat_workspace_bytes', 'tt_voxelize_workspace_bytes',
              'tt_rulebook_workspace_bytes', 'tt_conv2d_workspace_bytes', 'tt_loss_workspace_bytes', 'tt_camera_loss_workspace_bytes',
              'tt_deform_conv_workspace_bytes', 'tt_sparse_conv_train_workspace_bytes', 'tt_sparse_pairs_ordered_workspace_bytes',
              'tt_lift_splat_train_workspace_bytes', 'tt_loss_backward_workspace_bytes', 'tt_camera_loss_train_workspace_bytes',
              'tt_conv2d_train_workspace_bytes', 'tt_conv_transpose2d_train_workspace_bytes', 'tt_batch_norm_train_workspace_bytes'):
        getattr(lib, n).restype = C.c_size_t
    if os.environ.get('TT_DEBUG'):                               # kernel-experiment knobs (tt_debug_set) for whole test / bench runs
        check(lib.tt_debug_set(int(os.environ['TT_DEBUG'], 0)), 'tt_debug_set')
    _lib = lib
    return lib


EXPORTS = [
    'tt_version', 'tt_last_error', 'tt_launch_count', 'tt_voxel_pooling_workspace_bytes', 'tt_voxel_pooling_forward',
    'tt_lift_splat_workspace_bytes', 'tt_lift_splat', 'tt_conv2d', 'tt_conv2d_workspace_bytes', 'tt_nchw_to_nhwc', 'tt_nchw_to_nhwc_padded', 'tt_nhwc_to_nchw',
    'tt_maxpool3x3s2', 'tt_upsample2x_bilinear_ac', 'tt_global_avgpool', 'tt_broadcast_rows', 'tt_se_gate', 'tt_se_pool',
    'tt_se_apply', 'tt_anti_transpose', 'tt_copy2d', 'tt_layernorm', 'tt_eltwise', 'tt_fill', 'tt_dcn_im2col',
    'tt_voxelize_workspace_bytes', 'tt_voxelize_mean', 'tt_rulebook_workspace_bytes', 'tt_sparse_rulebook',
    'tt_sparse_conv', 'tt_sparse_to_bev', 'tt_conv2d_f16s', 'tt_split_f16', 'tt_merge_f16', 'tt_image_to_split8', 'tt_pointwise_f16s', 'tt_upsample2x_bilinear_ac_split', 'tt_f16s_saturation_count', 'tt_sparse_conv_f16s', 'tt_sparse_conv_os_f16s', 'tt_look_project', 'tt_look_rebatch', 'tt_msda_forward', 'tt_look_reduce', 'tt_msda_forward_frames', 'tt_look_reduce_frames', 'tt_gru_input',
    'tt_preprocess_u8', 'tt_lidar_stitch', 'tt_points_union', 'tt_voxel_pooling_backward', 'tt_ms_deform_attn_forward', 'tt_ms_deform_attn_backward',
    'tt_loss_workspace_bytes', 'tt_loss_reduce', 'tt_camera_loss_workspace_bytes', 'tt_camera_loss',
    'tt_deform_conv_workspace_bytes', 'tt_deform_conv_forward', 'tt_deform_conv_backward',
    'tt_sparse_conv_train_workspace_bytes', 'tt_sparse_conv_train_forward', 'tt_sparse_conv_train_backward',
    'tt_sparse_pairs_ordered_workspace_bytes', 'tt_sparse_pairs_ordered',
    'tt_lift_splat_train_workspace_bytes', 'tt_lift_splat_train_forward', 'tt_lift_splat_train_backward',
    'tt_loss_backward_workspace_bytes', 'tt_loss_backward',
    'tt_camera_loss_train_workspace_bytes', 'tt_camera_loss_train_forward', 'tt_camera_loss_train_backward',
    'tt_conv2d_train_workspace_bytes', 'tt_conv2d_train_forward', 'tt_conv2d_train_backward',
    'tt_conv_transpose2d_train_workspace_bytes', 'tt_conv_transpose2d_train_forward', 'tt_conv_transpose2d_train_backward',
    'tt_interp_bilinear_train_forward', 'tt_interp_bilinear_train_backward',
    'tt_batch_norm_train_workspace_bytes', 'tt_batch_norm_train_stats', 'tt_batch_norm_train_fold', 'tt_batch_norm_train_forward',
    'tt_batch_norm_train_backward_reduce', 'tt_batch_norm_train_backward',
]


def pack_loss_terms(terms):
    """list of term dicts (LossTerm's field names; pointers from `_p`) -> the tt_loss_term array tt_loss_reduce reads."""
    arr = (LossTerm * len(terms))()
    for a, t in zip(arr, terms):
        if len(t['shape']) > LOSS_MAX_DIM:
            raise TTError(f'loss term of {len(t["shape"])} dims (at most {LOSS_MAX_DIM})')
        a.pred, a.pred2, a.gt, a.gt2 = t['pred'], t['pred2'], t['gt'], t['gt2']
        a.ndim, a.kind, a.slot, a.aux, a.scale = len(t['shape']), t['kind'], t['slot'], t['aux'], t['scale']
        for d, (n, ps, gs) in enumerate(zip(t['shape'], t['pred_stride'], t['gt_stride'])):
            a.shape[d], a.pred_stride[d], a.gt_stride[d] = n, ps, gs
    return arr


def pack_loss_grads(grads):
    """list of gradient dicts (LossGrad's field names; pointers from `_p`) -> the tt_loss_grad array tt_loss_backward reads."""
    arr = (LossGrad * len(grads))()
    for a, g in zip(arr, grads):
        a.grad_pred, a.grad_pred2, a.up_slot, a.up_count = g['grad_pred'], g['grad_pred2'], g['up_slot'], g['up_count']
        for d, s in enumerate(g['grad_stride']):
            a.grad_stride[d] = s
    return arr


def camera_loss_desc(**fields):
    """CameraLossDesc's field names (pointers from `_p`; an absent half's pointers NULL) -> the descriptor tt_camera_loss reads."""
    d = CameraLossDesc()
    for k, v in fields.items():
        setattr(d, k, v)
    return d


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t, off=0):
    """device pointer of tensor `t` advanced by `off` elements (None -> NULL)."""
    if t is None:
        return C.c_void_p(0)
    if not t.is_cuda:
        raise TTError('tt_b200 ops need CUDA tensors (there is no CPU fallback)')
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def ref(struct):
    """pointer to a ctypes struct for a C-ABI call."""
    return C.byref(struct)


def require_cuda(dev):
    if torch.device(dev).type != 'cuda':
        raise TTError('thinktwice_b200 runs on a CUDA device only (no CPU fallback)')


def check(rc, name):
    if rc != 0:
        raise TTError(f'{name} failed ({rc}): {load().tt_last_error().decode()}')


def launch_count():
    return int(load().tt_launch_count())


def f3(v):
    return (C.c_float * 3)(*[float(x) for x in v])


def i3(v):
    return (C.c_int * 3)(*[int(x) for x in v])


def i4(v):
    v = list(v) + [0] * (4 - len(v))
    return (C.c_int * 4)(*[int(x) for x in v])


# ---------------------------------------------------------------------------------------------
# thin typed wrappers (pointer arithmetic for channel offsets is done by the callers through `_p`)
# ---------------------------------------------------------------------------------------------
def call(name, *args):
    check(getattr(load(), name)(*args, _stream()), name)
