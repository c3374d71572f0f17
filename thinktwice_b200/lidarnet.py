"""LiDAR -> BEV encoder on the H100 op library.

Mirror of the reference `LidarNet` / `SparseEncoder_fp32` (open_loop_training/code/model_code/backbones/
lidarnet.py:24-96, cfg configs/thinktwice.py:159-193): hard voxelisation + mean VFE, the sparse 3-D
encoder (rulebooks on the device, convolutions through the gather-mode implicit GEMM), SECOND and
SECONDFPN.  Site counts live in device scalars — there is no host synchronisation (the reference syncs
at lidarnet.py:90 `coors[-1, 0] + 1`).
"""
import ctypes as C

import torch
import torch.nn as nn

from . import lib
from .lib import ACT_RELU, RulebookDesc, VoxelizeDesc, _p
from .registry import BACKBONES, MIDDLE_ENCODERS


def _pow2(v):
    t = 1024
    while t < v:
        t <<= 1
    return t


@MIDDLE_ENCODERS.register_module()
class SparseEncoder_fp32:
    """Holds the static description of the sparse encoder (channels, strides, paddings)."""

    def __init__(self, in_channels, sparse_shape, output_channels, encoder_channels, encoder_paddings,
                 order=('conv', 'norm', 'act'), base_channels=16, block_type='basicblock'):
        assert block_type == 'basicblock' and tuple(order) == ('conv', 'norm', 'act')
        self.in_channels, self.sparse_shape, self.output_channels = in_channels, tuple(sparse_shape), output_channels
        self.encoder_channels, self.encoder_paddings, self.base_channels = encoder_channels, encoder_paddings, base_channels


def _t3(v):
    return tuple(v) if isinstance(v, (list, tuple)) else (v, v, v)


@BACKBONES.register_module()
class LidarNet(nn.Module):
    def __init__(self, bev_h=None, bev_w=None, pts_voxel_layer=None, pts_voxel_encoder=None, pts_middle_encoder=None,
                 pts_fusion_layer=None, pts_backbone=None, pts_neck=None, pts_bbox_head=None, train_cfg=None,
                 test_cfg=None, prefix='lidar_encoder.'):
        super().__init__()
        self.prefix = prefix
        self.vcfg = dict(pts_voxel_layer)
        self.num_features = pts_voxel_encoder['num_features']
        self.me = MIDDLE_ENCODERS.build(dict(pts_middle_encoder))
        self.bb_cfg, self.neck_cfg = dict(pts_backbone), dict(pts_neck)
        import numpy as np
        vs = np.asarray(self.vcfg['voxel_size'], np.float32)
        r = np.asarray(self.vcfg['point_cloud_range'], np.float32)
        self.grid = [int(v) for v in np.round((r[3:] - r[:3]) / vs)]          # (x, y, z)
        mv = self.vcfg['max_voxels']
        self.max_voxels = int(mv[1] if isinstance(mv, (list, tuple)) else mv)     # (train, eval) pair: eval
        self.sparse_form = 'os'    # 'os': output-stationary sparse convs for the wide layers (f16s engine); 'tap': tap-major pair lists

    def prepare(self, pk, eng):
        self.eng = eng
        p = self.prefix + 'pts_middle_encoder.'
        me = self.me
        # plan of sparse layers: ('subm'|'down', packed weights, kernel, stride, pad, residual?)
        self.stages = []
        self.w_in, self.k_in = pk.spconv(p + 'conv_input.0', p + 'conv_input.1')
        n_stage = len(me.encoder_channels)
        for i, blocks in enumerate(me.encoder_channels):
            st = []
            for j, cout in enumerate(blocks):
                q = f'{p}encoder_layers.encoder_layer{i + 1}.{j}.'
                if j == len(blocks) - 1 and i != n_stage - 1:
                    wc, k = pk.spconv(q + '0', q + '1')
                    st.append(('down', wc, k, (2, 2, 2), _t3(me.encoder_paddings[i][j])))
                else:
                    (w1, k), (w2, _) = pk.spconv(q + 'conv1', q + 'bn1'), pk.spconv(q + 'conv2', q + 'bn2')
                    st.append(('block', w1, w2))
            self.stages.append(st)
        self.w_out, self.k_out = pk.spconv(p + 'conv_out.0', p + 'conv_out.1')
        q = self.prefix + 'pts_backbone.blocks.'
        self.second = []
        for bi, n in enumerate(self.bb_cfg['layer_nums']):
            self.second.append([pk.conv(f'{q}{bi}.{3 * k}', bn=f'{q}{bi}.{3 * k + 1}', eps=1e-3) for k in range(n + 1)])
        q = self.prefix + 'pts_neck.deblocks.'
        self.deblocks = []
        for i, s in enumerate(self.neck_cfg['upsample_strides']):
            if s > 1:
                self.deblocks.append(('up', pk.convT(f'{q}{i}.0', bn=f'{q}{i}.1', eps=1e-3)))
            else:
                self.deblocks.append(('conv', pk.conv(f'{q}{i}.0', bn=f'{q}{i}.1', eps=1e-3)))

    # ------------------------------------------------------------------
    def _rulebook(self, tag, B, in_coords, in_count, cap_in, in_shape, k, s, p, subm, form='pairs'):
        """form: 'pairs' = tap-major (input row, output row) lists (tt_sparse_conv / _f16s); 'nbr' = per output row the input row
        under every tap (tt_sparse_conv_os_f16s, the output-stationary form the wide layers use on the f16s engine)."""
        e = self.eng
        out_shape = in_shape if subm else tuple((in_shape[i] + 2 * p[i] - k[i]) // s[i] + 1 for i in range(3))
        cells = B * out_shape[0] * out_shape[1] * out_shape[2]
        cap_out = cap_in if subm else min(cap_in * 8, cells)
        d = RulebookDesc()
        d.B = B
        d.in_shape, d.out_shape, d.k, d.s, d.p = lib.i3(in_shape), lib.i3(out_shape), lib.i3(k), lib.i3(s), lib.i3(p)
        d.subm, d.cap_in, d.cap_out = int(subm), cap_in, cap_out
        d.table_size = _pow2(2 * max(cap_in, cap_out))
        kvol = k[0] * k[1] * k[2]
        ws = e.buf('sp.ws', (lib.load().tt_rulebook_workspace_bytes(C.byref(d)),), dtype=torch.uint8)
        out_coords, out_count = e.buf(f'sp.{tag}.coords', (cap_out, 4), torch.int32), e.buf(f'sp.{tag}.count', (1,), torch.int32)
        pin = pout = pcount = nbr = None
        if form == 'nbr':
            nbr = e.buf(f'sp.{tag}.nbr', (cap_out, kvol), torch.int32)
        else:
            pin, pout = e.buf(f'sp.{tag}.pin', (kvol, cap_out), torch.int32), e.buf(f'sp.{tag}.pout', (kvol, cap_out), torch.int32)
            pcount = e.buf(f'sp.{tag}.pcount', (kvol,), torch.int32)
        lib.call('tt_sparse_rulebook', C.byref(d), _p(in_coords), _p(in_count), _p(out_coords), _p(out_count), _p(nbr), _p(pin), _p(pout),
                 _p(pcount), _p(ws))
        return dict(coords=out_coords, count=out_count, cap=cap_out, shape=out_shape, kvol=kvol, pairs_in=pin, pairs_out=pout,
                    pair_count=pcount, nbr=nbr)

    def forward(self, pts):
        """pts (B, P, 5) fp32 on the device -> [FMap (B, 84, 84, 512)] already in the Roach BEV orientation
        (the rot90(flip) of encoder_decoder_framework.py:246 is applied to the neck output here)."""
        e = self.eng
        B, P, F = pts.shape
        pts = pts.contiguous()
        v = self.vcfg
        d = VoxelizeDesc()
        d.B, d.P, d.F = B, P, F
        d.lower, d.vsize = lib.f3(v['point_cloud_range'][:3]), lib.f3(v['voxel_size'])
        d.grid = lib.i3(self.grid)
        d.zmax = self.me.sparse_shape[0]
        d.max_points, d.max_voxels = v['max_num_points'], self.max_voxels
        cap = B * P
        d.cap = cap
        ws = e.buf('vox.ws', (lib.load().tt_voxelize_workspace_bytes(C.byref(d)),), dtype=torch.uint8)
        feats = e.buf('vox.feats', (cap, F))
        coords = e.buf('vox.coords', (cap, 4), torch.int32)
        count = e.buf('vox.count', (1,), torch.int32)
        lib.call('tt_voxelize_mean', C.byref(d), _p(pts), _p(feats), _p(coords), _p(count), _p(ws))

        shape = self.me.sparse_shape
        # conv_input (SubM 5 -> 16); all SubM convs of one resolution share one rulebook (spconv indice_key)
        def form(cin):                                             # wide layers on the f16s engine: output-stationary
            return 'nbr' if (e.split and self.sparse_form == 'os' and cin >= 32) else 'pairs'
        rb = self._rulebook('l0', B, coords, count, cap, shape, self.k_in, (1, 1, 1), (1, 1, 1), True, form(self.stages[0][0][1].Cin))
        x, xs = e.sparse_feats('sp.l0.x', rb['cap'], self.w_in.Cout)
        e.sparse_conv(feats, self.w_in, rb, x, act=ACT_RELU, name='conv_input', out_s=xs)
        for i, st in enumerate(self.stages):
            for j, layer in enumerate(st):
                if layer[0] == 'block':
                    _, w1, w2 = layer
                    po = rb.get('nbr') is not None                   # planes-only rows: the output-stationary convs need no fp32 copy
                    t, ts = e.sparse_feats(f'sp.l{i}.t', rb['cap'], w1.Cout, f32=not po)
                    e.sparse_conv(x, w1, rb, t, act=ACT_RELU, name=f'{i}.{j}.conv1', feats_s=xs, out_s=ts)
                    o, os_ = e.sparse_feats(f'sp.l{i}.o{j % 2}', rb['cap'], w2.Cout, f32=not po)
                    e.sparse_conv(t, w2, rb, o, act=ACT_RELU, res=x, res_s=xs if x is None else None, name=f'{i}.{j}.conv2', feats_s=ts, out_s=os_)
                    x, xs = o, os_
                else:
                    _, wc, k, s, p = layer
                    rd = self._rulebook(f'd{i}', B, rb['coords'], rb['count'], rb['cap'], rb['shape'], k, s, p, False, form(wc.Cin))
                    # rulebook of the SubM convs at the new resolution
                    rb2 = self._rulebook(f'l{i + 1}', B, rd['coords'], rd['count'], rd['cap'], rd['shape'], (3, 3, 3), (1, 1, 1), (1, 1, 1), True, form(wc.Cout))
                    o, os_ = e.sparse_feats(f'sp.l{i + 1}.x', rd['cap'], wc.Cout, f32=rd.get('nbr') is None or rb2.get('nbr') is None)
                    e.sparse_conv(x, wc, rd, o, act=ACT_RELU, name=f'{i}.{j}.down', feats_s=xs, out_s=os_)
                    x, xs, rb = o, os_, rb2
        ro = self._rulebook('out', B, rb['coords'], rb['count'], rb['cap'], rb['shape'], self.k_out, (2, 1, 1), (0, 0, 0), False, form(self.w_out.Cin))
        o, _ = e.sparse_feats('sp.out.x', ro['cap'], self.w_out.Cout)
        x = e.sparse_conv(x, self.w_out, ro, o, act=ACT_RELU, name='conv_out', feats_s=xs)
        coords2, count2, cap2, shape2 = ro['coords'], ro['count'], ro['cap'], ro['shape']
        D, H, W = shape2
        Cs = self.w_out.Cout
        dense = e.fmap('lidar.dense', B, H, W, Cs * D)
        e.fill(dense.t, 0.0)
        lib.call('tt_sparse_to_bev', _p(x), _p(coords2), _p(count2), cap2, Cs, D, H, W, 0, _p(dense.t))
        e.sync_split(dense)
        return self._second(dense)

    def _second(self, x):
        e = self.eng
        outs = []
        for bi, convs in enumerate(self.second):
            stride = self.bb_cfg['layer_strides'][bi]
            for k, wc in enumerate(convs):
                x = e.conv(x, wc, name=f'sec.{bi}.{k % 2}' if k < len(convs) - 1 else f'sec.{bi}.out', stride=stride if k == 0 else 1,
                           pad=1, act=ACT_RELU)
            outs.append(x)
        c_tot = sum(self.neck_cfg['out_channels'])
        N, H, W = outs[0].N, outs[0].H * self.neck_cfg['upsample_strides'][0], outs[0].W * self.neck_cfg['upsample_strides'][0]
        cat = e.fmap('lidar.out', N, H, W, c_tot)
        off = 0
        for (kind, wc), xin, co in zip(self.deblocks, outs, self.neck_cfg['out_channels']):
            dst = cat.slice(off, co)
            if kind == 'conv':
                e.conv(xin, wc, out=dst, name='fpn3d.conv', act=ACT_RELU)
            else:
                for i in range(2):
                    for j in range(2):
                        e.conv(xin, wc[i][j], out=dst, name=f'fpn3d.up{i}{j}', act=ACT_RELU, scatter=(2, i, 2, j))
            off += co
        return [e.anti_transpose(cat, 'lidar.out.at')]                # framework:246 rot90(flip)

