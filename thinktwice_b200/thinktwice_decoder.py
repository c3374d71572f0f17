"""ThinkTwiceDecoder — coarse heads + K x (Prediction, Look, Refine) on the H100 op library.

Mirror of open_loop_training/code/model_code/dense_heads/thinktwice_decoder.py:262-489 (forward), :491-533 (the teacher-forced pass) and
:535-636 (loss: values for open-loop validation, no gradients),
with the Look module's SpatialCrossAttention / MSDeformableAttention3D
(multi_scale_deformable_attn_function.py:216-526) and SpatialGRU (dense_heads/utils.py:53-106).
Reference quirks kept bit-for-bit in semantics by default: batch-wide max_len, "zero the first B rows / divide by
B" (msda:338-342).  With `independent_frames` each frame gets B = 1 semantics instead (its own max_len, row 0 zeroed,
divisor 1), so a frame predicts what it predicts alone.  Dead work is skipped with identical outputs: PredictionModule.ffn
(thinktwice_decoder.py:44-46) and the LiDAR look branch (:179-186, replaced by zeros in the reference).
"""
import ctypes as C

import torch
import torch.nn as nn

from . import lib
from .engine import FMap
from .lib import (ACT_GELU, ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_SOFTPLUS, ACT_SOFTPLUS_CLAMP, LookDesc, MsdaDesc, _p)
from .registry import HEADS

NQ, ZL = 120, 15


class LazyPred(dict):
    """pred dict whose bulky feature stacks (refine_*_BEV_feature) are assembled on first access."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self._lazy, self._all_lazy, self._made = {}, {}, set()
        self.maps = {}              # the arena maps behind the outputs (ThinkTwiceDecoder.loss reads them in place)

    def lazy(self, key, fn):
        self._lazy[key] = fn
        self._all_lazy[key] = fn

    def __missing__(self, key):
        if key in self._lazy:
            self[key] = self._lazy.pop(key)()
            self._made.add(key)
            return self[key]
        raise KeyError(key)

    def __contains__(self, key):
        return dict.__contains__(self, key) or key in self._lazy

    def keys(self):
        return list(dict.keys(self)) + list(self._lazy.keys())

    def fresh(self):
        """new view over the same (static) output buffers with every lazy entry un-materialised (graph replays)."""
        o = LazyPred({k: v for k, v in dict.items(self) if k not in self._made})
        o._lazy = dict(self._all_lazy)
        o._all_lazy, o._made = self._all_lazy, set()
        return o


@HEADS.register_module()
class ThinkTwiceDecoder(nn.Module):
    def __init__(self, *args, config=None, bev_h=None, bev_w=None, BEV_feat_dim=256, flattened_BEV_feat_dim=256,
                 prefix='decoder.', **kwargs):
        super().__init__()
        self.config, self.bev_h, self.bev_w, self.prefix = config, bev_h, bev_w, prefix
        self.T = config['pred_len']
        self.K = config['refine_num']
        self.value_all_budget = 8 << 30     # bytes the merged value_proj output may take (else per-layer projection)
        self.independent_frames = False     # Look module: batch-coupled reference semantics (False) or B = 1 per frame (True)

    # ------------------------------------------------------------------ weights
    def prepare(self, pk, eng, parent):
        self.eng = eng
        p = self.prefix
        w = self.w = {}

        def mlp(name, n):
            return [pk.linear(f'{p}{name}.{2 * i}') for i in range(n)]
        for name, n in (('join_traj', 3), ('output_traj', 2), ('join_ctrl', 3), ('speed_branch', 3), ('value_branch_traj', 3),
                        ('value_branch_ctrl', 3), ('policy_head', 2), ('dist_mu', 2), ('dist_sigma', 2)):
            w[name] = mlp(name, n)
        w['fpn_linear'] = [pk.conv(f'{p}fpn_linear{i}') for i in range(4)]
        # fpn_linear is followed by value_proj with nothing in between (thinktwice_decoder.py:442-450 -> msda:474): the value tensor is
        # computed from the FPN maps directly with the composed map (Wv Wf) x + Wv bf + ..., so the projected maps `mlvl` are only read by
        # the fp32 bilinear gather of the look points
        Wf = [pk.sd[f'{p}fpn_linear{i}.weight'].double().reshape(256, -1) for i in range(4)]
        bf = [pk.sd[f'{p}fpn_linear{i}.bias'].double() for i in range(4)]
        self.temb, self.semb = pk.vec(p + 'temporal_embedding'), pk.vec(p + 'static_embedding')
        cams, lvls = pk.sd[p + 'cams_embeds'].double(), pk.sd[p + 'level_embeds'].double()
        # GRU input planes are laid out [state 32 | x 6 | pad 2] (vector-aligned); permute the conv weights to match
        gru_idx = list(range(6, 38)) + list(range(6)) + [-1, -1]
        self.layers = []
        for k in range(self.K):
            q = f'{p}decoder_layers.{k}.'
            g = q + 'prediction_module.spatial_gru.'
            L = {}
            for n in ('conv_update', 'conv_reset', 'conv_state_tilde'):
                L[n] = (pk.conv(f'{g}{n}.0', cin_index=gru_idx), pk.conv(f'{g}{n}.2'))
            L['conv_decoder'] = (pk.conv(g + 'conv_decoder.0'), pk.conv(g + 'conv_decoder.2'))
            c = q + 'look_module.cam_look_module.'
            L['q_ln'] = (pk.vec(c + 'query_linear.0.weight'), pk.vec(c + 'query_linear.0.bias'))
            L['q1'] = pk.linear(c + 'query_linear.1', cin_pad=1544)
            L['q3'] = pk.linear(c + 'query_linear.3')
            L['off'] = pk.linear(c + 'deformable_attention.sampling_offsets')
            L['aw'] = pk.linear(c + 'deformable_attention.attention_weights')
            # value_proj(x + cams_embeds[cam] + level_embeds[lvl]) = W x + (W (e_cam + e_lvl) + b): one bias per (cam, lvl).
            # The K layers' value projections depend only on the FPN maps, not on the cascade: they are packed as ONE
            # 256 -> K*256 projection per level (self.value_all, built after this loop) and run once, ahead of the cascade.
            Wv, bv = pk.sd[c + 'deformable_attention.value_proj.weight'].double(), pk.sd[c + 'deformable_attention.value_proj.bias'].double()
            L['_value_w'] = [Wv @ Wf[l] for l in range(4)]          # [level] -> (256, C_fpn_l)
            L['_value_b'] = [torch.stack([bv + Wv @ (bf[l] + cams[cam] + lvls[l]) for cam in range(4)]) for l in range(4)]    # [level] -> (4 cams, 256)
            L['value'] = [pk.linear(c + 'deformable_attention.value_proj', weight=L['_value_w'][l], bias=L['_value_b'][l].float().reshape(-1))
                          for l in range(4)]
            L['ffn_ln'] = (pk.vec(c + 'ffn.norm.weight'), pk.vec(c + 'ffn.norm.bias'))
            L['ffn1'], L['ffn2'] = pk.linear(c + 'ffn.w_1'), pk.linear(c + 'ffn.w_2')
            L['op_ln'] = (pk.vec(c + 'output_proj.0.weight'), pk.vec(c + 'output_proj.0.bias'))
            L['op1'], L['op3'] = pk.linear(c + 'output_proj.1'), pk.linear(c + 'output_proj.3')
            L['mlp_ln'] = (pk.vec(q + 'mlp.0.weight'), pk.vec(q + 'mlp.0.bias'))
            L['mlp1'], L['mlp4'] = pk.linear(q + 'mlp.1'), pk.linear(q + 'mlp.4')
            L['traj'] = [pk.linear(f'{q}traj_offset_module.{i}') for i in (0, 2, 4)]
            L['ctrl'] = [pk.linear(f'{q}ctrl_offset_module.{i}') for i in (0, 2, 4)]
            L['bev_up'] = (pk.conv(q + 'BEV_feat_update_module.0'), pk.conv(q + 'BEV_feat_update_module.2'))
            L['flat_up'] = (pk.linear(q + 'flattened_BEV_feat_update_module.0'), pk.linear(q + 'flattened_BEV_feat_update_module.2'))
            self.layers.append(L)
        # (K*256, C_fpn_l) per level: layer k owns output channels [256k, 256k+256)
        self.value_all = [pk.linear(p + 'value_proj_all', weight=torch.cat([L['_value_w'][l] for L in self.layers], 0),
                                    bias=torch.cat([L['_value_b'][l] for L in self.layers], 1).float().reshape(-1))
                          for l in range(4)]                            # per level: bias table [4 cams][K*256] (bias_n_mod = 4)
        for L in self.layers:
            del L['_value_w'], L['_value_b']

    def stage(self, lidar2img, ida):
        """host half: upload the (B, 4, 4, 4) projection matrices the Look module needs."""
        B = lidar2img.shape[0]
        self.eng.upload('look.l2i', lidar2img.reshape(B, 4, 16).float().contiguous())
        self.eng.upload('look.ida', ida.reshape(B, 4, 16).float().contiguous())

    # ------------------------------------------------------------------ helpers
    def _seq(self, x, ws, tag, last_act=ACT_NONE, out=None):
        e = self.eng
        for i, wl in enumerate(ws):
            last = i == len(ws) - 1
            x = e.linear(x, wl, out=out if last else None, name=f'{tag}.{i}', act=last_act if last else ACT_RELU)
        return x

    def _gru(self, L, bev, wp, ctrl_sp, tag):
        """SpatialGRU over T steps (dense_heads/utils.py:83-106); returns the future BEV maps (B*T, 21, 21, 32)."""
        e, T = self.eng, self.T
        B, H, W, Cs = bev.N, bev.H, bev.W, bev.C
        HW = H * W
        xs = e.fmap('gru.xs', B, H, W, 40, zero=True)               # [state | x_t | 0 0]
        cin = e.fmap('gru.cand_in', B, H, W, 40, zero=True)         # [(1 - r) * state | x_t | 0 0]
        state = xs.slice(0, Cs)
        e.copy_cols(bev, state)
        fut = e.fmap(tag + '.fut', B * T, H, W, Cs)
        for t in range(T):
            for buf in (xs, cin):
                lib.call('tt_gru_input', _p(wp.t), _p(ctrl_sp.t), t, T, _p(buf.t, 32), buf.ld, B, HW)
                e.sync_split(buf.slice(32, 8))
            u = e.conv(e.conv(xs, L['conv_update'][0], name='gru.u1', pad=1, act=ACT_RELU), L['conv_update'][1], name='gru.u', pad=1, act=ACT_SIGMOID)
            r = e.conv(e.conv(xs, L['conv_reset'][0], name='gru.r1', pad=1, act=ACT_RELU), L['conv_reset'][1], name='gru.r', pad=1, act=ACT_SIGMOID)
            e.eltwise(1, r, state, out=cin.slice(0, Cs))             # (1 - r) * state
            cand = e.conv(e.conv(cin, L['conv_state_tilde'][0], name='gru.c1', pad=1, act=ACT_RELU), L['conv_state_tilde'][1], name='gru.c', pad=1)
            e.eltwise(2, u, state, cand, out=state)                  # (1 - u) * state + u * cand
            d1 = e.conv(state, L['conv_decoder'][0], name='gru.d1', pad=1, act=ACT_RELU)
            out_t = fut.view(B, H, W, Cs, Cs, t * HW * Cs)           # image b of step t lives at index b*T + t
            e.conv(d1, L['conv_decoder'][1], out=out_t, name='gru.d', pad=1, y_nstride=T * HW * Cs)
        return fut

    def _values(self, mlvl, meta):
        """value_proj of every decoder layer over all keys of every (camera, level): ONE 256 -> K*256 projection per FPN level
        (msda:474 per layer in the reference: the FPN maps are read once instead of K times, 4 launches instead of 4K)."""
        e = self.eng
        B, cams, nk, KC = meta['B'], 4, meta['num_keys'], self.K * 256
        if B * cams * nk * KC * 4 > self.value_all_budget:           # e.g. B = 32: 21.8 GB for K = 5
            return None
        value = e.buf('look.value_all', (B * cams, nk, KC))
        for l, m in enumerate(mlvl):
            out = FMap(value, B * cams, m.H, m.W, KC, KC, meta['lvl_start'][l] * KC)
            e.conv(meta['fpn'][l], self.value_all[l], out=out, name=f'look.value{l}', y_nstride=nk * KC, bias_n_mod=cams)
        return value

    def _look(self, L, k, wp, ctrl_sp, meas, flat, mlvl, meta):
        """LookModule.forward (thinktwice_decoder.py:154-187), image branch."""
        e = self.eng
        B, cams, cap = meta['B'], 4, NQ
        d = meta['look_desc']
        ref_cam = e.buf('look.ref_cam', (B, cams, NQ, 2))
        order = e.buf('look.order', (B, cams, NQ), torch.int32)
        counts = e.buf('look.counts', (B, cams), torch.int32)
        max_len = e.buf('look.max_len', (1,), torch.int32)
        lib.call('tt_look_project', C.byref(d), _p(wp.t), _p(meta['l2i']), _p(meta['ida']), _p(ref_cam), _p(order), _p(counts), _p(max_len))
        rows = e.fmap('look.rows', B * cams * cap, 1, 1, 1543)
        ref_re = e.buf('look.ref_re', (B * cams * cap, 2))
        ptrs = (C.c_void_p * 4)(*[m.t.data_ptr() for m in mlvl])
        lib.call('tt_look_rebatch', C.byref(d), _p(wp.t), _p(ctrl_sp.t), _p(self.temb), _p(self.semb), _p(meas.t), _p(flat.t, flat.coff),
                 ptrs, _p(ref_cam), _p(order), _p(counts), _p(rows.t), rows.ld, _p(ref_re))
        # query_linear: LN(1543) -> 512 GELU -> 256 GELU (msda:251-257)
        q = e.layernorm(rows, *L['q_ln'], name='look.q_ln', out_ld=1544)
        q = e.linear(q.view(q.N, 1, 1, 1544), L['q1'], name='look.q1', act=ACT_GELU)
        q = e.linear(q, L['q3'], name='look.q', act=ACT_GELU)
        # value_proj (msda:474): computed for all layers at once before the cascade (_values; layer k reads its channel block) when the
        # K-fold value tensor fits the memory budget, else layer by layer into one reused buffer
        nk = meta['num_keys']
        value = meta['value_all']
        if value is None:
            value = e.buf('look.value', (B * cams, nk, 256))
            for l, m in enumerate(mlvl):                             # one launch per level over all B*cams images
                out = FMap(value, B * cams, m.H, m.W, 256, 256, meta['lvl_start'][l] * 256)
                e.conv(meta['fpn'][l], L['value'][l], out=out, name=f'look.value{l}', y_nstride=nk * 256, bias_n_mod=cams)
        off = e.linear(q, L['off'], name='look.off')
        aw = e.linear(q, L['aw'], name='look.aw')
        # tt_msda_forward writes the first max_len rows of each (frame, camera) only (tt_msda_forward_frames: max_len_b of its frame); the FFN below runs over all `cap` rows (static
        # shapes for graph replay) and tt_look_reduce reads the valid ones.  Zero-filled once, so that the rows no forward has written yet
        # hold zeros instead of stale memory, which look.ffn2's epilogue would split into fp16 planes and count as saturated
        att = e.fmap('look.att', B * cams * cap, 1, 1, 256, zero=True)
        md = meta['msda_desc']
        md.value_ld, md.value_coff = (self.K * 256, k * 256) if meta['value_all'] is not None else (0, 0)
        if self.independent_frames:                                  # rows bounded by each frame's own max_len (from `counts`)
            lib.call('tt_msda_forward_frames', C.byref(md), _p(value), _p(off.t), _p(aw.t), _p(ref_re), _p(counts), cams, _p(att.t))
        else:
            lib.call('tt_msda_forward', C.byref(md), _p(value), _p(off.t), _p(aw.t), _p(ref_re), _p(max_len), _p(att.t))
        # PositionwiseFeedForward (msda:197-214)
        h = e.layernorm(att, *L['ffn_ln'], name='look.ffn_ln')
        h = e.linear(h, L['ffn1'], name='look.ffn1', act=ACT_GELU)
        h = e.linear(h, L['ffn2'], name='look.ffn2', res=att)
        red = e.fmap('look.red', B, 1, 1, cams * 256)
        if self.independent_frames:
            lib.call('tt_look_reduce_frames', _p(h.t), B, cams, cap, 256, _p(counts), _p(red.t))
        else:
            lib.call('tt_look_reduce', _p(h.t), B, cams, cap, 256, _p(max_len), _p(red.t))
        o = e.layernorm(red, *L['op_ln'], name='look.op_ln')
        o = e.linear(o, L['op1'], name='look.op1', act=ACT_GELU)
        return e.linear(o, L['op3'], name='look.img')                # (B, 256)

    def _layer(self, L, k, wp, ctrl, cur_bev, cur_flat, meas, mlvl, meta, parent_module, tag):
        """ThinkTwiceDecoderLayer.forward (thinktwice_decoder.py:236-260) of layer k: the waypoint / control offsets (B*T rows), the
        future BEV maps (B*T, 21, 21, 32) and the updated BEV / flat features.  Its outputs are named after `tag`, so that the
        teacher-forced pass never overwrites a map of the main pass; the scratch in between is shared."""
        e, T = self.eng, self.T
        B = cur_flat.rows()
        ctrl_sp = e.eltwise(3, ctrl, name='dec.ctrl_sp', act=ACT_SOFTPLUS)
        fut = self._gru(L, cur_bev, wp, ctrl_sp, f'{tag}.l{k}')
        fflat, _ = parent_module.pyramid(fut, 'dec.py')               # grid2feat (:405-415)
        img_look = self._look(L, k, wp, ctrl_sp, meas, cur_flat, mlvl, meta)
        # mlp input rows (b, t): [future flat 256 | img look 256 | zeros 256 (dead LiDAR look) | temporal 128 | meas 128]
        mi = e.fmap('dec.mlp_in', B * T, 1, 1, 1024, zero=True)
        e.copy_cols(fflat, mi.slice(0, 256)); e.copy_cols(img_look, mi.slice(256, 256), rdiv=T)
        e.copy_cols(FMap(self.temb, T, 1, 1, 128), mi.slice(768, 128), rmod=T); e.copy_cols(meas, mi.slice(896, 128), rdiv=T)
        a = e.layernorm(mi, *L['mlp_ln'], name='dec.mlp_ln')
        a = e.linear(a, L['mlp1'], name='dec.mlp1', act=ACT_RELU)
        a = e.linear(a, L['mlp4'], name='dec.all_future', act=ACT_RELU)          # (B*T, 512)
        ti = e.fmap('dec.traj_in', B * T, 1, 1, 514); e.copy_cols(wp, ti.slice(0, 2)); e.copy_cols(a, ti.slice(2, 512))
        ci = e.fmap('dec.ctrl_in', B * T, 1, 1, 516); e.copy_cols(ctrl, ci.slice(0, 4)); e.copy_cols(a, ci.slice(4, 512))
        t_off = self._seq(ti, L['traj'], 'dec.toff')
        c_off = self._seq(ci, L['ctrl'], 'dec.coff')
        a_flat = a.view(B, 1, 1, T * 512)
        # BEV update (thinktwice_decoder.py:257): conv over [BEV 32 | all_future 2048 tiled] + residual
        bi = e.fmap('dec.bev_in', B, cur_bev.H, cur_bev.W, 32 + T * 512)
        e.copy_cols(cur_bev, bi.slice(0, 32)); e.copy_cols(a_flat, bi.slice(32, T * 512), rdiv=cur_bev.H * cur_bev.W)
        h = e.conv(bi, L['bev_up'][0], name='dec.bev_h', pad=1, act=ACT_RELU)
        new_bev = e.conv(h, L['bev_up'][1], name=f'{tag}.bev.{k}', pad=1, res=cur_bev)
        fi = e.fmap('dec.flat_in', B, 1, 1, 256 + T * 512); e.copy_cols(cur_flat, fi.slice(0, 256)); e.copy_cols(a_flat, fi.slice(256, T * 512))
        h = e.linear(fi, L['flat_up'][0], name='dec.flat_h', act=ACT_RELU)
        new_flat = e.linear(h, L['flat_up'][1], name=f'{tag}.flat.{k}', res=cur_flat)
        return t_off, c_off, fut, new_bev, new_flat

    # ------------------------------------------------------------------ forward
    def forward(self, flattend_BEV_feat, BEV_feat, measurement_feat, target_point, parent_module, teacher_forcing_data=None,
                look_feature_metadata=None):
        e, w, T, K = self.eng, self.w, self.T, self.K
        flat, bev, meas = flattend_BEV_feat, BEV_feat, measurement_feat
        B = flat.rows()
        lidar2img, ida, fpn, _lidar_hi = look_feature_metadata

        # ---- coarse prediction (thinktwice_decoder.py:424-438)
        cat = e.fmap('dec.cat384', B, 1, 1, 384)
        e.copy_cols(flat, cat.slice(0, 256)); e.copy_cols(meas, cat.slice(256, 128))
        speed = self._seq(flat, w['speed_branch'], 'dec.speed')
        jt = self._seq(cat, w['join_traj'], 'dec.jt', last_act=ACT_RELU)
        v_traj = self._seq(jt, w['value_branch_traj'], 'dec.vt')
        wp_all = e.fmap('dec.wp_all', B, 1, 1, (K + 1) * T * 2)
        ctrl_all = e.fmap('dec.ctrl_all', B, 1, 1, (K + 1) * T * 4)
        wp = self._seq(jt, w['output_traj'], 'dec.wp0')               # (B, T*2)
        jc = self._seq(cat, w['join_ctrl'], 'dec.jc', last_act=ACT_RELU)
        v_ctrl = self._seq(jc, w['value_branch_ctrl'], 'dec.vc')
        pol = self._seq(jc, w['policy_head'], 'dec.pol', last_act=ACT_RELU)
        mu = self._seq(pol, w['dist_mu'], 'dec.mu')
        sg = self._seq(pol, w['dist_sigma'], 'dec.sigma')
        ctrl = e.fmap('dec.ctrl', B * T, 1, 1, 4)                     # rows (b, t): [mu 2 | sigma 2]
        e.copy_cols(FMap(mu.t, B * T, 1, 1, 2), ctrl.slice(0, 2)); e.copy_cols(FMap(sg.t, B * T, 1, 1, 2), ctrl.slice(2, 2))
        wp = FMap(wp.t, B * T, 1, 1, 2)
        e.copy_cols(FMap(wp.t, B, 1, 1, T * 2), wp_all.slice(0, T * 2)); e.copy_cols(FMap(ctrl.t, B, 1, 1, T * 4), ctrl_all.slice(0, T * 4))

        # ---- Look-module inputs (thinktwice_decoder.py:442-450)
        mlvl = [e.conv(fpn[i], w['fpn_linear'][i], name=f'dec.mlvl{i}', fmt='f') for i in range(4)]
        meta = self._look_meta(B, mlvl)
        meta['fpn'] = fpn
        meta['value_all'] = self._values(mlvl, meta)

        cur_bev, cur_flat = bev, flat
        s_bev, s_flat, s_fut = [], [], []
        for k, L in enumerate(self.layers):
            t_off, c_off, fut, new_bev, new_flat = self._layer(L, k, wp, ctrl, cur_bev, cur_flat, meas, mlvl, meta, parent_module, 'dec')
            # next waypoints / controls (thinktwice_decoder.py:467-468)
            wp = e.eltwise(0, t_off, wp, name=f'dec.wp.{k % 2}')
            ctrl = e.eltwise(0, c_off, ctrl, name=f'dec.ctrl.{k % 2}')
            e.copy_cols(FMap(wp.t, B, 1, 1, T * 2), wp_all.slice((k + 1) * T * 2, T * 2))
            e.copy_cols(FMap(ctrl.t, B, 1, 1, T * 4), ctrl_all.slice((k + 1) * T * 4, T * 4))
            cur_bev, cur_flat = new_bev, new_flat
            s_bev.append(new_bev); s_flat.append(new_flat); s_fut.append(fut)

        # ---- outputs (thinktwice_decoder.py:479-489)
        ctrl_sp_all = e.eltwise(3, ctrl_all, name='dec.ctrl_sp_all', act=ACT_SOFTPLUS_CLAMP)
        cs = ctrl_sp_all.t.view(B, K + 1, T, 4)
        o = LazyPred()
        o.maps.update(wp_all=wp_all, ctrl_sp_all=ctrl_sp_all, speed=speed, v_traj=v_traj, v_ctrl=v_ctrl, jt=jt, jc=jc,
                      refine_bev=s_bev, refine_flat=s_flat)
        if teacher_forcing_data is not None:
            self._teacher(o, teacher_forcing_data, bev, flat, meas, mlvl, meta, parent_module)
        o['pred_speed'] = speed.t.view(B, 1)
        o['pred_value_traj'], o['pred_features_traj'] = v_traj.t.view(B, 1), jt.t.view(B, 256)
        o['pred_value_ctrl'], o['pred_features_ctrl'] = v_ctrl.t.view(B, 1), jc.t.view(B, 256)
        o['pred_wp'] = wp_all.t.view(B, K + 1, T, 2)
        o['mu_branches'], o['sigma_branches'] = cs[:, :, 0, :2], cs[:, :, 0, 2:]
        o['future_mu'], o['future_sigma'] = cs[:, :, 1:, :2], cs[:, :, 1:, 2:]
        H, W = bev.H, bev.W
        o.lazy('bev_feature', lambda: bev.nchw())
        o.lazy('refine_flattned_BEV_feature', lambda: torch.stack([f.t.view(B, 256) for f in s_flat], 1))
        o.lazy('refine_BEV_feature', lambda: torch.stack([f.nchw() for f in s_bev], 1))
        o.lazy('refine_future_BEV_feature', lambda: torch.stack(
            [f.nchw().reshape(B, T, 32, H, W) for f in s_fut], 1).reshape(B, T, K, 32, H, W).transpose(1, 2))  # quirky view (:481)
        return o

    def _teacher(self, o, data, bev, flat, meas, mlvl, meta, parent_module):
        """Teacher-forced pass (thinktwice_decoder.py:491-533): the K layers again from the coarse BEV / flat features, each fed the
        ground-truth waypoints and controls instead of the previous layer's prediction; only the BEV, flat and future features chain
        from layer to layer.  Adds the teacher_* outputs to `o`."""
        e, T, K = self.eng, self.T, self.K
        B = flat.rows()
        self.stage_teacher(data, B)
        wp = FMap(e.static('tf.wp'), B * T, 1, 1, 2)
        ctrl = e.eltwise(lib.ELT_INV_SOFTPLUS, FMap(e.static('tf.ctrl_sp'), B * T, 1, 1, 4), name='tf.ctrl')
        wp_off = e.fmap('tf.wp_off', B, 1, 1, K * T * 2)
        ctrl_off = e.fmap('tf.ctrl_off', B, 1, 1, K * T * 4)
        cur_bev, cur_flat = bev, flat
        t_bev, t_flat, t_fut = [], [], []
        for k, L in enumerate(self.layers):
            t_off, c_off, fut, cur_bev, cur_flat = self._layer(L, k, wp, ctrl, cur_bev, cur_flat, meas, mlvl, meta, parent_module, 'tf')
            e.copy_cols(FMap(t_off.t, B, 1, 1, T * 2), wp_off.slice(k * T * 2, T * 2))
            e.copy_cols(FMap(c_off.t, B, 1, 1, T * 4), ctrl_off.slice(k * T * 4, T * 4))
            t_bev.append(cur_bev); t_flat.append(cur_flat); t_fut.append(fut)
        H, W = bev.H, bev.W
        o['teacher_pred_wp_offset'] = wp_off.t.view(B, K, T, 2)
        o['teacher_pred_ctrl_offset_lis'] = ctrl_off.t.view(B, K, T, 4)
        o.lazy('teacher_future_BEV_feature', lambda: torch.stack([f.nchw().reshape(B, T, 32, H, W) for f in t_fut], 1))  # plain (:525)
        o.lazy('teacher_refine_flattned_BEV_feature', lambda: torch.stack([f.t.view(B, 256) for f in t_flat], 1))
        o.lazy('teacher_refine_BEV_feature', lambda: torch.stack([f.nchw() for f in t_bev], 1))
        o.maps.update(tf_wp_off=wp_off, tf_ctrl_off=ctrl_off, tf_bev=t_bev, tf_flat=t_flat, tf_fut=t_fut)

    def stage_teacher(self, data, B):
        """host half of the teacher-forced pass: the ground-truth waypoints (B, T, 2) and the softplus-space controls (B, T, 4) =
        [action_mu | action_sigma] at t = 0 and [future_action_mu | future_action_sigma][t - 1] after (thinktwice_decoder.py:496-498),
        from host or device memory into static device buffers.  inv_softplus runs on the device (_teacher)."""
        e = self.eng
        self._check_controls(data, B)
        now = torch.cat([data['action_mu'], data['action_sigma']], -1).float().unsqueeze(1)
        later = torch.cat([torch.stack(list(data['future_action_mu'][:-1]), 1), torch.stack(list(data['future_action_sigma'][:-1]), 1)], -1).float()
        e.upload('tf.wp', data['waypoints'].float().contiguous())
        e.upload('tf.ctrl_sp', torch.cat([now, later.to(now.device)], 1).contiguous())

    # ------------------------------------------------------------------ ground-truth checks
    # The kernels read the ground truth through strides derived from the PREDICTION's shape, so every ground-truth tensor is checked
    # against it first (the reference gets the same errors from F.smooth_l1_loss / torch.distributions.Beta).
    @staticmethod
    def _expect(name, t, shape):
        if t is None or tuple(t.shape) != tuple(shape):
            raise ValueError(f'{name}: expected shape {tuple(shape)}, got {None if t is None else tuple(t.shape)}')

    @staticmethod
    def _beta(name, t):
        """torch.distributions.Beta's argument check (validate_args): concentrations finite and > 0."""
        t = t.float()
        if not bool((torch.isfinite(t) & (t > 0)).all()):
            raise ValueError(f'{name}: Beta concentrations must be finite and > 0')

    def _check_controls(self, data, B):
        T = self.T
        self._expect('waypoints', data['waypoints'], (B, T, 2))
        for k in ('action_mu', 'action_sigma'):
            self._expect(k, data[k], (B, 2))
            self._beta(k, data[k])
        for k in ('future_action_mu', 'future_action_sigma'):
            if len(data[k]) != T:
                raise ValueError(f'{k}: expected {T} entries, got {len(data[k])}')
            for t, v in enumerate(data[k]):
                self._expect(f'{k}[{t}]', v, (B, 2))
                if t < T - 1:                                          # the last entry is not read (thinktwice_decoder.py:498, 575)
                    self._beta(f'{k}[{t}]', v)

    # ------------------------------------------------------------------ losses (thinktwice_decoder.py:535-620)
    DISTIL_WEIGHTS = {2: 0.25, 3: 1.0 / 3.0, 4: 1.0 / 4.0, 5: 1 / 11.0}
    WP_LOSS_WEIGHT = ACTION_LOSS_WEIGHT = 15.0

    def stage_supervision(self, batch, B, mid_BEV_feature):
        """host half of loss(): the ground truth it reads, checked against the shapes of what it is compared with, by name from host or
        device memory into static device buffers."""
        e, T = self.eng, self.T
        self._check_controls(batch, B)
        for k in ('speed', 'value'):                                   # (B, 1) after .view(-1, 1) in the reference (:543-544)
            if batch[k].numel() != B:
                raise ValueError(f'{k}: expected {B} values, got shape {tuple(batch[k].shape)}')
        self._expect('feature', batch['feature'], (B, 256))
        fm = {i: mid_BEV_feature[i] for i in self.DISTIL_WEIGHTS}
        for i, f in fm.items():
            self._expect(f'grid_feature[{i}]', batch['grid_feature'][i], (B, f.C, f.H, f.W))
        if len(batch['future_grid_feature']) != T:
            raise ValueError(f'future_grid_feature: expected {T} entries, got {len(batch["future_grid_feature"])}')
        for t, f in enumerate(batch['future_grid_feature']):
            self._expect(f'future_grid_feature[{t}][2]', f[2], (B, fm[2].C, fm[2].H, fm[2].W))
        e.upload('gt.speed', batch['speed'].to(dtype=torch.float32).reshape(B) / 12.)
        e.upload('gt.value', batch['value'].float().reshape(B).contiguous())
        e.upload('gt.feature', batch['feature'].float().contiguous())
        e.upload('gt.waypoints', batch['waypoints'].float().contiguous())
        for k in ('action_mu', 'action_sigma'):
            e.upload('gt.' + k, batch[k].float().contiguous())
        for k in ('future_action_mu', 'future_action_sigma'):
            e.upload('gt.' + k, torch.stack(list(batch[k][:-1]), 1).float().contiguous())            # (B, T - 1, 2)
        for i in self.DISTIL_WEIGHTS:
            e.upload(f'gt.grid{i}', batch['grid_feature'][i].float().contiguous())
        e.upload('gt.future_grid2', torch.stack([f[2] for f in batch['future_grid_feature']], 1).float().contiguous())   # (B, T, 32, 21, 21)

    def loss(self, batch, pred, mid_BEV_feature):
        """ThinkTwiceDecoder.loss: the reference's dict of 0-d fp32 device tensors ((B, 1) for value_loss), every term reduced by ONE
        tt_loss_reduce launch reading the arena maps in place.  `pred` is the output of a teacher-forced forward, `mid_BEV_feature`
        the fusion's pyramid maps [None, None, 21x21, 10x10, 4x4, 2x2].  Values only: no gradients."""
        e, T, K = self.eng, self.T, self.K
        m = pred.maps
        B = m['speed'].rows()
        if m.get('tf_bev') is None:
            raise ValueError('ThinkTwiceDecoder.loss needs the outputs of a teacher-forced forward')
        self.stage_supervision(batch, B, mid_BEV_feature)
        fw, vw = float(self.config['features_weight']), float(self.config['value_weight'])
        g = e.static
        terms, slots = [], {}

        def slot(name, n=1):                                           # the next n output slots, in the reference's key order
            slots[name] = (sum(c for _, c in slots.values()), n)
            return slots[name][0]

        def term(kind, name, scale, shape, pred, gt=None, pred2=None, gt2=None, aux=0, s=None):
            """pred / gt / pred2 / gt2: (tensor, element offset, element strides) over the logical `shape`; pred2 / gt2 share the strides of
            pred / gt"""
            terms.append(dict(kind=kind, slot=slots[name][0] if s is None else s, scale=scale, shape=shape, aux=aux,
                              pred=lib._p(pred[0], pred[1]), pred_stride=pred[2],
                              pred2=lib._p(pred2[0], pred2[1]) if pred2 else lib._p(None),
                              gt=lib._p(gt[0], gt[1]) if gt else lib._p(None), gt_stride=gt[2] if gt else [0] * len(shape),
                              gt2=lib._p(gt2[0], gt2[1]) if gt2 else lib._p(None)))

        def nchw(fm):                                                  # a channels-last map as a logical (N, C, H, W) tensor
            return fm.t, fm.coff, [fm.H * fm.W * fm.ld, 1, fm.W * fm.ld, fm.ld]

        def rows(fm, n):                                               # (B, n) rows of a (B, 1, 1, >= n) map
            return fm.t, fm.coff, [fm.ld, 1]

        ctrl = m['ctrl_sp_all'].t                                      # (B, K + 1, T, 4) softplus'd controls, [mu 2 | sigma 2]
        cst = [(K + 1) * T * 4, T * 4, 4, 1]
        wp = m['wp_all'].t                                             # (B, K + 1, T, 2)
        wst = [(K + 1) * T * 2, T * 2, 2, 1]
        gwp = g('gt.waypoints')
        L1, SL1, CLAMP, KL, ACT = lib.LOSS_L1, lib.LOSS_SMOOTH_L1, lib.LOSS_SMOOTH_L1_CLAMP, lib.LOSS_BETA_KL, lib.LOSS_ACTION_L1

        # open-loop statistics (:549-561): no 'loss' in their names, so _parse_losses logs them but leaves them out of the total
        for c, name in enumerate(('current_throttle_brake_offset', 'current_steer_offset')):
            slot(name)
            last = K * T * 4 + c                                       # mu_branches[:, -1, c] / sigma_branches[:, -1, c]
            term(ACT, name, 1.0 / B, [B], (ctrl, last, [cst[0]]), pred2=(ctrl, last + 2, [cst[0]]),
                 gt=(g('gt.action_mu'), c, [2]), gt2=(g('gt.action_sigma'), c, [2]), aux=c)
        for c, name in enumerate(('longitudinal_offset', 'lateral_offset')):
            slot(name)
            term(L1, name, 1.0 / (B * T), [B, T], (wp, K * T * 2 + c, [wst[0], 2]), gt=(gwp, c, [T * 2, 2]))
        slot('action_loss')
        term(KL, 'action_loss', self.ACTION_LOSS_WEIGHT / (B * (K + 1) * 2), [B, K + 1, 2], (ctrl, 0, [cst[0], cst[1], 1]),
             pred2=(ctrl, 2, None), gt=(g('gt.action_mu'), 0, [2, 0, 1]), gt2=(g('gt.action_sigma'), 0, None))
        slot('speed_loss')
        term(SL1, 'speed_loss', 1.0 / B, [B], (m['speed'].t, 0, [m['speed'].ld]), gt=(g('gt.speed'), 0, [1]))
        # value_loss (:570) is the (B, 1) tensor (mean_b sl1(v_traj) + sl1(v_ctrl)[b]) * value_weight: one slot per frame
        v0 = slot('value_loss', B)
        for b in range(B):
            term(SL1, 'value_loss', vw / B, [B], (m['v_traj'].t, 0, [m['v_traj'].ld]), gt=(g('gt.value'), 0, [1]), s=v0 + b)
            term(SL1, 'value_loss', vw, [1], (m['v_ctrl'].t, b * m['v_ctrl'].ld, [1]), gt=(g('gt.value'), b, [1]), s=v0 + b)
        slot('flattened_feature_loss')
        for f in (m['jt'], m['jc']):
            term(SL1, 'flattened_feature_loss', fw / (B * 256), [B, 256], rows(f, 256), gt=(g('gt.feature'), 0, [256, 1]))
        slot('future_action_loss')
        term(KL, 'future_action_loss', self.ACTION_LOSS_WEIGHT * 0.25 / (B * (K + 1) * (T - 1) * 2), [B, K + 1, T - 1, 2],
             (ctrl, 4, cst), pred2=(ctrl, 6, None), gt=(g('gt.future_action_mu'), 0, [(T - 1) * 2, 0, 2, 1]),
             gt2=(g('gt.future_action_sigma'), 0, None))
        slot('wp_loss')
        term(SL1, 'wp_loss', self.WP_LOSS_WEIGHT / (B * (K + 1) * T * 2), [B, K + 1, T, 2], (wp, 0, wst), gt=(gwp, 0, [T * 2, 0, 2, 1]))
        gc = lambda t: (t, 0, list(t.stride()))
        for i, wt in self.DISTIL_WEIGHTS.items():                      # encoder BEV features (:588-591)
            fm = mid_BEV_feature[i]
            name = f'BEV_feature_loss{i}'
            slot(name)
            term(CLAMP, name, wt / (fm.N * fm.C * fm.H * fm.W), [fm.N, fm.C, fm.H, fm.W], nchw(fm), gt=gc(g(f'gt.grid{i}')))

        def per_layer(name, maps, scale, gt, shape, view):             # a K-stacked prediction: one term per layer, one slot
            slot(name)
            for fm in maps:
                term(CLAMP, name, scale, shape, view(fm), gt=gt)
        bev = m['refine_bev'][0]
        n_bev = B * 32 * bev.H * bev.W
        grid2 = gc(g('gt.grid2'))
        per_layer('refine_BEV_feature_loss2', m['refine_bev'], self.DISTIL_WEIGHTS[2] / (K * n_bev), grid2, [B, 32, bev.H, bev.W], nchw)
        per_layer('refine_flattened_feature_loss', m['refine_flat'], fw * 0.1 / (K * B * 256), (g('gt.feature'), 0, [256, 1]), [B, 256],
                  lambda f: rows(f, 256))
        # teacher forcing (:600-619): zero-target offsets, future / refined features against the ground truth
        slot('teacher_wp_loss')
        term(SL1, 'teacher_wp_loss', 1.0 / (B * K * T * 2), [B, K * T * 2], rows(m['tf_wp_off'], K * T * 2))
        slot('teacher_action_loss')
        term(SL1, 'teacher_action_loss', 1.0 / (B * K * T * 4), [B, K * T * 4], rows(m['tf_ctrl_off'], K * T * 4))
        HW = bev.H * bev.W

        def fut_view(fm):                                              # (B*T, H, W, 32) channels-last -> (B, T, 32, H, W)
            return fm.t, fm.coff, [T * HW * fm.ld, HW * fm.ld, 1, bev.W * fm.ld, fm.ld]
        per_layer('teacher_future_BEV_feature_loss2', m['tf_fut'], self.DISTIL_WEIGHTS[2] / (K * T * n_bev), gc(g('gt.future_grid2')),
                  [B, T, 32, bev.H, bev.W], fut_view)
        per_layer('teacher_refine_BEV_feature_loss2', m['tf_bev'], self.DISTIL_WEIGHTS[2] / (K * n_bev), grid2, [B, 32, bev.H, bev.W], nchw)
        per_layer('teacher_refine_flattened_feature_loss', m['tf_flat'], fw / (K * B * 256), (g('gt.feature'), 0, [256, 1]), [B, 256],
                  lambda f: rows(f, 256))
        n_slots = sum(c for _, c in slots.values())
        out = e.buf('loss.out', (n_slots,))
        ws = e.buf('loss.ws', (int(lib.load().tt_loss_workspace_bytes(len(terms))),), torch.uint8)
        lib.call('tt_loss_reduce', lib.pack_loss_terms(terms), len(terms), lib._p(out), n_slots, lib._p(ws), C.c_size_t(ws.numel()))
        vals = out.clone()                                             # the caller owns its losses (the arena buffer is reused)
        d = {}
        for name, (s0, n) in slots.items():
            d[name] = vals[s0:s0 + n].view(B, 1) if name == 'value_loss' else vals[s0]
        return d

    def _look_meta(self, B, mlvl):
        e = self.eng
        H_img, W_img = self.config['img_size']
        d = LookDesc()
        d.B, d.num_cams, d.num_query, d.T = B, 4, NQ, self.T
        d.img_w, d.img_h, d.levels = float(W_img), float(H_img), 4
        d.lvl_h, d.lvl_w = lib.i4([m.H for m in mlvl]), lib.i4([m.W for m in mlvl])
        d.C, d.q_dim, d.emb_dim, d.meas_dim, d.flat_dim, d.max_len_cap = 256, 519, 128, 128, 256, NQ
        starts, acc = [], 0
        for m in mlvl:
            starts.append(acc); acc += m.H * m.W
        md = MsdaDesc()
        md.BN, md.rows_cap, md.heads, md.levels, md.points, md.dh = B * 4, NQ, 8, 4, 8, 32
        md.lvl_h, md.lvl_w, md.lvl_start, md.num_keys = d.lvl_h, d.lvl_w, lib.i4(starts), acc
        l2i, idm = e.static('look.l2i'), e.static('look.ida')      # staged by stage()
        return dict(B=B, look_desc=d, msda_desc=md, l2i=l2i, ida=idm, num_keys=acc, lvl_start=starts)
