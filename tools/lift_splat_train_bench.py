"""Training lift-splat benchmark at thinktwice.py shapes (N = 4, C = 256, D = 80, 28 x 56, rig matrices), default B = 8.

Variants, alternated rep by rep, CUDA-event medians:
  fused       : thinktwice_b200.ops.lift_splat (tt_lift_splat_train_forward / _backward), forward and forward + backward;
  composition : lss.py:583-615 in fp32 torch: softmax, outer product, permute + .contiguous(), thinktwice_b200.ops.voxel_pooling,
                geometry and voxel index included, forward and forward + backward;
  inference   : the inference tt_lift_splat on channels-last copies of the same tensors (forward only: it has no backward).
Also the torch.cuda.max_memory_allocated increment of each variant's forward + backward (forward for inference), and the card's
name and power limit read in the same run.  Usage: python tools/lift_splat_train_bench.py [--batch 8] [--reps 20] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from thinktwice_b200 import lib  # noqa: E402
from thinktwice_b200.ops.lift_splat import lift_splat  # noqa: E402
from thinktwice_b200.ops.voxel_pooling import voxel_pooling  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = 'not reported'
    return f'{name} ({q})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--json')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('lift_splat_train_bench needs a CUDA device')
    from oracle.camera import LSS as OLSS
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.lss import LSS
    from thinktwice_b200.synthetic import rig_metas
    cfg = Config.fromfile(DEFAULT_CONFIG)
    m = LSS(**{k: v for k, v in cfg.model['img_encoder'].items() if k != 'type'})
    B, N, D, fH, fW, Cc = a.batch, len(cfg.model['decoder']['config']['camera_names']), m.depth_channels, m.fH, m.fW, m.output_channels
    mats = LSS.build_mats([rig_metas(tuple(m.final_dim), m.queue_len) for _ in range(B)], N)
    s2e, intr, ida = (mats[k][:, -1].cuda() for k in ('sensor2ego_mats', 'intrin_mats', 'ida_mats'))
    g = torch.Generator().manual_seed(0)
    depth_feature = torch.randn(B * N, D + Cc, fH, fW, generator=g).cuda() * 3
    feat = torch.randn(B * N, Cc, fH, fW, generator=g).cuda()
    G = torch.randn(B, Cc, int(m.voxel_num[1]), int(m.voxel_num[0]), generator=g).cuda()
    ns = types.SimpleNamespace(frustum=m.frustum.cuda(), voxel_coord=m.voxel_coord.cuda(), voxel_size=m.voxel_size.cuda())
    vn = m.voxel_num.cuda()
    # the inference op's inputs: ida^-1 | sensor2ego @ intrin^-1 as LSS.stage makes them, the frustum floats, the grid
    h = lambda t: t.cpu()
    kmats = torch.stack([torch.inverse(h(ida)), h(s2e).matmul(torch.inverse(h(intr)))], 2).reshape(B * N, 32).cuda()
    d = lib.LiftSplatDesc()
    d.B, d.N, d.D, d.fH, d.fW, d.C = B, N, D, fH, fW, Cc
    d.ld_d, d.d_coff, d.ld_c, d.c_coff = D, 0, Cc, 0
    vs = m.voxel_size.float()
    d.lower, d.size = lib.f3((m.voxel_coord.float() - vs / 2.0).tolist()), lib.f3(vs.tolist())
    d.X, d.Y, d.Z = (int(v) for v in m.voxel_num)
    d.bev_ld, d.bev_coff, d.anti_transpose = Cc, 0, 0
    ws = torch.empty(lib.load().tt_lift_splat_workspace_bytes(C.byref(d)), dtype=torch.uint8, device='cuda')
    fu, fv, fd = m.frustum_u.cuda(), m.frustum_v.cuda(), m.frustum_d.cuda()

    def fused(backward):
        x, f = depth_feature.requires_grad_(backward), feat.requires_grad_(backward)
        out = lift_splat(x[:, :D], f, s2e, intr, ida, m.frustum, m.voxel_coord, m.voxel_size, m.voxel_num)
        if backward:
            out.backward(G)

    def composition(backward):
        x, f = depth_feature.requires_grad_(backward), feat.requires_grad_(backward)
        lifted = x[:, :D].softmax(1).unsqueeze(1) * f.unsqueeze(2)
        lifted = lifted.reshape(B, N, Cc, D, fH, fW).permute(0, 1, 3, 4, 5, 2).contiguous()
        idx = OLSS.geom_index(ns, OLSS.get_geometry(ns, s2e, intr, ida)).contiguous()
        out = voxel_pooling(idx, lifted, vn)
        if backward:
            out.backward(G)

    def inference(backward):
        bev = torch.empty(B, d.Y, d.X, Cc, device='cuda')
        dl = depth_feature[:, :D].permute(0, 2, 3, 1).contiguous()
        cl = feat.permute(0, 2, 3, 1).contiguous()
        lib.call('tt_lift_splat', C.byref(d), lib._p(dl), lib._p(cl), lib._p(kmats), lib._p(fu), lib._p(fv), lib._p(fd), lib._p(bev),
                 lib._p(ws))
    variants = {'fused': fused, 'composition': composition, 'inference': inference}
    res = dict(card=card(), batch=B, reps=a.reps, shape=dict(N=N, C=Cc, D=D, fH=fH, fW=fW), ms={}, peak_mib={})
    for mode in ('forward', 'forward+backward'):
        bw = mode != 'forward'
        names = [n for n in variants if not (bw and n == 'inference')]
        for n in names:                                              # peak memory of one call, from a fresh baseline
            depth_feature.grad = feat.grad = None
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            variants[n](bw)
            torch.cuda.synchronize()
            res['peak_mib'][f'{n} {mode}'] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        for _ in range(a.warmup):
            for n in names:
                variants[n](bw)
        ts = {n: [] for n in names}
        for _ in range(a.reps):
            for n in names:
                depth_feature.grad = feat.grad = None
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                variants[n](bw)
                e1.record()
                torch.cuda.synchronize()
                ts[n].append(e0.elapsed_time(e1))
        for n in names:
            res['ms'][f'{n} {mode}'] = sorted(ts[n])[len(ts[n]) // 2]
    print(f"card: {res['card']}   B = {B}, median of {a.reps} alternated reps")
    for k in res['ms']:
        print(f"  {k:32s} {res['ms'][k]:9.3f} ms   peak +{res['peak_mib'][k]:9.1f} MiB")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
