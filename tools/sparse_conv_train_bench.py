"""Time the trainable LiDAR SparseEncoder (thinktwice_b200/ops/sparse_conv.py) against a plain-torch sparse convolution.

usage: python tools/sparse_conv_train_bench.py [--batch 8] [--points 40000] [--reps 10] [--warmup 3] [--json OUT.json]

The input is the seeded synthetic cloud (thinktwice_b200.synthetic.make_batch) voxelised with tt_voxelize_mean, fed to the full
thinktwice.py middle encoder at B = 8 (the reference's per-GPU training batch).  Per convolution layer (on the rulebooks the
encoder's forward built) and for the whole encoder (rulebooks, BatchNorm and ReLU included), forward and forward + backward times are
CUDA-event medians over `reps` repetitions after warm-up, ours and the baseline alternated.  The baseline is a gather / mm / index_add_
sparse convolution in plain torch over the same ordered pair lists, fp32 with TF32 off.  Algorithmic TFLOP/s count 2 * Cin * Cout
multiply-adds per pair (x 3 for forward + backward)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch
from torch.autograd import Function

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from thinktwice_b200 import lib                                          # noqa: E402
from thinktwice_b200.lib import _p                                      # noqa: E402
from thinktwice_b200.ops import sparse_conv as sc                        # noqa: E402


class TorchSparseConv(Function):
    """the baseline: per tap, y[pout] += x[pin] W_t^T; backward gx[pin] += gy[pout] W_t, gW_t = gy[pout]^T x[pin]."""

    @staticmethod
    def forward(ctx, x, w, rb, geom):
        Cout, Cin = w.shape[0], w.shape[-1]
        W = w.reshape(Cout, -1, Cin)
        ctx.save_for_backward(x, w)
        ctx.rb = rb
        y = x.new_zeros(rb.n_out, Cout)
        for t, (pi, po) in enumerate(_pairs(rb)):
            y.index_add_(0, po, x[pi] @ W[:, t].t())
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w = ctx.saved_tensors
        Cout, Cin = w.shape[0], w.shape[-1]
        W = w.reshape(Cout, -1, Cin)
        gx, gw = torch.zeros_like(x), torch.zeros_like(W)
        for t, (pi, po) in enumerate(_pairs(ctx.rb)):
            g = gy[po]
            gx.index_add_(0, pi, g @ W[:, t])
            gw[:, t] = g.t() @ x[pi]
        return gx, gw.view_as(w), None, None


def _pairs(rb):
    if not hasattr(rb, 'torch_pairs'):
        pc = rb.pair_count.tolist() if rb.pair_count is not None else []
        rb.torch_pairs = [(rb.pairs_in[t, :c].long(), rb.pairs_out[t, :c].long()) for t, c in enumerate(pc) if c > 0]
        rb.n_pairs = sum(pc)
    return rb.torch_pairs


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = 'not reported'
    return f'{name} ({q})'


def voxelise(batch, points):
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.synthetic import make_batch
    import numpy as np
    cfg = Config.fromfile(DEFAULT_CONFIG)
    le = cfg.model['lidar_encoder']
    v = le['pts_voxel_layer']
    vs, r = np.asarray(v['voxel_size'], np.float32), np.asarray(v['point_cloud_range'], np.float32)
    pts = make_batch(cfg, batch, seed=0, num_points=points)['points'][:, 0].float().contiguous().cuda()
    B, P, F = pts.shape
    d = lib.VoxelizeDesc()
    d.B, d.P, d.F = B, P, F
    d.lower, d.vsize = lib.f3(r[:3]), lib.f3(vs)
    d.grid = lib.i3([int(g) for g in np.round((r[3:] - r[:3]) / vs)])
    mv = v['max_voxels']
    d.zmax, d.max_points, d.max_voxels, d.cap = le['pts_middle_encoder']['sparse_shape'][0], v['max_num_points'], int(mv[0]), B * P
    ws = torch.empty(lib.load().tt_voxelize_workspace_bytes(C.byref(d)), dtype=torch.uint8, device='cuda')
    feats = torch.empty(B * P, F, device='cuda')
    coords = torch.empty(B * P, 4, dtype=torch.int32, device='cuda')
    count = torch.empty(1, dtype=torch.int32, device='cuda')
    lib.call('tt_voxelize_mean', C.byref(d), _p(pts), _p(feats), _p(coords), _p(count), _p(ws))
    n = int(count.item())
    enc_cfg = {k: v for k, v in le['pts_middle_encoder'].items() if k != 'type'}
    return feats[:n].contiguous(), coords[:n].contiguous(), enc_cfg


def timed(fn, warmup, reps):
    """median ms of fn(ours) and fn(baseline), alternated."""
    for _ in range(warmup):
        fn(True); fn(False)
    ts = {True: [], False: []}
    for _ in range(reps):
        for which in (True, False):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn(which)
            b.record()
            torch.cuda.synchronize()
            ts[which].append(a.elapsed_time(b))
    med = {k: sorted(v)[len(v) // 2] for k, v in ts.items()}
    return med[True], med[False]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--points', type=int, default=40000)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--json')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('sparse_conv_train_bench needs a CUDA device')
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    feats, coords, enc_cfg = voxelise(a.batch, a.points)
    torch.manual_seed(0)
    enc = sc.SparseEncoder(**enc_cfg).cuda().train()
    # capture every conv's input and rulebook from one forward
    layers = []
    orig = sc.SparseConvFunction.apply

    def capture(x, w, rb, geom):
        layers.append((x.detach(), w, rb, geom))
        return orig(x, w, rb, geom)
    sc.SparseConvFunction.apply = capture
    enc(feats, coords, a.batch)
    sc.SparseConvFunction.apply = orig
    names = [n for n, m in enc.named_modules() if isinstance(m, sc.SparseConvolution)]
    rows = []
    for name, (x, w, rb, geom) in zip(names, layers):
        _pairs(rb)
        Cout, Cin = w.shape[0], w.shape[-1]
        xg = x.clone().requires_grad_(True)
        gy = torch.randn(rb.n_out, Cout, device='cuda')

        def fwd(ours):
            with torch.no_grad():
                (orig if ours else TorchSparseConv.apply)(x, w, rb, geom)

        def fb(ours):
            w.grad = None
            xg.grad = None
            (orig if ours else TorchSparseConv.apply)(xg, w, rb, geom).backward(gy)
        f_o, f_b = timed(fwd, a.warmup, a.reps)
        b_o, b_b = timed(fb, a.warmup, a.reps)
        flop = 2.0 * Cin * Cout * rb.n_pairs
        rows.append(dict(layer=name, Cin=Cin, Cout=Cout, sites_in=rb.n_in, sites_out=rb.n_out, pairs=rb.n_pairs, fwd_ms=f_o, fwd_base_ms=f_b,
                         fwd_bwd_ms=b_o, fwd_bwd_base_ms=b_b, fwd_tflops=flop / f_o / 1e9, fwd_bwd_tflops=3 * flop / b_o / 1e9))
    # the whole encoder, rulebooks, BatchNorm and ReLU included
    G = None

    def whole(ours, backward):
        nonlocal G
        sc.SparseConvFunction.apply = orig if ours else TorchSparseConv.apply
        try:
            enc.zero_grad(set_to_none=True)
            xg = feats.clone().requires_grad_(backward)
            if backward:
                y = enc(xg, coords, a.batch)
                if G is None:
                    G = torch.randn_like(y)
                (y * G).sum().backward()
            else:
                with torch.no_grad():
                    enc(xg, coords, a.batch)
        finally:
            sc.SparseConvFunction.apply = orig
    e_f = timed(lambda o: whole(o, False), a.warmup, a.reps)
    e_b = timed(lambda o: whole(o, True), a.warmup, a.reps)
    total_flop = sum(2.0 * r['Cin'] * r['Cout'] * r['pairs'] for r in rows)
    res = dict(card=card(), batch=a.batch, points=a.points, sites=int(feats.shape[0]), reps=a.reps, layers=rows,
               encoder=dict(fwd_ms=e_f[0], fwd_base_ms=e_f[1], fwd_bwd_ms=e_b[0], fwd_bwd_base_ms=e_b[1],
                            conv_flop=total_flop, fwd_tflops=total_flop / e_f[0] / 1e9, fwd_bwd_tflops=3 * total_flop / e_b[0] / 1e9))
    print(f"card: {res['card']}   B = {a.batch}, {res['sites']} voxels, median of {a.reps} alternated reps (ms)")
    print(f"{'layer':40s} {'Cin':>4s} {'Cout':>4s} {'pairs':>9s} {'fwd':>7s} {'base':>7s} {'f+b':>7s} {'base':>7s} {'TF/s f+b':>8s}")
    for r in rows:
        print(f"{r['layer']:40s} {r['Cin']:4d} {r['Cout']:4d} {r['pairs']:9d} {r['fwd_ms']:7.3f} {r['fwd_base_ms']:7.3f} "
              f"{r['fwd_bwd_ms']:7.3f} {r['fwd_bwd_base_ms']:7.3f} {r['fwd_bwd_tflops']:8.2f}")
    e = res['encoder']
    print(f"{'encoder':40s} {'':4s} {'':4s} {'':9s} {e['fwd_ms']:7.3f} {e['fwd_base_ms']:7.3f} {e['fwd_bwd_ms']:7.3f} "
          f"{e['fwd_bwd_base_ms']:7.3f} {e['fwd_bwd_tflops']:8.2f}")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
