"""Training-side deformable convolution: forward and forward + backward at the key sweep of the reference's largest per-GPU training
batch (8 frames x 4 cameras = 32 images x 512 x 28 x 56, groups 4: lss.py:189-197, thinktwice.py:80), ours
(thinktwice_b200.ops.deform_conv) alternated in one process with torchvision's CUDA deform_conv2d (whose kernels descend from the same
DCN code as mmcv's).  CUDA events over warmed-up repetitions; the card's name, power limit and SM clocks are read in the same run.

    python tools/deform_conv_bench.py [--reps 20] [--warmup 3] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

N, C, COUT, H, W, GROUPS = 32, 512, 512, 28, 56, 4


def work():
    """algorithmic work from the shapes: each of the three GEMMs (forward, grad_col, grad_weight) is 2 * K * 9 * (C / groups) * Cout
    flops over the K = N * H * W pixels; the columns are K * 9 * C floats."""
    K = N * H * W
    gemm = 2 * K * 9 * (C // GROUPS) * COUT            # forward, grad_col and grad_weight GEMMs each
    return dict(pixels=K, gflop_per_gemm=gemm / 1e9, column_bytes=K * 9 * C * 4)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f'nvidia-smi unavailable ({q.returncode})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('deform_conv_bench needs a CUDA device')
    from torchvision.ops import deform_conv2d as tv_dcn

    from thinktwice_b200.ops.deform_conv import deform_conv2d
    g = torch.Generator(device='cuda').manual_seed(0)
    x = torch.randn(N, C, H, W, device='cuda', generator=g).requires_grad_(True)
    off = (torch.randn(N, 18, H, W, device='cuda', generator=g) * 2).requires_grad_(True)
    w = (torch.randn(COUT, C // GROUPS, 3, 3, device='cuda', generator=g) * 0.03).requires_grad_(True)
    gy = torch.randn(N, COUT, H, W, device='cuda', generator=g)
    impls = {'ours': lambda: deform_conv2d(x, off, w, 1, 1, 1, GROUPS, 1, False, 128),
             'torchvision': lambda: tv_dcn(x, off, w, padding=1)}

    def fwd(f):
        with torch.no_grad():
            f()

    def fwd_bwd(f):
        x.grad = off.grad = w.grad = None
        f().backward(gy)
    times = {(k, m): [] for k in impls for m in ('forward', 'forward_backward')}
    for mode, step in (('forward', fwd), ('forward_backward', fwd_bwd)):
        for f in impls.values():
            for _ in range(a.warmup):
                step(f)
        torch.cuda.synchronize()
        for _ in range(a.reps):                               # alternate the two implementations rep by rep
            for k, f in impls.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step(f)
                e1.record()
                torch.cuda.synchronize()
                times[(k, mode)].append(e0.elapsed_time(e1))
    res = dict(shape=dict(N=N, C=C, Cout=COUT, H=H, W=W, groups=GROUPS), work=work(), card=card(), reps=a.reps,
               ms={f'{k}.{m}': dict(median=sorted(v)[len(v) // 2], min=min(v), max=max(v)) for (k, m), v in times.items()})
    wk = res['work']
    for k in impls:
        res['ms'][f'{k}.forward']['tflops'] = wk['gflop_per_gemm'] / res['ms'][f'{k}.forward']['median']      # GFLOP / ms = TFLOP/s
        res['ms'][f'{k}.forward_backward']['tflops'] = 3 * wk['gflop_per_gemm'] / res['ms'][f'{k}.forward_backward']['median']
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
