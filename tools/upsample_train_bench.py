"""Training-side upsampling: the layers of a training step that torch/cuDNN ran before convert_upsampling, at 32 camera images
(batch_size_per_gpu 8 x 4 cameras) and 8 LiDAR BEVs, forward alone and forward + backward, three ways alternated in one process:
  ours       thinktwice_b200.ops ConvTranspose2d / interpolate_bilinear (3xTF32 tensor cores; a gather backward without atomics);
  torch_fp32 cuDNN with cudnn.allow_tf32 = False, cudnn.benchmark = True (the bilinear op is the same for both torch rows);
  torch_tf32 torch's default: single-pass TF32 transposed convolutions, a 10-bit mantissa -- the LOWER-PRECISION reference point.
The layers: the UNet seg head's three k2s2 deconvs and its bilinear x2 (lss.py:246, 267), the ASPP pooling branch's 1 x 1 -> 28 x 56
bilinear broadcast, the SECONDFPN deblock (k2s2, no bias), and the whole UNet head (convolutions through convert_conv2d).  CUDA events
around each step, medians over alternated repetitions, the peak max_memory_allocated increment of one step, and for the bilinear layers
the achieved bytes/s (bytes the op must move: read the input, write the output; backward: read grad_y, write grad_x) against the H100
SXM's 3.35 TB/s HBM3.  The card's name, power limit and SM clocks are read in the same run.

    python tools/upsample_train_bench.py [--reps 7] [--warmup 2] [--out results.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12
IMAGES, BEVS = 32, 8


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f'nvidia-smi unavailable ({q.returncode})'


class Interp(nn.Module):
    def __init__(self, size, ours):
        super().__init__()
        self.size, self.ours = size, ours

    def forward(self, x):
        if self.ours:
            from thinktwice_b200.ops.interpolate import interpolate_bilinear
            return interpolate_bilinear(x, size=self.size)
        return F.interpolate(x, size=self.size, mode='bilinear', align_corners=True)


class Head(nn.Module):
    """oracle.camera.UNet on its four FPN maps."""

    def __init__(self):
        from oracle.camera import UNet
        super().__init__()
        self.unet = UNet(12, (256, 256, 256, 256))

    def forward(self, *feats):
        return self.unet(list(feats))


def cases(dev):
    """(name, module factory(ours), input shapes, bilinear bytes or None)."""
    def deconv(cin, cout, bias):
        return lambda: nn.ConvTranspose2d(cin, cout, 2, stride=2, bias=bias)
    cl = []
    for cin, cout, h, w in ((256, 256, 14, 28), (256, 256, 28, 56), (256, 128, 56, 112)):
        cl.append((f'up {cin}->{cout} {h}x{w}', deconv(cin, cout, True), [(IMAGES, cin, h, w)], None))
    cl.append(('deblock 256->256 42x42 (8 BEVs)', deconv(256, 256, False), [(BEVS, 256, 42, 42)], None))
    cl.append(('bilinear x2 128ch 112x224', lambda: nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True),
               [(IMAGES, 128, 112, 224)], (IMAGES * 128 * 112 * 224 * 4, IMAGES * 128 * 224 * 448 * 4)))
    cl.append(('broadcast 512ch 1x1->28x56', None, [(IMAGES, 512, 1, 1)], (IMAGES * 512 * 4, IMAGES * 512 * 28 * 56 * 4)))
    cl.append(('UNet head', Head, [(IMAGES, 256, 112, 224), (IMAGES, 256, 56, 112), (IMAGES, 256, 28, 56), (IMAGES, 256, 14, 28)], None))
    return cl


def build(factory, name, variant, dev):
    from thinktwice_b200.ops.conv2d import convert_conv2d
    from thinktwice_b200.ops.conv_transpose2d import convert_upsampling
    torch.manual_seed(0)
    m = Interp((28, 56), variant == 'ours') if factory is None else factory()
    m = m.to(dev).train()
    if variant == 'ours':
        m, _ = convert_conv2d(m)
        m, skipped = convert_upsampling(m)
        assert not skipped, skipped
    return m


def step(m, xs, backward):
    y = m(*xs)
    if backward:
        y.backward(y.detach())
    return y


def run(args):
    dev = 'cuda'
    torch.backends.cudnn.benchmark = True
    res = {'card': card(), 'images': IMAGES, 'bevs': BEVS, 'layers': {}}
    print(res['card'])
    for name, factory, shapes, nbytes in cases(dev):
        xs = [torch.randn(s, device=dev).contiguous(memory_format=torch.channels_last) for s in shapes]
        mods = {v: build(factory, name, v, dev) for v in ('ours', 'torch_fp32', 'torch_tf32')}
        row = {}
        for mode in ('fwd', 'fwd+bwd'):
            bwd = mode == 'fwd+bwd'
            inputs = [x.clone().requires_grad_(bwd) for x in xs]
            times = {v: [] for v in mods}
            peak = {}
            for rep in range(args.warmup + args.reps):
                for v, m in mods.items():
                    torch.backends.cudnn.allow_tf32 = v == 'torch_tf32'
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    base = torch.cuda.memory_allocated()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    with torch.set_grad_enabled(bwd):
                        y = step(m, inputs, bwd)
                    e1.record()
                    torch.cuda.synchronize()
                    del y
                    for t in inputs:
                        t.grad = None
                    m.zero_grad(set_to_none=True)
                    if rep >= args.warmup:
                        times[v].append(e0.elapsed_time(e1))
                        peak[v] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
            for v in mods:
                ms = statistics.median(times[v])
                r = {'ms': ms, 'peak_MiB': peak[v]}
                if nbytes is not None:
                    moved = nbytes[0] + nbytes[1] + (nbytes[1] + nbytes[0] if bwd else 0)
                    r['GB/s'] = moved / (ms * 1e-3) / 1e9
                    r['of_hbm'] = moved / (ms * 1e-3) / HBM
                row.setdefault(v, {})[mode] = r
        res['layers'][name] = row
        print(name, json.dumps(row))
        del mods, xs
        torch.cuda.empty_cache()
    torch.backends.cudnn.allow_tf32 = True
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('upsample_train_bench needs a CUDA device (nothing is measured without one)')
    res = run(args)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
