"""Training-side dense convolution: the converted camera trunk (oracle.camera ResNet-50 + PAFPN + neck_conv + DepthNet at thinktwice.py
sizes, BatchNorm in train mode, 32 key-sweep images of 448 x 896 = batch_size_per_gpu 8 x 4 cameras) and every distinct convolution
shape in it, forward alone and forward + backward, three ways alternated in one process:
  ours       thinktwice_b200.ops.conv2d.Conv2d after convert_conv2d (3xTF32 tensor cores, fp32-class);
  torch_fp32 cuDNN with cudnn.allow_tf32 = False, cudnn.benchmark = True;
  torch_tf32 cuDNN with TF32 on (torch's default for convolutions): single-pass TF32, a 10-bit mantissa -- the LOWER-PRECISION
             reference point, not an equal-accuracy comparison.
CUDA events around each step, medians over alternated repetitions, the peak max_memory_allocated increment of one step; the card's
name, power limit and SM clocks are read in the same run.  Layers the library refuses (the stem, the DCN's conv_offset) stay on
torch in every variant, and so does the DCN itself (the oracle's torchvision deform_conv2d).

    python tools/conv2d_train_bench.py [--images 32] [--reps 5] [--warmup 2] [--out results.json] [--table profiles/conv2d_train.md]
"""
import argparse
import copy
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, W, CAMS = 448, 896, 4


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f'nvidia-smi unavailable ({q.returncode})'


class Trunk(nn.Module):
    """the camera branch's key sweep up to the depth / context logits (lss.py:542-560), without the seg head and the lift-splat."""

    def __init__(self):
        from oracle.camera import PAFPN, DepthNet, ResNet50
        super().__init__()
        self.img_backbone, self.img_neck = ResNet50(), PAFPN()
        self.neck_conv = nn.Conv2d(256, 512, 1)
        self.depth_net = DepthNet(512, 512, 256, 80)

    def forward(self, x, mats):
        return self.depth_net(self.neck_conv(self.img_neck(self.img_backbone(x))[2]), mats)


def mats(n_img, dev):
    B = n_img // CAMS
    eye = torch.eye(4, device=dev).expand(B, 1, CAMS, 4, 4).clone()
    intr = eye.clone()
    intr[..., 0, 0] = intr[..., 1, 1] = 800.0
    intr[..., 0, 2], intr[..., 1, 2] = W / 2, H / 2
    return dict(intrin_mats=intr, ida_mats=eye.clone(), sensor2ego_mats=eye.clone())


class Tf32:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = self.on

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.old


def timed(step, variants, reps, warmup):
    """{variant: (median ms, peak MB above the allocation before the step)} for step(variant) alternated rep by rep."""
    for v in variants:
        for _ in range(warmup):
            step(v)
    torch.cuda.synchronize()
    times, peak = {v: [] for v in variants}, {v: 0.0 for v in variants}
    for _ in range(reps):
        for v in variants:
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(v)
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1))
            peak[v] = max(peak[v], (torch.cuda.max_memory_allocated() - base) / 2 ** 20)
    return {v: dict(ms=sorted(t)[len(t) // 2], peak_mb=round(peak[v], 1)) for v, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=32)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    ap.add_argument('--table', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('conv2d_train_bench needs a CUDA device')
    from thinktwice_b200.ops.conv2d import Conv2d, convert_conv2d
    torch.backends.cudnn.benchmark = True
    dev = 'cuda'
    torch.manual_seed(0)
    ref = Trunk().to(dev).train()
    ours, skipped = convert_conv2d(copy.deepcopy(ref))
    x = torch.randn(a.images, 3, H, W, device=dev)
    m = mats(a.images, dev)
    variants = {'ours': (ours, False), 'torch_fp32': (ref, False), 'torch_tf32': (ref, True)}
    res = dict(card=card(), images=a.images, reps=a.reps, skipped=[f'{n}: {why}' for n, _, why in skipped], trunk={}, layers=[])

    # distinct convolution shapes of the trunk at this batch
    shapes = {}

    def hook(mod, inp):
        key = (mod.in_channels, mod.out_channels, mod.kernel_size[0], mod.stride[0], mod.padding[0], mod.dilation[0], mod.bias is not None,
               *inp[0].shape[2:])
        shapes[key] = shapes.get(key, 0) + 1
    hs = [mod.register_forward_pre_hook(hook) for mod in ours.modules() if isinstance(mod, Conv2d)]
    with torch.no_grad():
        ours(x, m)
    for h in hs:
        h.remove()

    def trunk_step(backward):
        def step(v):
            model, tf32 = variants[v]
            with Tf32(tf32):
                if backward:
                    model.zero_grad(set_to_none=True)
                    model(x, m).float().sum().backward()
                else:
                    with torch.no_grad():
                        model(x, m)
        return step
    for mode, bwd in (('forward', False), ('forward_backward', True)):
        try:
            res['trunk'][mode] = timed(trunk_step(bwd), list(variants), a.reps, a.warmup)
        except torch.cuda.OutOfMemoryError as e:                  # reported, not retried at another size
            res['trunk'][mode] = f'out of memory: {str(e).splitlines()[0]}'
            torch.cuda.empty_cache()
        print(mode, res['trunk'][mode], flush=True)

    for (cin, cout, k, s, p, d, bias, h, w), count in sorted(shapes.items(), key=lambda kv: -kv[0][0] * kv[0][1] * kv[0][2] ** 2 * kv[0][7] * kv[0][8]):
        lo = Conv2d(cin, cout, k, stride=s, padding=p, dilation=d, bias=bias).to(dev)
        tl = nn.Conv2d(cin, cout, k, stride=s, padding=p, dilation=d, bias=bias).to(dev)
        tl.load_state_dict(lo.state_dict())
        xi = torch.randn(a.images, cin, h, w, device=dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        layer_v = {'ours': (lo, False), 'torch_fp32': (tl, False), 'torch_tf32': (tl, True)}
        oh, ow = (h + 2 * p - d * (k - 1) - 1) // s + 1, (w + 2 * p - d * (k - 1) - 1) // s + 1
        gy = torch.randn(a.images, cout, oh, ow, device=dev).contiguous(memory_format=torch.channels_last)
        row = dict(shape=f'{cin}->{cout} {k}x{k} s{s} p{p} d{d} {h}x{w}' + (' bias' if bias else ''), count=count,
                   gflop_fwd=round(2 * a.images * oh * ow * cout * cin * k * k / 1e9, 2))
        for mode, bwd in (('forward', False), ('forward_backward', True)):
            def step(v, bwd=bwd):
                layer, tf32 = layer_v[v]
                with Tf32(tf32):
                    if bwd:
                        xi.grad = None
                        layer.zero_grad(set_to_none=True)
                        layer(xi).backward(gy)
                    else:
                        with torch.no_grad():
                            layer(xi)
            row[mode] = timed(step, list(layer_v), a.reps, a.warmup)
        res['layers'].append(row)
        print(row, flush=True)
        del xi, gy, lo, tl
        torch.cuda.empty_cache()

    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')
    if a.table:
        with open(a.table, 'w') as f:
            f.write(table(res))


def table(res):
    out = [f'Card: {res["card"]}; {res["images"]} images of {H} x {W}; medians of {res["reps"]} alternated reps '
           '(`tools/conv2d_train_bench.py`).  torch_tf32 is single-pass TF32 (10-bit mantissa): the lower-precision reference point.', '']
    for mode in ('forward', 'forward_backward'):
        t = res['trunk'].get(mode)
        if isinstance(t, dict):
            out.append(f'Trunk {mode}: ' + ', '.join(f'{v} {r["ms"]:.1f} ms (+{r["peak_mb"]:.0f} MB)' for v, r in t.items()))
        else:
            out.append(f'Trunk {mode}: {t}')
    out += ['', '| layer | calls | GFLOP fwd | fwd ours / fp32 / tf32 (ms) | f+b ours / fp32 / tf32 (ms) | f+b ours vs fp32 |',
            '|---|---|---|---|---|---|']
    for r in res['layers']:
        f, b = r['forward'], r['forward_backward']
        out.append(f'| {r["shape"]} | {r["count"]} | {r["gflop_fwd"]} | {f["ours"]["ms"]:.2f} / {f["torch_fp32"]["ms"]:.2f} / '
                   f'{f["torch_tf32"]["ms"]:.2f} | {b["ours"]["ms"]:.2f} / {b["torch_fp32"]["ms"]:.2f} / {b["torch_tf32"]["ms"]:.2f} | '
                   f'{b["torch_fp32"]["ms"] / b["ours"]["ms"]:.2f}x |')
    return '\n'.join(out) + '\n'


if __name__ == '__main__':
    main()
