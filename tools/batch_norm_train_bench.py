"""Training-side batch norm: every distinct BatchNorm2d shape of the converted camera trunk (tools/conv2d_train_bench.py's Trunk: ResNet-50
+ PAFPN + neck_conv + DepthNet at thinktwice.py sizes, 32 images of 448 x 896, train mode), forward alone and forward + backward, in
three variants -- BN, BN + ReLU, BN + residual + ReLU -- two ways alternated in one process:
  ours   thinktwice_b200.ops.batch_norm.BatchNorm2d(x, residual=r, relu=...): 3 passes forward, 2 backward (+ 2 tiny folds);
  torch  channels_last F.batch_norm (cuDNN / ATen) followed by add_ and relu_.
Bytes moved are counted from shapes for the library's passes (fp32 rows read and written) and set against the 3.35 TB/s HBM3 figure
of the H100 SXM data sheet.  Then the whole trunk's forward + backward after convert_conv2d + convert_upsampling, with and without
convert_batchnorm.  CUDA events, medians over alternated repetitions; the card's name, power limit and SM clocks are read in the same
run.

    python tools/batch_norm_train_bench.py [--images 32] [--reps 5] [--warmup 2] [--out results.json] [--table profiles/batch_norm_train.md]
"""
import argparse
import copy
import json
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from conv2d_train_bench import H, W, Trunk, card, mats, timed  # noqa: E402

HBM = 3.35e12
VARIANTS = (('bn', False, False), ('bn+relu', True, False), ('bn+res+relu', True, True))


def bytes_moved(M, Cc, relu, res, backward):
    """fp32 bytes the library's passes read and write: stats (x), apply (x, r -> y); reduce (x, gy, r when masked by a residual
    ReLU), apply (x, gy, r -> grad_x, grad_r)."""
    e = 4 * M * Cc
    fwd = e * (1 + 2 + res)
    if not backward:
        return fwd
    rr = 1 if (res and relu) else 0
    return fwd + e * (2 + rr) + e * (2 + rr + 1 + res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=32)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    ap.add_argument('--table', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('batch_norm_train_bench needs a CUDA device')
    from thinktwice_b200.ops.batch_norm import BatchNorm2d, convert_batchnorm
    from thinktwice_b200.ops.conv2d import convert_conv2d
    from thinktwice_b200.ops.conv_transpose2d import convert_upsampling
    torch.backends.cudnn.benchmark = True
    dev = 'cuda'
    torch.manual_seed(0)
    base, _ = convert_conv2d(Trunk().to(dev).train())
    base, _ = convert_upsampling(base)
    ours, skipped, fused = convert_batchnorm(copy.deepcopy(base))
    x = torch.randn(a.images, 3, H, W, device=dev)
    m = mats(a.images, dev)
    res = dict(card=card(), images=a.images, reps=a.reps, skipped=[f'{n}: {why}' for n, _, why in skipped], fused=fused, trunk={},
               layers=[])

    shapes = {}

    def hook(mod, inp):
        if inp[0].dim() == 4:
            key = (mod.num_features, *inp[0].shape[2:])
            shapes[key] = shapes.get(key, 0) + 1
    hs = [mod.register_forward_pre_hook(hook) for mod in base.modules() if type(mod) is nn.BatchNorm2d]
    with torch.no_grad():
        base(x, m)
    for h in hs:
        h.remove()

    def trunk_step(v):
        model = {'ours': ours, 'torch': base}[v]
        model.zero_grad(set_to_none=True)
        model(x, m).float().sum().backward()
    try:
        res['trunk'] = timed(trunk_step, ['ours', 'torch'], a.reps, a.warmup)
    except torch.cuda.OutOfMemoryError as e:                      # reported, not retried at another size
        res['trunk'] = f'out of memory: {str(e).splitlines()[0]}'
    print('trunk forward_backward', res['trunk'], flush=True)
    del ours, base
    torch.cuda.empty_cache()

    for (Cc, h, w), count in sorted(shapes.items(), key=lambda kv: -kv[0][0] * kv[0][1] * kv[0][2]):
        M = a.images * h * w
        lo = BatchNorm2d(Cc).to(dev)
        tw, tb = lo.weight.detach().clone().requires_grad_(True), lo.bias.detach().clone().requires_grad_(True)
        trm, trv = lo.running_mean.clone(), lo.running_var.clone()
        xi = torch.randn(a.images, Cc, h, w, device=dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        ri = torch.randn_like(xi).requires_grad_(True)
        gy = torch.randn_like(xi)
        row = dict(shape=f'{Cc} @ {h}x{w}', count=count, M=M)
        for name, relu, resid in VARIANTS:
            for mode, bwd in (('forward', False), ('forward_backward', True)):
                def step(v, bwd=bwd, relu=relu, resid=resid):
                    r = ri if resid else None
                    with torch.set_grad_enabled(bwd):
                        if v == 'ours':
                            y = lo(xi, residual=r, relu=relu)
                        else:
                            y = F.batch_norm(xi, trm, trv, tw, tb, True, 0.1, 1e-5)
                            if resid:
                                y = y.add_(r)
                            if relu:
                                y = y.relu_()
                        if bwd:
                            xi.grad = ri.grad = lo.weight.grad = lo.bias.grad = tw.grad = tb.grad = None
                            y.backward(gy)
                t = timed(step, ['ours', 'torch'], a.reps, a.warmup)
                gb = bytes_moved(M, Cc, relu, resid, bwd)
                row[f'{name} {mode}'] = dict(ours_ms=t['ours']['ms'], torch_ms=t['torch']['ms'], gbytes=round(gb / 1e9, 3),
                                             roof=round(gb / HBM * 1e3 / t['ours']['ms'], 3))
        res['layers'].append(row)
        print(row, flush=True)
        del xi, ri, gy, lo
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
           '(`tools/batch_norm_train_bench.py`).  roof: the bytes the library\'s passes move over 3.35 TB/s, over our time.', '']
    t = res['trunk']
    if isinstance(t, dict):
        out.append('Trunk forward + backward (after convert_conv2d + convert_upsampling): '
                   f'with convert_batchnorm {t["ours"]["ms"]:.1f} ms (+{t["ours"]["peak_mb"]:.0f} MB), '
                   f'torch batch norm {t["torch"]["ms"]:.1f} ms (+{t["torch"]["peak_mb"]:.0f} MB)')
    else:
        out.append(f'Trunk forward + backward: {t}')
    out.append(f'Fused ReLUs: {len(res["fused"])}; left on torch: {", ".join(res["skipped"]) or "none"}')
    out += ['', '| BN shape | calls | variant | fwd ours / torch (ms) | fwd roof | f+b ours / torch (ms) | f+b roof | f+b speed-up |',
            '|---|---|---|---|---|---|---|---|']
    for r in res['layers']:
        for name, _, _ in VARIANTS:
            f, b = r[f'{name} forward'], r[f'{name} forward_backward']
            sp = b['torch_ms'] / b['ours_ms']
            out.append(f'| {r["shape"]} | {r["count"]} | {name} | {f["ours_ms"]:.3f} / {f["torch_ms"]:.3f} | {f["roof"]:.0%} | '
                       f'{b["ours_ms"]:.3f} / {b["torch_ms"]:.3f} | {b["roof"]:.0%} | {sp:.2f}x{" (slower)" if sp < 1 else ""} |')
    return '\n'.join(out) + '\n'


if __name__ == '__main__':
    main()
