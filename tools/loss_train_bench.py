"""Training losses benchmark at thinktwice.py shapes (N = 4 cameras, seg (BN, 12, 224, 448) against 448 x 896 labels, depth (BN, 80,
28, 56) as a view of an (80 + 64)-channel map against 448 x 896 depths, K = 5, T = 4), default B = 16.

Variants, alternated rep by rep, CUDA-event medians:
  ours  : thinktwice_b200.ops.losses.camera_losses (forward; forward + backward) and decoder_loss (forward + backward);
  torch : the fp32 torch composition of the reference's lines (tests/camera_loss_oracle.camera_loss, tests/loss_oracle.decoder_loss),
          TF32 off.
Also: the bytes each of our kernels must move (counted from the shapes) and the bandwidth that implies against the H100 SXM data
sheet's 3.35 TB/s; the torch.cuda.max_memory_allocated increment of each forward + backward; the decoder half's launch count (ours:
the library's counter; torch: CUDA kernels in a torch.profiler trace of one forward + backward); the card's name and power limit read
in the same run.  Usage: python tools/loss_train_bench.py [--batch 16] [--reps 20] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from thinktwice_b200 import lib  # noqa: E402
from thinktwice_b200.ops.losses import camera_losses, decoder_loss  # noqa: E402

HBM_TBS = 3.35    # NVIDIA H100 SXM data sheet, HBM3


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = 'not reported'
    return f'{name} ({q})'


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--json')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('loss_train_bench needs a CUDA device')
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    import camera_loss_oracle as CO
    import loss_oracle as LO
    import loss_train_reference as R
    from test_loss_train_gpu import camera_inputs, gpu_inputs, model_ns
    B = a.batch
    seg, depth, lab, dep = camera_inputs(B)
    seg.requires_grad_(); depth.requires_grad_()
    P, M, batch = gpu_inputs(B)
    batch32 = R.batch_as(batch, torch.float32, 'cuda')
    dec, model = R.decoder_module(), model_ns()
    leaves = [P[k] for k in R.PRED_KEYS] + M[2:]

    def cam_ours(bwd):
        d = camera_losses(model, dict(seg=lab, depth=dep), dict(seg=seg, depth=depth))
        if bwd:
            torch.autograd.grad(d['seg_loss'] + d['depth_loss'], (seg, depth))

    def cam_torch(bwd):
        d = CO.camera_loss(dict(use_seg=True, use_depth=True), dict(seg=lab, depth=dep), seg, depth, R.DBOUND)
        if bwd:
            torch.autograd.grad(d['seg_loss'] + d['depth_loss'], (seg, depth))

    def total(d):
        return sum(v.mean() for k, v in d.items() if 'loss' in k)

    def dec_ours():
        torch.autograd.grad(total(decoder_loss(dec, batch32, P, M)), leaves)

    def dec_torch():
        torch.autograd.grad(total(LO.decoder_loss(R.CONFIG, batch32, P, M)), leaves)

    variants = {'camera_fwd': (lambda: cam_ours(False), lambda: cam_torch(False)), 'camera_fwd_bwd': (lambda: cam_ours(True), lambda: cam_torch(True)),
                'decoder_fwd_bwd': (dec_ours, dec_torch)}
    for _ in range(a.warmup):
        for o, t in variants.values():
            o(); t()
    times = {k: ([], []) for k in variants}
    for _ in range(a.reps):
        for k, (o, t) in variants.items():
            times[k][0].append(timed(o))
            times[k][1].append(timed(t))
    res = dict(card=card(), batch=B, reps=a.reps)
    for k, (o, t) in times.items():
        res[k] = dict(ours_ms=statistics.median(o), torch_ms=statistics.median(t))
    # bytes our kernels must move: the forward reads every seg logit and label it uses once, every depth and depth logit once, and
    # writes one target byte per logit pixel; the backward reads the logits and targets once and writes the gradients once
    BN = 4 * B
    seg_px, dcell = BN * 224 * 448, BN * 28 * 56
    fwd_bytes = seg_px * (12 * 4 + 4 + 1) + dcell * (16 * 16 * 4 + 80 * 4 + 1)
    bwd_bytes = seg_px * (12 * 4 * 2 + 1) + dcell * (80 * 4 * 2 + 1)
    res['camera_fwd']['bytes'] = fwd_bytes
    res['camera_fwd_bwd']['bytes'] = fwd_bytes + bwd_bytes
    for k in ('camera_fwd', 'camera_fwd_bwd'):
        r = res[k]
        r['ours_TBs'] = r['bytes'] / (r['ours_ms'] * 1e-3) / 1e12
        r['share_of_datasheet_hbm'] = r['ours_TBs'] / HBM_TBS
    res['camera_peak_MiB'] = dict(ours=peak(lambda: cam_ours(True)), torch=peak(lambda: cam_torch(True)))
    res['decoder_peak_MiB'] = dict(ours=peak(dec_ours), torch=peak(dec_torch))
    n0 = lib.launch_count()
    dec_ours()
    torch.cuda.synchronize()
    ours_lib = lib.launch_count() - n0
    counts, kernel_ms = {}, {}
    for name, fn in (('ours', dec_ours), ('torch', dec_torch)):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA]
        counts[name] = sum(e.count for e in ev)
        kernel_ms[name] = sum(e.self_device_time_total for e in ev) / 1e3
        if name == 'ours':
            kernel_ms['ours_loss_kernels'] = {e.key[:60]: e.self_device_time_total / 1e3 for e in ev if 'loss' in e.key}
    res['decoder_launches'] = dict(ours_library=ours_lib, ours_all_cuda_ops=counts['ours'], torch_all_cuda_ops=counts['torch'])
    res['decoder_device_ms'] = kernel_ms
    print(json.dumps(res, indent=1))
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
