"""Time of one open-loop validation step — `forward(is_eval=True, **batch)` with the supervision keys: both sweeps encoded, the decoder's
main and teacher-forced passes, every loss term (one tt_loss_reduce launch), _parse_losses — against one eager `forward_inference` on
the same batch, in the same process, the two alternated step by step.  Full thinktwice.py config with depth / segmentation supervision
off, device-resident batch.  The card's name, power limit and SM clocks are read in the same call (nvidia-smi queries only).

    python tools/val_step_bench.py [--batch 16] [--steps 7]     -> one JSON line (milliseconds: median, min, max over --steps)

--camera-supervision: the config's use_depth / use_seg as shipped (on) and the camera ground truth in the batch.  The validation step
with seg_loss and depth_loss is then alternated with the same step with the two flags off, and the tt_camera_loss launch is timed alone
(CUDA events over --launches launches on the staged ground truth), next to the bytes it must read, computed from the shapes.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_state(index):
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        r = subprocess.run(['nvidia-smi', f'--id={index}', f'--query-gpu={q}', '--format=csv,noheader,nounits'], capture_output=True,
                           text=True, timeout=20)
        name, limit, sm, sm_max = [v.strip() for v in r.stdout.strip().split(',')]
        return dict(name=name, power_limit_w=float(limit), sm_mhz=float(sm), sm_max_mhz=float(sm_max))
    except Exception as ex:                                          # the numbers are still printed, marked as unqualified
        return dict(error=str(ex))


def main():
    import torch
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch, make_supervision
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--steps', type=int, default=7)
    ap.add_argument('--camera-supervision', action='store_true')
    ap.add_argument('--launches', type=int, default=50)
    args = ap.parse_args()
    cfg = Config.fromfile(DEFAULT_CONFIG)
    if not args.camera_supervision:
        for k in ('use_depth', 'use_seg'):
            cfg.merge_from_dict({f'model.train_cfg.{k}': False})
    m = build_model(cfg.model).prepare('cuda:0')
    batch = make_batch(cfg, args.batch, seed=0, num_points=40000, device='cuda')
    sup = make_supervision(cfg, args.batch, seed=0, device='cuda')
    if args.camera_supervision:
        from thinktwice_b200.synthetic import make_camera_supervision
        sup.update(make_camera_supervision(cfg, args.batch, seed=0, device='cuda'))

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3
    runs = {'inference_eager': lambda: m.forward_inference(batch), 'validation_step': lambda: m.forward(is_eval=True, **batch, **sup)}
    if args.camera_supervision:
        def without_camera():
            m.config['use_depth'] = m.config['use_seg'] = False
            try:
                m.forward(is_eval=True, **batch, **sup)
            finally:
                m.config['use_depth'] = m.config['use_seg'] = True
        runs['validation_step_no_camera'] = without_camera
    for fn in runs.values():                                         # the first call of each allocates its buffers
        timed(fn)
    ts = {k: [] for k in runs}
    state = [gpu_state(torch.cuda.current_device())]
    for _ in range(args.steps):                                      # alternated: both see the same host / clock conditions
        for k, fn in runs.items():
            ts[k].append(timed(fn))
    state.append(gpu_state(torch.cuda.current_device()))
    stat = lambda v: dict(median=round(sorted(v)[len(v) // 2], 2), min=round(min(v), 2), max=round(max(v), 2))
    out = {k + '_ms': stat(v) for k, v in ts.items()}
    out.update(batch=args.batch, steps=args.steps, gpu=state,
               ratio=round(out['validation_step_ms']['median'] / out['inference_eager_ms']['median'], 3))
    if args.camera_supervision:
        out['camera_loss_kernel'] = camera_kernel(m, batch, sup, args.launches)
    print(json.dumps(out))


def camera_kernel(m, batch, sup, launches):
    """tt_camera_loss alone on the ground truth the last step staged: milliseconds per launch (CUDA events around `launches` launches)
    and the bytes the launch must read (the C logits of each segmentation pixel, its label, each depth block, the D logits of a cell)."""
    import torch
    m.forward(is_eval=True, **batch, **sup)
    terms, cam = m._camera_terms(), m.last_cam_feat
    d = m.stage_camera_supervision(sup, cam, terms)
    m.launch_camera_loss(d)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        m.launch_camera_loss(d)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / launches
    sg, dp = cam['seg'], cam['depth']
    f, D = m.downsample_factor, m.img_encoder.depth_channels
    parts = dict(seg_logits=sg.N * sg.H * sg.W * sg.C * 4, seg_labels=sg.N * sg.H * sg.W * 4,
                 depth_gt=dp.N * dp.H * dp.W * f * f * 4, depth_logits=dp.N * dp.H * dp.W * D * 4)
    total = sum(parts.values())
    return dict(ms=round(ms, 4), launches=launches, bytes={k: v for k, v in parts.items()}, total_bytes=total,
                effective_tb_s=round(total / (ms * 1e-3) / 1e12, 3))


if __name__ == '__main__':
    main()
