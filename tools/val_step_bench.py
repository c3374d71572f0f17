"""Time of one open-loop validation step — `forward(is_eval=True, **batch)` with the supervision keys: both sweeps encoded, the decoder's
main and teacher-forced passes, every loss term (one tt_loss_reduce launch), _parse_losses — against one eager `forward_inference` on
the same batch, in the same process, the two alternated step by step.  Full thinktwice.py config with depth / segmentation supervision
off, device-resident batch.  The card's name, power limit and SM clocks are read in the same call (nvidia-smi queries only).

    python tools/val_step_bench.py [--batch 16] [--steps 7]     -> one JSON line (milliseconds: median, min, max over --steps)
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
    args = ap.parse_args()
    cfg = Config.fromfile(DEFAULT_CONFIG)
    for k in ('use_depth', 'use_seg'):
        cfg.merge_from_dict({f'model.train_cfg.{k}': False})
    m = build_model(cfg.model).prepare('cuda:0')
    batch = make_batch(cfg, args.batch, seed=0, num_points=40000, device='cuda')
    sup = make_supervision(cfg, args.batch, seed=0, device='cuda')

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3
    runs = {'inference_eager': lambda: m.forward_inference(batch), 'validation_step': lambda: m.forward(is_eval=True, **batch, **sup)}
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
    print(json.dumps(out))


if __name__ == '__main__':
    main()
