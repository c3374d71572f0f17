"""BASELINE.json configs[4]: decoder-depth sweep K in {1, 2, 3, 5, 10} at a fixed encoder, one H100 — frames/s at the throughput
batch (16 frames per forward: 32 do not fit 80 GB) and per-frame latency at B = 1, device-timed CUDA-graph replays with resident inputs.

  python tools/k_sweep.py [--batch 16] [--ks 1,2,3,5,10] > k_sweep.json

Weights: the bench's synthetic calibrated checkpoint (K = 5); decoder layers beyond the fifth keep the model's seeded init, layers
the checkpoint has but the model lacks are dropped — the encoder is identical in every run.  Parity per K is the test suite's job
(tests/test_model_gpu.py: K in {1, 2, 3, 10} on the plumbing shape, K = 5 on the full one); this tool only measures.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def measure(cfg, sd, K, B, steps, dev):
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    for c in (cfg.model.decoder.config, cfg.model.train_cfg, cfg.model.test_cfg):
        c['refine_num'] = K
    model = build_model(cfg.model)
    own = model.state_dict()
    model.load_state_dict({k: v for k, v in sd.items() if k in own and own[k].shape == v.shape}, strict=False)
    model.prepare(dev)
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in make_batch(cfg, B, seed=100).items()}
    model.forward_inference(batch)
    model.enable_cuda_graph()
    for _ in range(3):
        model.forward_inference(batch)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        pred = model.forward_inference(batch)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    ok = bool(torch.isfinite(pred['pred_wp']).all()) and tuple(pred['pred_wp'].shape) == (B, K + 1, 4, 2)
    sat = model.f16s_saturations()
    model.release_buffers()
    del model
    torch.cuda.empty_cache()
    return {'K': K, 'batch': B, 'ms_per_step': ms, 'frames_per_s': 1000.0 * B / ms, 'finite': ok, 'f16s_saturated_operands': sat}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--ks', default='1,2,3,5,10')
    args = ap.parse_args()
    from bench import synthetic_checkpoint
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    dev = torch.device('cuda:0')
    sd = torch.load(synthetic_checkpoint(0), map_location='cpu', weights_only=False)['state_dict']
    rows = []
    for K in [int(k) for k in args.ks.split(',')]:
        for B, steps in ((args.batch, 3), (1, 20)):
            try:
                rows.append(measure(Config.fromfile(DEFAULT_CONFIG), sd, K, B, steps, dev))
            except torch.OutOfMemoryError as ex:                      # K = 10 at B = 16 may not fit beside the arena: say so, keep going
                torch.cuda.empty_cache()
                rows.append({'K': K, 'batch': B, 'error': repr(ex)[:200]})
            print(rows[-1], file=sys.stderr, flush=True)
    base = {r['batch']: r for r in rows if r['K'] == 1 and 'ms_per_step' in r}
    for r in rows:
        if 'ms_per_step' in r and r['batch'] in base:
            r['ms_over_K1'] = r['ms_per_step'] - base[r['batch']]['ms_per_step']
    print(json.dumps({'workload': 'configs[4]: decoder-depth sweep at fixed encoder, thinktwice.py shape, 1 x H100, CUDA-graph replay, inputs resident',
                      'rows': rows}))


if __name__ == '__main__':
    main()
