"""Serving 16 agents from one GPU: what B = 1 semantics per frame cost with and without the independent-frames mode.

thinktwice.py configuration, 16 frames with ragged LiDAR clouds (40000 / 31000 / 5000 points, one frame with no point in range, passed
as a list of per-frame clouds), inputs resident on the device, CUDA-graph replay.  Three variants, alternated in one process:
  (a) coupled:     one B = 16 forward, reference batch semantics (a frame's result depends on the batch);
  (b) independent: one B = 16 forward with enable_independent_frames() (every frame as if alone);
  (c) sequential:  16 B = 1 forwards, one per frame (a second model instance, so neither arena is released).
Reports medians over the rounds of the per-step time of each variant, the device name and power limit read in the same process, and
the largest difference of (a) and (b) from (c) per output (relative to the output's largest magnitude over the 16 frames).
Weights: seeded random init with BatchNorm statistics calibrated by one oracle pass (as bench.py's synthetic checkpoint).

  python tools/batched_agents_bench.py [--rounds 5] [--steps 3] > batched_agents.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

LENGTHS = [40000, 31000, 5000, 40000, 31000, 5000, 40000, 40000, 31000, 5000, 40000, 31000, 5000, 40000, 31000, 40000]
EMPTY = 4                                    # this frame's cloud lies outside point_cloud_range: no voxel
OUTPUTS = ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed', 'pred_value_traj', 'pred_value_ctrl')


def device_info():
    idx = torch.cuda.current_device()
    info = {'device': torch.cuda.get_device_name(idx), 'power_limit_w': None, 'sm_max_mhz': None}
    try:
        r = subprocess.run(['nvidia-smi', f'--id={idx}', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader,nounits'],
                           capture_output=True, text=True, timeout=10).stdout.strip().split(',')
        info['power_limit_w'], info['sm_max_mhz'] = float(r[0]), float(r[1])
    except Exception as ex:                                            # reported as unknown, never guessed
        info['power_query_error'] = str(ex)
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5, help='alternations of (a), (b), (c); medians are taken over them (>= 3)')
    ap.add_argument('--steps', type=int, default=3, help='timed steps of each variant per round')
    ap.add_argument('--seed', type=int, default=50)
    args = ap.parse_args()
    assert args.rounds >= 3
    if not torch.cuda.is_available():
        raise SystemExit('batched_agents_bench.py measures on a CUDA device; none is present')
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, 0)
    calibrate_bn(oracle, make_batch(cfg, 1, seed=0))
    sd = oracle.state_dict()
    del oracle

    def model():
        m = build_model(cfg.model)
        m.load_state_dict(sd)
        return m.prepare('cuda:0').enable_cuda_graph()
    m16, m1 = model(), model()
    B = len(LENGTHS)
    host = make_batch(cfg, B, seed=args.seed, num_points=max(LENGTHS))
    clouds = [host['points'][j, :, :n].clone() for j, n in enumerate(LENGTHS)]
    clouds[EMPTY][..., 0] = 1000.0
    host['points'] = clouds
    dev = {k: ([x.cuda() for x in v] if k == 'points' else v.cuda() if torch.is_tensor(v) else v) for k, v in host.items()}
    singles = [{k: v[j:j + 1] for k, v in dev.items()} for j in range(B)]

    def coupled():
        m16.enable_independent_frames(False)
        return m16.forward_inference(dev)

    def independent():
        m16.enable_independent_frames(True)
        return m16.forward_inference(dev)

    def sequential():
        return [m1.forward_inference(s) for s in singles]
    variants = {'a_b16_coupled': coupled, 'b_b16_independent': independent, 'c_16x_b1': sequential}
    outs = {}
    for name, fn in variants.items():                                  # eager pass + capture, then one replay
        for _ in range(2):
            p = fn()
        torch.cuda.synchronize()
        if name == 'c_16x_b1':
            outs[name] = {k: torch.cat([q[k].float().cpu() for q in p], 0) for k in OUTPUTS}
        else:
            outs[name] = {k: p[k].float().cpu() for k in OUTPUTS}
    ms = {name: [] for name in variants}
    for _ in range(args.rounds):
        for name, fn in variants.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            for _ in range(args.steps):
                fn()
            t1.record()
            torch.cuda.synchronize()
            ms[name].append(t0.elapsed_time(t1) / args.steps)
    med = {name: statistics.median(v) for name, v in ms.items()}
    ref = outs['c_16x_b1']

    def diff(name):
        return {k: float((outs[name][k] - ref[k]).abs().max() / ref[k].abs().max().clamp_min(1e-12)) for k in OUTPUTS}
    res = dict(what='16 agents on one GPU, thinktwice.py, ragged LiDAR clouds, device-resident inputs, CUDA-graph replay; ms per step of 16 frames',
               **device_info(), rounds=args.rounds, steps_per_round=args.steps, frames=B, point_counts=LENGTHS, empty_frame=EMPTY,
               median_ms={k: round(v, 2) for k, v in med.items()},
               frames_per_s={k: round(1000.0 * B / v, 2) for k, v in med.items()},
               speedup_b_over_c=round(med['c_16x_b1'] / med['b_b16_independent'], 3),
               b_over_a_time=round(med['b_b16_independent'] / med['a_b16_coupled'], 3),
               all_ms={k: [round(x, 2) for x in v] for k, v in ms.items()},
               max_rel_diff_vs_c={'a_b16_coupled': diff('a_b16_coupled'), 'b_b16_independent': diff('b_b16_independent')})
    print(json.dumps(res))


if __name__ == '__main__':
    main()
