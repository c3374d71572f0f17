"""Run the kernel census (tests/kernel_census.py) outside pytest: one eager forward of the full thinktwice.py model (oracle weights,
calibrated BatchNorm) with every C ABI call checked against float64 on the activations it received, then the per-entry table and every
failing call (index, entry, layer, launches, impl, worst element).  The gate for kernel changes: every ratio must stay below 1.

From B = 8 up (or with --window) each convolution is checked on windows of whole images / >= 256 rows at the start and the end of its
N, and a call of another entry whose fp64 copies would pass 4 GB is counted as skipped: the B = 16 arena leaves no room for whole
copies.  At smaller B every tensor is checked whole, with the writes-outside-the-destination check.

usage: python tools/kernel_census.py [--batch B] [--independent] [--window] [--stop]
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import pytest
import torch

import kernel_census as KC


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=1)
    ap.add_argument('--independent', action='store_true', help='independent-frames Look mode')
    ap.add_argument('--window', action='store_true', help='windowed checks (the default from B = 8)')
    ap.add_argument('--stop', action='store_true', help='stop at the first failing call')
    ap.add_argument('--seed', type=int, default=0)
    args = ap.parse_args()
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, args.seed)
    calibrate_bn(oracle, make_batch(cfg, 1, seed=args.seed, num_points=40000))
    model = build_model(cfg.model)
    model.load_state_dict(oracle.state_dict())
    model.prepare('cuda:0')
    model.enable_independent_frames(args.independent)
    batch = make_batch(cfg, args.batch, seed=7 + args.batch, num_points=40000)
    window = args.window or args.batch >= 8
    t0 = time.time()
    with pytest.MonkeyPatch.context() as mp:
        census = KC.install(mp, KC.Census(model.eng, stop=args.stop, outside=not window, window=window, cap=(4 << 30) if window else None))
        try:
            model.forward_inference(batch)
            KC.inverse_softplus(model.eng)
        except KC.CensusError as e:
            print(e)
        torch.cuda.synchronize()
    ws, call, entry = census.peak
    print(f'{torch.cuda.get_device_name()}: B = {args.batch}, {"independent" if args.independent else "coupled"} Look, '
          f'{"windows" if window else "whole tensors"}, {census.calls} ABI calls, {time.time() - t0:.0f} s, largest per-call working set '
          f'{ws / 2 ** 30:.2f} GiB (call #{call} {entry}), f16s saturations {model.f16s_saturations()}')
    print(census.table())
    for f in census.failures:
        print('FAIL', f)
    return 1 if census.failures or census.unchecked else 0


if __name__ == '__main__':
    sys.exit(main())
