"""Error of the plumbing forward against the committed golden vectors under precision knobs (tt_debug_set).

usage: python tools/golden_err.py   -> one line per (variant, seed): worst key and its relative error, pred_speed error
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
from thinktwice_b200 import lib
from thinktwice_b200.config import Config, PLUMBING_CONFIG
from thinktwice_b200.registry import build_model
from thinktwice_b200.synthetic import make_batch

G = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')
KEYS = ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed', 'refine_flattned_BEV_feature')


def rel(a, b):
    return float(np.abs(np.asarray(a) - b).max() / (np.abs(b).max() + 1e-12))


def main():
    cfg = Config.fromfile(PLUMBING_CONFIG)
    variants = [('simt fp32', 1, 0), ('3xtf32', 3, 0), ('3xtf32 chunk4', 3, 0x20000), ('3xtf32 no-splitk', 3, 128)]
    for seed in (0, 1, 2):
        o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
        init_oracle_weights(o, seed)
        batch = make_batch(cfg, 1, seed=seed, num_points=2000)
        calibrate_bn(o, batch)
        ref = np.load(os.path.join(G, f'plumbing_seed{seed}.npz'))
        for name, impl, dbg in variants:
            lib.check(lib.load().tt_debug_set(dbg), 'tt_debug_set')
            m = build_model(cfg.model)
            m.load_state_dict(o.state_dict())
            m.prepare('cuda:0', impl=impl)
            pred = m.forward_inference(batch)
            errs = {k: rel(pred[k].cpu().numpy(), ref[k]) for k in KEYS}
            worst = max(errs, key=errs.get)
            print(f'seed {seed} {name:22s} worst {worst:28s} {errs[worst]:.2e}  pred_speed {errs["pred_speed"]:.2e}  pred_wp {errs["pred_wp"]:.2e}', flush=True)
    lib.load().tt_debug_set(0)


if __name__ == '__main__':
    main()
