"""Site counts and neighbour-table occupancy of every output-stationary sparse conv of one forward (full config, device).

usage: python tools/sparse_conv_stats.py [batch] [--seed S] [--times DUMP.json ...] [--json OUT.json]

For each wide LiDAR conv that runs in the output-stationary form (tt_sparse_conv_os_f16s) the rulebook's `count` and `nbr`
are read back after one forward.  Per layer:
  rows        output sites (min(count, cap))
  slots       non-empty (row, tap) entries of nbr;  algorithmic FLOPs = 2 * slots * Cin * Cout
  full        FLOPs of a tile walk over every tap: 128-row tiles x kvol taps (tap pairs at Cin = 32) x 64-half K slabs
              x Cout rounded up to the N tile (one of the three wgmma products of the scaled-split format)
  skip        the same with only the taps (tap pairs) that some row of the 128-row tile uses
  empty       fraction of (tile, tap) slots that no row of the tile uses
--times takes `bench.py --dump-convs` files and adds each layer's time and algorithmic TFLOP/s per file.  bench.py uses
seed 100 at B = 16, the default here.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from thinktwice_b200.config import Config, DEFAULT_CONFIG
from thinktwice_b200.registry import build_model
from thinktwice_b200.synthetic import make_batch

BM, KE = 128, 64


def layer_stats(nbr, count, cap, cin, cout):
    kvol = nbr.shape[1]
    n = min(int(count), cap)
    occ = (nbr[:n] >= 0)
    slots = int(occ.sum())
    tiles = (n + BM - 1) // BM
    pad = tiles * BM - n
    occ_t = torch.cat([occ, occ.new_zeros(pad, kvol)]).view(tiles, BM, kvol).any(1) if tiles else occ.new_zeros(0, kvol)
    tps = 2 if cin == 32 else 1
    if tps == 2:                                    # two taps share one 64-half K slab
        occ_k = torch.cat([occ_t, occ_t.new_zeros(tiles, kvol % 2)], 1).view(tiles, -1, 2).any(2)
        slabs = 1
    else:
        occ_k = occ_t
        slabs = (cin + KE - 1) // KE
    bn_old = 64
    bn_new = 128 if cout >= 128 else 64
    per_stage = lambda bn: 2 * BM * KE * bn * ((cout + bn - 1) // bn)
    return dict(rows=n, cap=cap, kvol=kvol, Cin=cin, Cout=cout, tiles=tiles, slots=slots,
                alg_flops=2 * slots * cin * cout,
                full_flops=tiles * occ_k.shape[1] * slabs * per_stage(bn_old),
                skip_flops=int(occ_k.sum()) * slabs * per_stage(bn_new),
                empty=float(1 - occ_t.float().mean()) if tiles else 0.0,
                empty_k=float(1 - occ_k.float().mean()) if tiles else 0.0,
                fill=slots / max(n * kvol, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('batch', type=int, nargs='?', default=16)
    ap.add_argument('--seed', type=int, default=100)
    ap.add_argument('--times', nargs='*', default=[])
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    cfg = Config.fromfile(DEFAULT_CONFIG)
    model = build_model(cfg.model)
    dev = torch.device('cuda:0')
    model.prepare(dev)
    e = model.eng
    seen = {}
    inner = e.sparse_conv

    def record(feats, pw, rule, out, *args, name=None, **kw):
        if rule.get('nbr') is not None:
            seen[name] = (pw.Cin, pw.Cout, rule)
        return inner(feats, pw, rule, out, *args, name=name, **kw)
    e.sparse_conv = record
    model.forward_inference(make_batch(cfg, a.batch, seed=a.seed, device=dev))
    torch.cuda.synchronize()
    e.sparse_conv = inner
    times = []
    for path in a.times:
        times.append({n: ms for n, _, ms in json.load(open(path))})
    rows = {}
    for name, (cin, cout, rule) in seen.items():
        rows[name] = layer_stats(rule['nbr'].cpu(), rule['count'].item(), rule['cap'], cin, cout)
        rows[name]['ms'] = [t.get(f'sparse.{name}') for t in times]
    hdr = '| layer | Cin→Cout | kvol | rows | tiles | fill | empty (tile, tap) | alg GFLOP | full-walk GFLOP | skip GFLOP |'
    hdr += ''.join(f' ms [{i}] | TFLOP/s [{i}] |' for i in range(len(times)))
    print(f'B = {a.batch}, seed {a.seed}')
    print(hdr)
    print('|' + '---|' * (hdr.count('|') - 1))
    tot = [0, 0, 0] + [0.0] * len(times)
    for name, r in rows.items():
        line = (f"| `{name}` | {r['Cin']}→{r['Cout']} | {r['kvol']} | {r['rows']} | {r['tiles']} | {r['fill']:.3f} | "
                f"{r['empty']:.3f} | {r['alg_flops'] / 1e9:.1f} | {r['full_flops'] / 1e9:.1f} | {r['skip_flops'] / 1e9:.1f} |")
        tot[0] += r['alg_flops']; tot[1] += r['full_flops']; tot[2] += r['skip_flops']
        for i, ms in enumerate(r['ms']):
            line += f" {ms:.3f} | {r['alg_flops'] / (ms * 1e-3) / 1e12:.1f} |" if ms else ' - | - |'
            tot[3 + i] += ms or 0.0
        print(line)
    line = f'| **all** | | | | | | | {tot[0] / 1e9:.1f} | {tot[1] / 1e9:.1f} | {tot[2] / 1e9:.1f} |'
    for i in range(len(times)):
        line += f' {tot[3 + i]:.3f} | {tot[0] / (tot[3 + i] * 1e-3) / 1e12:.1f} |' if tot[3 + i] else ' - | - |'
    print(line)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
