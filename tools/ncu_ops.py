#!/usr/bin/env python
"""One `ncu --set full` capture covering EVERY kernel family of the forward (north_star: "each kernel committed with an ncu
capture"), in a single application run:

  ncu --set full --clock-control none --import-source on --profile-from-start off -o gpurun_out/r2_ops \
      python tools/ncu_ops.py [--batch B] [--impl 3|4]

The forward launches ~700 kernels; profiling all of them with ~40 replays each would take the whole GPU budget.  This driver
runs warm-up steps unprofiled, then one eager step in which cudaProfilerStart/Stop brackets only the FIRST occurrence(s) of
each C-ABI op (and of a chosen list of dominant conv layers), so the report holds a few launches of every kernel.
tools/ncu_summary.py turns the report into *.md / *.json.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONV_LAYERS = {  # layer name -> occurrences to capture (the layers that dominate the step, plus one of each regime)
    'rs.stem': 1, 'rs.y1': 1, 'rs.y2': 2, 'rs.o0': 1, 'rs.c2': 1, 'rs.c5': 1, 'rs.idt': 1,
    'fpn.lat0': 1, 'fpn.int0': 1, 'fpn.down0': 1, 'dn.bb.t': 1, 'dn.aspp1': 1, 'dn.dcn.out': 1,
    'un.cat4.up00': 1, 'un.d2': 1, 'un.d0a': 1, 'seg': 1, 's2f.2': 1, 'img_feature': 1,
    'sec.0.0': 1, 'fu.f1': 1, 'look.value0': 1, 'look.q1': 1, 'gru.u1': 1, 'dec.bev_h': 1, 'dec.mlp1': 1, 'fu.py.fc0': 1,
}
SPARSE_LAYERS = {'conv_input': 1, '0.2.down': 1, '1.0.conv1': 1, '2.0.conv1': 1, '3.0.conv1': 1, 'conv_out': 1}
OP_COUNT = 1   # occurrences captured per C-ABI op name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=1)
    ap.add_argument('--impl', type=int, default=0)
    ap.add_argument('--ops-only', action='store_true', help='skip the conv layers (memory-bound / gather kernels only)')
    args = ap.parse_args()
    import torch
    from thinktwice_b200 import lib
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.engine import Engine
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    dev = torch.device('cuda', 0)
    model = build_model(cfg.model)
    model.prepare(dev, impl=args.impl)
    batch = make_batch(cfg, args.batch, seed=100)
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    for _ in range(2):
        model.forward_inference(batch)
    torch.cuda.synchronize()
    model.eng.overlap = False                                       # serial launches: one kernel at a time under the profiler

    rt = torch.cuda.cudart()
    seen = {}

    def bracket(key, limit, fn, *a, **k):
        n = seen.get(key, 0)
        seen[key] = n + 1
        if n >= limit:
            return fn(*a, **k)
        torch.cuda.synchronize()
        rt.cudaProfilerStart()
        try:
            return fn(*a, **k)
        finally:
            torch.cuda.synchronize()
            rt.cudaProfilerStop()

    orig_call, orig_conv, orig_sparse = lib.call, Engine.conv, Engine.sparse_conv
    in_conv = [0]

    def call(name, *a):
        if in_conv[0]:
            return orig_call(name, *a)
        return bracket('op:' + name, OP_COUNT, orig_call, name, *a)

    def conv(self, x, pw, out=None, name=None, **k):
        lim = 0 if args.ops_only else CONV_LAYERS.get(name, 0)
        in_conv[0] += 1
        try:
            return bracket('conv:' + str(name), lim, orig_conv, self, x, pw, out=out, name=name, **k)
        finally:
            in_conv[0] -= 1

    def sparse_conv(self, feats, pw, rule, out, **k):
        in_conv[0] += 1
        try:
            return bracket('sparse:' + str(k.get('name')), SPARSE_LAYERS.get(k.get('name'), 0), orig_sparse, self, feats, pw, rule, out, **k)
        finally:
            in_conv[0] -= 1

    lib.call, Engine.conv, Engine.sparse_conv = call, conv, sparse_conv
    model.forward_inference(batch)
    torch.cuda.synchronize()
    lib.call, Engine.conv, Engine.sparse_conv = orig_call, orig_conv, orig_sparse
    got = sorted(k for k, v in seen.items() if v and (k.startswith('op:') or CONV_LAYERS.get(k[5:], 0) or SPARSE_LAYERS.get(k[7:], 0)))
    print('captured:', ', '.join(got))
    missing = [n for n in CONV_LAYERS if 'conv:' + n not in seen] + [n for n in SPARSE_LAYERS if 'sparse:' + n not in seen]
    if missing and not args.ops_only:
        print('layer names never launched (rename in tools/ncu_ops.py):', missing)


if __name__ == '__main__':
    main()
