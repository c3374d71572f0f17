"""Per-layer-family comparison of two `bench.py --dump-convs` files (one serial eager B = 16 step each).

    python tools/conv_dump_compare.py BEFORE.json AFTER.json [--label-before X] [--label-after Y] > table.md

A family is a launch name with its indices removed and cut to its first two parts ('cam.rs.l3.2.c2' -> 'cam.rs'); the table gives
the launches, the algorithmic TFLOP of the family and its summed CUDA-event time in each file, largest families first."""
import argparse
import json
import re
from collections import OrderedDict


def family(name):
    parts = [p for p in re.split(r'[.#]', name) if p and not p.isdigit()]
    return '.'.join(re.sub(r'\d+$', '', p) or p for p in parts[:2]) or name


def load(path):
    fam = OrderedDict()
    for name, flops, ms in json.load(open(path)):
        f = fam.setdefault(family(name), [0, 0.0, 0.0])
        f[0] += 1
        f[1] += flops
        f[2] += ms
    return fam


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('before')
    ap.add_argument('after')
    ap.add_argument('--label-before', default='before')
    ap.add_argument('--label-after', default='after')
    a = ap.parse_args()
    b, n = load(a.before), load(a.after)
    keys = sorted(set(b) | set(n), key=lambda k: -(b.get(k, [0, 0, 0])[2]))
    print(f'| family | launches | TFLOP | {a.label_before} ms | {a.label_after} ms | speed-up | {a.label_after} TFLOP/s |')
    print('|---|---:|---:|---:|---:|---:|---:|')
    tot = [0, 0.0, 0.0, 0.0]
    for k in keys:
        cb, fb, mb = b.get(k, [0, 0.0, 0.0])
        ca, fa, ma = n.get(k, [0, 0.0, 0.0])
        tot[0] += ca; tot[1] += fa; tot[2] += mb; tot[3] += ma
        sp = f'{mb / ma:.2f}x' if ma > 0 else '-'
        rate = f'{fa / (ma * 1e-3) / 1e12:.0f}' if ma > 0 else '-'
        print(f'| `{k}` | {ca} | {fa / 1e12:.2f} | {mb:.2f} | {ma:.2f} | {sp} | {rate} |')
    print(f'| **all** | {tot[0]} | {tot[1] / 1e12:.2f} | {tot[2]:.2f} | {tot[3]:.2f} | {tot[2] / tot[3]:.2f}x | '
          f'{tot[1] / (tot[3] * 1e-3) / 1e12:.0f} |')


if __name__ == '__main__':
    main()
