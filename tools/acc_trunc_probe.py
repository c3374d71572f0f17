"""Probe how the tensor-core fp32 accumulator rounds (round 2 experiment, ~10 s of GPU time).

DESIGN.md §2: the dominant error of the 3xTF32 path is the truncating accumulate inside the tensor core.  If the
truncation is toward zero, draining `acc + n_acc * 0.5 ulp(acc) * sign(acc)` would centre the error and allow
4-8 K-slab chunks (8 % faster) at the accuracy of 2-slab chunks.  This script measures the SIGNED error of a single-pass
TF32 1x1 convolution (impl 2: hi*hi only, one accumulator chunk of up to 16 K-slabs) whose operands are exactly
TF32-representable, so every product is exact and the only rounding is the accumulate:

  * all-positive products  -> mean error / ulp(result)
  * all-negative products  -> mean error / ulp(result)
  * K = 32 ... 512 (number of accumulations = K / 8)

round-to-nearest: both means ~0;  toward zero: negative for positive sums, positive for negative sums, ~ -0.5 * K / 8 ulp;
toward -inf: negative for both.

usage: python tools/acc_trunc_probe.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from thinktwice_b200.engine import Engine, FMap
from thinktwice_b200.weights import Packer


def main():
    eng = Engine('cuda:0', impl=2)
    eng.tc_min_rows = 1
    g = torch.Generator().manual_seed(0)
    M, Cout = 1024, 64
    for K in (32, 64, 128, 256, 512):
        for sign in (1.0, -1.0):
            x = 1.0 + torch.randint(0, 1024, (M, K), generator=g).float() / 1024.0          # 11 significant bits: TF32-exact
            w = sign * (1.0 + torch.randint(0, 1024, (Cout, K), generator=g).float() / 1024.0)
            pw = Packer({'c.weight': w.view(Cout, K, 1, 1)}, torch.device('cuda:0'), tc_mode=2).conv('c')
            xm = FMap(x.cuda().contiguous(), M, 1, 1, K)
            y = eng.conv(xm, pw, name=f'probe.{K}').t.view(M, Cout).double().cpu()
            ref = x.double() @ w.double().t()                                               # exact in fp64
            ulp = torch.pow(2.0, torch.floor(torch.log2(ref.abs())) - 23)
            e = (y - ref) / ulp
            rn = (ref.float().double() - ref) / ulp                                         # what one final RN would leave
            print(f'K {K:4d} ({K // 8:3d} accumulations) sign {sign:+.0f}: mean err {float(e.mean()):+8.3f} ulp, '
                  f'rms {float(e.pow(2).mean().sqrt()):7.3f}, min {float(e.min()):+8.2f}, max {float(e.max()):+8.2f}'
                  f'   [single RN of the exact sum: mean {float(rn.mean()):+.3f}, rms {float(rn.pow(2).mean().sqrt()):.3f}]')


if __name__ == '__main__':
    main()
