"""Micro-benchmark of single conv shapes through the C ABI (diagnosis tool, not a test).  python tools/conv_bench.py"""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from thinktwice_b200 import lib
from thinktwice_b200.engine import Engine, FMap
from thinktwice_b200.weights import Packer

SHAPES = [  # name, N, H, W, Cin, Cout, k, stride, pad, residual
    ('rs.o0  1x1 64->256 @112x224 +res', 4, 112, 224, 64, 256, 1, 1, 0, True),
    ('rs.o0  same, no residual', 4, 112, 224, 64, 256, 1, 1, 0, False),
    ('rs.y1  1x1 256->64 @112x224', 4, 112, 224, 256, 64, 1, 1, 0, False),
    ('fpn.lat0 1x1 256->256 @112x224', 4, 112, 224, 256, 256, 1, 1, 0, False),
    ('fpn.int0 3x3 256->256 @112x224', 4, 112, 224, 256, 256, 3, 1, 1, False),
    ('dn.bb 3x3 512->512 @28x56', 4, 28, 56, 512, 512, 3, 1, 1, True),
    ('rs.l4 3x3 512->512 @14x28', 4, 14, 28, 512, 512, 3, 1, 1, False),
    ('rs.l4 1x1 2048->512 @14x28', 4, 14, 28, 2048, 512, 1, 1, 0, False),
]
if os.environ.get('SHAPES'):
    SHAPES = [SHAPES[int(i)] for i in os.environ['SHAPES'].split(',')]


def run(eng, x, pw, res, k, stride, pad, iters=20):
    for _ in range(3):
        eng.conv(x, pw, name='b.y', stride=stride, pad=pad, act=1, res=res)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        eng.conv(x, pw, name='b.y', stride=stride, pad=pad, act=1, res=res)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def main():
    dbg_list = [int(a) for a in sys.argv[1:]] or [0]
    L = lib.load()
    for name, N, H, W, Cin, Cout, k, stride, pad, use_res in SHAPES:
        g = torch.Generator().manual_seed(0)
        N = N * int(os.environ.get('NMUL', '1'))
        xt = torch.randn(N, H, W, Cin, generator=g).cuda()
        w = torch.randn(Cout, Cin, k, k, generator=g) * 0.05
        OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        res = FMap(torch.randn(N, OH, OW, Cout, generator=g).cuda(), N, OH, OW, Cout) if use_res else None
        gf = 2.0 * N * OH * OW * Cin * k * k * Cout / 1e9
        mb = (N * H * W * Cin + N * OH * OW * Cout * (2 if use_res else 1)) * 4 / 1e6
        line = f'{name:36s} {gf:7.1f} GF {mb:6.0f} MB(min)'
        for impl, tag in [(int(i), {1: 'simt', 2: 'tf32', 3: '3xtf32', 4: 'f16s'}[int(i)]) for i in os.environ.get('IMPLS', '1,3,4').split(',')]:
            eng = Engine('cuda:0', impl=impl); eng.tc_min_rows = 1
            pw = Packer({'c.weight': w}, torch.device('cuda:0'), tc_mode=impl if impl > 1 else 0).conv('c')
            x = FMap(xt, N, H, W, Cin)
            if impl == 4:                                              # input with a split companion, as a producing conv would leave it
                x = eng.fmap('b.x', N, H, W, Cin, split=True)
                x.t.copy_(xt)
                eng.sync_split(x)
            for dbg in (dbg_list if impl > 1 else [0]):
                lib.check(L.tt_debug_set(dbg), 'tt_debug_set')
                us = run(eng, x, pw, res, k, stride, pad)
                line += f' | {tag}{"/d%d" % dbg if dbg else ""} {us:7.1f}us {gf / us * 1e3:6.1f}TF/s'
            L.tt_debug_set(0)
        print(line, flush=True)


if __name__ == '__main__':
    main()
