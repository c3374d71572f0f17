"""SHA-256 of every output buffer of the f16s convolution kernel on seeded inputs (diagnosis tool, not a test).

Two builds of conv_f16s_kernel whose non-atomic outputs must be bitwise equal print the same digests:
    python tools/conv_digest.py
Cases: the tools/conv_bench.py shapes (N = 4) with bias and ReLU, on the tiles the host selects and with 64-column tiles forced;
residuals given as fp32 rows and as split planes; a nearest-upsampled (UP2) residual; a per-image bias table (bias_n_mod); and
output-stationary sparse convolutions (128- and 64-column tiles, the Cin = 32 tap-pair walk, fp32 / split / no residual) over a
seeded LiDAR-like cloud.  Split-K is switched off (debug bit 128): its partial sums are added with red.add in no fixed order."""
import hashlib
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from thinktwice_b200 import lib
from thinktwice_b200.engine import Engine, FMap, PackedConv
from thinktwice_b200.lidarnet import LidarNet
from thinktwice_b200.weights import Packer, f16s_split

NO_SPLITK, FORCE_BN64 = 128, 0x400000
SHAPES = [  # name, N, H, W, Cin, Cout, k, stride, pad, residual (tools/conv_bench.py)
    ('rs.o0', 4, 112, 224, 64, 256, 1, 1, 0, True),
    ('rs.o0.nores', 4, 112, 224, 64, 256, 1, 1, 0, False),
    ('rs.y1', 4, 112, 224, 256, 64, 1, 1, 0, False),
    ('fpn.lat0', 4, 112, 224, 256, 256, 1, 1, 0, False),
    ('fpn.int0', 4, 112, 224, 256, 256, 3, 1, 1, False),
    ('dn.bb', 4, 28, 56, 512, 512, 3, 1, 1, True),
    ('rs.l4.3x3', 4, 14, 28, 512, 512, 3, 1, 1, False),
    ('rs.l4.1x1', 4, 14, 28, 2048, 512, 1, 1, 0, False),
]


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def split_only(eng, name, t):
    """an FMap of the fp32 tensor t (N, H, W, C) that exists only as split planes"""
    N, H, W, C = t.shape
    fm = eng.fmap(name, N, H, W, C, fmt='fs')
    fm.t.copy_(t)
    eng.sync_split(fm)
    return FMap(None, N, H, W, C, fm.ld, 0, fm.s)


def dense_cases(eng, out):
    for name, N, H, W, Cin, Cout, k, stride, pad, use_res in SHAPES:
        g = torch.Generator().manual_seed(len(out))
        OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        x = eng.fmap('d.x', N, H, W, Cin, split=True)
        x.t.copy_(torch.randn(N, H, W, Cin, generator=g))
        eng.sync_split(x)
        pw = Packer({'c.weight': torch.randn(Cout, Cin, k, k, generator=g) * 0.05, 'c.bias': torch.randn(Cout, generator=g) * 0.1},
                    torch.device('cuda:0'), tc_mode=4).conv('c')
        r32 = torch.randn(N, OH, OW, Cout, generator=g).cuda()
        res = [('', None)]
        if use_res:
            res = [('+res', FMap(r32, N, OH, OW, Cout)), ('+res_s', split_only(eng, 'd.rs', r32))]
        for tag, r in res:
            for dbg, tile in ((NO_SPLITK, ''), (NO_SPLITK | FORCE_BN64, '/bn64')):
                lib.check(lib.load().tt_debug_set(dbg), 'tt_debug_set')
                y = eng.conv(x, pw, name='d.y', stride=stride, pad=pad, act=1, res=r)
                torch.cuda.synchronize()
                out.append((f'{name}{tag}{tile} y', digest(y.t)))
                out.append((f'{name}{tag}{tile} y#s', digest(y.s)))
        lib.check(lib.load().tt_debug_set(0), 'tt_debug_set')


def up2_and_bias_table_cases(eng, out):
    g = torch.Generator().manual_seed(100)
    N, H, W, Cin, Cout = 4, 56, 112, 256, 256
    x = eng.fmap('u.x', N, H, W, Cin, split=True)
    x.t.copy_(torch.randn(N, H, W, Cin, generator=g))
    eng.sync_split(x)
    pw = Packer({'c.weight': torch.randn(Cout, Cin, 1, 1, generator=g) * 0.05, 'c.bias': torch.randn(Cout, generator=g) * 0.1},
                torch.device('cuda:0'), tc_mode=4).conv('c')
    coarse = torch.randn(N, H // 2, W // 2, Cout, generator=g).cuda()
    lib.check(lib.load().tt_debug_set(NO_SPLITK), 'tt_debug_set')
    for tag, r in (('+up2', FMap(coarse, N, H // 2, W // 2, Cout)), ('+up2_s', split_only(eng, 'u.rs', coarse))):
        y = eng.conv(x, pw, name='u.y', act=1, res=r, res_mode=lib.RES_UP2)
        torch.cuda.synchronize()
        out.append((f'lat1x1{tag} y', digest(y.t)))
        out.append((f'lat1x1{tag} y#s', digest(y.s)))
    pw.bias = (torch.randn(4 * Cout, generator=g) * 0.1).cuda()       # per-image bias rows: image n takes row n % 4
    y = eng.conv(x, pw, name='u.yb', bias_n_mod=4)
    torch.cuda.synchronize()
    out.append(('lat1x1 bias_n_mod y', digest(y.t)))
    out.append(('lat1x1 bias_n_mod y#s', digest(y.s)))
    lib.check(lib.load().tt_debug_set(0), 'tt_debug_set')


def sparse_cases(eng, out):
    """output-stationary SubM 3x3x3 convolutions over a seeded cloud of unique voxels"""
    rng = np.random.default_rng(7)
    shape = (40, 200, 176)
    keys = np.unique(rng.integers(0, shape[0] * shape[1] * shape[2], 60000))
    coords = np.stack([np.zeros_like(keys), keys // (shape[1] * shape[2]), (keys // shape[2]) % shape[1], keys % shape[2]], 1)
    n = len(coords)
    c = torch.as_tensor(coords, dtype=torch.int32).cuda()
    rb = LidarNet._rulebook(types.SimpleNamespace(eng=eng), 'dg', 1, c, torch.tensor([n], dtype=torch.int32).cuda(), n, shape,
                            (3, 3, 3), (1, 1, 1), (1, 1, 1), True, 'nbr')
    g = torch.Generator().manual_seed(200)
    for cin, cout, rkind in ((64, 128, 'res'), (64, 64, 'res_s'), (32, 64, None), (128, 128, 'res_s')):
        x = torch.randn(n, cin, generator=g)
        hi, lo = f16s_split(x)
        x_s = torch.stack([hi.reshape(-1), lo.reshape(-1)]).cuda()
        w = torch.randn(cout, 27, cin, generator=g) / np.sqrt(27 * cin)
        b = torch.randn(cout, generator=g) * 0.1
        pw = PackedConv(w.permute(1, 2, 0).reshape(27 * cin, cout).contiguous().cuda(), b.cuda(), cin, cout,
                        w_h=torch.stack(f16s_split(w)).contiguous().cuda())
        r = torch.randn(n, cout, generator=g)
        res = r.cuda() if rkind == 'res' else None
        res_s = torch.stack([t.reshape(-1) for t in f16s_split(r)]).cuda() if rkind == 'res_s' else None
        y = torch.zeros(rb['cap'], cout, device='cuda:0')
        y_s = torch.zeros(2, rb['cap'] * cout, dtype=torch.float16, device='cuda:0')
        eng.sparse_conv(None, pw, rb, y, act=1, res=res, name='dg', feats_s=x_s, out_s=y_s, res_s=res_s)
        torch.cuda.synchronize()
        tag = f'os {cin}->{cout}' + (f' +{rkind}' if rkind else '')
        out.append((f'{tag} y', digest(y)))
        out.append((f'{tag} y#s', digest(y_s)))


def main():
    torch.manual_seed(0)
    eng = Engine('cuda:0', impl=4)
    eng.tc_min_rows = 1
    out = []
    dense_cases(eng, out)
    up2_and_bias_table_cases(eng, out)
    sparse_cases(eng, out)
    for name, h in out:
        print(f'{name:32s} {h}')
    print(f'{"all":32s} {hashlib.sha256("".join(h for _, h in out).encode()).hexdigest()}')


if __name__ == '__main__':
    main()
