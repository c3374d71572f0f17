"""Stores what the reference's own voxel-pooling kernel (open_loop_training/ops/voxel_pooling, compiled by oracle/build_ref.py
into oracle/_ref/libvoxel_pooling_ref.so) returns for the inputs of tests/test_ops_gpu.py::test_voxel_pooling_dropin_matches_oracle_and_reference_kernel,
so that the test keeps comparing with the reference where the reference build is absent.  Needs a GPU:

    python tests/golden/make_voxel_pool_golden.py        # -> tests/golden/ref_voxel_pool_<B>_<P>_<C>_<X>_<Y>.npz

Outputs larger than SAMPLE elements are stored at SAMPLE seeded positions (pooled features) / rows (pos_memo)."""
import ctypes as C
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
SHAPES = [(1, 5000, 64, 21, 21), (2, 20000, 256, 21, 21), (1, 30000, 80, 200, 200), (1, 100, 7, 5, 4)]
SAMPLE = 16384
SYMBOL = '_Z37voxel_pooling_forward_kernel_launcheriiiiiiPKiPKfPfPiP11CUstream_st'


def inputs(shape):
    from test_ops_gpu import _rand_geom
    B, P, Cc, X, Y = shape
    gen = torch.Generator().manual_seed(P)
    geom = _rand_geom(gen, B, P, X, Y)
    return geom, torch.randn(B, P, Cc, generator=gen)


def positions(n, seed):
    if n <= SAMPLE:
        return torch.arange(n)
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:SAMPLE].sort().values


def main():
    fn = getattr(C.CDLL(os.path.join(ROOT, 'oracle', '_ref', 'libvoxel_pooling_ref.so')), SYMBOL)
    for shape in SHAPES:
        B, P, Cc, X, Y = shape
        geom, feats = inputs(shape)
        g, f = geom.cuda().contiguous(), feats.cuda().contiguous()
        out = torch.zeros(B, Y, X, Cc, device='cuda')
        memo = -torch.ones(B, P, 3, dtype=torch.int32, device='cuda')
        fn(B, P, Cc, X, Y, 1, C.c_void_p(g.data_ptr()), C.c_void_p(f.data_ptr()), C.c_void_p(out.data_ptr()), C.c_void_p(memo.data_ptr()),
           C.c_void_p(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        out = out.permute(0, 3, 1, 2).contiguous().reshape(-1).cpu()      # (B, C, Y, X) as the product returns it
        memo = memo.reshape(B * P, 3).cpu()
        po, pm = positions(out.numel(), 1), positions(B * P, 2)
        np.savez_compressed(os.path.join(HERE, 'ref_voxel_pool_%d_%d_%d_%d_%d.npz' % shape), out_pos=po.int().numpy(), out=out[po].numpy(),
                            memo_rows=pm.int().numpy(), memo=memo[pm].numpy())


if __name__ == '__main__':
    main()
