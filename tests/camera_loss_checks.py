"""Crafted inputs and float64 references for tt_camera_loss (csrc/losses.cu), the camera branch's seg_loss / depth_loss.

tests/test_camera_losses_gpu.py runs these checks on the CUDA kernel; tests/test_camera_losses_cpu.py runs them on the torch emulation
of the C ABI (tests/emu_camera_losses.py) and shows that each one rejects a seeded bug of that emulation.  The references are the reference's
formulas (tests/camera_loss_oracle.py: get_downsampled_gt_seg / get_downsampled_gt_depth, FocalLoss, BCE-with-logits) evaluated in float64 on
the same logits, never a kernel's intermediate values.  The runner calls the C ABI through thinktwice_b200.lib, so it works on either
backend."""
import ctypes as C

import numpy as np
import torch

import camera_loss_oracle

REL = 2e-6                 # fp64 sums in a different order, the result rounded to fp32
D_BOUND = [1.0, 41.0, 0.5]  # thinktwice.py: D = 80 bins of 0.5 m


def make_case(seed, B, N, seg_HW, seg_classes, seg_ld, seg_coff, depth_hw, D, depth_ld, depth_coff, f=16, s=2, d_bound=D_BOUND):
    """random logits in channels-last buffers whose other channels are NaN (a kernel must not read them), labels with fractional
    parts and ignored pixels, depths over the bin range and beyond."""
    g = torch.Generator().manual_seed(seed)
    BN, (H, W), (dh, dw) = B * N, seg_HW, depth_hw
    h, w = H // s, W // s
    seg = torch.full((BN, h, w, seg_ld), float('nan'))
    seg[..., seg_coff:seg_coff + seg_classes] = 3 * torch.randn(BN, h, w, seg_classes, generator=g)
    lab = torch.randint(0, seg_classes, (B, N, H, W), generator=g).float() + 0.999 * torch.rand(B, N, H, W, generator=g)
    lab[torch.rand(B, N, H, W, generator=g) < 0.2] = 255.0
    dep = torch.full((BN, dh, dw, depth_ld), float('nan'))
    dep[..., depth_coff:depth_coff + D] = 3 * torch.randn(BN, dh, dw, D, generator=g)
    d0, d1, step = d_bound
    gt = (d0 - 2 * step) + (d1 - d0 + 6 * step) * torch.rand(B, N, dh * f, dw * f, generator=g)
    gt[torch.rand(B, N, dh * f, dw * f, generator=g) < 0.3] = 0.0
    return dict(seg=seg, seg_coff=seg_coff, seg_classes=seg_classes, seg_gt=lab, s=s,
                depth=dep, depth_coff=depth_coff, D=D, depth_gt=gt, f=f, d_bound=list(d_bound))


def crafted_cases():
    """name -> case.  'edges': +-100 logits, a non-zero coff, odd label rows, a frame whose pixels are all ignored, depth blocks with
    NaN, +-inf, zeros, negative values and minima exactly on bin values; 'ignored': every pixel ignored (seg_loss NaN) and no foreground
    cell (depth_loss 0); 'large': a thinktwice.py-sized frame pair, many grid-stride rounds per CTA."""
    d0, _, step = D_BOUND
    c = make_case(1, 2, 2, (33, 40), 12, 32, 4, (3, 4), 80, 96, 3)
    c['seg'][0, 0, :3, 4:16] = torch.tensor([100.0, -100.0, 100.0]).view(3, 1)
    c['seg'][1, 2, 5, 4:16] = -100.0
    c['seg'][1, 2, 5, 4 + 7] = 100.0
    c['seg_gt'][0, 1] = 255.0                                       # a frame whose pixels are all ignored
    c['depth'][0, 0, 0, 3:83] = 100.0
    c['depth'][0, 0, 1, 3:83] = -100.0
    gt, f = c['depth_gt'], c['f']
    edge = lambda v: (d0 - step) + v * step
    blocks = [(0.0, None), (edge(3.5), 'nan'), (edge(5.0), 'inf'), (edge(7.0), '-inf'), (-3.0, None), (edge(0), None), (edge(1), None),
              (edge(80), None), (edge(81), None), (edge(1 - 2 ** -10), None), (edge(81 - 2 ** -10), None), (edge(2), None)]
    for k, (v, extra) in enumerate(blocks):                         # frame 0, camera 0: one crafted block per cell
        cy, cx = divmod(k, 4)
        blk = gt[0, 0, cy * f:(cy + 1) * f, cx * f:(cx + 1) * f]
        if v == 0.0:
            blk.zero_()                                             # no measurement: 1e5, background
            continue
        blk.copy_(torch.full((f, f), 45.0))
        blk[3, 7] = v
        if extra == 'nan':
            blk[9, 2] = float('nan')                                # torch.min propagates it: background (fminf would keep 3.5)
        elif extra == 'inf':
            blk[0, 0] = float('inf')
        elif extra == '-inf':
            blk[15, 15] = float('-inf')                             # the minimum is -inf: below the range, background
    ign = make_case(2, 1, 2, (32, 32), 12, 32, 0, (2, 2), 80, 80, 0)
    ign['seg_gt'][:] = 255.0
    ign['depth_gt'][:] = 1e4                                        # beyond the last bin
    ign['depth_gt'][..., :16, :16] = -1.0                           # below the first
    ign['depth_gt'][..., 16:, 16:] = 0.0                            # no measurement
    large = make_case(3, 1, 2, (448, 896), 12, 32, 0, (28, 56), 80, 336, 0)
    return dict(edges=c, ignored=ign, large=large)


def reference(case):
    """(seg_loss, depth_loss) in float64 by the reference's formulas."""
    cfg = dict(use_seg=True, use_depth=True)
    B, N = case['seg_gt'].shape[:2]
    seg = case['seg'][..., case['seg_coff']:case['seg_coff'] + case['seg_classes']].permute(0, 3, 1, 2).double()
    depth = case['depth'][..., case['depth_coff']:case['depth_coff'] + case['D']].permute(0, 3, 1, 2).double()
    d = camera_loss_oracle.camera_loss(cfg, dict(seg=case['seg_gt'], depth=case['depth_gt']), seg, depth, case['d_bound'], case['f'], case['s'])
    return float(d['seg_loss']), float(d['depth_loss'])


def run(case, device, halves=('seg', 'depth')):
    """tt_camera_loss on `device` through thinktwice_b200.lib: out[0] = seg_loss, out[1] = depth_loss (NaN where a half is off)."""
    from thinktwice_b200 import lib
    dev = lambda t: t.contiguous().to(device)
    seg, dep = dev(case['seg']), dev(case['depth'])
    B, N, H, W = case['seg_gt'].shape
    sgt = dev(case['seg_gt'].reshape(B * N, H, W))
    dgt = dev(case['depth_gt'].reshape(B * N, *case['depth_gt'].shape[2:]))
    d0, _, step = case['d_bound']
    f = dict(BN=B * N, seg_logits=lib._p(None), seg_gt=lib._p(None), depth_logits=lib._p(None), depth_gt=lib._p(None))
    if 'seg' in halves:
        f.update(seg_logits=lib._p(seg), seg_gt=lib._p(sgt), seg_h=seg.shape[1], seg_w=seg.shape[2], seg_H=H, seg_W=W, seg_ld=seg.shape[3],
                 seg_coff=case['seg_coff'], seg_classes=case['seg_classes'], seg_ignore=255, seg_alpha=0.5, seg_gamma=2.0, seg_weight=10.0)
    if 'depth' in halves:
        f.update(depth_logits=lib._p(dep), depth_gt=lib._p(dgt), depth_h=dep.shape[1], depth_w=dep.shape[2], depth_factor=case['f'],
                 depth_ld=dep.shape[3], depth_coff=case['depth_coff'], depth_bins=case['D'], depth_offset=d0 - step, depth_step=step)
    desc = lib.camera_loss_desc(**f)
    out = torch.full((2,), float('nan'), device=device)
    ws = torch.empty(int(lib.load().tt_camera_loss_workspace_bytes(lib.ref(desc))), dtype=torch.uint8, device=device)
    lib.call('tt_camera_loss', lib.ref(desc), lib._p(out), lib._p(ws), C.c_size_t(ws.numel()))
    if out.is_cuda:
        torch.cuda.synchronize()
    return out.cpu().double().numpy()


def agree(got, want, what):
    if np.isnan(want) or np.isnan(got):
        assert np.isnan(want) and np.isnan(got), f'{what}: got {got!r}, want {want!r}'
        return
    assert abs(got - want) <= REL * abs(want), f'{what}: got {got!r}, want {want!r} (rel {abs(got - want) / max(abs(want), 1e-300):.2e})'


def check_case(name, case, device):
    """both halves against float64 (each alone and both in one launch); the launch repeated is bitwise equal."""
    ws, wd = reference(case)
    both = run(case, device)
    agree(both[0], ws, f'{name}: seg_loss')
    agree(both[1], wd, f'{name}: depth_loss')
    again = run(case, device)
    assert np.array_equal(both.view(np.int64), again.view(np.int64)), f'{name}: two launches differ: {both} vs {again}'
    alone_s, alone_d = run(case, device, ('seg',)), run(case, device, ('depth',))
    assert np.isnan(alone_s[1]) and np.isnan(alone_d[0]), f'{name}: a disabled half wrote its slot'
    agree(alone_s[0], ws, f'{name}: seg_loss alone')
    agree(alone_d[1], wd, f'{name}: depth_loss alone')
    return both, (ws, wd)


def check_all(device):
    out = {}
    for name, case in crafted_cases().items():
        out[name] = check_case(name, case, device)
    (gs, gd), (ws, wd) = out['ignored']
    assert np.isnan(ws) and wd == 0.0, 'the all-ignored / no-foreground case must give NaN / 0'
    return out
