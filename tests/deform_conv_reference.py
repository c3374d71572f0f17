"""float64 reference of mmcv's DCNv1 (3x3, stride 1, padding 1, deform_groups 1) for the deformable-convolution tests: torchvision's
deform_conv2d autograd on the CPU, with one correction, and the sums of absolute contributions the GPU tests bound their errors by.

The correction: mmcv's get_coordinate_weight returns 0 for a sample outside (-1, H) x (-1, W) (where the forward samples zero);
torchvision's has no such test and differentiates the bilinear footprint there too (nonzero for a sample in [-2, -1] or [H, H + 1],
e.g. every border tap at zero offset).  The reference's offset gradient is zeroed at those samples; tests/test_deform_conv_cpu.py pins
both the agreement everywhere else and the difference."""
import torch
from torchvision.ops import deform_conv2d as tv


def sample_coords(off):
    """float64 sampling coordinates (h, w) of every (image, tap, pixel): (N, 9, H, W) each."""
    N, _, H, W = off.shape
    off = off.double()
    taps = torch.arange(9)
    hs = off[:, 0::2] + (torch.arange(H).view(1, 1, H, 1) - 1 + (taps // 3).view(1, 9, 1, 1))
    ws = off[:, 1::2] + (torch.arange(W).view(1, 1, 1, W) - 1 + (taps % 3).view(1, 9, 1, 1))
    return hs, ws


def outside(off):
    """samples mmcv reads as zero: not (-1 < h < H and -1 < w < W); (N, 9, H, W)."""
    H, W = off.shape[2:]
    hs, ws = sample_coords(off)
    return ~((hs > -1) & (hs < H) & (ws > -1) & (ws < W))


def mmcv_offset_grad(goff, off):
    """torchvision's offset gradient with mmcv's border rule: zero at samples outside (-1, H) x (-1, W)."""
    mask = outside(off).repeat_interleave(2, dim=1)
    return goff.masked_fill(mask, 0.0)


def reference(x, off, w, gout, dtype=torch.float64):
    """forward and (grad_input, grad_offset, grad_weight) on the CPU in `dtype`."""
    t = [v.detach().cpu().to(dtype).requires_grad_(True) for v in (x, off, w)]
    y = tv(t[0], t[1], t[2], padding=1)
    y.backward(gout.detach().cpu().to(dtype))
    return y.detach(), t[0].grad, mmcv_offset_grad(t[1].grad, off.cpu()), t[2].grad


def abs_bounds(x, off, w, gout, groups):
    """float64 sum of |contribution| of every element of (output, grad_input, grad_offset, grad_weight).  For the output, grad_input
    and grad_weight that is the reference itself on |x|, |w|, |grad_output| (the bilinear weights are >= 0); for grad_offset,
    sum_c |grad_col| ((1 - lw) (|v_hl,wl| + |v_hh,wl|) + lw (|v_hl,wh| + |v_hh,wh|)) (dh; dw alike), |grad_col| = |w|^T |grad_output|."""
    ax, aw, ag = x.detach().cpu().double().abs(), w.detach().cpu().double().abs(), gout.detach().cpu().double().abs()
    ya, gxa, _, gwa = reference(ax, off, aw, ag)
    N, C, H, W = x.shape
    Cout, Cg = w.shape[:2]
    Cog = Cout // groups
    hs, ws = sample_coords(off.cpu())
    out = outside(off.cpu())
    goa = torch.zeros(N, 18, H, W, dtype=torch.float64)
    for n in range(N):
        img = ax[n].reshape(C, H * W)
        for t in range(9):
            i, j = divmod(t, 3)
            gcol = torch.cat([aw[g * Cog:(g + 1) * Cog, :, i, j].t() @ ag[n, g * Cog:(g + 1) * Cog].reshape(Cog, H * W)
                              for g in range(groups)])                        # (C, HW)
            h, wv = hs[n, t].reshape(-1), ws[n, t].reshape(-1)
            hl, wl = torch.floor(h), torch.floor(wv)
            lh, lw = h - hl, wv - wl

            def corner(a, b):
                ok = (a >= 0) & (a < H) & (b >= 0) & (b < W)
                idx = (a.clamp(0, H - 1) * W + b.clamp(0, W - 1)).long()
                return img[:, idx] * ok
            v1, v2, v3, v4 = corner(hl, wl), corner(hl, wl + 1), corner(hl + 1, wl), corner(hl + 1, wl + 1)
            bh = (gcol * ((1 - lw) * (v1 + v3) + lw * (v2 + v4))).sum(0)
            bw = (gcol * ((1 - lh) * (v1 + v2) + lh * (v3 + v4))).sum(0)
            keep = ~out[n, t].reshape(-1)
            goa[n, 2 * t] = (bh * keep).reshape(H, W)
            goa[n, 2 * t + 1] = (bw * keep).reshape(H, W)
    return ya, gxa, goa, gwa


def worst(got, ref, bound):
    """max over elements of |got - ref| / bound (elements whose bound is 0 must match exactly)."""
    err = (got.detach().cpu().double() - ref).abs()
    zero = bound == 0
    assert float(err[zero].max()) == 0 if bool(zero.any()) else True
    return float((err[~zero] / bound[~zero]).max())
