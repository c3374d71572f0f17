"""Float64 restatement of the training-side dense convolution's backward (thinktwice_b200/csrc/conv2d_train.cu): grad_x as one stride-1
convolution per output phase with the flipped, transposed sub-kernel of the taps that reach it, and grad_weight as a sum over output
pixels per tap of grad_y x the tap-shifted input.  `bug` seeds one mistake so the tests can show each is caught:
  'origin'     : every phase's row origin off by one;
  'zero_phase' : a phase no tap reaches is left unwritten (ones) instead of zeros;
  'unflipped'  : the sub-kernel taps in ascending instead of descending order;
  'tap_order'  : grad_weight's tap b decoded column-major, (b % KH, b // KH), instead of (b // KW, b % KW)."""
import math

import torch
import torch.nn.functional as F


def phase_dim(p, K, s, pad, dil, extent):
    """(first reaching tap k0, tap count n, origin, output extent) of phase p along one dimension, as make_phases computes it."""
    ext = (extent - p + s - 1) // s if extent > p else 0
    taps = [k for k in range(K - 1, -1, -1) if (p + pad - k * dil) % s == 0]
    if not taps:
        return 0, 0, 0, ext
    return taps[0], len(taps), (p + pad - taps[0] * dil) // s, ext


def phase_params(s, dil):
    """(tap step inside a phase, the phases' dilation)"""
    step = s // math.gcd(s, dil)
    return step, step * dil // s


def _window(t, org_h, org_w, rows, cols):
    """t[..., org_h : org_h + rows, org_w : org_w + cols] with zeros outside t."""
    H, W = t.shape[-2:]
    out = t.new_zeros(*t.shape[:-2], rows, cols)
    h0, h1 = max(org_h, 0), min(org_h + rows, H)
    w0, w1 = max(org_w, 0), min(org_w + cols, W)
    if h0 < h1 and w0 < w1:
        out[..., h0 - org_h:h1 - org_h, w0 - org_w:w1 - org_w] = t[..., h0:h1, w0:w1]
    return out


def grad_input(gy, w, H, W, stride, pad, dil, bug=None):
    """dL/dx of y = conv2d(x, w, stride, pad, dil) for x of H x W, from gy (N, Cout, OH, OW), in float64 by output phases."""
    gy, w = gy.double(), w.double()
    N, Cout = gy.shape[:2]
    Cin, KH, KW = w.shape[1:]
    s = stride
    step, pdil = phase_params(s, dil)
    gx = gy.new_zeros(N, Cin, H, W)
    for py in range(s):
        kh0, nh, oh_org, eh = phase_dim(py, KH, s, pad, dil, H)
        for px in range(s):
            kw0, nw, ow_org, ew = phase_dim(px, KW, s, pad, dil, W)
            if eh == 0 or ew == 0:
                continue
            if nh == 0 or nw == 0:
                if bug == 'zero_phase':
                    gx[:, :, py::s, px::s] = 1.0
                continue
            if bug == 'origin':
                oh_org += 1
            jh = torch.arange(nh) if bug != 'unflipped' else torch.arange(nh - 1, -1, -1)
            jw = torch.arange(nw) if bug != 'unflipped' else torch.arange(nw - 1, -1, -1)
            sub = w[:, :, kh0 - jh * step][:, :, :, kw0 - jw * step]          # (Cout, Cin, nh, nw), tap j -> weight tap k0 - j step
            win = _window(gy, oh_org, ow_org, eh + (nh - 1) * pdil, ew + (nw - 1) * pdil)
            gx[:, :, py::s, px::s] = F.conv2d(win, sub.transpose(0, 1), dilation=pdil)
    return gx


def grad_weight(x, gy, KH, KW, stride, pad, dil, bug=None):
    """dL/dw (Cout, Cin, KH, KW) in float64: per tap, the sum over output pixels of gy times the input pixel that tap reads."""
    x, gy = x.double(), gy.double()
    OH, OW = gy.shape[2:]
    gw = x.new_zeros(gy.shape[1], x.shape[1], KH, KW)
    for b in range(KH * KW):
        kh, kw = (b // KW, b % KW) if bug != 'tap_order' else (b % KH, b // KH)
        if kh >= KH or kw >= KW:
            continue
        win = _window(x, kh * dil - pad, kw * dil - pad, (OH - 1) * stride + 1, (OW - 1) * stride + 1)[:, :, ::stride, ::stride]
        gw[:, :, b // KW, b % KW] = torch.einsum('nohw,nihw->oi', gy, win)
    return gw
