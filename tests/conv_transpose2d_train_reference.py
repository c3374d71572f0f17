"""Float64 restatement of the training-side transposed convolution (thinktwice_b200/csrc/conv2d_train.cu, include/tt_b200.h §17) as the
adjoint of a Conv2d with the same weight tensor: the forward by output phases (the Conv2d's grad_x path), grad_x as the Conv2d's forward,
grad_weight as the Conv2d's weight gradient with x and grad_y exchanged.  `bug` seeds one mistake so the tests can show each is caught:
  'swapped_phase': phase (py, px) computed with the sub-kernel of phase (px, py);
  'flipped_tap'  : the sub-kernel taps in ascending instead of descending order."""
import torch
import torch.nn.functional as F

import conv2d_train_reference as R


def out_size(H, k, s, p, op):
    return (H - 1) * s - 2 * p + k + op


def forward(x, w, b, s, p, op, bug=None):
    """conv_transpose2d(x, w, b, s, p, op) in float64: w (Cin, Cout, k, k) is the weight of the adjoint Conv2d (Cout_conv = Cin), whose
    input gradient, by phases, is this output."""
    x, w = x.double(), w.double()
    N, Cin, H, W = x.shape
    Cout, KH, KW = w.shape[1:]
    OH, OW = out_size(H, KH, s, p, op), out_size(W, KW, s, p, op)
    step, pdil = R.phase_params(s, 1)
    y = x.new_zeros(N, Cout, OH, OW)
    for py in range(s):
        for px in range(s):
            qy, qx = (px, py) if bug == 'swapped_phase' else (py, px)
            kh0, nh, oh_org, eh = R.phase_dim(qy, KH, s, p, 1, OH)
            kw0, nw, ow_org, ew = R.phase_dim(qx, KW, s, p, 1, OW)
            eh, ew = R.phase_dim(py, KH, s, p, 1, OH)[3], R.phase_dim(px, KW, s, p, 1, OW)[3]
            if eh == 0 or ew == 0 or nh == 0 or nw == 0:
                continue
            jh = torch.arange(nh) if bug != 'flipped_tap' else torch.arange(nh - 1, -1, -1)
            jw = torch.arange(nw) if bug != 'flipped_tap' else torch.arange(nw - 1, -1, -1)
            sub = w[:, :, kh0 - jh * step][:, :, :, kw0 - jw * step]          # (Cin, Cout, nh, nw)
            win = R._window(x, oh_org, ow_org, eh + (nh - 1) * pdil, ew + (nw - 1) * pdil)
            y[:, :, py::s, px::s] = F.conv2d(win, sub.transpose(0, 1), dilation=pdil)
    if b is not None:
        y += b.double()[None, :, None, None]
    return y


def grad_input(gy, w, s, p):
    """dL/dx: the adjoint Conv2d's forward of gy, no bias."""
    return F.conv2d(gy.double(), w.double(), stride=s, padding=p)


def grad_weight(x, gy, k, s, p):
    """dL/dw (Cin, Cout, k, k): the adjoint Conv2d's weight gradient with x := gy and grad_y := x."""
    return R.grad_weight(gy, x, k, k, s, p, 1)
