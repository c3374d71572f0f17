"""Float64 restatement of the training-side bilinear interpolation, align_corners=True (thinktwice_b200/csrc/interp_train.cu,
include/tt_b200.h §17), as one weight matrix per dimension: y = A_h x A_w^T.  The forward builds A from ATen's arithmetic (output index o
reads rows i0 = (int)(scale o) and i0 + (i0 < in - 1) with weights 1 - l and l); the backward builds A^T the way the kernel gathers, row i
of A^T summing the contiguous range of outputs whose i0 is i - 1 or i.  `coord` is the dtype of the coordinate arithmetic: float64 is
torch's float64 op, float32 the coordinates the fp32 op (ATen's and the library's) computes and then weighs in float64.
`bug` seeds one mistake so the tests can show it is caught:
  'reach': the gather range of every input row one output short at its end."""
import numpy as np
import torch


def _scale(n_in, n_out, coord):
    return coord(n_in - 1) / coord(n_out - 1) if n_out > 1 else coord(0)


def _coord(scale, o, coord):
    return coord(scale * coord(o))


def forward_matrix(n_in, n_out, coord=np.float64):
    """A (n_out, n_in): y[o] = sum_i A[o, i] x[i] along one dimension."""
    A = np.zeros((n_out, n_in))
    s = _scale(n_in, n_out, coord)
    for o in range(n_out):
        r = _coord(s, o, coord)
        i0 = int(r)
        i1 = i0 + (1 if i0 < n_in - 1 else 0)
        l1 = coord(r - coord(i0))
        A[o, i0] += float(coord(1) - l1)
        A[o, i1] += float(l1)
    return torch.from_numpy(A)


def first_reaching(scale, t, n_out, coord):
    """the first output index o in [0, n_out] with (int)(scale o) >= t, as the kernel finds it."""
    return next((o for o in range(n_out) if int(_coord(scale, o, coord)) >= t), n_out)


def reach(i, n_in, n_out, coord=np.float64, bug=None):
    """the output indices reaching input index i: those with i0 in {i - 1, i}."""
    s = _scale(n_in, n_out, coord)
    lo, hi = first_reaching(s, i - 1, n_out, coord) if i > 0 else 0, first_reaching(s, i + 1, n_out, coord)
    return range(lo, hi - 1 if bug == 'reach' and hi > lo else hi)


def gather_matrix(n_in, n_out, coord=np.float64, bug=None):
    """A^T (n_in, n_out) row by row from the gather ranges, the weight of each output recomputed as the forward computes it."""
    A = forward_matrix(n_in, n_out, coord)
    G = torch.zeros(n_in, n_out, dtype=torch.float64)
    for i in range(n_in):
        for o in reach(i, n_in, n_out, coord, bug):
            G[i, o] = A[o, i]
    return G


def forward(x, OH, OW, coord=np.float64):
    H, W = x.shape[-2:]
    Ah, Aw = forward_matrix(H, OH, coord).to(x.device), forward_matrix(W, OW, coord).to(x.device)
    return torch.einsum('oh,nchw,pw->ncop', Ah, x.double(), Aw)


def backward(gy, H, W, coord=np.float64, bug=None):
    OH, OW = gy.shape[-2:]
    Gh, Gw = gather_matrix(H, OH, coord, bug).to(gy.device), gather_matrix(W, OW, coord, bug).to(gy.device)
    return torch.einsum('ho,ncop,wp->nchw', Gh, gy.double(), Gw)


def backward_abs(gy, H, W, coord=np.float32):
    """S of the backward: the float64 sum of |terms| of every grad_x element."""
    OH, OW = gy.shape[-2:]
    Gh, Gw = gather_matrix(H, OH, coord).abs().to(gy.device), gather_matrix(W, OW, coord).abs().to(gy.device)
    return torch.einsum('ho,ncop,wp->nchw', Gh, gy.double().abs(), Gw)
