"""The float64 reference of the training-side sparse convolution (thinktwice_b200/ops/sparse_conv.py) and its error bounds.

The reference is the oracle's explicit-rulebook `SparseConvBase` (oracle/lidar.py) run in float64 under autograd, on whatever device its
inputs are on: forward, grad_input and grad_weight.  `abs_bounds` runs the same computation on |x|, |W| and |gy|: per element the sum of
the absolute values of every term that element adds up, the S of the bound |got - ref| <= tol * S."""
import torch


def site_keys(coords, shape):
    D, H, W = shape
    c = coords.long()
    return ((c[:, 0] * D + c[:, 1]) * H + c[:, 2]) * W + c[:, 3]


def reference(x, coords, shape, B, w, k, s, p, subm, gy=None):
    """(y, out_coords, grad_x, grad_w) in float64; grad_x / grad_w are None without gy.  w: (Cout, kd, kh, kw, Cin)."""
    from oracle.lidar import SparseConvBase, SparseTensor
    conv = SparseConvBase(w.shape[-1], w.shape[0], k, stride=s, padding=p, subm=subm).to(x.device, torch.float64)
    with torch.no_grad():
        conv.weight.copy_(w.to(torch.float64))
    xx = x.detach().to(torch.float64).requires_grad_(gy is not None)
    out = conv(SparseTensor(xx, coords, shape, B))
    if gy is None:
        return out.feats.detach(), out.coords, None, None
    out.feats.backward(gy.to(torch.float64))
    return out.feats.detach(), out.coords, xx.grad, conv.weight.grad


def abs_bounds(x, coords, shape, B, w, k, s, p, subm, gy):
    y, _, gx, gw = reference(x.abs(), coords, shape, B, w.abs(), k, s, p, subm, gy.abs())
    return y, gx, gw


def worst(got, ref, bnd):
    """the largest |got - ref| / bnd (0 / 0 counts as 0; an error where bnd is 0 is infinite)."""
    err = (got.to(torch.float64) - ref.to(torch.float64)).abs()
    ratio = torch.where(bnd > 0, err / bnd.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, float('inf')), torch.zeros_like(err)))
    return float(ratio.max()) if ratio.numel() else 0.0
