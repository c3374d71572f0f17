"""float64 restatement of the training-side batch norm (include/tt_b200.h §18) on rows x [M][C]: the forward with batch statistics,
the running update (unbiased variance), and the backward with ReLU and residual, including SyncBatchNorm's semantics over an R-way split
of the rows (grad_x from the global sums, grad_weight / grad_bias from each rank's own rows).  `bug` seeds one mistake each:
'biased_running_var', 'global_grad_weight', 'mask_without_residual' (the ReLU mask taken from z before the residual is added)."""
import torch


def stats(x, eps):
    """(mean, invstd, biased var, unbiased var) per channel of the rows x."""
    n = x.shape[0]
    mean = x.mean(0)
    m2 = ((x - mean) ** 2).sum(0)
    return mean, 1.0 / torch.sqrt(m2 / n + eps), m2 / n, m2 / (n - 1)


def running(rm, rv, x, eps, factor, bug=None):
    mean, _, var_b, var_u = stats(x, eps)
    return (1 - factor) * rm + factor * mean, (1 - factor) * rv + factor * (var_b if bug == 'biased_running_var' else var_u)


def z_of(x, r, w, b, mean, invstd):
    z = w * ((x - mean) * invstd) + b
    return z if r is None else z + r


def forward(x, r, w, b, eps, relu):
    mean, invstd, _, _ = stats(x, eps)
    z = z_of(x, r, w, b, mean, invstd)
    return torch.relu(z) if relu else z


def backward(x, r, w, b, gy, eps, relu, splits=None, mask=None, bug=None):
    """(grad_x, grad_r, [grad_weight per rank], [grad_bias per rank]); splits: row counts of the ranks (one rank when None).
    mask: the ReLU's pass mask (by default z > 0 in float64)."""
    mean, invstd, _, _ = stats(x, eps)
    xhat = (x - mean) * invstd
    if relu:
        if mask is None:
            zm = z_of(x, None if bug == 'mask_without_residual' else r, w, b, mean, invstd)
            mask = zm > 0
        dz = gy * mask
    else:
        dz = gy
    n = x.shape[0]
    sdz, sdzx = dz.sum(0), (dz * xhat).sum(0)
    grad_x = w * invstd * (dz - sdz / n - xhat * sdzx / n)
    splits = [n] if splits is None else list(splits)
    gw, gb, lo = [], [], 0
    for m in splits:
        if bug == 'global_grad_weight':
            gw.append(sdzx.clone())
            gb.append(sdz.clone())
        else:
            gw.append((dz[lo:lo + m] * xhat[lo:lo + m]).sum(0))
            gb.append(dz[lo:lo + m].sum(0))
        lo += m
    return grad_x, (dz if r is not None else None), gw, gb
