"""float64 reference of the training lift-splat (include/tt_b200.h §14, csrc/lift_splat.cu): the cell of every bin with its
ambiguity, and the two gradients with their rounding bounds.  Shared by tests/test_lift_splat_train_cpu.py (which pins it against
the oracle composition under autograd and a literal loop) and tests/test_lift_splat_train_gpu.py.

Notation: pixel p of frame b, bins d < D, logits l, pi = softmax(l), context f (C channels), G = dL/dbev (B, C, Y, X), cell(p, d)
the cell the forward recorded (-1 outside the grid), g[p][d] = f[p] . G[b][:, cell(p, d)] (0 outside), S[p] = sum_d pi g.
  grad_logits[p][d] = pi[p][d] (g[p][d] - S[p]),   grad_context[p] = sum_d pi[p][d] G[b][:, cell(p, d)].

Bounds (u = 2^-24), all in multiples of u times sums of |terms|, on the recorded cells (so no ambiguity term):
  pi   : as ref_lift: expf(l - max) * (1 / sum) is within e_pi = (a + D + 14) u pi, a = max - l; a weight below fp32's normal
         range may flush, so it carries its whole pi plus 2^-148.
  g    : the kernel's dot runs ceil(C / 32) fmaf per lane and a 5-level butterfly: |dg| <= gamma(C/32 + 6) sum_c |f_c G_c| = gamma M.
  runs : a run's weight sums its n <= D bins in order ((n - 1) u) and the run count R <= D adds one rounding per run to grad_context
         and to S, so each bin's weight carries 2 D u pi on top of e_pi:
         |d grad_context_c| <= sum_d (e_pi + 2 D u pi) |G_c(cell(p, d))|.
  S    : |dS| <= sum_d [e_pi |g| + pi (2 D u |g| + gamma M)].
  grad_logits: the product pi (g - S) rounds twice after the subtraction:
         |d grad_logits| <= e_pi |g - S| + pi (gamma M + |dS| + 2 u |g - S|).
  Both bounds are widened by 1 % for the second-order terms, and by 2^-149 per rounding that may land in the subnormal range
  (grad_logits' last product; grad_context's at most D fmaf)."""
import types

import numpy as np
import torch

from camera_look_checks import U, gamma

TINY = 2.0 ** -126
UNDER = 2.0 ** -149      # absolute error of an fp32 rounding in the subnormal range (no flush to zero)


def ref_cells(s2e, intrin, ida, mats32, geo):
    """float64 cell of every bin and the per-bin restatement of ref_lift's geometry-error analysis.  s2e / intrin / ida (B, N, 4, 4)
    fp32, mats32 the [BN][32] matrices the kernel is given.  Returns dict(cell (pixels, D) int64 (-1 outside the grid),
    amb (pixels, D) bool, cand (pixels, D, 8) int64 (the cell or -1 of each corner of the error box), in_bins, amb_bins);
    pixels in the kernel's order (bn, h, w)."""
    from oracle.camera import LSS as OLSS
    B, N = s2e.shape[:2]
    D, fH, fW = geo['D'], geo['fH'], geo['fW']
    X, Y, Z = geo['X'], geo['Y'], geo['Z']
    lower, size = geo['lower'].astype(np.float64), geo['size'].astype(np.float64)
    hi_ = np.array([X, Y, Z])
    x = geo['frustum'].double().numpy()
    ns = types.SimpleNamespace(frustum=geo['frustum'].double())
    m32 = mats32.detach().cpu().double().numpy().reshape(B, N, 2, 4, 4)
    g4 = gamma(4)
    cells, ambs, cands = [], [], []

    def to_cell(i):
        ok = ((i >= 0) & (i < hi_)).all(-1)
        return np.where(ok, i[..., 1] * X + i[..., 0], -1)
    for b in range(B):
        g = OLSS.get_geometry(ns, s2e[b:b + 1].double(), intrin[b:b + 1].double(), ida[b:b + 1].double())[0].numpy()
        Mi = torch.inverse(ida[b].double()).numpy()
        Mc = s2e[b].double().matmul(torch.inverse(intrin[b].double())).numpy()
        dMi, dMc = np.abs(m32[b, :, 0] - Mi), np.abs(m32[b, :, 1] - Mc)
        ax = np.abs(x)
        A = np.einsum('nij,dhwj->ndhwi', np.abs(Mi), ax)
        eq = g4 * A + np.einsum('nij,dhwj->ndhwi', dMi, ax)
        P = np.stack([A[..., 0] * A[..., 2], A[..., 1] * A[..., 2], A[..., 2], A[..., 3]], -1)
        ep = np.stack([A[..., 0] * eq[..., 2] + A[..., 2] * eq[..., 0] + eq[..., 0] * eq[..., 2] + U * P[..., 0],
                       A[..., 1] * eq[..., 2] + A[..., 2] * eq[..., 1] + eq[..., 1] * eq[..., 2] + U * P[..., 1],
                       eq[..., 2], eq[..., 3]], -1)
        aMc = np.abs(Mc[:, :3])
        ee = (g4 * np.einsum('nij,ndhwj->ndhwi', aMc, P) + np.einsum('nij,ndhwj->ndhwi', aMc, ep)
              + np.einsum('nij,ndhwj->ndhwi', dMc[:, :3], P))
        t = (g - lower) / size
        et = ee / size + 2 * U * np.abs(t) + 1e-12
        t, et = (v.transpose(0, 2, 3, 1, 4).reshape(N * fH * fW, D, 3) for v in (t, et))
        idx, lo, hi = np.trunc(t).astype(np.int64), np.trunc(t - et).astype(np.int64), np.trunc(t + et).astype(np.int64)
        cells.append(to_cell(idx))
        ambs.append((lo != hi).any(-1))
        cands.append(np.stack([to_cell(np.where(np.array([(k >> i) & 1 for i in range(3)], bool), hi, lo)) for k in range(8)], -1))
    cell, amb, cand = np.concatenate(cells), np.concatenate(ambs), np.concatenate(cands)
    return dict(cell=cell, amb=amb, cand=cand, in_bins=int((cell >= 0).sum()), amb_bins=int((amb & (cand >= 0).any(-1)).sum()))


def check_bin_cell(got, ref, name='bin_cell'):
    """got (pixels, D) int: equal to the float64 cell, except that an ambiguous bin may hold any of its candidate cells (or -1
    when a candidate lies outside the grid).  Ambiguous bins must stay under 0.1 % of the in-grid bins."""
    got = np.asarray(got).astype(np.int64)
    amb, ins = ref['amb_bins'], ref['in_bins']
    assert amb <= 1e-3 * max(ins, 1), f'{name}: {amb} ambiguous bins of {ins} in the grid'
    bad = ~ref['amb'] & (got != ref['cell'])
    if bad.any():
        p, d = np.argwhere(bad)[0]
        raise AssertionError(f'{name}: pixel {p} bin {d}: cell {got[p, d]}, float64 cell {ref["cell"][p, d]}')
    bad = ref['amb'] & ~(ref['cand'] == got[..., None]).any(-1)
    if bad.any():
        p, d = np.argwhere(bad)[0]
        raise AssertionError(f'{name}: pixel {p} bin {d} (ambiguous): cell {got[p, d]} is none of {sorted(set(ref["cand"][p, d]))}')


def ref_grads(logits, context, cells, G):
    """float64 gradients on the recorded cells.  logits (BN, D, fH, fW), context (BN, C, fH, fW), cells (BN*fH*fW, D) int,
    G (B, C, Y, X); any device (the work follows `context`).  Returns dict(gl, gl_bound (BN, D, fH, fW), gc, gc_bound (BN, C, fH, fW))
    float64, computed one frame at a time with dense (pixels x cells) matrices: never the (pixels, D, C) tensor."""
    dev = context.device
    BN, D, fH, fW = logits.shape
    B, Cc, Y, X = G.shape
    N, ncell, HW = BN // B, X * Y, fH * fW
    P = N * HW
    gam = gamma(-(-Cc // 32) + 6)
    out = {k: [] for k in ('gl', 'gl_bound', 'gc', 'gc_bound')}
    cells = torch.as_tensor(np.asarray(cells), device=dev).long().reshape(BN * HW, D)
    for b in range(B):
        lg = logits[b * N:(b + 1) * N].to(dev).double().permute(0, 2, 3, 1).reshape(P, D)
        f = context[b * N:(b + 1) * N].to(dev).double().permute(0, 2, 3, 1).reshape(P, Cc)
        cell = cells[b * P:(b + 1) * P]
        Gb = G[b].to(dev).double().reshape(Cc, ncell).t()                     # (cells, C)
        a = lg.max(1, keepdim=True).values - lg
        e = torch.exp(-a)
        pi = e / e.sum(1, keepdim=True)
        epi = (a + D + 14) * U * pi + torch.where(pi < TINY, pi, torch.zeros_like(pi)) + 2.0 ** -148
        ins = (cell >= 0).double()
        ci = cell.clamp(min=0)
        g = (f @ Gb.t()).gather(1, ci) * ins                                  # (P, D)
        M = (f.abs() @ Gb.abs().t()).gather(1, ci) * ins
        S = (pi * g).sum(1, keepdim=True)
        W = torch.zeros(P, ncell, dtype=torch.float64, device=dev).scatter_add_(1, ci, pi * ins)
        Wb = torch.zeros_like(W).scatter_add_(1, ci, (epi + 2 * D * U * pi) * ins)
        dS = (epi * g.abs() + pi * (2 * D * U * g.abs() + gam * M)).sum(1, keepdim=True)
        gmS = g - S
        gl_b = 1.01 * (epi * gmS.abs() + pi * (gam * M + dS + 2 * U * gmS.abs())) + UNDER
        nchw = lambda v: v.reshape(N, fH, fW, -1).permute(0, 3, 1, 2)
        out['gl'].append(nchw(pi * gmS)); out['gl_bound'].append(nchw(gl_b))
        out['gc'].append(nchw(W @ Gb)); out['gc_bound'].append(nchw(1.01 * (Wb @ Gb.abs()) + D * UNDER))
    return {k: torch.cat(v) for k, v in out.items()}


def check_grads(gl, gc, ref, name='lift_splat_train'):
    """gl / gc: the kernel's grad_logits / grad_context (either may be None).  Every element within its bound (exactly the reference
    where the bound is 0).  Returns (largest |err| / bound of grad_logits, of grad_context)."""
    ratios = []
    for key, got, what in (('gl', gl, 'grad_logits'), ('gc', gc, 'grad_context')):
        if got is None:
            ratios.append(None)
            continue
        val, lim = ref[key], ref[key + '_bound']
        got = got.to(val.device).double()
        assert got.shape == val.shape, f'{name}: {what} {tuple(got.shape)}, expected {tuple(val.shape)}'
        err = (got - val).abs()
        over = ~(err <= lim)
        if over.any():
            i = tuple(int(v) for v in torch.nonzero(over)[0])
            raise AssertionError(f'{name}: {what} (image {i[0]}, channel {i[1]}, h {i[2]}, w {i[3]}): {float(got[i]):.7g}, expected '
                                 f'{float(val[i]):.7g} +- {float(lim[i]):.2e}')
        pos = lim > 0
        ratios.append(float((err[pos] / lim[pos]).max()) if pos.any() else 0.0)
    return tuple(ratios)


def run_forward(d, geo, logits, context, mats, bev, bin_cell, ws=None):
    """tt_lift_splat_train_forward through the C ABI; bev [B][Y][X][C], bin_cell [pixels][D] (or None)."""
    import ctypes as C
    from thinktwice_b200 import lib
    dev = context.device
    n = int(lib.load().tt_lift_splat_train_workspace_bytes(C.byref(d)))
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device=dev) if ws is None else ws
    fu, fv, fd = geo['fu'].to(dev), geo['fv'].to(dev), geo['fd'].to(dev)
    lib.call('tt_lift_splat_train_forward', C.byref(d), lib._p(logits), lib._p(context), lib._p(mats.to(dev)), lib._p(fu), lib._p(fv),
             lib._p(fd), lib._p(bev), lib._p(bin_cell), lib._p(ws), C.c_size_t(n))
    return ws


def run_backward(d, logits, context, bin_cell, G, gl, gc, ws=None):
    """tt_lift_splat_train_backward through the C ABI; G (B, C, Y, X) at its own strides, gl / gc outputs (or None)."""
    import ctypes as C
    from thinktwice_b200 import lib
    dev = context.device
    n = int(lib.load().tt_lift_splat_train_workspace_bytes(C.byref(d)))
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device=dev) if ws is None else ws
    lib.call('tt_lift_splat_train_backward', C.byref(d), lib._p(logits), lib._p(context), lib._p(bin_cell), lib._p(G),
             *[C.c_longlong(s) for s in G.stride()], lib._p(gl), lib._p(gc), lib._p(ws), C.c_size_t(n))
    return ws


def train_desc(geo, B, C_, depth_bstride=None):
    from thinktwice_b200 import lib
    d = lib.LiftSplatTrainDesc()
    d.B, d.N, d.D, d.fH, d.fW, d.C = B, geo['N'], geo['D'], geo['fH'], geo['fW'], C_
    d.depth_bstride = geo['D'] * geo['fH'] * geo['fW'] if depth_bstride is None else depth_bstride
    d.lower, d.size = lib.f3(geo['lower']), lib.f3(geo['size'])
    d.X, d.Y, d.Z = geo['X'], geo['Y'], geo['Z']
    return d
