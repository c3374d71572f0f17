"""Torch-on-CPU emulations of the open-loop loss entry points (include/tt_b200.h: tt_loss_reduce, tt_eltwise op 4) — TEST HARNESS ONLY.
`install(emu, monkeypatch)` adds them to an emu_lib.Emu instance, so that the product's host code for the teacher-forced pass and
ThinkTwiceDecoder.loss runs on the CPU like the rest of the forward (tests/test_losses_cpu.py).  The arithmetic is plain fp64 torch:
what is under test is the descriptor filling (pointers, strides, slots, scales) above the C ABI."""
import torch
from torch.distributions import Beta, kl_divergence

from emu_lib import _v


def _view(p, shape, stride):
    return torch.as_strided(p.flat(), shape, stride).double()


def _action(a, b, comp):
    x = torch.full_like(a, 0.5 if comp == 1 else 0.0)
    x = torch.where((a > 1) & (b > 1), (a - 1) / (a + b - 2), x)
    x = torch.where((a <= 1) & (b > 1), torch.zeros_like(x), x)
    x = torch.where((a > 1) & (b <= 1), torch.ones_like(x), x)
    x = torch.where((a <= 1) & (b <= 1), a / torch.clamp(a + b, min=1e-5), x)
    return x * 2 - 1


def term_operands(t):
    """(P, G, P2, G2) of one term as fp64 tensors of its logical shape (G zeros without gt; P2 / G2 None without them)."""
    shape = list(t['shape'])
    P = _view(t['pred'], shape, t['pred_stride'])
    G = _view(t['gt'], shape, t['gt_stride']) if t['gt'] else torch.zeros(shape, dtype=torch.float64, device=P.device)
    P2 = _view(t['pred2'], shape, t['pred_stride']) if t['pred2'] else None
    G2 = _view(t['gt2'], shape, t['gt_stride']) if t['gt2'] else None
    return P, G, P2, G2


def term_values(t):
    """the per-element values of one term (before its scale), fp64, over its logical shape."""
    P, G, P2, G2 = term_operands(t)
    if t['kind'] in (0, 1):
        d = (P - G).abs()
        v = torch.where(d < 1, 0.5 * d * d, d - 0.5)
        if t['kind'] == 1:
            v = v.clamp(-5.0, 5.0)
    elif t['kind'] == 2:
        v = (P - G).abs()
    elif t['kind'] == 3:                                               # NaN outside the Beta domain, as the kernel
        ok = torch.stack([x.isfinite() & (x > 0) for x in (G, G2, P, P2)]).all(0)
        one = torch.ones_like(G)
        v = kl_divergence(Beta(torch.where(ok, G, one), torch.where(ok, G2, one)), Beta(torch.where(ok, P, one), torch.where(ok, P2, one)))
        v = torch.where(ok, v, torch.full_like(v, float('nan')))
    else:
        v = (_action(P.float(), P2.float(), t['aux']).double() - _action(G.float(), G2.float(), t['aux']).double()).abs()
    return v


def tt_loss_reduce(emu, terms, n_terms, out, n_slots, ws, ws_bytes, stream):
    emu.launches += 1
    acc = torch.zeros(n_slots, dtype=torch.float64, device=out.t.device)
    for t in terms[:n_terms]:
        acc[t['slot']] += t['scale'] * term_values(t).sum()
    out.flat()[:n_slots] = acc.to(out.t.dtype)
    return 0


def tt_eltwise(emu, op, act, a, a_ld, b, b_ld, c, c_ld, y, y_ld, rows, cols, stream):
    if _v(op) != 4:
        return emu._eltwise(op, act, a, a_ld, b, b_ld, c, c_ld, y, y_ld, rows, cols, stream)
    from emu_lib import _act
    emu.launches += 1
    A = torch.as_strided(a.flat(), (rows, cols), (a_ld, 1))
    torch.as_strided(y.flat(), (rows, cols), (y_ld, 1)).copy_(_act(A + torch.log(-torch.expm1(-A)), _v(act)))
    return 0


def install(emu, monkeypatch=None):
    """monkeypatch None: the entries only, lib untouched (the kernel census's float64 reference, which decodes the product's
    tt_loss_term array into term dicts itself)."""
    emu._eltwise = emu.tt_eltwise
    for fn in (tt_loss_reduce, tt_eltwise):
        setattr(emu, fn.__name__, fn.__get__(emu))
    if monkeypatch is not None:
        from thinktwice_b200 import lib
        monkeypatch.setattr(lib, 'pack_loss_terms', lambda terms: terms)     # the emulation reads the term dicts themselves
    return emu
