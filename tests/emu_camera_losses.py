"""Torch-on-CPU emulation of tt_camera_loss (include/tt_b200.h section 11) — TEST HARNESS ONLY.  `install(emu, monkeypatch)` adds it to an
emu_lib.Emu instance (next to tests/emu_losses.py's entries), so that the product's host code for seg_loss / depth_loss runs on the CPU
(tests/test_camera_losses_cpu.py).  The arithmetic is plain fp64 torch following the kernel's contract: what is under test is the ground
truth checks, the staging and the descriptor filling above the C ABI."""
from types import SimpleNamespace

import torch
import torch.nn.functional as F

# A seeded bug (tests/test_camera_losses_cpu.py shows that tests/camera_loss_checks.py rejects each): None, or one of
#   'nan_dropping_min'  the block minimum skips NaN (fminf) instead of propagating it (torch.min)
#   'ce_all_pixels'     the cross-entropy mean divides by every pixel, not by the non-ignored ones
#   'no_max1'           depth_loss divides by the foreground count without max(1, .)
#   'bin_off_by_one'    the hot column is the bin itself, not bin - 1
#   'read_past_C'       the log-sum-exp reads one channel past the classes
#   'per_pixel_focal'   the focal transform is applied per pixel, then averaged
BUG = None


def nearest_index(out, n):
    """ATen's nearest source index (the kernel's formula): identity, k >> 1 for a 2x upscale, else floor(k * (float)n / out) clamped."""
    k = torch.arange(out)
    if out == n:
        return k
    if out == 2 * n:
        return k >> 1
    scale = torch.tensor(n, dtype=torch.float32) / out
    return torch.clamp(torch.floor(k.float() * scale).long(), max=n - 1)


def camera_terms(d):
    """the sums and counts of tt_camera_loss in fp64: {'seg': (CE sum, valid pixels, bad labels, total pixels, per-pixel focal mean),
    'depth': (BCE sum, foreground cells)}."""
    out = {}
    if d.seg_logits:
        BN, h, w = d.BN, d.seg_h, d.seg_w
        C = d.seg_classes + (BUG == 'read_past_C')
        logits = torch.as_strided(d.seg_logits.flat(), (BN, h, w, C), (h * w * d.seg_ld, w * d.seg_ld, d.seg_ld, 1), d.seg_coff).double()
        gt = d.seg_gt.flat()[:BN * d.seg_H * d.seg_W].view(BN, d.seg_H, d.seg_W)
        lab = gt[:, nearest_index(h, d.seg_H)][:, :, nearest_index(w, d.seg_W)]
        bad = ~(lab.abs() < 2147483648.0)                                # NaN / inf / no int: torch raises
        t = torch.where(bad, torch.zeros_like(lab), lab).long()          # .long() truncates toward zero
        keep = (t != d.seg_ignore) & ~bad
        bad = bad | (keep & ((t < 0) | (t >= d.seg_classes)))
        keep = keep & ~bad
        tc = t.clamp(0, d.seg_classes - 1)[..., None]                   # 8 frames at a time: the temporaries of a B = 16 batch stay small
        ce = torch.cat([torch.logsumexp(q, -1) - q.gather(-1, i)[..., 0] for q, i in zip(logits.split(8), tc.split(8))])
        pt = torch.exp(-ce[keep])
        focal = (-((1 - pt) ** d.seg_gamma) * d.seg_alpha * -ce[keep]).mean()
        out['seg'] = (ce[keep].sum(), int(keep.sum()), int(bad.sum()), lab.numel(), focal)
    if d.depth_logits:
        BN, h, w, f, D = d.BN, d.depth_h, d.depth_w, d.depth_factor, d.depth_bins
        logits = torch.as_strided(d.depth_logits.flat(), (BN, h, w, D), (h * w * d.depth_ld, w * d.depth_ld, d.depth_ld, 1),
                                  d.depth_coff).double()
        gt = d.depth_gt.flat()[:BN * h * f * w * f].view(BN, h * f, w * f)
        blocks = gt.reshape(BN, h, f, w, f).permute(0, 1, 3, 2, 4).reshape(BN, h, w, f * f)
        mn = torch.where(blocks == 0.0, torch.full_like(blocks, 1e5), blocks)
        if BUG == 'nan_dropping_min':
            mn = torch.where(mn.isnan(), torch.full_like(mn, float('inf')), mn)
        mn = mn.min(-1).values                                           # torch.min: NaN propagates
        v = (mn - torch.tensor(d.depth_offset, dtype=torch.float32)) / torch.tensor(d.depth_step, dtype=torch.float32)
        b = torch.where((v >= 0) & (v < D + 1), v, torch.zeros_like(v)).long()
        fg = b >= 1
        onehot = F.one_hot(b, D + 1)
        target = (onehot[..., :D] if BUG == 'bin_off_by_one' else onehot[..., 1:]).double()
        bce = F.binary_cross_entropy_with_logits(logits, target, reduction='none').sum(-1)
        out['depth'] = (bce[fg].sum(), int(fg.sum()))
    return out


def camera_finish(d, sums):
    """(seg_loss, depth_loss) from camera_terms' sums, as the kernel's last CTA computes them (None for a half that is off)."""
    seg = depth = None
    if 'seg' in sums:
        s, n, bad, total, focal = sums['seg']
        if BUG == 'ce_all_pixels':
            n = total
        ce = float('nan') if bad or not n else float(s) / n
        logpt = torch.tensor(-ce, dtype=torch.float64)
        seg = -((1 - torch.exp(logpt)) ** d.seg_gamma) * d.seg_alpha * logpt * d.seg_weight
        if BUG == 'per_pixel_focal':
            seg = focal * d.seg_weight
    if 'depth' in sums:
        s, n = sums['depth']
        if BUG == 'no_max1':
            depth = s / n if n else torch.tensor(float('nan'))
        else:
            depth = s / max(1, n)
    return seg, depth


def tt_camera_loss_workspace_bytes(emu, d):
    return 256


def tt_camera_loss(emu, d, out, ws, ws_bytes, stream):
    emu.launches += 1
    seg, depth = camera_finish(d, camera_terms(d))
    o = out.flat()
    if seg is not None:
        o[0] = float(seg)
    if depth is not None:
        o[1] = float(depth)
    return 0


def install(emu, monkeypatch=None):
    """monkeypatch None: the entries only, lib untouched (the kernel census's float64 reference, which decodes the product's
    tt_camera_loss_desc itself)."""
    for fn in (tt_camera_loss, tt_camera_loss_workspace_bytes):
        setattr(emu, fn.__name__, fn.__get__(emu))
    if monkeypatch is not None:
        from thinktwice_b200 import lib
        monkeypatch.setattr(lib, 'camera_loss_desc', lambda **f: SimpleNamespace(**f))   # the emulation reads the fields themselves
    return emu
