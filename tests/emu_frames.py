"""Torch-on-CPU emulations of the independent-frames Look entry points (include/tt_b200.h: tt_msda_forward_frames,
tt_look_reduce_frames) — TEST HARNESS ONLY.  `install(emu)` adds them to an emu_lib.Emu instance, so that the product's host code
for the independent-frames mode runs on the CPU like the rest of the forward (tests/test_independent_frames_cpu.py)."""
import torch

from emu_lib import NULL, Ptr, _desc


def frame_max_len(counts, B, cams):
    """max_len_b = max over cams of counts[b][cam]."""
    return [int(v) for v in counts.flat()[:B * cams].view(B, cams).amax(1)]


def tt_msda_forward_frames(emu, d, value, off, logits, ref, counts, cams, out, stream):
    """tt_msda_forward on rows r < max_len_b of each frame b only; the other rows of `out` are left as they are."""
    dd = _desc(d)
    BN, cap, E = dd.BN, dd.rows_cap, dd.heads * dd.dh
    assert cams > 0 and BN % cams == 0
    full = torch.empty(BN * cap * E, dtype=out.t.dtype, device=out.t.device)
    emu.tt_msda_forward(d, value, off, logits, ref, NULL, Ptr(full), stream)
    src, dst = full.view(BN, cap, E), out.flat()[:BN * cap * E].view(BN, cap, E)
    for b, ml in enumerate(frame_max_len(counts, BN // cams, cams)):
        dst[b * cams:(b + 1) * cams, :ml] = src[b * cams:(b + 1) * cams, :ml]
    return 0


def tt_look_reduce_frames(emu, rows, B, cams, cap, Cc, counts, out, stream):
    """msda:338-342 at B = 1 for every frame: rows 1 <= r < max_len_b summed, divisor 1."""
    emu.launches += 1
    r = rows.flat()[:B * cams * cap * Cc].view(B, cams, cap, Cc)
    o = out.flat()[:B * cams * Cc].view(B, cams * Cc)
    for b, ml in enumerate(frame_max_len(counts, B, cams)):
        o[b] = r[b, :, 1:min(ml, cap)].double().sum(1).float().reshape(cams * Cc)
    return 0


def install(emu):
    for fn in (tt_msda_forward_frames, tt_look_reduce_frames):
        setattr(emu, fn.__name__, fn.__get__(emu))
    return emu
