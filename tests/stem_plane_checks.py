"""Bitwise checker of the row-packed stem's operand planes that tt_preprocess_u8 writes (include/tt_b200.h section 8): shared by the
full-shape GPU test (tests/test_preprocess_gpu.py) and its negative controls on the CPU (tests/test_preprocess_cpu.py)."""
import torch

SENTINEL = 0x7E5A                   # fp16 bits of a quiet NaN with a payload: never a value split_h writes, so any write over it shows


def sentinel_planes(split_plane, device):
    """(2 * split_plane,) fp16 planes pre-filled with the sentinel bits: hi at 0, lo' at split_plane."""
    return torch.full((2 * split_plane,), SENTINEL, dtype=torch.int16, device=device).view(torch.float16)


def split_h(v):
    """csrc/preprocess.cu split_h in torch: hi = RN_f16(clamp(v, +-65504)), lo' = RN_f16((clamp(v) - hi) * 2048).  The difference and
    the scaling are exact in fp32, so the kernel's bits are reproduced exactly."""
    c = v.float().clamp(-65504.0, 65504.0)
    hi = c.half()
    return hi, ((c - hi.float()) * 2048.0).half()


def stem_plane_failures(planes, split_plane, v, pad):
    """planes: the (2 * split_plane,) fp16 buffer after one call with n = v.shape[0] images; v: the (n, 3, H0, W0) fp32 NCHW result of the
    same call; pad = (pad_H, pad_W, top, left).  Returns the list of violated properties (empty: the planes are right):
      * channels 0-2 of every interior pixel: bitwise split_h(v) in the hi and lo' planes;
      * channels 3-7 of every interior pixel: +0;
      * every border pixel of every slot, and the guard gap after the n-th slot of each plane: still the sentinel."""
    n, _, H0, W0 = v.shape
    pH, pW, top, left = pad
    slot = pH * pW * 8
    bits = planes.view(torch.int16).view(2, split_plane)
    slots = bits[:, :n * slot].view(2, n, pH, pW, 8)
    inner = slots[:, :, top:top + H0, left:left + W0]
    hi, lo = split_h(v.permute(0, 2, 3, 1))
    out = []
    for p, (name, want) in enumerate((('hi', hi), ("lo'", lo))):
        bad = (inner[p, ..., :3] != want.view(torch.int16)).nonzero()
        if bad.numel():
            out.append(f'{name} plane differs from split_h of the NCHW value at {bad.shape[0]} elements, first (n, y, x, c) = {bad[0].tolist()}')
    bad = (inner[..., 3:] != 0).nonzero()
    if bad.numel():
        out.append(f'pad channels 3-7 not +0 at {bad.shape[0]} elements, first (plane, n, y, x, c) = {bad[0].tolist()}')
    border = torch.ones(pH, pW, dtype=torch.bool, device=bits.device)
    border[top:top + H0, left:left + W0] = False
    bad = (slots[:, :, border] != SENTINEL).nonzero()
    if bad.numel():
        out.append(f'border pixels written at {bad.shape[0]} elements, first (plane, n, border pixel, c) = {bad[0].tolist()}')
    bad = (bits[:, n * slot:] != SENTINEL).nonzero()
    if bad.numel():
        out.append(f'guard gap after slot {n - 1} written at {bad.shape[0]} elements, first (plane, offset) = {bad[0].tolist()}')
    return out
