"""Weight preparation: reference-format state_dict -> kernel-layout tensors on the device.

Done once at load time (eval mode): BatchNorm running statistics are folded into the preceding (or, for
BN-after-ReLU, the following) linear map, weights are repacked K-major as [taps*Cin_g][Cout] for the
implicit-GEMM kernels, and transposed convolutions are split into their four 1x1 phases.
"""
import torch

from .engine import PackedConv


def bn_affine(sd, n, eps):
    s = sd[n + '.weight'].double() / torch.sqrt(sd[n + '.running_var'].double() + eps)
    t = sd[n + '.bias'].double() - sd[n + '.running_mean'].double() * s
    return s, t


def _rn_tf32(w):
    u = w.contiguous().view(torch.int32)
    u = u + 0xFFF + ((u >> 13) & 1)
    return (u & ~0x1FFF).view(torch.float32)


def tf32_split(w, rn=True):
    """w (fp32) -> (hi, lo) with hi = RN_tf32(w), lo = RN_tf32(w - hi): both exactly TF32-representable — the same
    split the tensor-core kernel applies to the activations in shared memory (csrc/gemm_conv_tc.cu: split_rn)."""
    w = w.float().contiguous()
    hi = _rn_tf32(w)
    return hi, _rn_tf32(w - hi)


F16S_SCALE = 2048.0


def f16s_split(w):
    """w (fp32 / fp64) -> (hi, lo') halves with hi = RN_f16(w), lo' = RN_f16((w - hi) * 2048): the scaled-split operand format of
    csrc/gemm_conv_f16s.cu (w = hi + lo' / 2048 to 2^-22 relative).  Weights must lie inside the fp16 range."""
    w = w.float().contiguous()
    if w.numel() and float(w.abs().max()) > 65504.0:
        raise ValueError('f16s weight packing: |w| exceeds the fp16 range')
    hi = w.half()
    lo = ((w - hi.float()) * F16S_SCALE).half()
    return hi, lo


class Packer:
    def __init__(self, sd, device, tc_mode=0):
        self.sd = {k: v.detach().cpu() for k, v in sd.items()}
        self.device = device
        self.tc_mode = tc_mode      # 0: SIMT only; 2 / 3: also pack [2][Cout][taps][Cin] TF32 hi/lo planes; 4: scaled-split fp16 planes

    def _tc(self, w_ohwi):
        """w_ohwi: (Cout, taps, Cin) float64 -> device tensor [2][Cout][taps][Cin] or None."""
        Cout, taps, Cin = w_ohwi.shape
        if self.tc_mode not in (2, 3) or Cin % 4 or Cout % 4 or Cout < 32:
            return None
        hi, lo = tf32_split(w_ohwi.float())
        return torch.stack([hi, lo]).contiguous().to(self.device)

    def _h(self, w_ohwi):
        """w_ohwi: (Cout, taps, Cin) float64 -> device tensor [2][Cout][taps][Cin8] halves (Cin zero-padded to 8) or None."""
        Cout, taps, Cin = w_ohwi.shape
        if self.tc_mode != 4 or Cout % 4 or Cout < 32:
            return None
        c8 = -(-Cin // 8) * 8
        w = w_ohwi.float()
        if c8 != Cin:
            w = torch.cat([w, w.new_zeros(Cout, taps, c8 - Cin)], 2)
        hi, lo = f16s_split(w)
        return torch.stack([hi, lo]).contiguous().to(self.device)

    def _dev(self, t):
        return None if t is None else t.float().contiguous().to(self.device)

    @staticmethod
    def _reindex(w, index):
        """input-channel gather along dim 1; index -1 inserts a zero channel."""
        idx = torch.as_tensor(index, dtype=torch.long)
        out = w.new_zeros((w.shape[0], idx.numel()) + tuple(w.shape[2:]))
        ok = idx >= 0
        out[:, ok] = w[:, idx[ok]]
        return out

    def conv(self, n, bn=None, eps=1e-5, groups=1, cin_pad=None, cin_index=None, cout_pad=None):
        """Conv2d weight (Cout, Cin_g, KH, KW) [+bias] followed by BN `bn` -> PackedConv."""
        w = self.sd[n + '.weight'].double()
        b = self.sd.get(n + '.bias')
        b = b.double() if b is not None else None
        if bn is not None:
            s, t = bn_affine(self.sd, bn, eps)
            w = w * s.view(-1, 1, 1, 1)
            b = t if b is None else b * s + t
        if cin_index is not None:
            w = self._reindex(w, cin_index)
        if cout_pad is not None and cout_pad > w.shape[0]:           # zero output channels: lifts a thin conv onto the tensor cores
            w = torch.cat([w, w.new_zeros((cout_pad - w.shape[0],) + tuple(w.shape[1:]))], 0)
            if b is not None:
                b = torch.cat([b, b.new_zeros(cout_pad - b.shape[0])])
        Cout, Cg, KH, KW = w.shape
        if cin_pad is not None and cin_pad > Cg:
            assert groups == 1
            w = torch.cat([w, w.new_zeros(Cout, cin_pad - Cg, KH, KW)], 1)
            Cg = cin_pad
        packed = w.permute(2, 3, 1, 0).reshape(KH * KW * Cg, Cout)
        ohwi = w.permute(0, 2, 3, 1).reshape(Cout, KH * KW, Cg)
        w_tc = self._tc(ohwi) if groups == 1 else None
        return PackedConv(self._dev(packed), self._dev(b), Cg * groups, Cout, KH, KW, groups, w_tc, self._h(ohwi) if groups == 1 else None)

    def conv_rowpacked(self, n, bn=None, eps=1e-5, cpad=4, kslab=32):
        """thin-channel Conv2d (Cout, Cin<=cpad, KH, KW) [+BN] as a KH x 1 conv whose "channels" are the KW*cpad floats
        of a tap row, contiguous in a channels-last image with `cpad` floats per pixel (tt_conv_desc.x_hstride).
        K per kernel row = kslab (>= KW*cpad, zero weights in the tail): the 7x7x3 stem becomes 7 full 32-float K slabs
        instead of 49 slabs with 3 of 32 lanes in use."""
        w = self.sd[n + '.weight'].double()
        b = self.sd.get(n + '.bias')
        b = b.double() if b is not None else None
        if bn is not None:
            s, t = bn_affine(self.sd, bn, eps)
            w = w * s.view(-1, 1, 1, 1)
            b = t if b is None else b * s + t
        Cout, Cin, KH, KW = w.shape
        assert Cin <= cpad and KW * cpad <= kslab
        wk = w.new_zeros(Cout, KH, kslab)                                # [co][kh][kw * cpad + c]
        wk.view(Cout, KH, kslab // cpad, cpad)[:, :, :KW, :Cin] = w.permute(0, 2, 3, 1)
        pc = PackedConv(self._dev(wk.permute(1, 2, 0).reshape(KH * kslab, Cout)), self._dev(b), kslab, Cout, KH, 1,
                        w_tc=self._tc(wk), w_h=self._h(wk))
        pc.alg_k = KH * KW * Cin
        return pc

    def conv_group_gemms(self, n, groups):
        """grouped Conv2d weight (Cout, Cin_g, KH, KW) -> one dense GEMM per group over im2col columns laid out
        [group][tap][Cin_g] (tt_dcn_im2col): list of PackedConv with Cin = KH*KW*Cin_g, Cout = Cout/groups."""
        w = self.sd[n + '.weight'].double()
        assert self.sd.get(n + '.bias') is None
        Cout, Cg, KH, KW = w.shape
        Co = Cout // groups
        out = []
        for g in range(groups):
            wg = w[g * Co:(g + 1) * Co].permute(0, 2, 3, 1).reshape(Co, KH * KW * Cg)      # K = (tap, cin)
            out.append(PackedConv(self._dev(wg.t()), None, KH * KW * Cg, Co, w_tc=self._tc(wg.reshape(Co, 1, KH * KW * Cg)),
                                  w_h=self._h(wg.reshape(Co, 1, KH * KW * Cg))))
        return out

    def linear(self, n, bn_after=None, eps=1e-5, in_affine=None, cin_pad=None, weight=None, bias=None, cin_index=None):
        """Linear (Cout, Cin).  in_affine=(s, t): the input is s*x + t (a folded BatchNorm1d in front);
        bn_after: BatchNorm1d applied to the output."""
        w = (self.sd[n + '.weight'] if weight is None else weight).double()
        b = self.sd.get(n + '.bias') if bias is None else bias
        b = b.double() if b is not None else torch.zeros(w.shape[0], dtype=torch.float64)
        if b.numel() != w.shape[0]:                                 # per-image bias table: no folding allowed
            assert in_affine is None and bn_after is None
        if in_affine is not None:
            s, t = in_affine
            b = b + w @ t
            w = w * s.view(1, -1)
        if bn_after is not None:
            s, t = bn_affine(self.sd, bn_after, eps)
            w = w * s.view(-1, 1)
            b = b * s + t
        if cin_index is not None:
            w = self._reindex(w, cin_index)
        Cout, Cin = w.shape
        if cin_pad is not None and cin_pad > Cin:
            w = torch.cat([w, w.new_zeros(Cout, cin_pad - Cin)], 1)
            Cin = cin_pad
        return PackedConv(self._dev(w.t()), self._dev(b), Cin, Cout, w_tc=self._tc(w.reshape(Cout, 1, Cin)), w_h=self._h(w.reshape(Cout, 1, Cin)))

    def conv1x1_as_linear(self, n, **kw):
        w = self.sd[n + '.weight']
        return self.linear(n, weight=w.reshape(w.shape[0], -1), **kw)

    def convT(self, n, bn=None, eps=1e-5):
        """ConvTranspose2d k2s2 (Cin, Cout, 2, 2) -> four PackedConv, phase (i, j) writes pixel (2h+i, 2w+j)."""
        w = self.sd[n + '.weight'].double()
        b = self.sd.get(n + '.bias')
        b = b.double() if b is not None else None
        if bn is not None:
            s, t = bn_affine(self.sd, bn, eps)
            w = w * s.view(1, -1, 1, 1)
            b = t if b is None else b * s + t
        Cin, Cout = w.shape[:2]
        bd = self._dev(b)
        return [[PackedConv(self._dev(w[:, :, i, j]), bd, Cin, Cout, w_tc=self._tc(w[:, :, i, j].t().reshape(Cout, 1, Cin)),
                            w_h=self._h(w[:, :, i, j].t().reshape(Cout, 1, Cin)))
                 for j in range(2)] for i in range(2)]

    def spconv(self, n, bn, eps=1e-3):
        """spconv weight (Cout, kd, kh, kw, Cin) + BatchNorm1d -> PackedConv with K = (tap, cin)."""
        w = self.sd[n + '.weight'].double()
        s, t = bn_affine(self.sd, bn, eps)
        w = w * s.view(-1, 1, 1, 1, 1)
        Cout, kd, kh, kw, Cin = w.shape
        packed = w.reshape(Cout, kd * kh * kw, Cin).permute(1, 2, 0).reshape(kd * kh * kw * Cin, Cout)
        pc = PackedConv(self._dev(packed), self._dev(t), Cin, Cout, w_tc=self._tc(w.reshape(Cout, kd * kh * kw, Cin)) if Cin >= 32 else None,
                        w_h=self._h(w.reshape(Cout, kd * kh * kw, Cin)) if Cin >= 32 else None)
        return pc, (kd, kh, kw)

    def vec(self, n):
        return self._dev(self.sd[n])
