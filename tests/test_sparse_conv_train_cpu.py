"""CPU side of the training-side sparse convolution (include/tt_b200.h §13, thinktwice_b200/ops/sparse_conv.py): the ctypes descriptor,
the library's and the modules' refusals of what the reference does not build, CPU tensors refused, the trainable SparseEncoder's
parameter names, and the float64 reference the GPU tests compare against pinned to a masked dense convolution and to a literal loop."""
import ctypes as C
import itertools
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

from sparse_conv_reference import reference, site_keys
from thinktwice_b200 import lib
from thinktwice_b200.ops import sparse_conv as sc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the thinktwice.py middle encoder (configs/thinktwice.py, pts_middle_encoder)
CFG = dict(in_channels=5, sparse_shape=[41, 672, 672], output_channels=128, encoder_channels=((16, 16, 32), (32, 32, 64), (64, 64, 128), (128, 128)),
           encoder_paddings=((0, 0, 1), (0, 0, 1), (0, 0, [0, 1, 1]), (0, 0)))
# the convolutions the reference builds: (kernel, stride, padding, subm)
LAYERS = [((3, 3, 3), (1, 1, 1), (1, 1, 1), True), ((3, 3, 3), (2, 2, 2), (1, 1, 1), False), ((3, 3, 3), (2, 2, 2), (0, 1, 1), False),
          ((3, 1, 1), (2, 1, 1), (0, 0, 0), False)]


def test_ctypes_descriptor_matches_the_c_header(tmp_path):
    fields = [n for n, _ in lib.SparseConvTrainDesc._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "tt_b200.h"\nint main(void) {\n' +
                   ''.join(f'  printf("%zu\\n", offsetof(tt_sparse_conv_train_desc, {n}));\n' for n in fields) +
                   '  printf("%zu\\n", sizeof(tt_sparse_conv_train_desc));\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [getattr(lib.SparseConvTrainDesc, n).offset for n in fields] + [C.sizeof(lib.SparseConvTrainDesc)]


def test_new_entries_are_exported():
    assert {'tt_sparse_conv_train_workspace_bytes', 'tt_sparse_conv_train_forward', 'tt_sparse_conv_train_backward',
            'tt_sparse_pairs_ordered_workspace_bytes', 'tt_sparse_pairs_ordered'} <= set(lib.EXPORTS)


REFUSED = [(dict(dilation=2), 'dilation'), (dict(groups=2), 'groups'), (dict(bias=True), 'bias'), (dict(transposed=True), 'transposed'),
           (dict(inverse=True), 'inverse'), (dict(kernel_size=5), 'kvol'), (dict(kernel_size=(3, 3, 1)), 'kernel_size'),
           (dict(stride=3), 'stride'), (dict(padding=2), 'padding'), (dict(subm=True, stride=2), 'stride'), (dict(subm=True, stride=1, padding=0), 'padding')]


@pytest.mark.parametrize('kw,named', REFUSED)
def test_the_library_refuses_what_the_reference_does_not_build(kw, named):
    """checked before any pointer or device is touched: the refusal works without a GPU."""
    geom = dict(kernel_size=3, stride=2, padding=1, subm=False)
    geom.update(kw)
    d = sc.conv_desc(16, 32, n_in=100, n_out=100, pair_cap=100, **geom)
    L = lib.load()
    assert L.tt_sparse_conv_train_workspace_bytes(C.byref(d)) == 0
    null = C.c_void_p(0)
    for call in (lambda: L.tt_sparse_conv_train_forward(C.byref(d), null, null, null, null, null, null, null, null, C.c_size_t(0), null),
                 lambda: L.tt_sparse_conv_train_backward(C.byref(d), null, null, null, null, null, null, null, null, null, null, null,
                                                         C.c_size_t(0), null)):
        assert call() == -3                                          # TT_ERR_UNSUPPORTED
        assert named in L.tt_last_error().decode()


@pytest.mark.parametrize('k,s,p,subm', LAYERS)
def test_the_library_accepts_what_the_reference_builds(k, s, p, subm):
    d = sc.conv_desc(5, 16, k, s, p, subm=subm, n_in=10, n_out=10, pair_cap=10)
    assert lib.load().tt_sparse_conv_train_workspace_bytes(C.byref(d)) > 0


@pytest.mark.parametrize('make,named', [
    (lambda: sc.SubMConv3d(16, 16, 3, padding=1, bias=False, dilation=2), 'dilation'),
    (lambda: sc.SubMConv3d(16, 16, 3, padding=1, bias=False, groups=2), 'groups'),
    (lambda: sc.SubMConv3d(16, 16, 3, padding=1), 'bias'),                                  # spconv's default is bias=True
    (lambda: sc.SparseConvTranspose3d(16, 16, 3, stride=2, padding=1, bias=False), 'transposed'),
    (lambda: sc.SparseInverseConv3d(16, 16, 3, indice_key='spconv1', bias=False), 'inverse'),
    (lambda: sc.SparseConv3d(16, 16, 5, stride=2, padding=2, bias=False), 'kvol'),
    (lambda: sc.SparseConv3d(16, 16, 3, stride=1, padding=1, bias=False), 'stride')])
def test_the_modules_refuse_what_the_library_refuses(make, named):
    with pytest.raises(lib.TTError, match=named):
        make()


def test_cpu_tensors_are_refused():
    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    idx = torch.tensor([[0, 1, 2, 3], [0, 1, 2, 4]], dtype=torch.int32)
    x = sc.SparseConvTensor(torch.randn(2, 4), idx, [5, 6, 7], 1)
    with pytest.raises(lib.TTError):
        sc.SubMConv3d(4, 8, 3, padding=1, bias=False)(x)
    with pytest.raises(lib.TTError):
        sc.SparseConv3d(4, 8, 3, stride=2, padding=1, bias=False)(x)
    with pytest.raises(lib.TTError):
        sc.SparseEncoder(**CFG)(torch.randn(2, 5), idx, 1)


def test_encoder_state_dict_keys_equal_the_oracles_and_round_trip():
    from oracle.lidar import SparseEncoder as OracleEncoder
    torch.manual_seed(0)
    ours, ref = sc.SparseEncoder(**CFG), OracleEncoder(**CFG)
    assert [(k, tuple(v.shape)) for k, v in ours.state_dict().items()] == [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    ours.load_state_dict(ref.state_dict())
    for k, v in ours.state_dict().items():
        assert torch.equal(v, ref.state_dict()[k]), k
    back = OracleEncoder(**CFG)
    back.load_state_dict(ours.state_dict())
    for k, v in back.state_dict().items():
        assert torch.equal(v, ours.state_dict()[k]), k
    # the SubM convs of one resolution share a rulebook; the strided ones have their own keys
    keys = [(n, m.indice_key) for n, m in ours.named_modules() if isinstance(m, sc.SparseConvolution)]
    assert keys[0] == ('conv_input.0', 'subm1') and keys[-1] == ('conv_out.0', 'spconv_down2')
    assert ('encoder_layers.encoder_layer3.2.0', 'spconv3') in keys and ('encoder_layers.encoder_layer4.1.conv2', 'subm4') in keys


def test_sparse_sequential_dispatch_and_dense_on_the_cpu():
    """SparseSequential hands a SparseConvTensor to SparseModules and `.features` to the others; dense() is differentiable."""
    calls = []

    class Probe(sc.SparseModule):
        def forward(self, x):
            calls.append(type(x).__name__)
            return x
    idx = torch.tensor([[0, 0, 1, 2], [1, 3, 0, 0]], dtype=torch.int32)
    f = torch.randn(2, 3, requires_grad=True)
    x = sc.SparseConvTensor(f, idx, [4, 3, 3], 2)
    y = sc.SparseSequential(Probe(), torch.nn.ReLU(), Probe())(x)
    assert calls == ['SparseConvTensor', 'SparseConvTensor'] and torch.equal(y.features, F.relu(f))
    d = y.dense()
    assert d.shape == (2, 3, 4, 3, 3) and torch.equal(d[1, :, 3, 0, 0], F.relu(f[1]))
    d.sum().backward()
    assert torch.equal(f.grad, (f > 0).float())


# ----------------------------------------------------------------------------------------- the float64 reference, pinned
def _cloud(B, shape, n, seed, border=True):
    g = torch.Generator().manual_seed(seed)
    D, H, W = shape
    keys = torch.randperm(B * D * H * W, generator=g)[:n]
    c = torch.stack([keys // (D * H * W), (keys // (H * W)) % D, (keys // W) % H, keys % W], 1)
    if border:                                     # corners of the grid
        c = torch.cat([c, torch.tensor([[0, 0, 0, 0], [B - 1, D - 1, H - 1, W - 1], [0, D - 1, 0, W - 1]])])
        c = torch.unique(c, dim=0)
    return c.int()


def _dense_reference(x, coords, shape, B, w, k, s, p, subm, gy):
    """the sparse conv as autograd of a masked dense F.conv3d (spconv and torch both correlate: input = out * s - p + tap)."""
    D, H, W = shape
    c = coords.long()
    xx = x.detach().double().requires_grad_(True)
    ww = w.detach().double().requires_grad_(True)
    X = xx.new_zeros(B, D, H, W, x.shape[1]).index_put((c[:, 0], c[:, 1], c[:, 2], c[:, 3]), xx).permute(0, 4, 1, 2, 3)
    Y = F.conv3d(X, ww.permute(0, 4, 1, 2, 3), stride=s, padding=p)
    if subm:
        oc = c
    else:
        m = torch.zeros(B, 1, D, H, W, dtype=torch.float64)
        m[c[:, 0], 0, c[:, 1], c[:, 2], c[:, 3]] = 1
        reach = F.conv3d(m, torch.ones(1, 1, *k, dtype=torch.float64), stride=s, padding=p)[:, 0]
        oc = torch.nonzero(reach > 0)
    y = Y.permute(0, 2, 3, 4, 1)[oc[:, 0], oc[:, 1], oc[:, 2], oc[:, 3]]
    y.backward(gy.double())
    return y.detach(), oc, xx.grad, ww.grad


def _literal(x, coords, shape, w, k, s, p, subm, gy_of):
    """forward and both gradients as loops over every (output site, tap) pair; gy_of(out_coords) gives the output gradient."""
    sites = {tuple(int(v) for v in r): i for i, r in enumerate(coords)}
    taps = list(itertools.product(*(range(v) for v in k)))
    if subm:
        outs = [tuple(int(v) for v in r) for r in coords]
    else:
        oshape = [(shape[a] + 2 * p[a] - k[a]) // s[a] + 1 for a in range(3)]
        cand = set()
        for r in sites:
            for t in taps:
                num = [r[1 + a] + p[a] - t[a] for a in range(3)]
                if all(n >= 0 and n % s[a] == 0 and n // s[a] < oshape[a] for a, n in enumerate(num)):
                    cand.add((r[0],) + tuple(n // s[a] for a, n in enumerate(num)))
        outs = sorted(cand)
    oc = torch.tensor(outs, dtype=torch.long).view(-1, 4)
    gy = gy_of(oc)
    xd, wd = x.double(), w.double()
    y, gx, gw = torch.zeros(len(outs), w.shape[0], dtype=torch.float64), torch.zeros_like(xd), torch.zeros_like(wd)
    for o, r in enumerate(outs):
        for t in taps:
            src = (r[0],) + tuple(r[1 + a] * s[a] - p[a] + t[a] for a in range(3))
            i = sites.get(src)
            if i is None:
                continue
            W_t = wd[:, t[0], t[1], t[2], :]
            y[o] += W_t @ xd[i]
            gx[i] += W_t.t() @ gy[o]
            gw[:, t[0], t[1], t[2], :] += torch.outer(gy[o], xd[i])
    return y, oc, gx, gw


@pytest.mark.parametrize('k,s,p,subm', LAYERS)
def test_the_float64_reference_equals_a_masked_dense_conv_and_a_literal_loop(k, s, p, subm):
    B, shape, Cin, Cout = 2, (7, 6, 5), 3, 4
    coords = _cloud(B, shape, 40, seed=sum(k) + sum(p))
    g = torch.Generator().manual_seed(11)
    x = torch.randn(coords.shape[0], Cin, generator=g, dtype=torch.float64)
    w = torch.randn(Cout, *k, Cin, generator=g, dtype=torch.float64)
    y0, oc0, _, _ = reference(x, coords, shape, B, w, k, s, p, subm)
    gy_tab = torch.randn(B, *[max(shape)] * 3, Cout, generator=g, dtype=torch.float64)

    def gy_of(oc):
        oc = oc.long()
        return gy_tab[oc[:, 0], oc[:, 1], oc[:, 2], oc[:, 3]]
    ref = reference(x, coords, shape, B, w, k, s, p, subm, gy_of(oc0))
    dense = _dense_reference(x, coords, shape, B, w, k, s, p, subm, gy_of(oc0))
    lit = _literal(x, coords, shape, w, k, s, p, subm, gy_of)
    out_shape = shape if subm else [(shape[a] + 2 * p[a] - k[a]) // s[a] + 1 for a in range(3)]
    for other in (dense, lit):
        assert torch.equal(site_keys(ref[1], out_shape).sort()[0], site_keys(other[1], out_shape).sort()[0])
        o1, o2 = site_keys(ref[1], out_shape).argsort(), site_keys(other[1], out_shape).argsort()
        assert torch.allclose(ref[0][o1], other[0][o2], rtol=1e-12, atol=1e-12)
        assert torch.allclose(ref[2], other[2], rtol=1e-12, atol=1e-12)
        assert torch.allclose(ref[3], other[3], rtol=1e-12, atol=1e-12)
    if subm:
        assert torch.equal(ref[1], coords.long())                         # SubM: the input sites in input order
    else:
        keys = site_keys(ref[1], out_shape)
        assert bool((keys[1:] > keys[:-1]).all())                          # strided: ascending (b, z, y, x)
