"""Training-side batch norm on the GPU (include/tt_b200.h §18, thinktwice_b200/ops/batch_norm.py) against float64.

Every output element is held to |got - ref| <= 1e-5 * S, S the float64 sum of |terms| of that element (the §16 convention): y, the
running statistics, grad_x, grad_r, grad_weight and grad_bias of every distinct batch norm of one thinktwice.py forward of the oracle
(collected with hooks; the camera trunk at 32 images, the sparse encoder at its full site counts, the BEV fusion and SE blocks, SECOND
and output_fc at 8 samples), each plain, with ReLU and with residual + ReLU.  The ReLU mask of the float64 reference is the one the op
defines: the sign of its fp32 z, read from y.  Also: an R-way split emulated on one GPU, a two-process SyncBatchNorm over gloo against
torch.nn.SyncBatchNorm, bitwise repeatability, eval mode, momentum None, empty inputs, NULL gradients, the ValueError, and the oracle's
ResNet-50 under autograd after convert_conv2d + convert_upsampling + convert_batchnorm."""
import copy
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

import batch_norm_train_reference as RB
from thinktwice_b200 import lib
from thinktwice_b200.ops import batch_norm as bn
from thinktwice_b200.ops import conv2d as cv
from thinktwice_b200.ops import conv_transpose2d as ct

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
WORST = {}


@pytest.fixture(scope='module', autouse=True)
def report():
    yield
    if WORST:
        print('\n[batch_norm_train] worst |err| / (1e-5 S): ' + ', '.join(f'{k} {v:.3g}' for k, v in sorted(WORST.items())))


def _ratio(name, got, ref, S):
    err = (got.double() - ref).abs()
    bound = 1e-5 * S
    r = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), r)
    assert r <= 1.0, (name, r)
    assert bool((err[S == 0] == 0).all()), name


def _layer_shapes():
    """{(kind, C, eps, momentum, rows per sample or None, H, W): where} of every batch norm of one thinktwice.py oracle forward."""
    from oracle.model import EncoderDecoder as Oracle, init_oracle_weights
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(o, 0)
    o.eval()
    seen = {}
    for name, m in o.named_modules():
        if isinstance(m, nn.modules.batchnorm._BatchNorm) and m.num_features % 4 == 0:
            def hook(mod, inp, name=name):
                x = inp[0]
                where = 'trunk' if name.startswith('img_encoder') else 'sparse' if 'middle_encoder' in name else 'bev'
                key = (x.dim(), mod.num_features, mod.eps, mod.momentum, *((x.shape[0],) if where == 'sparse' else (None,)),
                       *(tuple(x.shape[2:]) if x.dim() == 4 else (None, None)))
                seen.setdefault(key, where)
            m.register_forward_pre_hook(hook)
    with torch.no_grad():
        o.forward_inference(make_batch(cfg, 1, seed=0, num_points=40000))
    return seen


def _make(dim, Cc, eps, momentum, g):
    m = (bn.BatchNorm2d if dim == 4 else bn.BatchNorm1d)(Cc, eps=eps, momentum=momentum).cuda()
    with torch.no_grad():
        m.weight.copy_(1 + 0.3 * torch.randn(Cc, generator=g, device='cuda'))
        m.bias.copy_(0.3 * torch.randn(Cc, generator=g, device='cuda'))
        m.running_mean.copy_(torch.randn(Cc, generator=g, device='cuda'))
        m.running_var.copy_(torch.rand(Cc, generator=g, device='cuda') + 0.5)
    return m


def _input(shape, g):
    Cc = shape[1]
    view = (1, Cc) + (1,) * (len(shape) - 2)
    x = torch.randn(shape, generator=g, device='cuda') * (0.5 + torch.rand(Cc, generator=g, device='cuda')).view(view) \
        + 2 * torch.randn(Cc, generator=g, device='cuda').view(view)
    return x.contiguous(memory_format=torch.channels_last) if len(shape) == 4 else x


def _rows(t):
    return bn._rows(t)[0]


def check(shape, eps, momentum, relu, res, tag, seed=0, train=True):
    g = torch.Generator(device='cuda').manual_seed(seed)
    m = _make(len(shape), shape[1], eps, momentum, g).train(train)
    rm0, rv0 = m.running_mean.double(), m.running_var.double()
    x = _input(shape, g).requires_grad_(True)
    r = _input(shape, g).requires_grad_(True) if res else None
    y = m(x, residual=r, relu=relu)
    gy = _input(shape, g)
    y.backward(gy)
    xd, gyd, yf = _rows(x.detach()).double(), _rows(gy).double(), _rows(y.detach())
    rd = _rows(r.detach()).double() if res else None
    w, b = m.weight.detach().double(), m.bias.detach().double()
    if train:
        mean, invstd, _, _ = RB.stats(xd, eps)
    else:
        mean, invstd = rm0, 1.0 / torch.sqrt(m.running_var.float() + eps).double()
    xh = (xd - mean) * invstd
    mag = (xd.abs() + mean.abs()) * invstd
    z = w * xh + b + (rd if res else 0)
    _ratio(f'{tag} y', yf, torch.relu(z) if relu else z, w.abs() * mag + b.abs() + (rd.abs() if res else 0))
    mask = ~(yf <= 0) if relu else torch.ones_like(yf, dtype=torch.bool)
    dz = gyd * mask
    n = xd.shape[0]
    if train:
        f = momentum if momentum is not None else 1.0 / float(m.num_batches_tracked)
        want_m, want_v = RB.running(rm0, rv0, xd, eps, f)
        _ratio(f'{tag} running_mean', m.running_mean, want_m, (1 - f) * rm0.abs() + f * xd.abs().mean(0))
        _ratio(f'{tag} running_var', m.running_var, want_v, (1 - f) * rv0.abs() + f * ((xd - mean) ** 2).sum(0) / (n - 1))
        gx, gr, gw, gb = RB.backward(xd, rd, w, b, gyd, eps, relu, mask=mask)
        sdz, sdzx = dz.sum(0), (dz * xh).sum(0)
        S_gx = w.abs() * invstd * (dz.abs() + sdz.abs() / n + mag * (sdzx.abs() / n))
    else:
        gx, gw, gb = w * invstd * dz, [(dz * xh).sum(0)], [dz.sum(0)]
        S_gx = (w * invstd * dz).abs()
        assert torch.equal(m.running_mean.double(), rm0) and torch.equal(m.running_var.double(), rv0)
    _ratio(f'{tag} grad_x', _rows(x.grad), gx, S_gx)
    if res:
        assert torch.equal(_rows(r.grad).double(), dz), tag                # grad_r is dz, exactly
    _ratio(f'{tag} grad_weight', m.weight.grad, gw[0], (dz.abs() * mag).sum(0))
    _ratio(f'{tag} grad_bias', m.bias.grad, gb[0], dz.abs().sum(0))


VARIANTS = [(False, False, 'plain'), (True, False, 'relu'), (True, True, 'res+relu')]


def test_every_batch_norm_of_the_model_against_float64():
    shapes = _layer_shapes()
    where = set(shapes.values())
    assert where == {'trunk', 'sparse', 'bev'}
    assert (4, 256, 1e-5, 0.1, None, 112, 224) in shapes and (2, 512, 1e-5, 0.1, None, None, None) in shapes   # layer1 bn3, output_fc
    for (dim, Cc, eps, mom, rows, H, W), w in sorted(shapes.items(), key=str):
        shape = (32, Cc, H, W) if w == 'trunk' else (8, Cc, H, W) if dim == 4 else (rows, Cc) if w == 'sparse' else (8, Cc)
        for relu, res, name in VARIANTS:
            check(shape, eps, mom, relu, res, f'{w} {name}')
            torch.cuda.empty_cache()


@pytest.mark.parametrize('shape', [(3, 4, 5, 7), (2, 2052, 3, 3), (5, 12), (1000, 1028), (70001, 16), (7, 8, 1, 1)])
def test_corner_shapes_against_float64(shape):
    for relu, res, name in VARIANTS:
        check(shape, 1e-3, 0.01, relu, res, f'corner {name}')


def test_eval_mode_with_gradients_and_momentum_none():
    for relu, res, name in VARIANTS:
        check((4, 64, 9, 11), 1e-5, 0.1, relu, res, f'eval {name}', train=False)
    g = torch.Generator(device='cuda').manual_seed(5)
    m = _make(4, 32, 1e-5, None, g)
    for step in range(3):
        x = _input((2, 32, 6, 5), g)
        rm0, rv0 = m.running_mean.double(), m.running_var.double()
        m(x)
        want_m, want_v = RB.running(rm0, rv0, _rows(x).double(), 1e-5, 1.0 / (step + 1))
        assert int(m.num_batches_tracked) == step + 1
        assert torch.allclose(m.running_mean.double(), want_m, rtol=1e-6, atol=1e-6)
        assert torch.allclose(m.running_var.double(), want_v, rtol=1e-6, atol=1e-6)


def test_empty_input_and_the_value_error():
    m = bn.BatchNorm2d(16).cuda().eval()
    x = torch.empty(0, 16, 5, 5, device='cuda', requires_grad=True)
    n0 = lib.launch_count()
    y = m(x, relu=True)
    y.backward(torch.empty_like(y))
    torch.cuda.synchronize()
    assert y.shape == x.shape and lib.launch_count() == n0
    assert torch.equal(m.weight.grad, torch.zeros_like(m.weight)) and torch.equal(m.bias.grad, torch.zeros_like(m.bias))
    m.train()
    with pytest.raises(ValueError, match='Expected more than 1 value per channel when training, got input size 1'):
        bn.BatchNorm1d(8).cuda()(torch.randn(1, 8, device='cuda'))
    with pytest.raises(ValueError, match='got input size 1'):
        m(torch.randn(1, 16, 1, 1, device='cuda'))
    with pytest.raises(ValueError, match='got input size 0'):
        m(torch.randn(0, 16, 3, 3, device='cuda'))


def _run(m, x, r, gy, relu, want):
    """forward + backward with only the gradients in `want` requested; returns the gradients (None where not requested)."""
    xi = x.clone().requires_grad_('x' in want)
    ri = r.clone().requires_grad_('r' in want)
    m.weight.requires_grad_('w' in want)
    m.bias.requires_grad_('b' in want)
    m.weight.grad = m.bias.grad = None
    y = m(xi, residual=ri, relu=relu)
    if y.requires_grad:
        y.backward(gy)
    return y.detach(), xi.grad, ri.grad, m.weight.grad, m.bias.grad


def test_repeatable_bitwise_and_null_gradients_skipped():
    g = torch.Generator(device='cuda').manual_seed(3)
    shape = (32, 256, 56, 112)
    m = _make(4, 256, 1e-5, 0.1, g)
    x, r, gy = _input(shape, g), _input(shape, g), _input(shape, g)
    state = copy.deepcopy(m.state_dict())
    full = _run(m, x, r, gy, True, 'xrwb')
    m.load_state_dict(state)
    again = _run(m, x, r, gy, True, 'xrwb')
    for a, c in zip(full, again):
        assert torch.equal(a, c)
    for want in ('x', 'r', 'w', 'b', 'xb', ''):
        m.load_state_dict(state)
        got = _run(m, x, r, gy, True, want)
        assert torch.equal(got[0], full[0])
        for k, name in enumerate('xrwb'):
            assert (got[k + 1] is None) == (name not in want), (want, name)
            if got[k + 1] is not None:
                assert torch.equal(got[k + 1], full[k + 1]), (want, name)


def _emulated(x, r, w, b, gy, splits, relu, eps=1e-5, f=0.1):
    """The library's five calls with the rows split over len(splits) emulated ranks on one GPU (the gathers: a stack)."""
    Cc, R, n = x.shape[1], len(splits), x.shape[0]
    parts = list(x.split(splits)), list(r.split(splits)), list(gy.split(splits))
    rm, rv = torch.zeros(Cc, device='cuda'), torch.ones(Cc, device='cuda')
    recs = torch.empty(R, 3 * Cc, dtype=torch.float64, device='cuda')
    for k, xk in enumerate(parts[0]):
        d = bn._desc(xk.shape[0], Cc, R, True, True, relu, eps, f, n)
        ws, nb = bn._workspace(d, 'cuda')
        lib.call('tt_batch_norm_train_stats', C.byref(d), lib._p(xk), lib._p(recs[k]), lib._p(ws), C.c_size_t(nb))
    mean, invstd = torch.empty(Cc, device='cuda'), torch.empty(Cc, device='cuda')
    lib.call('tt_batch_norm_train_fold', C.byref(d), lib._p(recs), lib._p(rm), lib._p(rv), lib._p(mean), lib._p(invstd))
    ys, gws, gbs, brecs = [], [], [], torch.empty(R, 2 * Cc, dtype=torch.float64, device='cuda')
    for k, (xk, rk, gk) in enumerate(zip(*parts)):
        d = bn._desc(xk.shape[0], Cc, R, True, True, relu, eps, f, n)
        ys.append(torch.empty_like(xk))
        lib.call('tt_batch_norm_train_forward', C.byref(d), lib._p(xk), lib._p(rk), lib._p(w), lib._p(b), lib._p(mean), lib._p(invstd),
                 lib._p(ys[-1]))
        gws.append(torch.empty_like(w))
        gbs.append(torch.empty_like(b))
        ws, nb = bn._workspace(d, 'cuda')
        lib.call('tt_batch_norm_train_backward_reduce', C.byref(d), lib._p(xk), lib._p(rk), lib._p(w), lib._p(b), lib._p(mean),
                 lib._p(invstd), lib._p(gk), lib._p(brecs[k]), lib._p(gws[-1]), lib._p(gbs[-1]), lib._p(ws), C.c_size_t(nb))
    gxs, grs = [], []
    for k, (xk, rk, gk) in enumerate(zip(*parts)):
        d = bn._desc(xk.shape[0], Cc, R, True, True, relu, eps, f, n)
        gxs.append(torch.empty_like(xk))
        grs.append(torch.empty_like(xk))
        lib.call('tt_batch_norm_train_backward', C.byref(d), lib._p(xk), lib._p(rk), lib._p(w), lib._p(b), lib._p(mean), lib._p(invstd),
                 lib._p(gk), lib._p(brecs), lib._p(gxs[-1]), lib._p(grs[-1]))
    return torch.cat(ys), rm, rv, torch.cat(gxs), torch.cat(grs), gws, gbs


@pytest.mark.parametrize('splits', [(5000,), (1700, 3300), (2100, 0, 2900)])
def test_an_emulated_r_way_split_against_float64_of_the_whole_batch(splits):
    g = torch.Generator(device='cuda').manual_seed(7)
    Cc, n = 48, sum(splits)
    x, r, gy = _input((n, Cc), g), _input((n, Cc), g), _input((n, Cc), g)
    w, b = 1 + 0.3 * torch.randn(Cc, generator=g, device='cuda'), 0.3 * torch.randn(Cc, generator=g, device='cuda')
    y, rm, rv, gx, gr, gws, gbs = _emulated(x, r, w, b, gy, splits, True)
    xd, rd, gyd, wd, bd = x.double(), r.double(), gy.double(), w.double(), b.double()
    mean, invstd, _, _ = RB.stats(xd, 1e-5)
    xh, mag = (xd - mean) * invstd, (xd.abs() + mean.abs()) * invstd
    z = wd * xh + bd + rd
    _ratio('split y', y, torch.relu(z), wd.abs() * mag + bd.abs() + rd.abs())
    want_m, want_v = RB.running(torch.zeros_like(mean), torch.ones_like(mean), xd, 1e-5, 0.1)
    assert torch.allclose(rm.double(), want_m, rtol=1e-6, atol=1e-7) and torch.allclose(rv.double(), want_v, rtol=1e-6, atol=1e-7)
    mask = y > 0
    dz = gyd * mask
    rgx, rgr, rgw, rgb = RB.backward(xd, rd, wd, bd, gyd, 1e-5, True, splits=splits, mask=mask)
    S = wd.abs() * invstd * (dz.abs() + dz.sum(0).abs() / n + mag * ((dz * xh).sum(0).abs() / n))
    _ratio('split grad_x', gx, rgx, S)
    assert torch.equal(gr.double(), rgr)
    lo = 0
    for k, m in enumerate(splits):
        dzk, magk = dz[lo:lo + m], mag[lo:lo + m]
        _ratio('split grad_weight (per rank)', gws[k], rgw[k], (dzk.abs() * magk).sum(0))
        _ratio('split grad_bias (per rank)', gbs[k], rgb[k], dzk.abs().sum(0))
        lo += m
    if len(splits) == 1:                                              # one rank: the same as the module
        m = bn.BatchNorm1d(Cc).cuda()
        with torch.no_grad():
            m.weight.copy_(w)
            m.bias.copy_(b)
        assert torch.equal(m(x, residual=r, relu=True), y)


def test_two_process_sync_batch_norm_over_gloo_matches_torch(tmp_path):
    world = 2
    env = dict(os.environ)
    procs = []
    try:
        for rank in range(world):
            procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, 'batch_norm_sync_worker.py'), str(rank), str(world),
                                           str(tmp_path / 'store'), str(tmp_path / f'out{rank}.json')], env=env))
        codes = [p.wait(timeout=600) for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    assert codes == [0] * world
    worst = 0.0
    for rank in range(world):
        res = json.loads((tmp_path / f'out{rank}.json').read_text())
        assert len(res) >= 12, res
        for k, v in res.items():
            assert v <= 1e-4, (rank, k, v)
            worst = max(worst, v)
    print(f'\n[batch_norm_train] two-process SyncBatchNorm vs torch.nn.SyncBatchNorm: worst max-relative difference {worst:.2e}')


def test_resnet50_under_autograd_after_all_three_converters():
    """The oracle's ResNet-50 in train mode at 4 images of 224 x 448, every parameter and input gradient against the float64 module.
    A ReLU whose input is within rounding of zero passes or stops a gradient depending on the last bit, and the trunk's depth makes
    the largest elementwise error chaotic (a 1e-7 relative perturbation of the input moves torch fp32's own worst max-norm error by 3x),
    so the measure is each gradient's relative L2 error, averaged over all of them.  It is held to max(1e-4, 2 x torch fp32's) (TF32
    off): as close as fp32.  The worst single gradient is printed beside it."""
    from oracle.camera import ResNet50
    torch.manual_seed(0)
    ref = ResNet50().cuda().train()
    f32 = copy.deepcopy(ref)
    ours, _ = cv.convert_conv2d(copy.deepcopy(ref))
    ours, _ = ct.convert_upsampling(ours)
    ours, skipped, _ = bn.convert_batchnorm(ours)
    assert skipped == [] and not any(type(m) is nn.BatchNorm2d for m in ours.modules())
    ref = ref.double()
    x = torch.randn(4, 3, 224, 448, device='cuda')
    wts = [torch.randn(o.shape, device='cuda', dtype=torch.float64) for o in ref(x.double())]

    def run(model, dtype):
        xi = x.to(dtype, copy=True).requires_grad_(True)
        sum((o * wt.to(dtype)).sum() for o, wt in zip(model(xi), wts)).backward()
        g = {n: p.grad.double() for n, p in model.named_parameters()}
        g['input'] = xi.grad.double()
        return g
    want = run(ref, torch.float64)
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        g_f32, got = run(f32, torch.float32), run(ours, torch.float32)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
    rel = {n: [float((h[n] - want[n]).norm() / want[n].norm()) for h in (got, g_f32)] for n in want}
    mean = [sum(r[k] for r in rel.values()) / len(rel) for k in (0, 1)]
    n = max(rel, key=lambda k: rel[k][0])
    print(f'\n[batch_norm_train] ResNet-50 relative L2 gradient error, mean over {len(rel)} gradients (ours, torch fp32): '
          f'{mean[0]:.2e}, {mean[1]:.2e}; worst: {n} {tuple(f"{v:.2e}" for v in rel[n])}')
    WORST['resnet50 autograd err / bound'] = mean[0] / max(1e-4, 2 * mean[1])
    assert mean[0] <= max(1e-4, 2 * mean[1]), mean
