"""The training losses on the GPU (thinktwice_b200/ops/losses.py; include/tt_b200.h §10b, §15) at thinktwice.py shapes: values
against float64 torch and the inference kernels, every gradient element within EPS x the largest term of its formula
(tests/loss_train_reference.py), crafted edge cases, bitwise repeatability, skipped gradients, empty batches, launch counts, autograd
through small layers, and the camera half's peak memory against the torch composition."""
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import camera_loss_checks as CK
import camera_loss_oracle as CO
import loss_train_reference as R
from thinktwice_b200 import lib
from thinktwice_b200.ops.losses import camera_losses, decoder_loss

pytestmark = pytest.mark.gpu
DEV = 'cuda'
N_CAM, D, EXTRA, F_DEPTH = 4, 80, 64, 16


def model_ns():
    return SimpleNamespace(use_seg=True, use_depth=True, downsample_factor=F_DEPTH, seg_downsample_factor=2, dbound=list(R.DBOUND),
                           depth_channels=D, seg_loss_func=SimpleNamespace(alpha=R.ALPHA, gamma=R.GAMMA, ignore_index=R.IGNORE, weight=None))


def camera_inputs(B, seed=0):
    """seg logits (BN, 12, 224, 448); depth logits as the [:, :80] view of an (80 + 64)-channel map whose other channels are NaN;
    448 x 896 labels (a quarter ignored, frame 0 all ignored when B > 1) and depths (zeros, a NaN pixel, frame 1 without foreground)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    BN = B * N_CAM
    seg = torch.randn(BN, 12, 224, 448, generator=g, device=DEV) * 3
    full = torch.full((BN, D + EXTRA, 28, 56), float('nan'), device=DEV)
    full[:, :D] = torch.randn(BN, D, 28, 56, generator=g, device=DEV) * 2
    lab = torch.randint(0, 12, (B, N_CAM, 448, 896), generator=g, device=DEV).float()
    lab[torch.rand(lab.shape, generator=g, device=DEV) < 0.25] = R.IGNORE
    dep = 0.5 + 0.5 * torch.randint(-2, 100, (B, N_CAM, 448, 896), generator=g, device=DEV).float()
    dep[torch.rand(dep.shape, generator=g, device=DEV) < 0.02] = 0.0
    dep[0, 0, 5, 7] = float('nan')
    if B > 1:
        lab[0, 1] = R.IGNORE                                           # an all-ignored image
        dep[1, 2] = 100.0                                              # an image without a foreground cell
    return seg, full[:, :D], lab, dep


@pytest.mark.parametrize('B', [1, 8])
def test_camera_losses_values_and_gradients(B):
    seg, depth, lab, dep = camera_inputs(B)
    seg.requires_grad_(); depth.requires_grad_()
    n0 = lib.launch_count()
    out = camera_losses(model_ns(), dict(seg=lab, depth=dep), dict(seg=seg, depth=depth))
    assert list(out) == ['seg_loss', 'depth_loss'] and lib.launch_count() - n0 == 1
    up = (0.7, -1.3)
    (out['seg_loss'] * up[0] + out['depth_loss'] * up[1]).backward()
    assert lib.launch_count() - n0 == 2
    (rs, rd), gs, gd = R.camera_ref(seg, depth, lab, dep, f=F_DEPTH, up=up)
    vs, vd = float(out['seg_loss']), float(out['depth_loss'])
    assert abs(vs - rs) <= 2e-6 * abs(rs) and abs(vd - rd) <= 2e-6 * abs(rd), (vs, rs, vd, rd)
    case = dict(seg=seg.detach().permute(0, 2, 3, 1), depth=depth.detach().permute(0, 2, 3, 1), seg_gt=lab, depth_gt=dep,
                d_bound=R.DBOUND, f=F_DEPTH, seg_coff=0, seg_classes=12, depth_coff=0, D=D)
    inf = CK.run(case, DEV)
    ulp = lambda v: abs(float(torch.tensor(v).float().nextafter(torch.tensor(float('inf'))) - torch.tensor(v).float()))
    assert abs(vs - inf[0]) <= ulp(inf[0]) and abs(vd - inf[1]) <= ulp(inf[1]), (vs, inf[0], vd, inf[1])
    ss, sd = R.camera_scale(seg, depth, lab, dep, f=F_DEPTH, up=up)
    r_seg, r_dep = R.ratio(seg.grad, gs, R.EPS * ss), R.ratio(depth.grad, gd, R.EPS * sd)
    print(f'[camera B={B}] worst err / bound: grad_seg {r_seg:.3f}, grad_depth {r_dep:.3f}; seg_loss rel err {abs(vs - rs) / abs(rs):.2e}')
    assert r_seg <= 1 and r_dep <= 1
    if B > 1:
        assert (seg.grad[1] == 0).all() and (depth.grad[6] == 0).all()   # the all-ignored image, the image without foreground


def test_camera_backward_is_bitwise_repeatable_and_skips_null_gradients():
    seg, depth, lab, dep = camera_inputs(1, seed=3)
    seg.requires_grad_(); depth.requires_grad_()
    out = camera_losses(model_ns(), dict(seg=lab, depth=dep), dict(seg=seg, depth=depth))
    total = out['seg_loss'] + out['depth_loss']
    a = torch.autograd.grad(total, (seg, depth), retain_graph=True)
    b = torch.autograd.grad(total, (seg, depth))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    s2 = seg.detach().clone()                                          # no gradient for the seg logits: only grad_depth is written
    out = camera_losses(model_ns(), dict(seg=lab, depth=dep), dict(seg=s2, depth=depth))
    (g,) = torch.autograd.grad(out['seg_loss'] + out['depth_loss'], (depth,))
    assert torch.equal(g, a[1])
    with torch.no_grad():
        n0 = lib.launch_count()
        out = camera_losses(model_ns(), dict(seg=lab, depth=dep), dict(seg=seg, depth=depth))
        assert lib.launch_count() - n0 == 1 and out['seg_loss'].grad_fn is None


def test_camera_empty_batch_launches_nothing_and_bad_labels_raise():
    m = model_ns()
    seg = torch.zeros(0, 12, 224, 448, device=DEV, requires_grad=True)
    depth = torch.zeros(0, D, 28, 56, device=DEV, requires_grad=True)
    n0 = lib.launch_count()
    out = camera_losses(m, dict(seg=torch.zeros(0, 4, 448, 896), depth=torch.zeros(0, 4, 448, 896)), dict(seg=seg, depth=depth))
    (out['seg_loss'].nan_to_num() + out['depth_loss']).backward()
    assert lib.launch_count() == n0 and float(out['depth_loss']) == 0.0
    seg, depth, lab, dep = camera_inputs(1)
    for v in (12.0, -1.0, float('nan')):
        bad = lab.clone()
        bad[0, 0, 10, 10] = v
        with pytest.raises(ValueError, match='seg'):
            camera_losses(m, dict(seg=bad, depth=dep), dict(seg=seg, depth=depth))
    with pytest.raises(ValueError, match='depth'):
        camera_losses(m, dict(seg=lab, depth=dep[..., :-16]), dict(seg=seg, depth=depth))
    with pytest.raises(lib.TTError, match='float32'):
        camera_losses(m, dict(seg=lab, depth=dep), dict(seg=seg.double(), depth=depth))


def test_camera_peak_memory_against_torch():
    """forward + backward at B = 8: the peak allocation above the inputs, ours against the fp32 torch composition"""
    seg, depth, lab, dep = camera_inputs(8)
    seg.requires_grad_(); depth.requires_grad_()

    def peak(fn):
        seg.grad = depth.grad = None
        torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        d = fn()
        (d['seg_loss'] + d['depth_loss']).backward()
        torch.cuda.synchronize()
        return (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    ours = peak(lambda: camera_losses(model_ns(), dict(seg=lab, depth=dep), dict(seg=seg, depth=depth)))
    theirs = peak(lambda: CO.camera_loss(dict(use_seg=True, use_depth=True), dict(seg=lab, depth=dep), seg, depth, R.DBOUND))
    print(f'[camera B=8] peak increment of forward + backward: ours {ours:.1f} MiB, torch {theirs:.1f} MiB')
    assert ours < theirs


# ------------------------------------------------------------------------------------------------------------------ decoder
def gpu_inputs(B, seed=0, views=False):
    pred, mid, batch = R.make_inputs(B, seed=seed, quarter=True)
    pred['mu_branches'][0, 0] = torch.tensor([1e-3, 900.0], dtype=torch.float64)   # Beta parameters near 0 and large
    pred['sigma_branches'][0, 0] = torch.tensor([700.0, 2e-3], dtype=torch.float64)
    batch['action_mu'][0] = torch.tensor([1.5e-3, 1200.0], dtype=torch.float64)
    rb, g2 = pred['refine_BEV_feature'], batch['grid_feature'][2]
    rb[0, 0, 0, 0, :6] = g2[0, 0, 0, :6] + torch.tensor([0, 1, -1, 5.5, -5.5, 5.75], dtype=torch.float64)   # smooth-L1 / clamp edges
    P = {k: v.float().to(DEV) for k, v in pred.items()}
    if views:                                                          # non-contiguous predictions, read in place
        P['pred_features_traj'] = torch.randn(256, B, device=DEV).t()
        P['pred_features_traj'].copy_(pred['pred_features_traj'].float())
        wide = torch.full((B, 5, 2 * 256), float('nan'), device=DEV)
        wide[..., ::2] = pred['refine_flattned_BEV_feature'].float().to(DEV)
        P['refine_flattned_BEV_feature'] = wide[..., ::2]
    for v in P.values():
        v.requires_grad_()
    M = [None, None] + [m.float().to(DEV).requires_grad_() for m in mid[2:]]
    return P, M, batch


@pytest.mark.parametrize('B,views', [(1, False), (8, True)])
def test_decoder_loss_values_and_gradients(B, views):
    P, M, batch = gpu_inputs(B, seed=B, views=views)
    n0 = lib.launch_count()
    out = decoder_loss(R.decoder_module(), batch, P, M)
    assert lib.launch_count() - n0 == 1
    vals, G, w = R.decoder_ref({k: v.detach() for k, v in P.items()}, [m if m is None else m.detach() for m in M], batch)
    assert list(out) == list(vals) and out['value_loss'].shape == (B, 1)
    for k in out:
        assert out[k].shape == vals[k].shape
        assert torch.allclose(out[k].double().cpu(), vals[k].detach(), rtol=2e-6, atol=1e-9), k
        assert out[k].requires_grad == (k not in R.OFFSETS), k
    total = sum((out[k] * w[k].float().to(DEV)).sum() for k in out if k not in R.OFFSETS)
    leaves = [P[k] for k in R.PRED_KEYS] + M[2:]
    got = torch.autograd.grad(total, leaves, retain_graph=True)
    assert lib.launch_count() - n0 == 2
    again = torch.autograd.grad(total, leaves)
    assert all(torch.equal(a, b) for a, b in zip(got, again))
    S = R.decoder_scale({k: v.detach() for k, v in P.items()}, [m if m is None else m.detach() for m in M], batch, w)
    names = list(R.PRED_KEYS) + [f'mid{i}' for i in (2, 3, 4, 5)]
    worst = {k: R.ratio(g, G[k], R.EPS * S[k]) for k, g in zip(names, got)}
    k = max(worst, key=worst.get)
    print(f'[decoder B={B}] worst err / bound {worst[k]:.3f} ({k})')
    assert worst[k] <= 1


def test_decoder_loss_refuses_bad_beta_and_shapes():
    P, M, batch = gpu_inputs(2)
    bad = dict(batch, action_sigma=batch['action_sigma'].clone())
    bad['action_sigma'][0, 0] = 0.0
    with pytest.raises(ValueError, match='Beta'):
        decoder_loss(R.decoder_module(), bad, P, M)
    bad = dict(batch, future_action_mu=[t.clone() for t in batch['future_action_mu']])
    bad['future_action_mu'][0][1, 1] = float('inf')
    with pytest.raises(ValueError, match='Beta'):
        decoder_loss(R.decoder_module(), bad, P, M)
    with pytest.raises(ValueError, match='broadcast'):
        decoder_loss(R.decoder_module(), dict(batch, feature=batch['feature'][:, :128]), P, M)
    with pytest.raises(lib.TTError, match='float32'):
        decoder_loss(R.decoder_module(), batch, dict(P, pred_speed=P['pred_speed'].double()), M)


def test_end_to_end_through_autograd_within_twice_torchs_error():
    """small layers produce the logits and predictions; a _parse_losses-style total is backpropagated.  Each parameter gradient's error
    against the float64 composition must stay within 2x the fp32 torch composition's own error (plus a floor at fp32 resolution)."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device=DEV).manual_seed(7)
    _, _, lab, dep = camera_inputs(1, seed=7)
    xs = torch.randn(4, 8, 224, 448, generator=g, device=DEV)
    xd = torch.randn(4, 8, 28, 56, generator=g, device=DEV)
    P0, M0, batch = gpu_inputs(2, seed=9)
    feat = torch.randn(2, 64, generator=g, device=DEV)
    conv_s = torch.nn.Conv2d(8, 12, 1).to(DEV)
    conv_d = torch.nn.Conv2d(8, D + EXTRA, 1).to(DEV)
    lin = torch.nn.Linear(64, 256).to(DEV)
    params = list(conv_s.parameters()) + list(conv_d.parameters()) + list(lin.parameters())

    def run(ours, dtype):
        cast = lambda t: t.to(dtype)
        seg = F.conv2d(cast(xs), cast(conv_s.weight), cast(conv_s.bias)) * 3
        depth = F.conv2d(cast(xd), cast(conv_d.weight), cast(conv_d.bias))[:, :D] * 3
        P = {k: cast(v.detach()) for k, v in P0.items()}
        P['pred_features_traj'] = F.linear(cast(feat), cast(lin.weight), cast(lin.bias))
        M = [None, None] + [cast(m.detach()) for m in M0[2:]]
        if ours:
            d = decoder_loss(R.decoder_module(), batch, P, M)
            d.update(camera_losses(model_ns(), dict(seg=lab, depth=dep), dict(seg=seg, depth=depth)))
        else:
            d = R.LO.decoder_loss(R.CONFIG, R.batch_as(batch, dtype, DEV), P, M)
            d.update(CO.camera_loss(dict(use_seg=True, use_depth=True), dict(seg=lab, depth=dep), seg, depth, R.DBOUND))
        total = sum(v.mean() for k, v in d.items() if 'loss' in k)
        return torch.autograd.grad(total, params)
    ref = run(False, torch.float64)
    fp32 = run(False, torch.float32)
    ours = run(True, torch.float32)
    for name, r, t, o in zip(('conv_s.w', 'conv_s.b', 'conv_d.w', 'conv_d.b', 'lin.w', 'lin.b'), ref, fp32, ours):
        r = r.cpu()
        e_t, e_o = float((t.double().cpu() - r).abs().max()), float((o.double().cpu() - r).abs().max())
        floor = 1e-6 * float(r.abs().max())
        print(f'[e2e] {name}: ours {e_o:.3e}, torch fp32 {e_t:.3e}')
        assert e_o <= 2 * e_t + floor, name
