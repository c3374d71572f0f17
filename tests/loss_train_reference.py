"""Float64 gradient references for the training losses (thinktwice_b200/ops/losses.py, include/tt_b200.h §10b and §15) — TEST
INFRASTRUCTURE ONLY.

  * camera_ref / decoder_ref   float64 autograd of tests/camera_loss_oracle.camera_loss and tests/loss_oracle.decoder_loss
  * camera_formula / decoder_formula   the same gradients as literal per-element expressions (the header's formulas), which
                                the CPU tests pin against the autograd references and mutate into seeded bugs
  * camera_scale / decoder_scale   the largest term of each gradient element's formula; GPU results are held to EPS * scale
  * ratio                       worst |got - ref| / bound (NaN must meet NaN)
"""
from collections import OrderedDict
from types import SimpleNamespace

import torch
import torch.nn.functional as F

import camera_loss_oracle as CO
import loss_oracle as LO

EPS = 4e-6                    # fp32 softmax / sigmoid / rounding of a product of O(1) terms, with room for the C-term sums
DBOUND = (1.0, 41.0, 0.5)     # thinktwice.py d_bound
ALPHA, GAMMA, IGNORE, SEG_W = 0.5, 2.0, 255, 10.0


def ratio(got, ref, bound):
    got, ref = got.double().cpu(), ref.double().cpu()
    both_nan = torch.isnan(got) & torch.isnan(ref)
    err = torch.where(both_nan, torch.zeros_like(ref), (got - ref).abs())
    err = torch.where(torch.isnan(err), torch.full_like(err, float('inf')), err)
    r = err / bound.double().cpu().clamp_min(1e-30)
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------------------------------- camera
def seg_labels(seg_gt, s):
    return CO.downsampled_gt_seg(seg_gt, s)


def depth_bins(depth_gt, f, D, dbound=DBOUND, nan_is_background=True):
    """(B*N*h*w,) bins 0..D (0 = background), in fp32 as the reference computes them: the min over each f x f block (0 -> 1e5
    first; a NaN pixel makes the block NaN, hence background), then the bin value."""
    B, N, H, W = depth_gt.shape
    g = depth_gt.float().reshape(B * N, H // f, f, W // f, f).permute(0, 1, 3, 2, 4).reshape(B * N, H // f, W // f, f * f)
    g = torch.where(g == 0, torch.full_like(g, 1e5), g)
    if not nan_is_background:
        g = torch.where(torch.isnan(g), torch.full_like(g, float('inf')), g)
    m = g.amin(-1)
    v = (m - (dbound[0] - dbound[2])) / dbound[2]
    v = torch.where((v < D + 1) & (v >= 0), v, torch.zeros_like(v))
    return v.long().reshape(-1)


def camera_ref(seg, depth, seg_gt, depth_gt, f=16, s=2, up=(1.0, 1.0)):
    """float64 autograd of camera_loss_oracle.camera_loss: ((seg_loss, depth_loss), grad_seg, grad_depth) for the upstream `up`."""
    sg = seg.detach().double().requires_grad_()
    dp = depth.detach().double().requires_grad_()
    batch = dict(seg=seg_gt.float(), depth=depth_gt.float())      # the reference's ground truth is fp32
    d = CO.camera_loss(dict(use_seg=True, use_depth=True), batch, sg, dp, DBOUND, f=f, s=s)
    (d['seg_loss'] * up[0] + d['depth_loss'] * up[1]).backward()
    return (float(d['seg_loss'].detach()), float(d['depth_loss'].detach())), sg.grad, dp.grad


def _focal_prime(ce, second=True):
    e = torch.exp(-ce)
    u = 1 - e
    return ALPHA * (u ** GAMMA + (GAMMA * ce * e * u ** (GAMMA - 1) if second else 0))


def camera_formula(seg, depth, seg_gt, depth_gt, f=16, s=2, up=(1.0, 1.0), bug=None):
    """the header's per-element gradients: grad_seg = g0 w f'(ce) (softmax - onehot) / n on counted pixels, grad_depth = g1 (sigmoid -
    onehot) / max(1, n_fg) on foreground cells.  `bug` names a seeded mistake."""
    x = seg.detach().double()
    BN, Cn, h, w = x.shape
    lab = seg_labels(seg_gt.double(), s).reshape(BN, h, w)
    counted = lab != IGNORE
    if bug == 'gradient on ignored pixels':
        counted = torch.ones_like(counted)
    p = torch.softmax(x, 1)
    onehot = F.one_hot(torch.where(lab == IGNORE, 0, lab), Cn).permute(0, 3, 1, 2).double() * (lab != IGNORE)[:, None]
    n = int((lab != IGNORE).sum())
    ce = (-(torch.log_softmax(x, 1) * onehot).sum(1))[lab != IGNORE].sum() / n if n else torch.tensor(float('nan'), dtype=torch.float64)
    k0 = up[0] * SEG_W * _focal_prime(ce, bug != "f' second term missing") / max(n, 1)
    gs = torch.where(counted[:, None], k0 * (p - onehot), torch.zeros_like(p))
    y = depth.detach().double()
    D, dh, dw = y.shape[1:]
    bins = depth_bins(depth_gt, f, D, nan_is_background=bug != 'NaN block treated as foreground').reshape(BN, dh, dw)
    fg = bins > 0
    nfg = int(fg.sum())
    oh = F.one_hot(bins, D + 1)[..., 1:].permute(0, 3, 1, 2).double()
    mask = torch.ones_like(fg) if bug == 'gradient on background cells' else fg
    gd = torch.where(mask[:, None], up[1] * (torch.sigmoid(y) - oh) / max(1, nfg), torch.zeros_like(y))
    return gs, gd


def camera_scale(seg, depth, seg_gt, depth_gt, f=16, s=2, up=(1.0, 1.0)):
    """per element: |g0 w f'(ce) / n| (softmax + onehot) and |g1 / max(1, n_fg)| (sigmoid + onehot), the formula's largest terms"""
    x = seg.detach().double()
    BN, Cn, h, w = x.shape
    lab = seg_labels(seg_gt.double(), s).reshape(BN, h, w)
    valid = lab != IGNORE
    n = int(valid.sum())
    onehot = F.one_hot(torch.where(valid, lab, 0), Cn).permute(0, 3, 1, 2).double() * valid[:, None]
    ce = (-(torch.log_softmax(x, 1) * onehot).sum(1))[valid].sum() / max(n, 1)
    k0 = abs(up[0] * SEG_W * float(_focal_prime(ce)) / max(n, 1))
    ss = k0 * (torch.softmax(x, 1) + onehot) + 1e-30
    y = depth.detach().double()
    D = y.shape[1]
    bins = depth_bins(depth_gt, f, D).reshape(y.shape[0], *y.shape[2:])
    k1 = abs(up[1]) / max(1, int((bins > 0).sum()))
    oh = F.one_hot(bins, D + 1)[..., 1:].permute(0, 3, 1, 2).double()
    sd = k1 * (torch.sigmoid(y) + oh) + 1e-30
    return ss, sd


# ------------------------------------------------------------------------------------------------------------------ decoder
PRED_KEYS = ('mu_branches', 'sigma_branches', 'pred_speed', 'pred_value_traj', 'pred_value_ctrl', 'pred_features_traj',
             'pred_features_ctrl', 'future_mu', 'future_sigma', 'pred_wp', 'refine_BEV_feature', 'refine_flattned_BEV_feature',
             'teacher_pred_wp_offset', 'teacher_pred_ctrl_offset_lis', 'teacher_future_BEV_feature', 'teacher_refine_BEV_feature',
             'teacher_refine_flattned_BEV_feature')
OFFSETS = ('current_throttle_brake_offset', 'current_steer_offset', 'longitudinal_offset', 'lateral_offset')
CONFIG = dict(value_weight=0.001, features_weight=0.05)      # thinktwice.py
DISTIL_SHAPES = {2: (32, 21, 21), 3: (64, 10, 10), 4: (128, 4, 4), 5: (256, 2, 2)}


def decoder_module(config=CONFIG):
    """the attributes decoder_loss reads from the reference's ThinkTwiceDecoder"""
    return SimpleNamespace(action_loss_weight=15.0, wp_loss_weight=15.0, distil_index=[2, 3, 4, 5],
                           distil_kl_loss_weight_dict=dict(LO.DISTIL), config=SimpleNamespace(**config))


def make_inputs(B, K=5, T=4, seed=0, quarter=False):
    """seeded (pred, mid, batch) at the teacher-forced pass's shapes.  quarter: every value a multiple of 1/4 (exact differences)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, lo=-3.0, hi=3.0: lo + (hi - lo) * torch.rand(*s, generator=g, dtype=torch.float64)
    q = (lambda t: torch.round(t * 4) / 4) if quarter else (lambda t: t)
    beta = lambda *s: 0.05 + 20 * torch.rand(*s, generator=g, dtype=torch.float64) ** 2
    pred = dict(mu_branches=beta(B, K + 1, 2), sigma_branches=beta(B, K + 1, 2), pred_speed=q(r(B, 1)), pred_value_traj=q(r(B, 1)),
                pred_value_ctrl=q(r(B, 1)), pred_features_traj=q(r(B, 256)), pred_features_ctrl=q(r(B, 256)),
                future_mu=beta(B, K + 1, T - 1, 2), future_sigma=beta(B, K + 1, T - 1, 2), pred_wp=q(r(B, K + 1, T, 2, hi=9.0)),
                refine_BEV_feature=q(r(B, K, 32, 21, 21, lo=-8, hi=10)), refine_flattned_BEV_feature=q(r(B, K, 256, lo=-8, hi=10)),
                teacher_pred_wp_offset=q(r(B, K, T, 2)), teacher_pred_ctrl_offset_lis=q(r(B, K, T, 4)),
                teacher_future_BEV_feature=q(r(B, K, T, 32, 21, 21, lo=-8, hi=10)), teacher_refine_BEV_feature=q(r(B, K, 32, 21, 21, lo=-8, hi=10)),
                teacher_refine_flattned_BEV_feature=q(r(B, K, 256, lo=-8, hi=10)))
    mid = [None, None] + [q(r(B, *DISTIL_SHAPES[i], lo=-8, hi=10)) for i in (2, 3, 4, 5)]
    batch = dict(speed=q(r(B, lo=0, hi=12)), value=q(r(B)), feature=q(r(B, 256, lo=0, hi=1)), waypoints=q(r(B, T, 2, hi=9.0)),
                 action_mu=beta(B, 2), action_sigma=beta(B, 2), future_action_mu=[beta(B, 2) for _ in range(T)],
                 future_action_sigma=[beta(B, 2) for _ in range(T)],
                 grid_feature=[None, None] + [q(r(B, *DISTIL_SHAPES[i], lo=0, hi=2)) for i in (2, 3, 4, 5)],
                 future_grid_feature=[[None, None, q(r(B, *DISTIL_SHAPES[2], lo=0, hi=2))] for _ in range(T)])
    return pred, mid, batch_as(batch, torch.float32, 'cpu', torch.float64)     # ground truth exact in fp32, as the op stages it


def batch_as(batch, dtype, device, then=None):
    """every tensor of the batch in `dtype` on `device` (and then in `then`)"""
    def cv(v):
        if torch.is_tensor(v):
            v = v.detach().to(device, dtype)
            return v.to(then) if then is not None else v
        if isinstance(v, list):
            return [cv(x) for x in v]
        return v
    return {k: cv(v) for k, v in batch.items()}


def upstream(values, seed=1):
    """a random weight per loss element (the total is sum w * value): upstream gradients that tell every slot apart"""
    g = torch.Generator().manual_seed(seed)
    return OrderedDict((k, 0.5 + torch.rand(tuple(v.shape), generator=g, dtype=torch.float64)) for k, v in values.items())


def decoder_ref(pred, mid, batch, w=None, config=CONFIG):
    """float64 autograd of loss_oracle.decoder_loss: (values, grads by pred key / 'mid{i}', the upstream weights used)"""
    P = {k: pred[k].detach().double().cpu().requires_grad_() for k in PRED_KEYS}
    M = [None, None] + [mid[i].detach().double().cpu().requires_grad_() for i in (2, 3, 4, 5)]
    bt = _to64(batch)
    d = LO.decoder_loss(config, bt, P, M)
    w = w if w is not None else upstream(d)
    total = sum((d[k] * w[k]).sum() for k in d if k not in OFFSETS)      # the offsets are computed under no_grad by the reference
    total.backward()
    grads = {k: P[k].grad for k in PRED_KEYS}
    grads.update({f'mid{i}': M[i].grad for i in (2, 3, 4, 5)})
    return d, grads, w


def _to64(batch):
    def cv(v):
        if torch.is_tensor(v):
            return v.detach().double().cpu()
        if isinstance(v, list):
            return [cv(x) for x in v]
        return v
    return {k: cv(v) for k, v in batch.items()}


def sl1p(d):
    return torch.clamp(d, -1.0, 1.0)


def _sl1(d):
    a = d.abs()
    return torch.where(a < 1, 0.5 * a * a, a - 0.5)


def clamp_pass(d, bug=None):
    v = _sl1(d)
    return ((v >= -5) & (v < 5)) if bug == 'clamp boundary excluded' else ((v >= -5) & (v <= 5))


def _kl_grads(a1, b1, a2, b2):
    ps = torch.special.digamma
    c = ps(a1 + b1) - ps(a2 + b2)
    return ps(a2) - ps(a1) + c, ps(b2) - ps(b1) + c


def decoder_formula(pred, mid, batch, w, config=CONFIG, bug=None):
    """the header's per-element gradients of every prediction for upstream weights w (tt_loss_backward's formulas)"""
    P = {k: pred[k].detach().double().cpu() for k in PRED_KEYS}
    bt = _to64(batch)
    vw, fw = config['value_weight'], config['features_weight']
    B = P['pred_speed'].shape[0]
    G = {}
    a1, b1 = bt['action_mu'][:, None], bt['action_sigma'][:, None]
    ga, gb = _kl_grads(a1, b1, P['mu_branches'], P['sigma_branches'])
    u = w['action_loss'] * 15.0 / P['mu_branches'].numel()
    G['mu_branches'], G['sigma_branches'] = u * ga, u * gb
    fa = torch.stack(bt['future_action_mu'][:-1], 1)[:, None]
    fb = torch.stack(bt['future_action_sigma'][:-1], 1)[:, None]
    ga, gb = _kl_grads(fa, fb, P['future_mu'], P['future_sigma'])
    u = w['future_action_loss'] * 15.0 * 0.25 / P['future_mu'].numel()
    G['future_mu'], G['future_sigma'] = u * ga, u * gb
    G['pred_speed'] = w['speed_loss'] * sl1p(P['pred_speed'] - (bt['speed'].float().view(-1, 1) / 12.).double()) / B
    gv = bt['value'].view(-1, 1)
    wv = w['value_loss'].view(-1)
    up_traj = wv[:1].sum() if bug == 'v_traj fed by one slot' else wv.sum()
    G['pred_value_traj'] = up_traj * vw / B * sl1p(P['pred_value_traj'] - gv)
    G['pred_value_ctrl'] = wv.view(-1, 1) * vw * sl1p(P['pred_value_ctrl'] - gv)
    for k in ('pred_features_traj', 'pred_features_ctrl'):
        G[k] = w['flattened_feature_loss'] * fw / P[k].numel() * sl1p(P[k] - bt['feature'])
    G['pred_wp'] = w['wp_loss'] * 15.0 / P['pred_wp'].numel() * sl1p(P['pred_wp'] - bt['waypoints'][:, None])

    def clamped(x, gt, scale):
        d = x - gt
        return torch.where(clamp_pass(d, bug), scale / x.numel() * torch.ones_like(d), torch.zeros_like(d)) * sl1p(d)
    for i in (2, 3, 4, 5):
        G[f'mid{i}'] = clamped(mid[i].detach().double().cpu(), bt['grid_feature'][i], w[f'BEV_feature_loss{i}'] * LO.DISTIL[i])
    g2 = bt['grid_feature'][2][:, None]
    G['refine_BEV_feature'] = clamped(P['refine_BEV_feature'], g2, w['refine_BEV_feature_loss2'] * LO.DISTIL[2])
    G['refine_flattned_BEV_feature'] = clamped(P['refine_flattned_BEV_feature'], bt['feature'][:, None],
                                               w['refine_flattened_feature_loss'] * fw * 0.1)
    G['teacher_pred_wp_offset'] = w['teacher_wp_loss'] / P['teacher_pred_wp_offset'].numel() * sl1p(P['teacher_pred_wp_offset'])
    G['teacher_pred_ctrl_offset_lis'] = (w['teacher_action_loss'] / P['teacher_pred_ctrl_offset_lis'].numel() *
                                         sl1p(P['teacher_pred_ctrl_offset_lis']))
    gf = torch.stack([f[2] for f in bt['future_grid_feature']], 1)[:, None]
    G['teacher_future_BEV_feature'] = clamped(P['teacher_future_BEV_feature'], gf, w['teacher_future_BEV_feature_loss2'] * LO.DISTIL[2])
    G['teacher_refine_BEV_feature'] = clamped(P['teacher_refine_BEV_feature'], g2, w['teacher_refine_BEV_feature_loss2'] * LO.DISTIL[2])
    G['teacher_refine_flattned_BEV_feature'] = clamped(P['teacher_refine_flattned_BEV_feature'], bt['feature'][:, None],
                                                       w['teacher_refine_flattened_feature_loss'] * fw)
    return G


def decoder_scale(pred, mid, batch, w, config=CONFIG):
    """per element: the largest term of its formula, |u| * (|s'(d)| for the smooth-L1 kinds, sum of |psi| for the Beta KL)"""
    P = {k: pred[k].detach().double().cpu() for k in PRED_KEYS}
    bt = _to64(batch)
    ones = {k: torch.ones_like(v) for k, v in w.items()}
    S = {k: v.abs() for k, v in decoder_formula(pred, mid, batch, ones, config).items()}
    ps = lambda x: torch.special.digamma(x).abs()
    B = P['pred_speed'].shape[0]
    for (m, s, gm, gs, key, wt) in (('mu_branches', 'sigma_branches', bt['action_mu'][:, None], bt['action_sigma'][:, None], 'action_loss', 15.0),
                                    ('future_mu', 'future_sigma', torch.stack(bt['future_action_mu'][:-1], 1)[:, None],
                                     torch.stack(bt['future_action_sigma'][:-1], 1)[:, None], 'future_action_loss', 15.0 * 0.25)):
        a2, b2 = P[m], P[s]
        common = ps(gm + gs) + ps(a2 + b2)
        u = wt / a2.numel() * float(w[key].abs().max())
        S[m] = u * (ps(a2) + ps(gm) + common)
        S[s] = u * (ps(b2) + ps(gs) + common)
    wmax = max(float(v.abs().max()) for v in w.values())
    S = {k: v * wmax + 1e-30 for k, v in S.items()}
    S['pred_value_traj'] = S['pred_value_traj'] * B               # fed by B slots
    return S
