"""Independent-frames mode (EncoderDecoder.enable_independent_frames) on the CPU, through the torch emulation of the C ABI
(tests/emu_lib.py, with the two per-frame Look entries from tests/emu_frames.py): frame j of an independent-mode batch must equal
the oracle run on frame j alone at B = 1, while the default batch-coupled mode keeps the reference's batch semantics.  The kernels behind the two new entry points are the GPU suite's job
(tests/test_independent_frames_gpu.py)."""
import numpy as np
import pytest
import torch

KEYS = ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed', 'refine_flattned_BEV_feature',
        'refine_BEV_feature', 'refine_future_BEV_feature')
TOL = 5e-4                                                             # fp32 oracle vs fp64-contraction emulation (as the other emulated tests)
B, SEED, POINTS = 4, 1, 1500


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-12))


@pytest.fixture
def emu(emulated):
    """the emulated C ABI with the per-frame Look entries installed."""
    import emu_frames
    return emu_frames.install(emulated)


def frame_err(batched, alone, j, k):
    """max |frame j of a batched output - frame j's own B = 1 output|, relative to the output's largest magnitude over the frames
    (a per-frame scalar such as pred_speed can be near zero in one frame)."""
    scale = max(float(ref[k].abs().max()) for ref in alone) + 1e-12
    return float((batched[k][j:j + 1].double() - alone[j][k].double()).abs().max()) / scale


def frame(batch, j):
    return {k: v[j:j + 1] for k, v in batch.items()}


@pytest.fixture(scope='module')
def plumbing():
    """oracle + product weights for the plumbing config, the B = 4 batch and the oracle's per-frame B = 1 and B = 4 results."""
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(PLUMBING_CONFIG)
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(o, SEED)
    batch = make_batch(cfg, B, seed=SEED, num_points=POINTS)
    calibrate_bn(o, batch)
    alone = []
    with torch.no_grad():
        for j in range(B):
            keep = {}
            ref = o.forward_inference(frame(batch, j), keep=keep)
            # the Look module's reduced feature of the last layer at B = 1: row 0 zeroed, divisor 1, rows < max_len (msda:338-342).
            # output_proj starts with a LayerNorm, which hides a wrong divisor from every model output: the sum is checked itself
            rows = keep['dec_keep']['layers'][-1]['sca_rows']
            ref['look_sum'] = rows[:, :, 1:].sum(2).reshape(1, -1)
            alone.append(ref)
        coupled = o.forward_inference(batch)
    return dict(cfg=cfg, oracle=o, batch=batch, alone=alone, coupled=coupled)


def product(plumbing, independent):
    from thinktwice_b200.registry import build_model
    m = build_model(plumbing['cfg'].model)
    m.load_state_dict(plumbing['oracle'].state_dict())
    m.prepare('cpu', impl=4)
    return m.enable_independent_frames(independent)


def worst_frame_error(m, pred, alone):
    """largest relative error over every output of every frame, and over the last Look module's reduced feature, against that
    frame's B = 1 reference; and where it is."""
    got = {k: pred[k] for k in KEYS}
    got['look_sum'] = m.eng.static_named('look.red').reshape(B, -1)
    errs = {(j, k): frame_err(got, alone, j, k) for j in range(B) for k in KEYS + ('look_sum',)}
    where = max(errs, key=errs.get)
    return errs[where], where


def test_independent_frames_match_each_frame_alone(emu, plumbing):
    m = product(plumbing, True)
    pred = m.forward_inference(plumbing['batch'])
    err, where = worst_frame_error(m, pred, plumbing['alone'])
    assert err < TOL, (err, where)
    # the per-frame row bound is what is under test: the frames' max_len_b must really differ
    ml = m.eng.static_named('look.counts').view(B, 4).amax(1).tolist()
    assert len(set(ml)) > 1, ml
    # and the coupled reference semantics really give other results for this batch
    err_c = max(frame_err(plumbing['coupled'], plumbing['alone'], j, k) for j in range(B) for k in KEYS)
    assert err_c > 10 * TOL, err_c


def _reduce_batch_max_len(self, rows, B_, cams, cap, Cc, counts, out, stream):
    """mutant: the per-frame sum bounded by the batch-wide max_len."""
    ml = int(counts.flat()[:B_ * cams].max())
    r = rows.flat()[:B_ * cams * cap * Cc].view(B_, cams, cap, Cc)
    out.flat()[:B_ * cams * Cc].view(B_, cams * Cc).copy_(r[:, :, 1:min(ml, cap)].double().sum(2).float().reshape(B_, cams * Cc))
    return 0


def _reduce_divide_by_b(self, rows, B_, cams, cap, Cc, counts, out, stream):
    """mutant: the per-frame bound, but the coupled divisor B."""
    import emu_frames
    emu_frames.tt_look_reduce_frames(self, rows, B_, cams, cap, Cc, counts, out, stream)
    out.flat()[:B_ * cams * Cc].div_(B_)
    return 0


@pytest.mark.parametrize('mutant', [_reduce_batch_max_len, _reduce_divide_by_b])
def test_the_per_frame_check_rejects_a_coupled_reduction(emu, plumbing, mutant, monkeypatch):
    monkeypatch.setattr(emu, 'tt_look_reduce_frames', mutant.__get__(emu))
    m = product(plumbing, True)
    err, where = worst_frame_error(m, m.forward_inference(plumbing['batch']), plumbing['alone'])
    assert err > TOL, (mutant.__name__, err, where)


def test_coupled_mode_still_matches_the_oracle_batch(emu, plumbing):
    m = product(plumbing, False)
    pred = m.forward_inference(plumbing['batch'])
    for k in KEYS:
        assert rel(pred[k], plumbing['coupled'][k]) < TOL, k


def _ragged(batch, lengths):
    """a list of per-frame (1, P_b, 5) clouds cut from the batch, and the same clouds zero-padded as mmcv's collate pads them."""
    clouds = [batch['points'][j, :, :n].clone() for j, n in enumerate(lengths)]
    padded = torch.zeros(len(lengths), 1, max(lengths), batch['points'].shape[-1])
    for j, c in enumerate(clouds):
        padded[j, :, :c.shape[1]] = c
    return clouds, padded


def test_ragged_cloud_list_in_coupled_mode_equals_the_collated_tensor(emu, plumbing):
    batch = plumbing['batch']
    clouds, padded = _ragged(batch, [POINTS, 900, POINTS, 300])
    m = product(plumbing, False)
    pred = m.forward_inference(dict(batch, points=padded))
    want = {k: pred[k].clone() for k in KEYS}
    got = m.forward_inference(dict(batch, points=clouds))
    for k in KEYS:
        assert torch.equal(got[k], want[k]), k


def test_ragged_cloud_list_in_independent_mode_gives_each_short_frame_its_own_result(emu, plumbing):
    batch, o = plumbing['batch'], plumbing['oracle']
    lengths = [POINTS, 900, POINTS, 300]
    clouds, padded = _ragged(batch, lengths)
    m = product(plumbing, True)
    got = m.forward_inference(dict(batch, points=clouds))
    pred = {k: got[k].clone() for k in KEYS}
    for j in (1, 3):                                                   # the short clouds: no phantom voxel from the padding
        one = dict(frame(batch, j), points=clouds[j][None])
        with torch.no_grad():
            ref = o.forward_inference(one)
        alone = m.forward_inference(one)
        refs = list(plumbing['alone'])
        refs[j] = ref
        for k in KEYS:
            assert frame_err(pred, refs, j, k) < TOL, (j, k)
            assert rel(pred[k][j:j + 1], alone[k]) < 1e-4, (j, k)        # the product alone: CPU op order varies with B
    # the collated tensor is taken as given: its zero rows are points, which put a voxel at the origin of frame 3
    with torch.no_grad():
        ref_padded = o.forward_inference(dict(frame(batch, 3), points=padded[3:4]))
    got = m.forward_inference(dict(batch, points=padded))
    assert rel(got['pred_wp'][3:4], ref_padded['pred_wp']) < TOL


def test_new_entry_points_fail_loudly_without_cuda():
    from thinktwice_b200 import lib
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.registry import build_model
    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    assert {'tt_msda_forward_frames', 'tt_look_reduce_frames'} <= set(lib.EXPORTS)
    m = build_model(Config.fromfile(PLUMBING_CONFIG).model)
    assert m.enable_independent_frames() is m and m.decoder.independent_frames
    with pytest.raises(lib.TTError):
        m.prepare('cpu')
    rows, counts, out = torch.zeros(4, 120, 256), torch.zeros(1, 4, dtype=torch.int32), torch.zeros(1, 1024)
    with pytest.raises(lib.TTError):
        lib.call('tt_look_reduce_frames', lib._p(rows), 1, 4, 120, 256, lib._p(counts), lib._p(out))
    d = lib.MsdaDesc()
    d.BN, d.rows_cap, d.heads, d.levels, d.points, d.dh = 4, 120, 8, 4, 8, 32
    with pytest.raises(lib.TTError):
        lib.call('tt_msda_forward_frames', lib.ref(d), lib._p(torch.zeros(4, 10, 256)), lib._p(torch.zeros(480, 512)),
                 lib._p(torch.zeros(480, 256)), lib._p(torch.zeros(480, 2)), lib._p(counts), 4, lib._p(torch.zeros(480, 256)))
