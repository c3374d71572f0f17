"""The kernel census (tests/kernel_census.py) over the open-loop validation forward, `forward(is_eval=True, **batch)`: the full
thinktwice.py config with its shipped flags (seg and depth supervision on), oracle weights and calibrated BatchNorm, supervision and
camera ground truth from thinktwice_b200.synthetic.  Every call of the network, of the teacher-forced decoder pass (buffers tf.*,
tt_eltwise op 4 on the real ground-truth controls), tt_loss_reduce and tt_camera_loss is checked against float64 on the operands it
received: at B = 1 and B = 2 in both Look modes with whole tensors and nothing outside each destination changed, and at B = 16 on
windows (tests/test_kernel_census_gpu.py), so the teacher layers >= 1 at the throughput batch are checked per element.  The logged
losses of a census run equal those of a run without it.  Plus the inference path whose call sequence differs from a cold forward: a
warm tick of the streaming BEV cache."""
import time

import pytest
import torch

import kernel_census as KC
from test_kernel_census_gpu import CAP, full                          # noqa: F401  (the module-scoped model fixture)

pytestmark = pytest.mark.gpu

EXACT = 1e-5                     # tests/test_losses_gpu.py: a loss against the same loss computed another way on the same outputs


def relerr(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-6))


def validation_batch(cfg, B, seed):
    from thinktwice_b200.synthetic import make_batch, make_camera_supervision, make_supervision
    batch = make_batch(cfg, B, seed=seed, num_points=40000)
    batch.update(make_supervision(cfg, B, seed=seed))
    batch.update(make_camera_supervision(cfg, B, seed=seed))
    return batch


def run_census(full, B, independent, window=False):
    cfg, model = full
    assert model.config['use_seg'] and model.config['use_depth']
    model.enable_independent_frames(independent)
    batch = validation_batch(cfg, B, seed=60 + B)
    plain = model.forward(is_eval=True, **batch)['log_vars']
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    with pytest.MonkeyPatch.context() as mp:
        census = KC.install(mp, KC.Census(model.eng, outside=not window, window=window, cap=CAP if window else None))
        out = model.forward(is_eval=True, **batch)
        torch.cuda.synchronize()
    ws, call, entry = census.peak
    peak = max(census.max_allocated, torch.cuda.max_memory_allocated())   # (the census resets the peak counter at every checked call)
    print(f'\n{torch.cuda.get_device_name()}, validation forward B = {B}, {"independent" if independent else "coupled"} Look, '
          f'{"windows" if window else "whole tensors"}: {census.calls} ABI calls, {time.time() - t0:.1f} s; peak device memory '
          f'{peak / 2 ** 30:.1f} GiB; largest per-call working set {ws / 2 ** 30:.2f} GiB (call #{call} {entry})')
    print(census.table())
    print(census.layer_table('tf.'))
    print(census.layer_table('loss.'))
    census.assert_clean()
    assert model.f16s_saturations() == 0
    assert {'tt_loss_reduce', 'tt_camera_loss', 'tt_eltwise'} <= set(census.stats)
    assert ('tt_eltwise', 'tf.ctrl') in census.layers                  # the inverse softplus of the ground-truth controls
    K = model.decoder.K
    tf = {layer for _, layer in census.layers if layer.startswith('tf.')}
    assert tf >= {f'tf.{m}' for k in range(K) for m in (f'l{k}.fut', f'bev.{k}', f'flat.{k}')}, sorted(tf)
    assert list(out['log_vars']) == list(plain)
    bad = {k: relerr(out['log_vars'][k], v) for k, v in plain.items() if not relerr(out['log_vars'][k], v) <= EXACT}
    assert not bad, bad                                                # the census changes timing, not results
    return census


def test_b1_validation_forward_every_call_matches_fp64(full):
    run_census(full, 1, False)


@pytest.mark.parametrize('independent', [False, True])
def test_b2_validation_forward_every_call_matches_fp64_and_writes_nothing_outside(full, independent):
    c = run_census(full, 2, independent)
    assert ('tt_msda_forward_frames' if independent else 'tt_msda_forward') in c.stats


def test_warm_streaming_tick_every_call_matches_fp64(full):
    """two consecutive eager ticks at B = 2 with the streaming BEV cache; the census covers the second, which copies the cached
    key-frame BEV into the history slot instead of rerunning the history sweep."""
    from thinktwice_b200 import lib
    from thinktwice_b200.synthetic import make_batch
    cfg, model = full
    model.enable_independent_frames(False)
    ticks = [make_batch(cfg, 2, seed=s, num_points=40000) for s in (81, 82)]
    ticks[1]['img'][:, 0] = ticks[0]['img'][:, 1]                      # tick 1's history sweep is tick 0's key frame
    model.enable_streaming_bev_cache()
    try:
        n0 = lib.launch_count()
        model.forward_inference(ticks[0])
        cold = lib.launch_count() - n0
        assert model.img_encoder.cache_ready(2)
        with pytest.MonkeyPatch.context() as mp:
            census = KC.install(mp, KC.Census(model.eng))
            model.forward_inference(ticks[1])
            torch.cuda.synchronize()
            warm = lib.launch_count() - n0 - cold                     # (+ the census's own fp32 upsample per split upsample call)
    finally:
        model.enable_streaming_bev_cache(False)
    print(f'\nwarm streaming tick, B = 2: {census.calls} ABI calls, {warm} launches (the cold tick: {cold})')
    print(census.table())
    census.assert_clean()
    assert model.f16s_saturations() == 0
    assert warm < cold


def test_b16_validation_forward_windows_of_every_call_match_fp64(full):
    c = run_census(full, 16, False, window=True)
    assert c.peak[0] < CAP
    assert c.stats['tt_conv2d_f16s'][0] > 100
