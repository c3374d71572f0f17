"""Every convolution and glue-kernel call of a thinktwice.py forward, checked call by call against float64 on the activations it
actually received (tests/kernel_census.py): the full config with oracle weights and calibrated BatchNorm, eagerly, at B = 1 (the
latency config: under-filled layers run split-K) and B = 2 in both Look modes, with whole tensors compared and every element of each
destination buffer outside the written region required bitwise unchanged; and at B = 16 (the throughput config: 128-column tiles,
offsets past 2^31 in the arena), where each convolution is checked on windows of whole images or >= 256 rows at the start and the
end of its N (every bias_n_mod residue in each) and a call of another entry whose fp64 copies would pass 4 GB is counted as skipped."""
import time

import pytest
import torch

import kernel_census as KC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def full():
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, 0)
    calibrate_bn(oracle, make_batch(cfg, 1, seed=0, num_points=40000))
    model = build_model(cfg.model)
    model.load_state_dict(oracle.state_dict())
    model.prepare('cuda:0')
    return cfg, model


CAP = 4 << 30


def run_census(full, B, independent, window=False):
    from thinktwice_b200.synthetic import make_batch
    cfg, model = full
    model.enable_independent_frames(independent)
    batch = make_batch(cfg, B, seed=7 + B, num_points=40000)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    with pytest.MonkeyPatch.context() as mp:
        census = KC.install(mp, KC.Census(model.eng, outside=not window, window=window, cap=CAP if window else None))
        model.forward_inference(batch)
        KC.inverse_softplus(model.eng)
        torch.cuda.synchronize()
    ws, call, entry = census.peak
    print(f'\n{torch.cuda.get_device_name()}, B = {B}, {"independent" if independent else "coupled"} Look, '
          f'{"windows" if window else "whole tensors"}: {census.calls} ABI calls, {time.time() - t0:.0f} s; largest per-call working set '
          f'{ws / 2 ** 30:.2f} GiB (call #{call} {entry}), {torch.cuda.memory_allocated() / 2 ** 30:.1f} GiB allocated after the forward')
    print(census.table())
    census.assert_clean()
    assert model.f16s_saturations() == 0
    return census


def test_b1_every_call_matches_fp64(full):
    c = run_census(full, 1, False)
    assert c.stats['tt_conv2d_f16s'][0] > 100


@pytest.mark.parametrize('independent', [False, True])
def test_b2_every_call_matches_fp64_and_writes_nothing_outside_its_destination(full, independent):
    c = run_census(full, 2, independent)
    assert ('tt_msda_forward_frames' if independent else 'tt_msda_forward') in c.stats


def test_b16_windows_of_every_call_match_fp64(full):
    c = run_census(full, 16, False, window=True)
    assert c.peak[0] < CAP
    assert c.stats['tt_conv2d_f16s'][0] > 100 and c.stats['tt_eltwise'][0] > 0
