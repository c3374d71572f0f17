"""The kernel census (tests/kernel_census.py) over the open-loop validation forward, `forward(is_eval=True, **batch)`, on the emulated
C ABI at the plumbing size (two Look layers, seg and depth supervision on): a B = 2 forward passes it in both Look modes, with the
teacher-forced pass, tt_loss_reduce and tt_camera_loss checked call by call; and each mutated emulator entry below is rejected by the
check meant for it, with a message naming the call."""
import pytest

import emu_camera_losses
import emu_frames
import emu_lib
import emu_losses
import kernel_census as KC
from emu_lib import _desc

B = 2


@pytest.fixture
def validation(emulated, monkeypatch):
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch, make_camera_supervision, make_supervision
    emu_camera_losses.install(emu_losses.install(emu_frames.install(emulated), monkeypatch), monkeypatch)
    emu_lib._by_addr.clear()
    cfg = Config.fromfile(PLUMBING_CONFIG)
    cfg.merge_from_dict({'model.train_cfg.use_seg': True, 'model.train_cfg.use_depth': True})
    for c in (cfg.model.decoder.config, cfg.model.train_cfg, cfg.model.test_cfg):
        c['refine_num'] = 2                                            # two Look layers in each pass, two teacher layers
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(o, 1)
    batch = make_batch(cfg, B, seed=1, num_points=1500)
    calibrate_bn(o, batch)
    batch.update(make_supervision(cfg, B, seed=1))
    batch.update(make_camera_supervision(cfg, B, seed=1))
    m = build_model(cfg.model)
    m.load_state_dict(o.state_dict())
    m.prepare('cpu', impl=4)

    def run(independent=False, census=None):
        m.enable_independent_frames(independent)
        census = KC.install(monkeypatch, census or KC.Census(m.eng))
        return census, m.forward(is_eval=True, **batch)
    yield emulated, m, batch, run
    emu_lib._by_addr.clear()


def test_b2_validation_forward_passes_the_census(validation):
    emu, m, batch, run = validation
    for independent in (False, True):
        census, out = run(independent)
        print(census.table())
        print(census.layer_table('tf.'))
        census.assert_clean()
        assert {'tt_loss_reduce', 'tt_camera_loss', 'tt_eltwise', 'tt_conv2d_f16s'} <= set(census.stats)
        assert census.stats['tt_loss_reduce'][0] == 1 and census.stats['tt_camera_loss'][0] == 1
        tf = {(k, layer) for k, layer in census.layers if layer.startswith('tf.')}
        assert ('tt_eltwise', 'tf.ctrl') in tf                         # the teacher's inverse softplus on the ground-truth controls
        for k in range(2):                                             # both teacher layers: GRU output, BEV and flat updates
            assert {layer for _, layer in tf} >= {f'tf.l{k}.fut', f'tf.bev.{k}', f'tf.flat.{k}'}
        assert {'seg_loss', 'depth_loss', 'teacher_wp_loss'} <= set(out['log_vars'])


# ---------------------------------------------------------------------------------------------------------- mutants
# As in tests/test_kernel_census_cpu.py: every call is compared with a reference computed from the operands it received, so the mutants
# share one forward, each on a call of its own.  The forward makes one tt_loss_reduce call; the two further loss mutants get theirs from
# ThinkTwiceDecoder.loss run again on the same teacher-forced outputs.
from test_kernel_census_cpu import Mutants                           # noqa: E402


def _reach(shape, stride):
    return sum((n - 1) * s for n, s in zip(shape, stride))


def mut_gt_pred_strides(M):
    """tt_loss_reduce reads one term's ground truth with the prediction's strides (a term whose pred and gt layouts differ and whose
    gt buffer holds every element so read: the channels-last BEV maps against NCHW ground truth)."""
    def make(orig):
        def f(terms, n_terms, out, n_slots, ws, ws_bytes, stream):
            i = next((i for i, t in enumerate(terms[:n_terms]) if t['gt'] and list(t['gt_stride']) != list(t['pred_stride'])
                      and _reach(t['shape'], t['pred_stride']) < t['gt'].flat().numel()), None)
            if M.claim('loss_gt_read_with_pred_strides', i is not None):
                terms = list(terms)
                terms[i] = dict(terms[i], gt_stride=list(terms[i]['pred_stride']))
            return orig(terms, n_terms, out, n_slots, ws, ws_bytes, stream)
        return f
    M.wrap('tt_loss_reduce', make)


def mut_last_range(M):
    """tt_loss_reduce drops the last of the 16 element ranges of its largest term."""
    def make(orig):
        def f(terms, n_terms, out, n_slots, ws, ws_bytes, stream):
            h = M.claim('loss_last_range_dropped')
            rc = orig(terms, n_terms, out, n_slots, ws, ws_bytes, stream)
            if h:
                t = max(terms[:n_terms], key=lambda t: emu_losses.term_values(t).numel())
                v = emu_losses.term_values(t).reshape(-1)
                out.flat()[t['slot']] -= float(t['scale'] * v[15 * -(-v.numel() // 16):].sum())
            return rc
        return f
    M.wrap('tt_loss_reduce', make)


def mut_next_slot(M):
    """tt_loss_reduce adds one term (the first with a non-zero sum) into the next slot as well."""
    def make(orig):
        def f(terms, n_terms, out, n_slots, ws, ws_bytes, stream):
            if M.claim('loss_term_into_next_slot'):
                t = next(t for t in terms[:n_terms] if t['slot'] + 1 < n_slots and float(emu_losses.term_values(t).sum()) != 0)
                terms = list(terms[:n_terms]) + [dict(t, slot=t['slot'] + 1)]
                n_terms += 1
            return orig(terms, n_terms, out, n_slots, ws, ws_bytes, stream)
        return f
    M.wrap('tt_loss_reduce', make)


def mut_camera_bin(M):
    """tt_camera_loss with the depth target one bin off (emu_camera_losses' seeded bug, set for the product's call only: the census's
    reference reads the same module)."""
    def make(orig):
        def f(d, out, ws, ws_bytes, stream):
            if not M.claim('camera_bin_off_by_one'):
                return orig(d, out, ws, ws_bytes, stream)
            emu_camera_losses.BUG = 'bin_off_by_one'
            try:
                return orig(d, out, ws, ws_bytes, stream)
            finally:
                emu_camera_losses.BUG = None
        return f
    M.wrap('tt_camera_loss', make)


def mut_inverse_softplus_skipped(M):
    """tt_eltwise op 4 returns its input (the teacher's ground-truth controls left in softplus space)."""
    def make(orig):
        def f(op, act, a, a_ld, b, b_ld, c, c_ld, y, y_ld, rows, cols, stream):
            if M.claim('inverse_softplus_skipped', emu_lib._v(op) == 4):
                op = 3
            return orig(op, act, a, a_ld, b, b_ld, c, c_ld, y, y_ld, rows, cols, stream)
        return f
    M.wrap('tt_eltwise', make)


def mut_teacher_y_nstride(M):
    """a teacher-layer convolution with a per-image output stride (the GRU decoder conv writing step t of every frame into tf.l0.fut)
    that ignores y_nstride: its images land contiguously."""
    def make(orig):
        def f(d, io, stream):
            dd = _desc(d)
            y = io.y if io.y else io.y_split
            if not M.claim('teacher_conv_ignores_y_nstride', dd.y_nstride != 0 and bool(y) and M.census.namer(y.t).startswith('tf.')):
                return orig(d, io, stream)
            k, dd.y_nstride = dd.y_nstride, 0
            try:
                return orig(d, io, stream)
            finally:
                dd.y_nstride = k
        return f
    M.wrap('tt_conv2d_f16s', make)


# mutant -> (installer, the entry its failure names, the words of the check that must reject it)
MUTANTS = {
    'loss_gt_read_with_pred_strides': (mut_gt_pred_strides, 'tt_loss_reduce', 'beyond the bound'),
    'loss_last_range_dropped': (mut_last_range, 'tt_loss_reduce', 'beyond the bound'),
    'loss_term_into_next_slot': (mut_next_slot, 'tt_loss_reduce', 'beyond the bound'),
    'camera_bin_off_by_one': (mut_camera_bin, 'tt_camera_loss', 'beyond the bound'),
    'inverse_softplus_skipped': (mut_inverse_softplus_skipped, 'tt_eltwise', 'beyond the bound'),
    'teacher_conv_ignores_y_nstride': (mut_teacher_y_nstride, 'tt_conv2d_f16s', 'write outside the destination'),
}


def test_each_validation_mutant_is_rejected_by_its_check_and_named(validation, monkeypatch):
    emu, m, batch, run = validation
    M = Mutants(emu, monkeypatch)
    for install, _, _ in MUTANTS.values():
        install(M)
    M.census = KC.Census(m.eng)
    run(census=M.census)
    for _ in range(2):
        m.decoder.loss(batch, m.last_train['pred'], m.last_train['mid'])
    fails = M.census.failures
    by_call = {}
    for f in fails:
        by_call.setdefault(int(f.split()[1].lstrip('#')), []).append(f)
    for mutant, (_, entry, what) in MUTANTS.items():
        assert M.hits.get(mutant), f'{mutant}: the validation forward makes no call it applies to'
        msgs = [f for i in M.hits[mutant] for f in by_call.get(i, [])]
        print(mutant, '->', msgs[0] if msgs else None)
        assert any(entry in f and what in f for f in msgs), (mutant, msgs)
        assert all('[?]' not in f and '[outside the arena]' not in f for f in msgs), msgs
    hit = {i for v in M.hits.values() for i in v}
    assert set(by_call) <= hit, [f for i, v in by_call.items() if i not in hit for f in v]      # nothing else fails
    assert not M.census.unchecked
