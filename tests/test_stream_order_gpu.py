"""The order of the forward's calls across streams (the LiDAR side stream, the pipelined forward's copy stream, CUDA-graph fork / join).

1. The happens-before audit (tests/stream_audit.py) of two consecutive forwards on different frames in every multi-stream configuration:
   no two accesses to one storage from different streams, one a write, may be unordered, and no caching-allocator block may be used
   off its allocation stream without record_stream.  The forwards run on a non-default stream, so a call on the legacy default stream
   (NULL) is a finding too.  Negative controls delete one wait from a recorded clean trace (nothing broken is executed) and require
   the conflict it guards.
2. Adversarial schedules, run only once the audit of this module passed: the same forwards with `torch.cuda._sleep` injected before
   every call of one lane and one long sleep (twice the other lane's measured time) at its first call, eagerly and captured into the
   CUDA graphs, against the serial run (Engine.overlap = False).  Each run must show from its timestamps that the delayed lane really
   finished last, and match the serial run to 1e-4 relative (the red.add accumulation order differs from run to run)."""
import numpy as np
import pytest
import torch

import stream_audit as A

pytestmark = pytest.mark.gpu
TOL = 1e-4
AUDITED = set()                          # audits of this module that passed (the adversarial runs need them)
OUT_KEYS = ('pred_wp', 'mu_branches', 'sigma_branches', 'pred_speed', 'refine_BEV_feature')


def relerr(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def _model(cfg, seed, batch):
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.registry import build_model
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, seed)
    calibrate_bn(oracle, batch)
    model = build_model(cfg.model)
    model.load_state_dict(oracle.state_dict())
    model.prepare('cuda:0')
    return model


@pytest.fixture(scope='module')
def full():
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    return cfg, _model(cfg, 0, make_batch(cfg, 1, seed=0, num_points=40000))


def plumbing_q2(seed, loss=False):
    """the plumbing config with two sweeps (a history sweep for the pipelined forward and the streaming cache)."""
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(PLUMBING_CONFIG)
    cfg.model['img_encoder']['queue_len'] = 2
    cfg.model['train_cfg']['queue_length'] = 2
    if loss:
        for k in ('use_depth', 'use_seg'):
            cfg.merge_from_dict({f'model.train_cfg.{k}': False, f'model.decoder.config.{k}': False})
    return cfg, _model(cfg, seed, make_batch(cfg, 1, seed=seed, num_points=1500))


def frames(cfg, B, seeds, points, where='cuda'):
    from thinktwice_b200.synthetic import make_batch
    out = []
    for s in seeds:
        b = make_batch(cfg, B, seed=s, num_points=points)
        if where == 'cuda':
            b = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in b.items()}
        elif where == 'pinned':
            b = {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in b.items()}
        out.append(b)
    return out


# ---------------------------------------------------------------------------------------------------------- the audit
def record(model, run):
    """run() recorded on a new non-default main stream, with the side, copy and capture streams four different CUDA streams: the
    Recorder."""
    torch.cuda.synchronize()
    with pytest.MonkeyPatch.context() as mp:
        main = A.distinct_streams(mp, model.eng)
        rec = A.Recorder(model.eng, main)
        mode = A.install(mp, rec)
        with torch.cuda.stream(main), mode:
            rec.active = True
            try:
                run()
            finally:
                rec.active = False
        torch.cuda.synchronize()
    return rec


def audit_clean(model, run, label, lanes=('main', 'side')):
    rec = record(model, run)
    findings, lines = A.audit(rec)
    print(f'\n[{label}] {rec.fwd} forwards, ops recorded: {dict(rec.ops)}, streams: {sorted(set(rec.roles.values()))}')
    print('\n'.join(lines))
    for f in findings[:30]:
        print('  FINDING', f)
    assert not rec.unknown, '\n'.join(rec.unknown[:10])
    assert not findings, f'{len(findings)} findings, first: {findings[0]}'
    assert rec.fwd >= 2 and rec.ops['Access'] > 100
    seen = set(rec.roles.values())
    assert set(lanes) <= seen, (lanes, seen)                        # the configuration really ran on those streams
    AUDITED.add(label)
    return rec


def expect_conflicts(rec, drop, names, label):
    """the clean trace re-analysed without the waits `drop` selects: findings on each of the buffers `names` (prefixes)."""
    findings, _ = A.audit(rec, drop=drop)
    hit = sorted({f.name for f in findings})
    print(f'[{label}] without the wait: {len(findings)} findings on {hit}')
    for f in findings[:3]:
        print('  ', f)
    for n in names:
        assert any(h.startswith(n) for h in hit), (label, n, hit)
    return findings


def two_forwards(model, batches, each=None):
    def run():
        for b in batches:
            model.forward_inference(b)
            if each:
                each()
    return run


@pytest.mark.parametrize('B,independent', [(1, False), (2, False), (2, True)])
def test_audit_one_stream_eager(full, B, independent):
    cfg, model = full
    model.use_graph = False
    model.enable_independent_frames(independent)
    try:
        rec = audit_clean(model, two_forwards(model, frames(cfg, B, (31, 32), 40000)), f'one-stream B={B} independent={independent}')
    finally:
        model.enable_independent_frames(False)
    if B == 1:                                                         # negative control: no side.join() in _device_forward
        expect_conflicts(rec, lambda op: op.where is not None and op.where.has('_device_forward', 'side.join()'), ['lidar.out.at'],
                         'side.join() deleted')


def test_audit_one_stream_b16_bench_configuration(full):
    cfg, model = full
    model.use_graph = False
    audit_clean(model, two_forwards(model, frames(cfg, 16, (33, 34), 40000)), 'one-stream B=16')
    model.release_buffers()


def test_audit_one_graph_capture_and_replay(full):
    cfg, model = full
    model.enable_cuda_graph()
    try:
        rec = audit_clean(model, two_forwards(model, frames(cfg, 1, (35, 36), 40000)), 'one graph', lanes=('main', 'side', 'capture'))
        assert any('(graph replay)' in op.what for op in rec.trace if isinstance(op, A.Access))
    finally:
        model.use_graph = False


def test_audit_streaming_cache_warm_tick():
    cfg, model = plumbing_q2(4)
    ticks = frames(cfg, 1, (41, 42), 1500)
    ticks[1]['img'][:, 0] = ticks[0]['img'][:, 1]
    model.enable_streaming_bev_cache()
    rec = audit_clean(model, two_forwards(model, ticks), 'streaming cache')
    assert model.img_encoder.cache_ready(1)


def pipelined_audit(model, batches, label, graph):
    if graph:
        model.enable_cuda_graph()
    try:
        rec = audit_clean(model, two_forwards(model, batches), label, lanes=('main', 'side', 'copy') + (('capture',) if graph else ()))
    finally:
        model.use_graph = False
    assert any(op.where is not None and op.where.phase == '_pipelined_forward' for op in rec.trace if isinstance(op, A.Wait))
    return rec


def pipelined_controls(rec, T):
    code = lambda c: (lambda op: op.where is not None and op.where.frames and op.where.frames[0][1] == c)
    expect_conflicts(rec, code('main.wait_event(ev_lidar)'), ['lidar.out.at'], 'main.wait_event(ev_lidar) deleted')
    expect_conflicts(rec, code('main.wait_event(ev_key)'), [f'in.img.{T - 1}'], 'main.wait_event(ev_key) deleted')
    # the next forward's key-frame upload (copy stream) against this forward's reader of in.img.{T-1}: copy.wait_event(ev_done) is one
    # edge between them, the next forward's copy.wait_event(ev_hist) (recorded on main after this forward's readers) is another
    alone = A.audit(rec, drop=code('copy.wait_event(ev_done)'))[0]
    print(f'[copy.wait_event(ev_done) deleted] {len(alone)} findings: copy.wait_event(ev_hist) of the next forward orders the upload too')
    both = lambda op: code('copy.wait_event(ev_done)')(op) or (code('copy.wait_event(ev_hist)')(op) and op.where.fwd > 1)
    f = expect_conflicts(rec, both, [f'in.img.{T - 1}'], 'copy.wait_event(ev_done) and the next copy.wait_event(ev_hist) deleted')
    assert any(x.name == f'in.img.{T - 1}' and {x.a.where.fwd, x.b.where.fwd} == {1, 2} for x in f)


@pytest.mark.parametrize('graph', [False, True])
def test_audit_pipelined_plumbing(graph):
    cfg, model = plumbing_q2(6)
    rec = pipelined_audit(model, frames(cfg, 2, (61, 62), 1500, 'pinned'), f'pipelined plumbing graph={graph}', graph)
    if not graph:
        pipelined_controls(rec, 2)


@pytest.mark.parametrize('graph', [False, True])
def test_audit_pipelined_full_b2(full, graph):
    cfg, model = full
    rec = pipelined_audit(model, frames(cfg, 2, (63, 64), 40000, 'pinned'), f'pipelined full B=2 graph={graph}', graph)
    if not graph:
        pipelined_controls(rec, 2)


def test_audit_pipelined_raw_frames():
    from thinktwice_b200.preprocess import AgentPreprocessor
    cfg, model = plumbing_q2(8)
    fH, fW = cfg.model['img_encoder']['final_dim']
    N = cfg.model['num_cams']
    conf = {'resize_lim': (0.56, 0.6255), 'final_dim': (fH, fW), 'rot_lim': (0, 0), 'H': 300, 'W': 400, 'rand_flip': True,
            'bot_pct_lim': (0.0, 0.0)}
    model.attach_preprocessor(AgentPreprocessor(dict(undistort=False, num_cams=N), conf, 'cuda:0'))
    batches = []
    for t, b in enumerate(frames(cfg, 2, (81, 82), 1500, 'cpu')):
        b.pop('img')
        b['img_raw'] = torch.from_numpy(np.random.default_rng(90 + t).integers(0, 256, size=(2, 2, N, 300, 400, 3), dtype=np.uint8))
        batches.append({k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in b.items()})
    rec = pipelined_audit(model, batches, 'pipelined raw frames', False)
    assert any(op.what.startswith('tt_preprocess_u8.') for op in rec.trace if isinstance(op, A.Access))


@pytest.mark.parametrize('order', ['validation_first', 'inference_first'])
def test_audit_validation_and_inference_mixed(order):
    from thinktwice_b200.synthetic import make_supervision
    cfg, model = plumbing_q2(10, loss=True)
    b1, = frames(cfg, 2, (101,), 1500, 'cpu')
    b1.update(make_supervision(cfg, 2, seed=101))
    b2, = frames(cfg, 2, (102,), 1500, 'pinned')

    def run():
        if order == 'validation_first':
            model.forward(**b1)
            model.forward_inference(b2)
        else:
            model.forward_inference(b2)
            model.forward(**b1)
    audit_clean(model, run, f'validation / inference, {order}')


# ---------------------------------------------------------------------------------------------------------- adversarial schedules
class SpinInjector:
    """torch.cuda._sleep before every ABI call of lane `target` ('side' / 'main') and one long sleep at its first call after the fork,
    or (target 'copy') one long sleep before the key-frame upload on the copy stream.  Records a timing event after every call per lane
    and, at the meeting point (_phase_tail), which lane finished last."""

    def __init__(self, model, target, long_cycles, small_cycles=2000):
        self.model, self.e, self.target, self.long, self.small = model, model.eng, target, int(long_cycles), small_cycles
        self.first, self.last, self.meet = {}, {}, []
        self.on = True
        self.reset()

    def lane(self, handle):
        e = self.e
        if e._side is not None and handle == e._side.cuda_stream:
            return 'side'
        cs = torch.cuda.graph.default_capture_stream
        if cs is not None and handle == cs.cuda_stream:
            return 'side' if e.lane == 1 else 'main'
        return 'main'

    def reset(self):
        self.side_started = self.long_done = False

    def before(self, name, args):
        lane = self.lane(args[-1].value or 0)
        if lane == 'side':
            self.side_started = True
        if self.on and lane == self.target:
            if not self.long_done and self.side_started:                # the first call of the lane after the fork
                torch.cuda._sleep(self.long)
                self.long_done = True
            torch.cuda._sleep(self.small)
        if lane not in self.first and not torch.cuda.is_current_stream_capturing():
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.first[lane] = ev

    def after(self, name, args):
        if not torch.cuda.is_current_stream_capturing():
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.last[self.lane(args[-1].value or 0)] = ev

    def install(self, mp):
        import thinktwice_b200.encoder_decoder_framework as fw
        inj = self
        A.install_abi(mp, self.before, self.after)
        for m in ('_device_forward', '_pipelined_forward', '_capture_pipeline'):
            orig = getattr(fw.EncoderDecoder, m)

            def wrapped(model, *a, _orig=orig, **k):
                inj.reset()
                return _orig(model, *a, **k)
            mp.setattr(fw.EncoderDecoder, m, wrapped)
        tail = fw.EncoderDecoder._phase_tail

        def phase_tail(model, *a, **k):
            if not torch.cuda.is_current_stream_capturing():
                inj.meet.append((inj.last.get('main'), inj.last.get('side')))
            return tail(model, *a, **k)
        mp.setattr(fw.EncoderDecoder, '_phase_tail', phase_tail)
        sweep = fw.EncoderDecoder._stage_sweep

        def stage_sweep(model, img, t):
            if inj.on and inj.target == 'copy' and inj.e._copy is not None and torch.cuda.current_stream() == inj.e._copy:
                torch.cuda._sleep(inj.long)
            return sweep(model, img, t)
        mp.setattr(fw.EncoderDecoder, '_stage_sweep', stage_sweep)


def calibrate():
    """GPU cycles of torch.cuda._sleep per millisecond, from CUDA events."""
    torch.cuda._sleep(1000)
    n = 20_000_000
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    torch.cuda._sleep(n)
    b.record()
    b.synchronize()
    return n / a.elapsed_time(b)


def outputs(model, pred):
    out = {k: pred[k].clone() for k in OUT_KEYS}
    out['cam_bev'] = model.last_cam_feat['bev'].nchw().clone()
    out['lidar.out.at'] = model.eng.static_named('lidar.out.at').clone()
    return out


@pytest.fixture(scope='module')
def adversarial(full):
    """inputs, the serial outputs, the sleep calibration and the lane times of an unperturbed overlapped run."""
    for k in ('one-stream B=2 independent=False', 'one graph', 'pipelined full B=2 graph=False', 'pipelined full B=2 graph=True'):
        if k not in AUDITED:
            pytest.skip(f'the audit "{k}" has not passed in this session: no perturbed schedule is run')
    cfg, model = full
    model.use_graph = False
    resident = frames(cfg, 2, (71, 72), 40000)
    pinned = frames(cfg, 2, (71, 72), 40000, 'pinned')
    model.eng.overlap = False
    try:
        serial = [outputs(model, model.forward_inference(b)) for b in resident]
    finally:
        model.eng.overlap = True
    torch.cuda.synchronize()
    per_ms = calibrate()
    lanes = {}
    with pytest.MonkeyPatch.context() as mp:
        A.distinct_streams(mp, model.eng)
        inj = SpinInjector(model, None, 0)
        inj.on = False
        inj.install(mp)
        model.forward_inference(resident[0])
        torch.cuda.synchronize()
        for lane in ('main', 'side'):
            lanes[lane] = inj.first[lane].elapsed_time(inj.last[lane])
    print(f'\n{torch.cuda.get_device_name()}: torch.cuda._sleep runs {per_ms / 1e6:.3f} Gcycles per second; lane times of the B=2 '
          f'overlapped forward: main {lanes["main"]:.2f} ms, side {lanes["side"]:.2f} ms')
    return dict(model=model, resident=resident, pinned=pinned, serial=serial, per_ms=per_ms, lanes=lanes)


MODES = [(form, target, graph) for form, targets in (('one-stream', ('side', 'main')), ('pipelined', ('side', 'main', 'copy')))
         for target in targets for graph in (False, True)]


@pytest.mark.parametrize('form,target,graph', MODES)
def test_adversarial_schedule_matches_the_serial_run(adversarial, form, target, graph):
    S = adversarial
    model = S['model']
    other = 'side' if target == 'main' else 'main'
    long_ms = 2 * S['lanes'][other]
    inputs = S['resident'] if form == 'one-stream' else S['pinned']
    got, ticks, replay_ms = [], [], []
    if graph:
        model.enable_cuda_graph()
    try:
        with pytest.MonkeyPatch.context() as mp:
            A.distinct_streams(mp, model.eng)
            inj = SpinInjector(model, target, long_ms * S['per_ms'])
            inj.install(mp)
            for i, b in enumerate(inputs):
                model._pipe_trace = [] if form == 'pipelined' else None
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                pred = model.forward_inference(b)
                t1.record()
                got.append(outputs(model, pred))
                torch.cuda.synchronize()
                replay_ms.append(t0.elapsed_time(t1))
                if form == 'pipelined':
                    ticks.append({lab: ev for lab, ev, _ in model._pipe_trace})
    finally:
        model._pipe_trace = None
        model.use_graph = False
    # the schedule moved: the delayed lane finished after the other one where they meet
    if form == 'pipelined':
        late, early = {'side': ('lidar_done', 'key_sweep_done'), 'main': ('key_sweep_done', 'lidar_done'),
                       'copy': ('key_uploaded', 'history_sweeps_done')}[target]
        for t in ticks:
            lag = t['start'].elapsed_time(t[late]) - t['start'].elapsed_time(t[early])
            print(f'[{form} delay {target} graph={graph}] long sleep {long_ms:.2f} ms; {late} {lag:.2f} ms after {early}')
            assert lag > 0, (late, early, lag)
    elif not graph:
        for main_ev, side_ev in inj.meet:
            d, o = (side_ev, main_ev) if target == 'side' else (main_ev, side_ev)
            lag = o.elapsed_time(d)
            print(f'[{form} delay {target}] long sleep {long_ms:.2f} ms; the {target} lane finished {lag:.2f} ms after the {other} lane')
            assert lag > 0, lag
    else:                                                              # inside one graph: the replay carries the long sleep
        print(f'[{form} delay {target} graph] long sleep {long_ms:.2f} ms; replay {replay_ms[1]:.2f} ms')
        assert replay_ms[1] > long_ms
    for i, (g, want) in enumerate(zip(got, S['serial'])):
        for k, v in want.items():
            err = relerr(g[k], v)
            assert err < TOL, (i, k, err)
