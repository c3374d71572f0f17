"""The happens-before analysis of tests/stream_audit.py on synthetic traces, and its reading of include/tt_b200.h: what the GPU audit
(tests/test_stream_order_gpu.py) concludes rests on these rules."""
import stream_audit as A
from stream_audit import Access, Alloc, HostSync, Record, RecordStream, Wait

MAIN, SIDE, COPY = 1, 2, 3
ROLES = {MAIN: 'main', SIDE: 'side', COPY: 'copy'}
BUF, OTHER = (100, 0), (200, 0)


def acc(stream, write, key=BUF, what=None):
    return Access(stream, key, write, what or ('write' if write else 'read') + f'@{ROLES[stream]}', A.Where())


def conflicts(trace, **kw):
    return [f for f in A.analyse(trace, roles=ROLES, **kw) if f.kind == 'conflict']


def test_a_missing_wait_is_flagged_in_both_orders():
    assert len(conflicts([acc(SIDE, True), acc(MAIN, False)])) == 1         # main reads what side wrote, no edge
    assert len(conflicts([acc(MAIN, False), acc(SIDE, True)])) == 1         # side overwrites what main still reads
    assert len(conflicts([acc(MAIN, True), acc(SIDE, True)])) == 1         # write / write
    f = conflicts([acc(SIDE, True, what='tt_conv2d.y'), acc(MAIN, False, what='tt_copy2d.src')])[0]
    f.name = 'lidar.out.at'
    assert 'lidar.out.at' in str(f) and 'tt_conv2d.y' in str(f) and 'tt_copy2d.src' in str(f) and 'side' in str(f) and 'main' in str(f)


def test_a_wait_orders_the_accesses_recorded_before_the_event():
    ok = [acc(SIDE, True), Record(0, SIDE), Wait(MAIN, 0), acc(MAIN, False)]
    assert not conflicts(ok)
    late = [Record(0, SIDE), acc(SIDE, True), Wait(MAIN, 0), acc(MAIN, False)]   # the write comes after the record
    assert len(conflicts(late)) == 1
    assert len(conflicts(ok, drop=lambda op: isinstance(op, Wait))) == 1     # the same trace with its wait deleted


def test_ordering_is_transitive_through_a_third_stream():
    trace = [acc(SIDE, True), Record(0, SIDE), Wait(COPY, 0), Record(1, COPY), Wait(MAIN, 1), acc(MAIN, True)]
    assert not conflicts(trace)
    assert len(conflicts(trace, drop=lambda op: isinstance(op, Wait) and op.stream == COPY)) == 1


def test_a_wait_orders_against_the_record_latest_when_it_was_issued():
    first = [acc(SIDE, True, key=OTHER), Record(0, SIDE), Wait(MAIN, 0), acc(SIDE, True), Record(0, SIDE), acc(MAIN, False)]
    assert len(conflicts(first)) == 1                                        # the wait was issued before the second record
    second = [acc(SIDE, True, key=OTHER), Record(0, SIDE), acc(SIDE, True), Record(0, SIDE), Wait(MAIN, 0), acc(MAIN, False)]
    assert not conflicts(second)
    assert not conflicts([Wait(MAIN, 7), acc(SIDE, True), acc(MAIN, True, key=OTHER)])   # waiting on a never-recorded event: no-op


def test_read_read_sharing_and_same_stream_reuse_pass():
    assert not conflicts([acc(SIDE, False), acc(MAIN, False), acc(COPY, False)])
    assert not conflicts([acc(MAIN, True), acc(MAIN, False), acc(MAIN, True)])
    assert not conflicts([acc(SIDE, True, key=OTHER), acc(MAIN, True)])    # different storages


def test_a_host_sync_orders_everything_issued_before_it():
    assert not conflicts([acc(SIDE, True), acc(COPY, True, key=OTHER), HostSync('device'), acc(MAIN, True), acc(MAIN, True, key=OTHER)])
    assert not conflicts([acc(SIDE, True), HostSync(('stream', SIDE)), acc(MAIN, False)])
    assert len(conflicts([acc(SIDE, True), HostSync(('stream', COPY)), acc(MAIN, False)])) == 1   # synchronised the wrong stream
    assert not conflicts([acc(SIDE, True), Record(3, SIDE), HostSync(('event', 3)), acc(MAIN, False)])
    assert len(conflicts([HostSync('device'), acc(SIDE, True), acc(MAIN, False)])) == 1          # only what came before it


def test_the_allocator_rule():
    K = (300, 1)
    hazard = [Alloc(K, MAIN, 'clone'), acc(MAIN, True, key=K), Record(0, MAIN), Wait(SIDE, 0), acc(SIDE, False, key=K)]
    f = A.analyse(hazard, roles=ROLES)
    assert [x.kind for x in f] == ['allocator'] and 'side' in str(f[0])     # ordered, but the block may be reused under side's read
    assert not A.analyse(hazard + [RecordStream(K, SIDE)], roles=ROLES)
    assert not A.analyse(hazard, roles=ROLES, arena=frozenset([K]))        # engine arena buffers live as long as the engine
    assert not A.analyse([Alloc(K, SIDE, 'empty'), acc(SIDE, True, key=K), acc(SIDE, False, key=K)], roles=ROLES)


def test_the_header_has_a_prototype_for_every_export():
    from thinktwice_b200 import lib
    protos, _ = A.parse_header()
    assert not set(lib.EXPORTS) - set(protos)
    for name in lib.EXPORTS:
        kinds = [k for _, k in protos[name]]
        if name not in ('tt_version', 'tt_last_error', 'tt_launch_count') and not name.endswith('_workspace_bytes'):
            assert kinds[-1] == 'stream', name                               # the stream is every kernel entry's last argument


def test_the_header_classifies_known_parameters():
    protos, structs = A.parse_header()
    io = structs['tt_f16s_io']
    assert io['y'] == io['y_split'] == 'w'
    assert io['x_split'] == io['w_split'] == io['bias'] == io['res'] == io['res_split'] == io['res2_split'] == 'r'
    assert io['x_plane'] is None and io['y_plane'] is None
    assert dict(protos['tt_conv2d_f16s']) == {'d': ('struct', 'tt_conv_desc', 'r'), 'io': ('struct', 'tt_f16s_io', 'r'), 'stream': 'stream'}
    conv = dict(protos['tt_conv2d'])
    assert conv['x'] == conv['w'] == conv['m_count'] == 'r' and conv['y'] == conv['workspace'] == 'w'
    assert dict(protos['tt_look_rebatch'])['mlvl'] == 'rr'
    split = dict(protos['tt_split_f16'])
    assert split['x'] == split['row_count'] == 'r' and split['y_split'] == 'w' and split['rows'] is None
    vox = dict(protos['tt_voxelize_mean'])
    assert vox['points'] == 'r' and vox['feats'] == vox['coords'] == vox['count'] == vox['workspace'] == 'w'
    assert structs['tt_loss_term']['pred'] == structs['tt_loss_term']['gt2'] == 'r'
    assert all(k is None for k in structs['tt_conv_desc'].values())


def test_two_roles_on_one_cuda_stream_fail_the_recording():
    """torch's pooled streams repeat: an engine side stream that is the recording's main stream would serialise the lanes unseen."""
    class S:
        def __init__(self, h):
            self.cuda_stream = h

    class Eng:
        _side, _copy = S(7), S(9)
    rec = A.Recorder(Eng(), S(7))
    try:
        rec.role(7)
    except A.AuditError as ex:
        assert 'main and side' in str(ex)
    else:
        raise AssertionError('aliased streams were not reported')
    assert rec.role(9) == 'copy' and rec.role(11) is None
