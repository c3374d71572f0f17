"""A happens-before audit of the multi-stream forward — TEST HARNESS ONLY.

`Recorder` (installed with `install()`) records one or more forwards as a trace of
  * storage accesses: every pointer of every C ABI call, attributed to its storage and classified read / write by the `const` of its
    parameter (or struct field) in include/tt_b200.h, on the stream whose handle the call was given; and every aten op on a CUDA tensor
    (a TorchDispatchMode: uploads, fills, clones, temporaries), writes from the schema's alias_info, on the current stream;
  * ordering edges: torch.cuda.Event.record / wait (Stream.wait_event and wait_stream go through them), torch.cuda.synchronize,
    Event.synchronize, Stream.synchronize;
  * caching-allocator blocks the forward allocates (with their stream) and record_stream calls.
A CUDA graph's capture is audited as it is recorded (its fork / join events are the graph's dependencies); a replay re-issues the accesses
the capture recorded, on the replay stream.

`analyse(trace)` keeps a vector clock per stream (no implicit ordering between streams: torch's streams are non-blocking) and reports
  (a) unordered conflicts: two accesses to one storage from different streams, at least one a write, neither happening before the other;
  (b) allocator hazards: a block allocated during the trace and used on a stream other than its allocation stream without record_stream
      (arena buffers of the engine excepted: they live as long as the engine).
The result depends only on the launch sequence, not on how the GPU happened to schedule it.  `analyse(trace, drop=...)` re-analyses a
recorded clean trace with some of its waits deleted: the negative controls of tests/test_stream_order_gpu.py.
"""
import ctypes as C
import linecache
import os
import re
import sys
from bisect import bisect_right
from collections import defaultdict

import torch
import torch.utils._python_dispatch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'tt_b200.h')
PKG = os.path.join(ROOT, 'thinktwice_b200') + os.sep
NOT_KERNELS = {'tt_version', 'tt_last_error', 'tt_launch_count', 'tt_debug_set'}
PHASES = ('_phase_lidar', '_phase_history', '_phase_key', '_phase_tail', '_stage_sweep', 'stage', 'stage_mats', '_own', 'fresh',
          'forward_train', 'get_fusion_feat', '_device_forward', '_pipelined_forward', '_capture_pipeline', 'forward_inference')


class AuditError(AssertionError):
    pass


# ---------------------------------------------------------------------------------------------------------- the header
def parse_header(path=HEADER):
    """(prototypes, structs).  prototypes: entry -> [(parameter, kind)]; structs: name -> {field: kind}.  kind of a parameter / field:
    'r' = pointer to const (read), 'w' = pointer to non-const (written; a `void*` workspace too), ('struct', name, 'r' | 'w') = pointer
    to a struct of the header, 'rr' = pointer to const pointers (read), 'stream' = the tt_stream_t, None = a value."""
    text = open(path).read()
    text = re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)
    text = re.sub(r'//[^\n]*', ' ', text)
    structs = {}
    for body, name in re.findall(r'typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;', text, flags=re.S):
        fields = {}
        for decl in body.split(';'):
            decl = ' '.join(decl.split())
            if not decl:
                continue
            if '*' in decl:
                fields[re.findall(r'(\w+)\s*$', decl)[0]] = 'r' if decl.startswith('const ') else 'w'
            else:
                typ, _, names = decl.partition(' ')
                while names.split(' ', 1)[0] in ('long', 'int', 'char', 'short'):   # multi-word types
                    names = names.split(' ', 1)[1]
                for nm in names.split(','):
                    fields[re.sub(r'\[.*', '', nm).strip()] = None
        structs[name] = fields
    protos = {}
    for name, params in re.findall(r'\b(tt_\w+)\s*\(([^()]*)\)\s*;', text):
        out = []
        params = ' '.join(params.split())
        if params != 'void':
            for p in params.split(','):
                p = p.strip()
                pname = re.findall(r'(\w+)\s*$', p)[0]
                typ = p[:-len(pname)].strip()
                base = typ.replace('const', '').replace('*', '').strip()
                if base == 'tt_stream_t':
                    kind = 'stream'
                elif typ.count('*') >= 2:
                    kind = 'rr' if typ.startswith('const ') else 'w'
                elif '*' in typ and base in structs:
                    kind = ('struct', base, 'r' if typ.startswith('const ') else 'w')
                elif '*' in typ:
                    kind = 'r' if typ.startswith('const ') else 'w'
                else:
                    kind = None
                out.append((pname, kind))
        protos[name] = out
    return protos, structs


_HEADER = None


def header():
    global _HEADER
    if _HEADER is None:
        _HEADER = parse_header()
    return _HEADER


# ---------------------------------------------------------------------------------------------------------- the trace
class Access:
    __slots__ = ('stream', 'key', 'write', 'what', 'where', 'seq')

    def __init__(self, stream, key, write, what, where):
        self.stream, self.key, self.write, self.what, self.where = stream, key, write, what, where


class Record:
    __slots__ = ('event', 'stream', 'where')

    def __init__(self, event, stream, where=None):
        self.event, self.stream, self.where = event, stream, where


class Wait:
    __slots__ = ('stream', 'event', 'where')

    def __init__(self, stream, event, where=None):
        self.stream, self.event, self.where = stream, event, where


class HostSync:
    """the host waits: scope 'device' (torch.cuda.synchronize, a capture's end), ('stream', s) or ('event', e)."""
    __slots__ = ('scope', 'where')

    def __init__(self, scope, where=None):
        self.scope, self.where = scope, where


class Alloc:
    __slots__ = ('key', 'stream', 'what', 'where')

    def __init__(self, key, stream, what='', where=None):
        self.key, self.stream, self.what, self.where = key, stream, what, where


class RecordStream:
    __slots__ = ('key', 'stream')

    def __init__(self, key, stream):
        self.key, self.stream = key, stream


class Where:
    """where an op was issued: forward index, framework phase, and the product frames (innermost first) as (function, source line)."""
    __slots__ = ('fwd', 'phase', 'frames')

    def __init__(self, fwd=0, phase='', frames=()):
        self.fwd, self.phase, self.frames = fwd, phase, tuple(frames)

    def has(self, function, code):
        return any(f == function and c == code for f, c in self.frames)

    def __str__(self):
        top = ' < '.join(f'{f}: {c}' for f, c in self.frames[:2]) if self.frames else 'test code'
        return f'forward {self.fwd}, {self.phase or "-"}, {top}'


def _join(a, b):
    for k, v in b.items():
        if a.get(k, 0) < v:
            a[k] = v


class Finding:
    def __init__(self, kind, key, a, b=None, text=''):
        self.kind, self.key, self.a, self.b, self.text = kind, key, a, b, text
        self.name = '?'

    def __str__(self):
        return self.text.replace('%NAME%', self.name)


def analyse(trace, drop=None, roles=None, arena=frozenset()):
    """findings of a trace (a list of the op objects above).  drop(op) -> True deletes that Wait.  roles: stream -> role name for the
    messages; arena: storage keys exempt from the allocator rule."""
    roles = roles or {}
    role = lambda s: roles.get(s, f'stream {s}')
    vc = {}                              # stream -> {stream: ops of that stream that happen before its next op}
    host = {}                            # what the host has seen complete
    events = {}                          # event -> clock of its latest record
    hist = defaultdict(lambda: defaultdict(lambda: ([], [])))   # key -> stream -> (seq list, accesses)
    alloc, used, rs = {}, defaultdict(set), defaultdict(set)
    findings, seen = [], set()

    def clock(s):
        c = vc.get(s)
        if c is None:
            c = vc[s] = {}
        _join(c, host)
        return c

    for op in trace:
        if isinstance(op, Access):
            c = clock(op.stream)
            c[op.stream] = c.get(op.stream, 0) + 1
            op.seq = c[op.stream]
            used[op.key].add(op.stream)
            for s, (seqs, accs) in hist[op.key].items():
                if s == op.stream:
                    continue
                for a in accs[bisect_right(seqs, c.get(s, 0)):]:        # the accesses of s that do not happen before op
                    if not (a.write or op.write):
                        continue
                    sig = (op.key, a.what, op.what, a.where.fwd if a.where else 0, op.where.fwd if op.where else 0)
                    if sig in seen:
                        continue
                    seen.add(sig)
                    rw = lambda x: 'writes' if x.write else 'reads'
                    findings.append(Finding('conflict', op.key, a, op, (
                        f'unordered conflict on %NAME%: {a.what} {rw(a)} it on {role(a.stream)} ({a.where}) and {op.what} {rw(op)} it on '
                        f'{role(op.stream)} ({op.where}); neither happens before the other')))
            seqs, accs = hist[op.key][op.stream]
            seqs.append(op.seq)
            accs.append(op)
        elif isinstance(op, Record):
            events[op.event] = dict(clock(op.stream))
        elif isinstance(op, Wait):
            if drop is not None and drop(op):
                continue
            _join(clock(op.stream), events.get(op.event, {}))
        elif isinstance(op, HostSync):
            if op.scope == 'device':
                for c in vc.values():
                    _join(host, c)
            elif op.scope[0] == 'stream':
                _join(host, vc.get(op.scope[1], {}))
            else:
                _join(host, events.get(op.scope[1], {}))
        elif isinstance(op, Alloc):
            alloc[op.key] = op
            used.pop(op.key, None)
            rs.pop(op.key, None)
        elif isinstance(op, RecordStream):
            rs[op.key].add(op.stream)
    for key, a in alloc.items():
        if key in arena:
            continue
        other = used.get(key, set()) - {a.stream} - rs.get(key, set())
        if other:
            findings.append(Finding('allocator', key, a, None, (
                f'allocator hazard on %NAME%: allocated by {a.what} on {role(a.stream)} ({a.where}), used on '
                f'{", ".join(sorted(role(s) for s in other))} without record_stream')))
    return findings


# ---------------------------------------------------------------------------------------------------------- recording
def _storage(t):
    s = t.untyped_storage()
    return s.data_ptr(), s.nbytes()


class Recorder:
    """eng: the product's Engine (stream roles, buffer names, arena).  main: the stream the test launches the forward on."""

    def __init__(self, eng, main):
        self.eng, self.main = eng, main
        self.trace = []
        self.gen = defaultdict(int)              # storage address -> allocations seen at that address (a key is (address, generation))
        self.table = {}                          # device address handed out by lib._p -> storage key
        self.roles = {main.cuda_stream: 'main'}
        self.unknown = []                        # ABI calls / ops on a stream of no known role
        self.fwd, self._depth = 0, 0
        self.capturing = None                    # list collecting the accesses of the graph being captured
        self.graphs = {}                         # id(CUDAGraph) -> its accesses
        self.events = {}                         # id(event) -> a small int (events die and ids are reused: keep them alive)
        self._keep = []
        self.active = False
        self.ops = defaultdict(int)

    # ------------------------------------------------------------------ naming
    def role(self, handle):
        handle = int(handle or 0)
        r = self.roles.get(handle)
        if r is None or r == 'main':
            e = self.eng
            streams = (('main', self.main), ('side', e._side), ('copy', e._copy), ('capture', torch.cuda.graph.default_capture_stream))
            names = [n for n, st in streams if st is not None and st.cuda_stream == handle]
            if len(names) > 1:
                # torch hands out pooled streams round robin, so two torch.cuda.Stream() objects can be one CUDA stream: the lanes would
                # run serialised and the audit could not tell them apart (distinct_streams() sets up a recording without that)
                raise AuditError(f'the {" and ".join(names)} streams are one CUDA stream ({handle:#x})')
            if names:
                self.roles[handle] = r = names[0]
        return r

    def stream_of(self, handle, what):
        handle = int(handle or 0)
        if self.role(handle) is None and self.active:
            self.unknown.append(f'{what} on stream handle {handle:#x} ({"NULL: the legacy default stream" if not handle else "no known role"}) '
                                f'at {self.where()}')
        return handle

    def key(self, t):
        ptr, _ = _storage(t)
        return (ptr, self.gen[ptr])

    def where(self):
        frames, phase = [], ''
        f = sys._getframe(2)
        while f is not None:
            fn = f.f_code.co_filename
            if fn.startswith(PKG):
                frames.append((f.f_code.co_name, linecache.getline(fn, f.f_lineno).split('#')[0].strip()))
                if not phase and f.f_code.co_name in PHASES:
                    phase = f.f_code.co_name
            f = f.f_back
        return Where(self.fwd, phase, frames)

    def arena(self):
        """storage key -> engine buffer name, for the buffers the engine owns now."""
        e, names = self.eng, {}
        for k, b in e.bufs.items():
            names[self.key(b)] = k[0] if k[0] != 'late#s' else 'late split companion'
        for lane, b in e._scratch.items():
            names[self.key(b)] = f'scratch[lane {lane}]'
        for lane, b in e.conv_ws.items():
            names[self.key(b)] = f'conv workspace[lane {lane}]'
        for b in e._ws_retired:
            names.setdefault(self.key(b), 'retired workspace')
        return names

    def _lookup(self, addr):
        """a device address not handed out by lib._p (a host array of device pointers): the engine buffer that contains it."""
        for b in list(self.eng.bufs.values()) + list(self.eng._scratch.values()):
            ptr, n = _storage(b)
            if ptr <= addr < ptr + n:
                return (ptr, self.gen[ptr])
        return None

    def resolve(self, addr, what):
        if not addr:
            return None
        k = self.table.get(addr)
        if k is None:
            k = self._lookup(addr)
        if k is None:
            raise AuditError(f'{what}: device pointer {addr:#x} was not handed out by lib._p and lies in no engine buffer')
        return k

    # ------------------------------------------------------------------ events
    def add(self, op):
        if self.active:
            self.trace.append(op)
            self.ops[type(op).__name__] += 1
            if self.capturing is not None and isinstance(op, Access):
                self.capturing.append(op)

    def ev(self, event):
        i = self.events.get(id(event))
        if i is None:
            i = self.events[id(event)] = len(self.events)
            self._keep.append(event)
        return i

    def abi(self, name, args):
        """the accesses of one C ABI call."""
        protos, structs = header()
        params = protos.get(name)
        if params is None:
            raise AuditError(f'{name}: no prototype in include/tt_b200.h')
        if len(params) != len(args):
            raise AuditError(f'{name}: {len(args)} arguments, the prototype has {len(params)}')
        s = args[-1]
        handle = s.value if isinstance(s, C.c_void_p) else s
        stream = self.stream_of(handle, name)
        where = self.where()
        acc = []

        def ptr(v, what, kind):
            addr = v.value if isinstance(v, C.c_void_p) else v
            if isinstance(addr, int) or addr is None:
                k = self.resolve(addr, what)
                if k is not None:
                    acc.append(Access(stream, k, kind == 'w', what, where))
            else:
                raise AuditError(f'{what}: a pointer argument of type {type(v).__name__}')

        for (pname, kind), v in zip(params, args):
            what = f'{name}.{pname}'
            if kind in ('r', 'w'):
                if type(v).__name__ == 'CArgObject':                    # byref of a host value (tt_f16s_saturation_count's out_host)
                    continue
                ptr(v, what, kind)
            elif kind == 'rr':
                for i, p in enumerate(v):
                    ptr(p, f'{what}[{i}]', 'r')
            elif isinstance(kind, tuple):
                sname = kind[1]
                fields = [(f, k) for f, k in structs[sname].items() if k is not None]
                if not fields:
                    continue
                objs = list(v) if isinstance(v, C.Array) else [getattr(v, '_obj', v)]
                for o in objs:
                    for f, k in fields:
                        ptr(getattr(o, f), f'{what}.{f}', k)
        for a in acc:
            self.add(a)
        if name == 'tt_f16s_saturation_count':                         # reads a device counter back: the host waits for the stream
            self.add(HostSync(('stream', stream), where))

    def aten(self, func, args, kwargs, out):
        schema = func._schema
        rets = schema.returns
        if rets and all(r.alias_info is not None and not r.alias_info.is_write for r in rets):
            return                                                     # a view: no data is touched
        stream = None
        where = None
        tensors_in = []
        host_out = False
        ins = set()
        for i, a in enumerate(schema.arguments):
            v = args[i] if i < len(args) else kwargs.get(a.name, None)
            vals = v if isinstance(v, (list, tuple)) else [v]
            for t in vals:
                if isinstance(t, torch.Tensor) and t.is_cuda and t.untyped_storage().nbytes():
                    w = a.alias_info is not None and a.alias_info.is_write
                    tensors_in.append((t, w, a.name))
                    ins.add(_storage(t)[0])
                elif isinstance(t, torch.Tensor) and not t.is_cuda and w_is(a):
                    host_out = True
        if func is torch.ops.aten._local_scalar_dense.default:
            host_out = True                                            # .item(): the host reads the value
        outs = out if isinstance(out, (list, tuple)) else [out]
        fresh = []
        for t in outs:
            if isinstance(t, torch.Tensor):
                if t.is_cuda and t.untyped_storage().nbytes() and _storage(t)[0] not in ins:
                    fresh.append(t)
                elif not t.is_cuda and tensors_in:
                    host_out = True
        if not tensors_in and not fresh:
            return
        stream = self.stream_of(torch.cuda.current_stream().cuda_stream, str(func))
        where = self.where()
        name = str(func).replace('aten.', '').replace('.default', '')
        for t in fresh:
            ptr = _storage(t)[0]
            self.gen[ptr] += 1
            k = (ptr, self.gen[ptr])
            self.add(Alloc(k, stream, name, where))
            if not name.startswith('empty'):
                self.add(Access(stream, k, True, name, where))
        for t, w, an in tensors_in:
            self.add(Access(stream, self.key(t), w, f'{name}({an})', where))
        if host_out and tensors_in:                                    # device -> host (.item(), .cpu()): the host waits for the stream
            self.add(HostSync(('stream', stream), where))


def w_is(a):
    return a.alias_info is not None and a.alias_info.is_write


class _Mode(torch.utils._python_dispatch.TorchDispatchMode):
    def __init__(self, rec):
        super().__init__()
        self.rec = rec

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        rec = self.rec
        if func is torch.ops.aten.record_stream.default:
            t, s = args
            if rec.active:
                rec.trace.append(RecordStream(rec.key(t), int(s.cuda_stream)))
            return func(*args, **kwargs)
        out = func(*args, **kwargs)
        if rec.active:
            rec.aten(func, args, kwargs, out)
        return out


class _Proxy:
    def __init__(self, real, before, after):
        self._real, self._before, self._after, self._cache = real, before, after, {}

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if not name.startswith('tt_') or name in NOT_KERNELS or name.endswith('_workspace_bytes'):
            return fn
        if name not in self._cache:
            before, after = self._before, self._after

            def call(*args):
                before(name, args)
                rc = fn(*args)
                if after is not None:
                    after(name, args)
                return rc
            self._cache[name] = call
        return self._cache[name]


def install_abi(monkeypatch, before, after=None):
    """route every kernel entry of the C ABI through before(name, args) and after(name, args) around the real entry."""
    from thinktwice_b200 import lib
    real = lib.load()
    monkeypatch.setattr(lib, 'load', lambda: _Proxy(real, before, after))
    return real


def distinct_streams(monkeypatch, eng):
    """give the engine's side and copy streams, torch's graph capture stream and a new main stream four different CUDA streams (torch's
    pooled streams repeat after a while, so separately created Stream objects may share one); returns the main stream."""
    taken = set()

    def fresh():
        for _ in range(256):
            s = torch.cuda.Stream()
            if s.cuda_stream not in taken:
                taken.add(s.cuda_stream)
                return s
        raise AuditError('torch hands out fewer than four distinct CUDA streams')
    eng._side, eng._copy = fresh(), fresh()
    monkeypatch.setattr(torch.cuda.graph, 'default_capture_stream', fresh())
    return fresh()


def install(monkeypatch, rec):
    """record every ABI call, aten op and ordering edge into `rec` (rec.active switches recording on); returns the dispatch mode to
    enter around the recorded forwards."""
    from thinktwice_b200 import lib
    import thinktwice_b200.encoder_decoder_framework as fw
    import thinktwice_b200.engine as engine
    import thinktwice_b200.lidarnet as lidarnet
    import thinktwice_b200.lss as lss
    import thinktwice_b200.preprocess as pre
    import thinktwice_b200.thinktwice_decoder as dec
    install_abi(monkeypatch, lambda name, args: rec.abi(name, args) if rec.active else None)
    orig_p = lib._p

    def _p(t, off=0):
        r = orig_p(t, off)
        if t is not None and r.value:
            rec.table[r.value] = rec.key(t)
        return r
    monkeypatch.setattr(lib, '_p', _p)
    for mod in (engine, lss, lidarnet, dec, fw, pre):
        monkeypatch.setattr(mod, '_p', _p, raising=False)

    E, S = torch.cuda.Event, torch.cuda.Stream
    ev_record, ev_wait, ev_sync, st_sync, dev_sync = E.record, E.wait, E.synchronize, S.synchronize, torch.cuda.synchronize

    def record(self, stream=None):
        s = stream if stream is not None else torch.cuda.current_stream()
        rec.add(Record(rec.ev(self), rec.stream_of(s.cuda_stream, 'Event.record'), rec.where() if rec.active else None))
        return ev_record(self, stream)

    def wait(self, stream=None):
        s = stream if stream is not None else torch.cuda.current_stream()
        rec.add(Wait(rec.stream_of(s.cuda_stream, 'Event.wait'), rec.ev(self), rec.where() if rec.active else None))
        return ev_wait(self, stream)

    def event_sync(self):
        rec.add(HostSync(('event', rec.ev(self))))
        return ev_sync(self)

    def stream_sync(self):
        rec.add(HostSync(('stream', int(self.cuda_stream))))
        return st_sync(self)

    def device_sync(device=None):
        rec.add(HostSync('device'))
        return dev_sync(device)
    monkeypatch.setattr(E, 'record', record)
    monkeypatch.setattr(E, 'wait', wait)
    monkeypatch.setattr(E, 'synchronize', event_sync)
    monkeypatch.setattr(S, 'synchronize', stream_sync)
    monkeypatch.setattr(torch.cuda, 'synchronize', device_sync)

    # CUDA graphs: the capture is audited as recorded, then ends like a host sync (captured work never runs by itself); a replay re-issues
    # the captured accesses on the replay stream
    G = torch.cuda.graph
    g_enter, g_exit, replay = G.__enter__, G.__exit__, torch.cuda.CUDAGraph.replay

    def enter(self):
        r = g_enter(self)
        rec.capturing = rec.graphs[id(self.cuda_graph)] = []
        rec._keep.append(self.cuda_graph)
        return r

    def exit_(self, *exc):
        r = g_exit(self, *exc)
        rec.capturing = None
        rec.add(HostSync('device'))
        return r

    def replay_(self):
        accs = rec.graphs.get(id(self))
        if accs is None:
            raise AuditError('replay of a graph captured outside the audit')
        s = rec.stream_of(torch.cuda.current_stream().cuda_stream, 'CUDAGraph.replay')
        where = rec.where()
        for a in accs:
            rec.add(Access(s, a.key, a.write, f'{a.what} (graph replay)', where))
        return replay(self)
    monkeypatch.setattr(G, '__enter__', enter)
    monkeypatch.setattr(G, '__exit__', exit_)
    monkeypatch.setattr(torch.cuda.CUDAGraph, 'replay', replay_)

    def counted(fn):
        def forward(model, *a, **k):
            rec._depth += 1
            if rec._depth == 1:
                rec.fwd += 1
            try:
                return fn(model, *a, **k)
            finally:
                rec._depth -= 1
        return forward
    for m in ('forward_inference', 'forward_train'):
        monkeypatch.setattr(fw.EncoderDecoder, m, counted(getattr(fw.EncoderDecoder, m)))
    return _Mode(rec)


def report(rec, findings):
    """the findings with buffer names, and the table of the storages each lane touched."""
    names = rec.arena()
    roles = {h: r for h, r in rec.roles.items()}
    for f in findings:
        f.name = names.get(f.key, f'a storage outside the arena ({f.key[0]:#x})')
    lanes = defaultdict(lambda: defaultdict(str))                     # storage -> role -> 'r' / 'w' / 'rw'
    for op in rec.trace:
        if isinstance(op, Access) and not op.what.endswith('(graph replay)'):   # a replay runs the captured lanes on one stream
            r = roles.get(op.stream, '?')
            m = lanes[op.key][r]
            c = 'w' if op.write else 'r'
            if c not in m:
                lanes[op.key][r] = ''.join(sorted(m + c))
    per = defaultdict(lambda: [0, 0])
    shared = []
    for k, rr in lanes.items():
        for r in rr:
            per[r][0] += 1
        if len({'main' if r == 'capture' else r for r in rr}) > 1:    # a graph's capture stream is the main lane of that graph
            shared.append((names.get(k, f'outside the arena {k[0]:#x}'), dict(rr)))
    lines = ['lane       storages', *[f'{r:10s} {n:8d}' for r, (n, _) in sorted(per.items())],
             f'storages touched by more than one lane ({len(shared)}; the capture stream counts as main):']
    for n, rr in sorted(shared):
        lines.append(f'  {n:40s} ' + '  '.join(f'{r}:{m}' for r, m in sorted(rr.items())))
    return lines


def audit(rec, drop=None):
    """(findings, report lines) of a recording."""
    names = rec.arena()
    findings = analyse(rec.trace, drop=drop, roles=rec.roles, arena=frozenset(names))
    lines = report(rec, findings)
    return findings, lines
