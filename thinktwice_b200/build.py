"""In-tree build of libtt_b200.so (nvcc, sm_90a only).  Used by __graft_entry__.build()."""
import glob
import hashlib
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libtt_b200.so')
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr']


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, 'rb') as f:
            h.update(f.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    srcs = sorted(glob.glob(os.path.join(CSRC, '*.cu')))
    deps = srcs + glob.glob(os.path.join(CSRC, '*.cuh')) + [os.path.join(HERE, '..', 'include', 'tt_b200.h')]
    stamp = os.path.join(HERE, 'build', 'stamp')
    dig = _digest(deps)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    os.makedirs(os.path.join(HERE, 'build'), exist_ok=True)
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    objs, procs = [], []
    for s in srcs:
        o = os.path.join(HERE, 'build', os.path.basename(s)[:-3] + '.o')
        objs.append(o)
        cmd = [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', s, '-o', o]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            print(' '.join(cmd)); print(out)
        if p.returncode:
            raise RuntimeError('nvcc failed: ' + ' '.join(cmd))
    cmd = [nvcc, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', LIB] + objs
    subprocess.check_call(cmd)
    with open(stamp, 'w') as f:
        f.write(dig)
    return LIB


if __name__ == '__main__':
    import sys
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
