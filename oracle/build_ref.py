"""Build the REAL reference kernel as a checker (TEST INFRASTRUCTURE ONLY).

The reference's only native source, open_loop_training/ops/voxel_pooling/src/voxel_pooling_forward_cuda.cu,
has no torch dependency: its launcher `voxel_pooling_forward_kernel_launcher(...)` is plain C++/CUDA.  It is
compiled here straight from /root/reference (never copied) into oracle/_ref/libvoxel_pooling_ref.so (git-ignored,
travels with gpurun) so GPU tests can compare tt_voxel_pooling_forward against the reference's own code.
The reference's Python side (mmcv/mmdet3d/spconv based) cannot be built or imported in this image — see DESIGN.md.
"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = '/root/reference/open_loop_training/ops/voxel_pooling/src/voxel_pooling_forward_cuda.cu'
OUT = os.path.join(HERE, '_ref', 'libvoxel_pooling_ref.so')


def build(force=False):
    if not os.path.exists(SRC):
        if os.path.exists(OUT):
            return OUT
        raise FileNotFoundError(SRC)
    if os.path.exists(OUT) and not force and os.path.getmtime(OUT) >= max(os.path.getmtime(SRC), os.path.getmtime(__file__)):   # (flags live here)
        return OUT
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    subprocess.check_call([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-shared', '-Xcompiler', '-fPIC',
                           '-o', OUT, SRC])
    return OUT


if __name__ == '__main__':
    print(build())
