"""Build libubnerf_b200.so (hand-written sm_90a CUDA + the C ABI of include/ubnerf_b200.h) in-tree.

    python -m unboundednerfpytorch_b200.build [--force]

nvcc cross-compiles without a GPU.  The library links the CUDA runtime statically and has no torch /
Python dependency: it is the drop-in boundary (INTEGRATION.md).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libubnerf_b200.so')
SOURCES = ['ray_ops.cu', 'alpha_ops.cu', 'grid_sweep.cu', 'trilinear.cu', 'march.cu', 'march_feature.cu', 'march_ndc.cu', 'shade.cu', 'shade_tc.cu', 'ray_gen.cu', 'loss.cu', 'grid_utils.cu', 'render_tma.cu', 'tensorf.cu', 'bounds.cu']
HEADERS = ['common.cuh', 'trilinear.cuh', 'march_common.cuh', 'ray_gen.cuh', 'tensorf.cuh', os.path.join('..', '..', 'include', 'ubnerf_b200.h')]
NVCC_FLAGS = ['-std=c++17', '-O3', '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo',
              '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden', '--cudart', 'static']


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.sep not in cand or os.path.exists(cand)):
            return cand
    raise RuntimeError('nvcc not found')


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every .cu of the package for sm_90a into one shared object. Returns its path."""
    if not (force or _stale()):
        return LIB
    objdir = os.path.join(HERE, 'build')
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    procs = []
    for s in SOURCES:
        obj = os.path.join(objdir, s.replace('.cu', '.o'))
        cmd = [nvcc, '-c', os.path.join(CSRC, s), '-o', obj] + NVCC_FLAGS
        if verbose:
            cmd += ['-Xptxas', '-v']
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True), obj))
    objs = []
    for s, p, obj in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError(f'nvcc failed on {s}')
        objs.append(obj)
    cmd = [nvcc, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '--cudart', 'static']
    subprocess.check_call(cmd)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
