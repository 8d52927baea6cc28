"""CPU: the fused Fourier-slab render (k_render_fourier<P>, csrc/render_fourier.cu) compiles for sm_90a at every slab count it takes
without local-memory spills and within one CTA of 12 warps per SM (168 registers).  Its only stack frame is the 32 bytes of
libdevice's sinf / cosf slow path (the large-argument range reduction of the view embedding and the Fourier coordinates, the only
code that touches local memory), the frame render.cu's rgbnet kernels carry too."""
import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT

CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
SLOW_PATH_FRAME = 32          # bytes, measured: libdevice's trig slow path


def _nvcc():
    from unboundednerfpytorch_b200 import build
    try:
        return build._nvcc()
    except RuntimeError:
        return None


def _cuobjdump():
    return shutil.which('cuobjdump') or ('/usr/local/cuda/bin/cuobjdump' if os.path.exists('/usr/local/cuda/bin/cuobjdump') else None)


@pytest.mark.skipif(_nvcc() is None or _cuobjdump() is None, reason='needs nvcc and cuobjdump')
def test_render_fourier_has_no_spills_and_fits_12_warps(tmp_path):
    from unboundednerfpytorch_b200 import build
    cubin = tmp_path / 'k.cubin'
    flags = [f for f in build.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC', '-fvisibility=hidden', '--cudart', 'static')]
    res = subprocess.run([_nvcc(), '-cubin', os.path.join(CSRC, 'render_fourier.cu'), '-o', str(cubin), '-Xptxas', '-v'] + flags,
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    log = res.stdout + res.stderr
    sass = subprocess.run([_cuobjdump(), '-sass', str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, body = part.split('\n', 1)
        funcs[name.strip()] = body
    for P in (7, 9, 11):
        name = f'_ZN3ubn3rfo16k_render_fourierILi{P}EEEvNS_3rnd4ArgsE'
        assert name in funcs, (name, sorted(funcs))
        m = re.search(r'Function properties for ' + re.escape(name) + r'\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                      r'(\d+) bytes spill loads', log)
        assert m, log[-2000:]
        frame, st, ld = map(int, m.groups())
        assert (st, ld) == (0, 0), f'P={P}: spills {st} / {ld}'
        assert frame <= SLOW_PATH_FRAME, f'P={P}: stack frame {frame}'
        m = re.search(r'Compiling entry function \'' + re.escape(name) + r'[^\n]*\n(?:[^\n]*\n){0,2}?[^\n]*Used (\d+) registers', log)
        assert m and int(m.group(1)) * 32 * 12 <= 65536, f'P={P}: registers do not fit 12 warps'
        assert re.search(r'\bHMMA\.1688\.F32\.TF32\b', funcs[name]), f'P={P}: the rgbnet is not on the tensor cores'
