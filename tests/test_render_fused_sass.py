"""CPU: the fused render kernels (k_render_contracted, csrc/render.cu) compile for sm_90a without local-memory spills.  The sigmoid
kernel has no stack frame at all; the rgbnet kernels carry only the 32-byte frame of libdevice's sinf / cosf (the view embedding),
whose large-argument path is the only code that touches local memory."""
import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT

CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
# (C, viewbase_pe, rgbnet)
INSTANCES = [(12, 4, 1), (3, 8, 1), (3, 0, 0)]

def _nvcc():
    from unboundednerfpytorch_b200 import build
    try:
        return build._nvcc()
    except RuntimeError:
        return None


def _cuobjdump():
    return shutil.which('cuobjdump') or ('/usr/local/cuda/bin/cuobjdump' if os.path.exists('/usr/local/cuda/bin/cuobjdump') else None)


@pytest.mark.skipif(_nvcc() is None or _cuobjdump() is None, reason='needs nvcc and cuobjdump')
def test_render_kernels_have_no_spills(tmp_path):
    from unboundednerfpytorch_b200 import build
    cubin = tmp_path / 'k.cubin'
    flags = [f for f in build.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC', '-fvisibility=hidden', '--cudart', 'static')]
    res = subprocess.run([_nvcc(), '-cubin', os.path.join(CSRC, 'render.cu'), '-o', str(cubin), '-Xptxas', '-v'] + flags,
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    log = res.stdout + res.stderr
    sass = subprocess.run([_cuobjdump(), '-sass', str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, body = part.split('\n', 1)
        funcs[name.strip()] = body
    for C, pe, net in INSTANCES:
        name = f'_ZN3ubn3rnd19k_render_contractedILi{C}ELi{pe}ELb{net}EEEvNS0_4ArgsE'
        assert name in funcs, (name, sorted(funcs))
        m = re.search(r'Function properties for ' + re.escape(name) + r'\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                      r'(\d+) bytes spill loads', log)
        assert m, log[-2000:]
        frame, st, ld = map(int, m.groups())
        assert (st, ld) == (0, 0), f'{name}: spills {st} / {ld}'
        if not net:
            assert frame == 0 and not re.search(r'\b(LDL|STL)\b', funcs[name]), f'{name}: stack frame {frame}'
        else:
            assert frame <= 32, f'{name}: stack frame {frame}'
