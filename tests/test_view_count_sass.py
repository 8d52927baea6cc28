"""CPU: the contracted view-count scatter (k_view_scatter_ones_contracted, grid_utils.cu) compiles for sm_90a without
local-memory spills and with no stack frame, and sends each (x, y) edge of a cell out through the 64-bit vector reduction."""
import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT

CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
KERNEL = r'k_view_scatter_ones_contracted'


def _nvcc():
    from unboundednerfpytorch_b200 import build
    try:
        return build._nvcc()
    except RuntimeError:
        return None


def _cuobjdump():
    return shutil.which('cuobjdump') or ('/usr/local/cuda/bin/cuobjdump' if os.path.exists('/usr/local/cuda/bin/cuobjdump') else None)


@pytest.mark.skipif(_nvcc() is None or _cuobjdump() is None, reason='needs nvcc and cuobjdump')
def test_view_scatter_ones_contracted_has_no_spills(tmp_path):
    from unboundednerfpytorch_b200 import build
    cubin = tmp_path / 'k.cubin'
    flags = [f for f in build.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC', '-fvisibility=hidden', '--cudart', 'static')]
    res = subprocess.run([_nvcc(), '-cubin', os.path.join(CSRC, 'grid_utils.cu'), '-o', str(cubin), '-Xptxas', '-v'] + flags,
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    sass = subprocess.run([_cuobjdump(), '-sass', str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, body = part.split('\n', 1)
        funcs[name.strip()] = body
    names = [n for n in funcs if re.search(KERNEL, n)]
    assert len(names) == 1, sorted(funcs)
    name = names[0]
    body = funcs[name]
    assert not re.search(r'\b(LDL|STL)\b', body), f'{name}: local-memory access'
    assert re.search(r'\bREDG?\.E\.ADD\.F32x2\b', body), f'{name}: no vector reduction in the scatter'
    log = res.stdout + res.stderr
    m = re.search(r'Function properties for ' + re.escape(name) + r'\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                  r'(\d+) bytes spill loads', log)
    assert m and m.groups() == ('0', '0', '0'), f'{name}: {m.groups() if m else log[-2000:]}'
