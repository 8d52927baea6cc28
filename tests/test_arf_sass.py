"""CPU: the colour-transfer kernels of csrc/color.cu (ubn_color_moments, ubn_color_affine) compile for sm_90a with no stack
frame, no spills and no local-memory access (ptxas -v, cuobjdump -sass)."""
import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT


def _tools():
    from unboundednerfpytorch_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        return None, None
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    return nvcc, (cuobjdump if os.path.exists(cuobjdump) else None)


@pytest.mark.skipif(None in _tools(), reason='needs nvcc and cuobjdump')
def test_color_kernels_have_no_spills_or_stack(tmp_path):
    from unboundednerfpytorch_b200 import build
    nvcc, cuobjdump = _tools()
    flags = [f for f in build.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC', '-fvisibility=hidden', '--cudart', 'static')]
    cubin = tmp_path / 'color.cubin'
    res = subprocess.run([nvcc, '-cubin', os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc', 'color.cu'), '-o', str(cubin),
                          '-Xptxas', '-v'] + flags, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    assert 'warning' not in log.lower(), log
    props = dict((m.group(1), tuple(int(v) for v in m.groups()[1:])) for m in re.finditer(
        r'Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', log))
    names = sorted(props)
    assert len(names) == 4 and all(re.search(r'k_color_(moments|moments_close|affine|affine_scalar)E', n) for n in names), names
    for name, sizes in props.items():
        assert sizes == (0, 0, 0), (name, sizes)
    sass = subprocess.run([cuobjdump, '-sass', str(cubin)], capture_output=True, text=True, check=True).stdout
    assert not re.search(r'\b(LDL|STL)\b', sass), 'local-memory access in color.cu'
