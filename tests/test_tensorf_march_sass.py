"""CPU: the box march's TensoRF kernels -- pass A with a TensoRF density (k_march_density_fwd<BoxSampler, -1 / -4>), the backward's
second launch (k_march_box_tensorf_scatter<1 / 4>), its closing launch and the points-writing pass B (k_march_box_points) --
compile for sm_90a without local-memory spills and with no stack frame."""
import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT

CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
KERNELS = {'march.cu': [r'k_march_density_fwdINS_10BoxSamplerELin1E', r'k_march_density_fwdINS_10BoxSamplerELin4E',
                        r'k_march_box_tensorf_scatterILi1E', r'k_march_box_tensorf_scatterILi4E', r'k_tensorf_bwd_finish'],
           'march_ndc.cu': [r'k_march_box_points']}


def _nvcc():
    from unboundednerfpytorch_b200 import build
    try:
        return build._nvcc()
    except RuntimeError:
        return None


def _cuobjdump():
    return shutil.which('cuobjdump') or ('/usr/local/cuda/bin/cuobjdump' if os.path.exists('/usr/local/cuda/bin/cuobjdump') else None)


@pytest.mark.skipif(_nvcc() is None or _cuobjdump() is None, reason='needs nvcc and cuobjdump')
@pytest.mark.parametrize('source', sorted(KERNELS))
def test_tensorf_march_kernels_have_no_spills(tmp_path, source):
    from unboundednerfpytorch_b200 import build
    cubin = tmp_path / 'k.cubin'
    flags = [f for f in build.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC', '-fvisibility=hidden', '--cudart', 'static')]
    res = subprocess.run([_nvcc(), '-cubin', os.path.join(CSRC, source), '-o', str(cubin), '-Xptxas', '-v'] + flags,
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    sass = subprocess.run([_cuobjdump(), '-sass', str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, body = part.split('\n', 1)
        funcs[name.strip()] = body
    log = res.stdout + res.stderr
    for pat in KERNELS[source]:
        names = [n for n in funcs if re.search(pat, n)]
        assert len(names) == 1, (pat, sorted(funcs))
        name = names[0]
        assert not re.search(r'\b(LDL|STL)\b', funcs[name]), f'{name}: local-memory access'
        m = re.search(r'Function properties for ' + re.escape(name) + r'\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                      r'(\d+) bytes spill loads', log)
        assert m and m.groups() == ('0', '0', '0'), f'{name}: {m.groups() if m else log[-2000:]}'
