"""CPU: both instantiations of the warpgroup-MMA dW2 kernel (k_shade_dw2_wgmma, 3xTF32 and single pass) run their products on
HGMMA, without local-memory spills and without a stack frame (the producer / consumer register split of setmaxnreg must fit)."""
import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT

CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
KERNELS = ('_ZN3ubn2tc17k_shade_dw2_wgmmaILb1EEE', '_ZN3ubn2tc17k_shade_dw2_wgmmaILb0EEE')


def _nvcc():
    from unboundednerfpytorch_b200 import build
    try:
        return build._nvcc()
    except RuntimeError:
        return None


@pytest.mark.skipif(_nvcc() is None or shutil.which('cuobjdump') is None and not os.path.exists('/usr/local/cuda/bin/cuobjdump'),
                    reason='needs nvcc and cuobjdump')
def test_dw2_wgmma_sass_has_hgmma_and_no_spills(tmp_path):
    from unboundednerfpytorch_b200 import build
    cubin = tmp_path / 'shade_tc.cubin'
    flags = [f for f in build.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC', '-fvisibility=hidden', '--cudart', 'static')]
    res = subprocess.run([_nvcc(), '-cubin', os.path.join(CSRC, 'shade_tc.cu'), '-o', str(cubin), '-Xptxas', '-v'] + flags,
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    sass = subprocess.run([cuobjdump, '-sass', str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, body = part.split('\n', 1)
        funcs[name.strip()] = body
    log = res.stdout + res.stderr
    for prefix in KERNELS:
        match = [n for n in funcs if n.startswith(prefix)]
        assert len(match) == 1, (prefix, sorted(funcs))
        body = funcs[match[0]]
        assert 'HGMMA' in body, f'{match[0]}: no warpgroup MMA'
        assert not re.search(r'\b(LDL|STL)\b', body), f'{match[0]}: local-memory spill'
        m = re.search(r'Function properties for ' + re.escape(prefix) + r'\S*\s*\n\s*(\d+) bytes stack frame', log)
        assert m and int(m.group(1)) == 0, f'{prefix}: stack frame in {log[-2000:]}'
        m = re.search(r'Compiling entry function \'' + re.escape(prefix) + r'[^\n]*\n(?:[^\n]*\n){0,2}?[^\n]*Used (\d+) registers', log)
        assert m and int(m.group(1)) * 384 <= 65536, f'{prefix}: registers do not fit 384 threads'
