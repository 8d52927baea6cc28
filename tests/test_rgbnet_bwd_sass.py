"""CPU: the default instantiations of the rgbnet backward (k_shade_bwd_tc 3xTF32 / 8 warps / panel saves / ReLU masks, and
k_shade_dw2_tc 3xTF32 / panel / masks) compile without shared-memory float atomics -- sm_90 has no native shared fp32 add, so
those become ATOMS.CAST compare-and-swap loops that serialise the warps of a CTA -- and without local-memory spills."""
import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT

CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
DEFAULTS = ('_ZN3ubn2tc14k_shade_bwd_tcILb1ELi8ELb1ELb1ELb0EEE', '_ZN3ubn2tc14k_shade_dw2_tcILb1ELb1ELb1EEE')


def _nvcc():
    from unboundednerfpytorch_b200 import build
    try:
        return build._nvcc()
    except RuntimeError:
        return None


@pytest.mark.skipif(_nvcc() is None or shutil.which('cuobjdump') is None and not os.path.exists('/usr/local/cuda/bin/cuobjdump'),
                    reason='needs nvcc and cuobjdump')
def test_rgbnet_backward_sass_has_no_shared_cas_and_no_spills(tmp_path):
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
    for prefix in DEFAULTS:
        match = [n for n in funcs if n.startswith(prefix)]
        assert len(match) == 1, (prefix, sorted(funcs))
        body = funcs[match[0]]
        assert 'HMMA' in body
        assert 'ATOMS.CAST' not in body, f'{match[0]}: shared-memory CAS loop'
        assert not re.search(r'\b(LDL|STL)\b', body), f'{match[0]}: local-memory spill'
    # ptxas: no stack frame for either kernel
    log = res.stdout + res.stderr
    for prefix in DEFAULTS:
        m = re.search(r'Function properties for ' + re.escape(prefix) + r'\S*\s*\n\s*(\d+) bytes stack frame', log)
        assert m and int(m.group(1)) == 0, f'{prefix}: stack frame in {log[-2000:]}'
