"""CPU: the width-64 rgbnet kernels (k_shade_fwd_tc_w / k_shade_bwd_tc_w / k_shade_dw2_tc_w at kF = 9, kW = 64: DirectMPIGO of
llff_default) run on the tensor cores and compile without shared-memory float atomics (ATOMS.CAST compare-and-swap loops on
sm_90), without local-memory spills and with no stack frame, at the warps per CTA and CTAs per SM they are launched with."""
import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT

CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
# (kernel, the template arguments that select the default 3xTF32 instantiation: kF, kW, then kSave + kThree / kThree)
DEFAULTS = (('k_shade_fwd_tc_w', 'ILi9ELi64ELb1ELb1E'), ('k_shade_bwd_tc_w', 'ILi9ELi64ELb1E'), ('k_shade_dw2_tc_w', 'ILi64ELb1E'))


def _nvcc():
    from unboundednerfpytorch_b200 import build
    try:
        return build._nvcc()
    except RuntimeError:
        return None


def _cuobjdump():
    return shutil.which('cuobjdump') or ('/usr/local/cuda/bin/cuobjdump' if os.path.exists('/usr/local/cuda/bin/cuobjdump') else None)


@pytest.mark.skipif(_nvcc() is None or _cuobjdump() is None, reason='needs nvcc and cuobjdump')
def test_rgbnet_w64_sass_has_hmma_no_shared_cas_and_no_spills(tmp_path):
    from unboundednerfpytorch_b200 import build
    cubin = tmp_path / 'shade_tc.cubin'
    flags = [f for f in build.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC', '-fvisibility=hidden', '--cudart', 'static')]
    res = subprocess.run([_nvcc(), '-cubin', os.path.join(CSRC, 'shade_tc.cu'), '-o', str(cubin), '-Xptxas', '-v'] + flags,
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    sass = subprocess.run([_cuobjdump(), '-sass', str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, body = part.split('\n', 1)
        funcs[name.strip()] = body
    log = res.stdout + res.stderr
    w64 = [n for n in funcs if re.match(r'_ZN3ubn2tc\d+k_shade_(fwd|bwd|dw2)_tc_wI', n)]
    assert len(w64) == 8, sorted(w64)        # forward: saves x 3xTF32 / single pass; launch 1 and dW2: 3xTF32 / single pass
    for kernel, args in DEFAULTS:
        match = [n for n in w64 if n.startswith(f'_ZN3ubn2tc{len(kernel)}{kernel}{args}')]
        assert len(match) == 1, (kernel, sorted(w64))
    for name in w64:
        body = funcs[name]
        assert 'HMMA' in body, name
        assert 'ATOMS.CAST' not in body, f'{name}: shared-memory CAS loop'
        assert not re.search(r'\b(LDL|STL)\b', body), f'{name}: local-memory spill'
        m = re.search(r'Function properties for ' + re.escape(name) + r'\s*\n\s*(\d+) bytes stack frame', log)
        assert m and int(m.group(1)) == 0, f'{name}: stack frame in {log[-2000:]}'
