"""CPU: every instantiation of the warpgroup-MMA rgbnet forward (k_shade_fwd_wgmma: 3xTF32 and single pass, with panel saves,
row-major saves and no saves) runs its products on HGMMA, without local-memory spills and without a stack frame, and its
registers fit 384 threads at launch (setmaxnreg then splits them between the producer and the two consumer warpgroups)."""
import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT

CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
KERNELS = tuple(f'_ZN3ubn2tc17k_shade_fwd_wgmmaILb{three}ELb{save}ELb{panel}EEE'
                for three in (1, 0) for save, panel in ((1, 1), (1, 0), (0, 0)))

# the setmaxnreg split of k_shade_fwd_wgmma (namespace fg of shade_tc.cu)
PRODUCER_REGS, CONSUMER_REGS = map(int, re.search(r'namespace fg \{.*?kProducerRegs = (\d+), kConsumerRegs = (\d+);',
                                                   open(os.path.join(CSRC, 'shade_tc.cu')).read(), re.S).groups())


def _nvcc():
    from unboundednerfpytorch_b200 import build
    try:
        return build._nvcc()
    except RuntimeError:
        return None


@pytest.mark.skipif(_nvcc() is None or shutil.which('cuobjdump') is None and not os.path.exists('/usr/local/cuda/bin/cuobjdump'),
                    reason='needs nvcc and cuobjdump')
def test_fwd_wgmma_sass_has_hgmma_and_no_spills(tmp_path):
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
        # layer 1: 2 k-steps, layer 2: 16, three products per k-step at 3xTF32
        want = 3 * 18 if 'wgmmaILb1E' in prefix else 18
        n = len(re.findall(r'\bHGMMA\.64x128x8\.F32\.TF32\b', body))
        assert n == want, f'{match[0]}: {n} HGMMA.64x128x8 instead of {want}'
        assert not re.search(r'\b(LDL|STL)\b', body), f'{match[0]}: local-memory spill'
        m = re.search(r'Function properties for ' + re.escape(prefix) + r'\S*\s*\n\s*(\d+) bytes stack frame', log)
        assert m and int(m.group(1)) == 0, f'{prefix}: stack frame in {log[-2000:]}'
        m = re.search(r'Compiling entry function \'' + re.escape(prefix) + r'[^\n]*\n(?:[^\n]*\n){0,2}?[^\n]*Used (\d+) registers', log)
        assert m and int(m.group(1)) * 384 <= 65536, f'{prefix}: registers do not fit 384 threads'
        # setmaxnreg only moves registers within the launch allotment: the consumers' increase waits until the producer's
        # decrease has freed enough, so the split must not need more than the kernel was launched with
        assert int(m.group(1)) * 384 >= 128 * PRODUCER_REGS + 256 * CONSUMER_REGS, \
            f'{prefix}: {m.group(1)} registers at launch cannot be split into {PRODUCER_REGS} / {CONSUMER_REGS}'
