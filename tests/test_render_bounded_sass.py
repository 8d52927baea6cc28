"""CPU: the fused render kernels of DirectVoxGO and DirectMPIGO (k_render_box / k_render_ndc, csrc/render_bounded.cu) compile for
sm_90a without local-memory spills, within the registers their CTA size allows.  The sigmoid and viewbase_pe 0 instances have no
stack frame at all (no sinf / cosf; the NDC act_shift grid is read at its one slab); the viewbase_pe 4 instances carry only the
32-byte frame of libdevice's sinf / cosf (the view embedding), whose large-argument path is the only code that touches local
memory."""
import os
import re
import subprocess

import pytest

from tests.test_render_fused_sass import _cuobjdump, _nvcc
from tests.util import ROOT

CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
# (kernel, C, viewbase_pe, rgbnet, width, warps per CTA)
INSTANCES = [('box', 12, 4, 1, 128, 12), ('box', 9, 4, 1, 64, 16), ('box', 3, 0, 0, 128, 12),
             ('ndc', 9, 0, 1, 64, 16), ('ndc', 3, 0, 0, 128, 12)]


@pytest.mark.skipif(_nvcc() is None or _cuobjdump() is None, reason='needs nvcc and cuobjdump')
def test_bounded_render_kernels_have_no_spills(tmp_path):
    from unboundednerfpytorch_b200 import build
    cubin = tmp_path / 'k.cubin'
    flags = [f for f in build.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC', '-fvisibility=hidden', '--cudart', 'static')]
    res = subprocess.run([_nvcc(), '-cubin', os.path.join(CSRC, 'render_bounded.cu'), '-o', str(cubin), '-Xptxas', '-v'] + flags,
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    log = res.stdout + res.stderr
    sass = subprocess.run([_cuobjdump(), '-sass', str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, body = part.split('\n', 1)
        funcs[name.strip()] = body
    assert len(funcs) == len(INSTANCES), sorted(funcs)
    for kind, C, pe, net, width, warps in INSTANCES:
        name = f'_ZN3ubn3rnd12k_render_{kind}ILi{C}ELi{pe}ELb{net}ELi{width}EEEvNS0_4ArgsE'
        assert name in funcs, (name, sorted(funcs))
        m = re.search(r'Function properties for ' + re.escape(name) + r'\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                      r'(\d+) bytes spill loads\s*\n\s*ptxas info\s*: Used (\d+) registers', log)
        assert m, log[-2000:]
        frame, st, ld, regs = map(int, m.groups())
        assert (st, ld) == (0, 0), f'{name}: spills {st} / {ld}'
        assert regs * 32 * warps <= 65536, f'{name}: {regs} registers do not fit {warps} warps per SM'
        if not net or pe == 0:
            assert frame == 0 and not re.search(r'\b(LDL|STL)\b', funcs[name]), f'{name}: stack frame {frame}'
        else:
            assert frame <= 32, f'{name}: stack frame {frame}'
