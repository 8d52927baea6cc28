"""CPU: the 9-channel pass-B kernels compile for sm_90a without local-memory spills.

* k_march_feature_narrow<9, P> / k_march_feature_bwd_narrow<9, P> (the contracted march, P in {1, 3, 5, 7, 9, 11}): no stack frame
  at P = 1; at P > 1 only the 32-byte frame of libdevice sinf's large-argument path, as the C = 3 / 15 instantiations.
* k_march_ndc_feature<BoxSampler, 9, *> (the box march): no spills; the forward has no stack frame, and the scatter the same frame
  as the NDC march's 9-channel scatter, whose red_add_record<9> it shares (the run-time channel index of that loop keeps the
  36-byte record in local memory)."""
import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT

CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
SINF_FRAME = 32


def _nvcc():
    from unboundednerfpytorch_b200 import build
    try:
        return build._nvcc()
    except RuntimeError:
        return None


def _cuobjdump():
    return shutil.which('cuobjdump') or ('/usr/local/cuda/bin/cuobjdump' if os.path.exists('/usr/local/cuda/bin/cuobjdump') else None)


def _compile(tmp_path, source):
    """(SASS by function name, {function name: (stack frame, spill stores, spill loads)}) of one source file."""
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
    props = {}
    for m in re.finditer(r'Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                         r'(\d+) bytes spill loads', log):
        props[m.group(1)] = tuple(int(v) for v in m.groups()[1:])
    return funcs, props


def _one(funcs, pat):
    names = [n for n in funcs if re.search(pat, n)]
    assert len(names) == 1, (pat, sorted(funcs))
    return names[0]


needs_toolkit = pytest.mark.skipif(_nvcc() is None or _cuobjdump() is None, reason='needs nvcc and cuobjdump')


@needs_toolkit
def test_contracted_c9_kernels_have_no_spills(tmp_path):
    funcs, props = _compile(tmp_path, 'march_feature.cu')
    for P in (1, 3, 5, 7, 9, 11):
        for kind in ('k_march_feature_narrow', 'k_march_feature_bwd_narrow'):
            name = _one(funcs, rf'{len(kind)}{kind}ILi9ELi{P}E')
            frame, stores, loads = props[name]
            assert (stores, loads) == (0, 0), f'{kind}<9, {P}>: spills {props[name]}'
            if P == 1:
                assert frame == 0, f'{kind}<9, 1>: {frame}-byte stack frame'
                assert not re.search(r'\b(LDL|STL)\b', funcs[name]), f'{kind}<9, 1>: local-memory access'
            else:
                assert frame == SINF_FRAME, f'{kind}<9, {P}>: {frame}-byte stack frame (sinf needs {SINF_FRAME})'


@needs_toolkit
def test_box_c9_kernels_have_no_spills(tmp_path):
    funcs, props = _compile(tmp_path, 'march_ndc.cu')
    fwd = _one(funcs, r'k_march_ndc_featureINS_10BoxSamplerELi9ELb0E')
    bwd = _one(funcs, r'k_march_ndc_featureINS_10BoxSamplerELi9ELb1E')
    ndc_bwd = _one(funcs, r'k_march_ndc_featureINS_10NdcSamplerELi9ELb1E')
    assert props[fwd] == (0, 0, 0), props[fwd]
    assert not re.search(r'\b(LDL|STL)\b', funcs[fwd]), 'box C = 9 gather: local-memory access'
    assert props[bwd][1:] == (0, 0), props[bwd]
    assert props[bwd][0] == props[ndc_bwd][0], (props[bwd], props[ndc_bwd])
