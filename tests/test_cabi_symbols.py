"""CPU: the C-ABI library builds, loads (no GPU needed for dlopen) and exports every symbol the header declares."""
import ctypes
import os
import re

from tests.util import ROOT


def _declared():
    src = open(os.path.join(ROOT, 'include', 'ubnerf_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(ubn_[a-z0-9_]+)\s*\(', src)))


def test_header_symbols_exported():
    from unboundednerfpytorch_b200 import build, _cabi
    path = build.build()
    lib = ctypes.CDLL(path)
    names = _declared()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f'{n} declared in include/ubnerf_b200.h but not exported'
    # the ctypes binding covers exactly the declared surface
    assert sorted(_cabi.exported_symbols()) == names


def test_abi_version_and_counters():
    from unboundednerfpytorch_b200 import _cabi
    lib = _cabi.load()
    assert lib.ubn_abi_version() == _cabi.ABI_VERSION == 3
    _cabi.reset_launch_count()
    assert _cabi.launch_count() == 0


def test_only_sm90a_code_in_library():
    """The shipped library carries sm_90a SASS only (no multi-arch fatbin, no PTX-JIT fallback for other GPUs)."""
    import subprocess
    from unboundednerfpytorch_b200 import build
    out = subprocess.run(['cuobjdump', '-lelf', build.build()], capture_output=True, text=True).stdout
    archs = set(re.findall(r'sm_(\d+a?)', out))
    assert archs == {'90a'}, archs
