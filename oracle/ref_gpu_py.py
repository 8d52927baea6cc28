"""oracle/ref_gpu_py.py -- TEST INFRASTRUCTURE ONLY: the reference's GPU path in Python.

Imports the reference's UNMODIFIED Python files, staged by __graft_entry__.build() into git-ignored oracle/_ref/py/FourierGrid/,
as a package of their own (``_ref_gpu_FourierGrid``) whose bare-name extension modules (render_utils_cuda, total_variation_cuda,
adam_upd_cuda, ub360_utils_cuda) are the reference's OWN CUDA extension built into oracle/_ref/*.so.  The two un-vendored
third-party packages the files import are pure-torch stand-ins here (torch_scatter.segment_coo / scatter_add as ATen index_add,
torch_efficient_distloss.flatten_eff_distloss as oracle/cpu_ref.py restates it).  So a model from this package runs the
reference's GPU path op for op: ATen grid_sample / cuBLAS / index_add plus the reference's kernels, none of this library's.

The package is separate from the ``FourierGrid`` package that tests import over ``legacy.install()`` (this library behind the same
bare names), so both can live in one process.  Models of these files allocate with the default tensor type, as
run_FourierGrid.py:87 sets it to CUDA; callers do the same (``default_cuda``)."""
import importlib
import importlib.util
import os
import sys
import types
import warnings

import torch

from oracle.cpu_ref import flatten_eff_distloss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, 'oracle', '_ref')
PY = os.path.join(REF, 'py', 'FourierGrid')
PKG = '_ref_gpu_FourierGrid'
EXTENSIONS = ('render_utils_cuda', 'total_variation_cuda', 'adam_upd_cuda', 'ub360_utils_cuda')

_cache = None


def missing():
    """None when everything is in place, else what is missing."""
    for n in EXTENSIONS:
        if not os.path.exists(os.path.join(REF, f'{n}.so')):
            return f'oracle/_ref/{n}.so'
    if not os.path.exists(os.path.join(PY, 'dmpigo.py')):
        return 'oracle/_ref/py/FourierGrid/dmpigo.py'
    return None


def _extension(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, f'{name}.so'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _segment_coo(src, index, out=None, dim_size=None, reduce='sum'):
    assert reduce == 'sum'
    if out is None:
        out = torch.zeros((dim_size if dim_size is not None else int(index.max()) + 1, *src.shape[1:]), dtype=src.dtype,
                          device=src.device)
    return out.index_add_(0, index, src)


def _scatter_add(src, index, dim=0, out=None, dim_size=None):
    assert dim == 0
    return _segment_coo(src, index, out, dim_size)


def load():
    """-> namespace(dmpigo, masked_adam, flatten_eff_distloss) of the reference's GPU path; raises if oracle/_ref is incomplete."""
    global _cache
    if _cache is not None:
        return _cache
    why = missing()
    if why is not None:
        raise FileNotFoundError(f'{why} is missing (built by __graft_entry__.build() where the reference checkout exists)')
    ts = types.ModuleType('torch_scatter')
    ts.segment_coo, ts.scatter_add = _segment_coo, _scatter_add
    td = types.ModuleType('torch_efficient_distloss')
    td.flatten_eff_distloss = flatten_eff_distloss
    bare = {n: _extension(n) for n in EXTENSIONS}
    bare.update(torch_scatter=ts, torch_efficient_distloss=td)
    saved = {k: sys.modules.get(k) for k in bare}
    sys.modules.update(bare)                 # bound by the staged files at import time, then restored
    try:
        spec = importlib.util.spec_from_file_location(PKG, os.path.join(PY, '__init__.py'), submodule_search_locations=[PY])
        pkg = importlib.util.module_from_spec(spec)
        sys.modules[PKG] = pkg
        spec.loader.exec_module(pkg)
        dmpigo = importlib.import_module(PKG + '.dmpigo')
        masked_adam = importlib.import_module(PKG + '.masked_adam')
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    _cache = types.SimpleNamespace(dmpigo=dmpigo, masked_adam=masked_adam, flatten_eff_distloss=flatten_eff_distloss)
    return _cache


def default_cuda(on, device='cuda:0'):
    """run_FourierGrid.py:87 `torch.set_default_tensor_type('torch.cuda.FloatTensor')` (deprecated in torch 2.x, still there)."""
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        try:
            torch.set_default_tensor_type('torch.cuda.FloatTensor' if on else 'torch.FloatTensor')
        except Exception:
            torch.set_default_device(device if on else 'cpu')
