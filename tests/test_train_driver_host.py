"""CPU: the model surface the reference's drivers use.  Every method run_train.py / run_render.py call on ``model`` that the
reference's own model class defines exists on the matching class of ``models`` with the same parameter names -- the list is
read from the staged sources (oracle/_ref/py, written by __graft_entry__.build()) with ``ast``, not kept by hand -- and
``legacy.install_models`` rebinds the reference modules' names and puts them back."""
import ast
import inspect
import os
import types

import pytest

from tests.util import ROOT

STAGED = os.path.join(ROOT, 'oracle', '_ref', 'py', 'FourierGrid')
DRIVERS = ('run_train.py', 'run_render.py')
CLASSES = {'FourierGridModel': 'FourierGrid_model.py', 'DirectContractedVoxGO': 'dcvgo.py', 'DirectVoxGO': 'dvgo.py',
           'DirectMPIGO': 'dmpigo.py'}


def _parse(name):
    path = os.path.join(STAGED, name)
    if not os.path.exists(path):
        pytest.skip(f'{name} is not staged under oracle/_ref/py (needs a reference checkout at build time)')
    with open(path) as f:
        return ast.parse(f.read())


def _driver_calls():
    """{method name: [driver files]} of every `model.<name>(...)` call in the drivers."""
    calls = {}
    for f in DRIVERS:
        for n in ast.walk(_parse(f)):
            if (isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and isinstance(n.func.value, ast.Name)
                    and n.func.value.id == 'model'):
                calls.setdefault(n.func.attr, []).append(f)
    return calls


def _reference_methods(cls_name):
    """{method name: [parameter names]} the reference class itself defines."""
    for n in _parse(CLASSES[cls_name]).body:
        if isinstance(n, ast.ClassDef) and n.name == cls_name:
            return {m.name: [a.arg for a in m.args.args + m.args.kwonlyargs] for m in n.body if isinstance(m, ast.FunctionDef)}
    raise AssertionError(f'{cls_name} not found in the staged {CLASSES[cls_name]}')


def test_driver_calls_are_found():
    calls = _driver_calls()
    # the calls this surface was built for must be among those the parser finds, or the check below proves nothing
    for name in ('gather_training_rays', 'update_occupancy_cache_lt_nviews', 'export_geometry_for_visualize',
                 'scale_volume_grid', 'voxel_count_views', 'maskout_near_cam_vox'):
        assert name in calls, name


@pytest.mark.parametrize('cls_name', list(CLASSES))
def test_every_driver_call_exists_on_the_fused_class(cls_name):
    from unboundednerfpytorch_b200 import models
    ours = getattr(models, cls_name)
    ref = _reference_methods(cls_name)
    calls = _driver_calls()
    checked = []
    for name in sorted(calls):
        if name not in ref:          # nn.Module's own (to, state_dict) or a method the reference class lacks as well
            continue
        assert hasattr(ours, name), f'{cls_name}.{name} (called by {calls[name]}) is missing'
        params = list(inspect.signature(getattr(ours, name)).parameters)
        assert params[1:len(ref[name])] == ref[name][1:], (cls_name, name, params, ref[name])
        checked.append(name)
    assert checked


def test_install_models_patches_and_restores():
    from unboundednerfpytorch_b200 import legacy, masked_adam, models
    run_train = types.ModuleType('run_train')
    run_train.FourierGridModel = ref_fg = object()
    run_train.unrelated = 'kept'
    dcvgo = types.ModuleType('dcvgo')
    dcvgo.DirectContractedVoxGO = ref_dc = object()
    utils = types.ModuleType('utils')
    utils.create_optimizer_or_freeze_model = ref_opt = object()
    utils.MaskedAdam = ref_adam = object()
    patch = legacy.install_models(run_train, dcvgo, utils)
    assert run_train.FourierGridModel is models.FourierGridModel
    assert dcvgo.DirectContractedVoxGO is models.DirectContractedVoxGO
    assert not hasattr(dcvgo, 'DirectVoxGO')                 # only names a module defines are touched
    assert utils.create_optimizer_or_freeze_model is masked_adam.create_optimizer_or_freeze_model
    assert utils.MaskedAdam is masked_adam.MaskedAdam
    assert run_train.unrelated == 'kept'
    patch.restore()
    assert (run_train.FourierGridModel, dcvgo.DirectContractedVoxGO) == (ref_fg, ref_dc)
    assert (utils.create_optimizer_or_freeze_model, utils.MaskedAdam) == (ref_opt, ref_adam)
    with legacy.install_models(dcvgo):
        assert dcvgo.DirectContractedVoxGO is models.DirectContractedVoxGO
    assert dcvgo.DirectContractedVoxGO is ref_dc


def test_optimizer_factory_takes_the_reference_verbose_keyword():
    import torch
    from unboundednerfpytorch_b200 import masked_adam
    model = torch.nn.Module()
    model.density = torch.nn.Parameter(torch.zeros(3))
    cfg = {'lrate_decay': 20, 'lrate_density': 0.1, 'skip_zero_grad_fields': []}
    opt = masked_adam.create_optimizer_or_freeze_model(model, cfg, global_step=0, verbose=True)
    assert len(opt.param_groups) == 1 and opt.param_groups[0]['lr'] == pytest.approx(0.1)
