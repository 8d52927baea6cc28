"""The four extension modules the reference imports by bare name (grid.py:10-11, dvgo.py:13, dcvgo.py:15,
masked_adam.py:3, FourierGrid_model.py:17-18).  ``install()`` makes ``import render_utils_cuda`` etc. resolve
to this package instead of the reference's ``python setup.py install`` build (README.md:138-144).

``install_models(*modules)`` goes one step further: it points the reference modules' own names for the model classes and the
optimizer factory at this package's, so run_train.py / run_render.py / FourierGrid_ckpt_manager.py run unedited on the fused
models (INTEGRATION.md §3).  ``install_metrics(*modules)`` does the same for the evaluation score utils.rgb_ssim, and
``install_arf(*modules)`` for the stylizer class ARF of arf.py."""
import importlib
import sys

NAMES = ('render_utils_cuda', 'total_variation_cuda', 'adam_upd_cuda', 'ub360_utils_cuda')


def install():
    mods = {}
    for n in NAMES:
        m = importlib.import_module(f'unboundednerfpytorch_b200.legacy.{n}')
        sys.modules[n] = m
        mods[n] = m
    return mods


def model_names():
    """{module-level name in the reference: this package's object}.  run_train.py imports FourierGridModel by name (:10) and
    reaches the other three through the dvgo / dcvgo / dmpigo modules (:36-50, :191-196); FourierGrid_ckpt_manager.py and
    load_everything.py do the same; utils.py binds MaskedAdam and create_optimizer_or_freeze_model (:12, :26)."""
    from .. import masked_adam, models
    return {
        'FourierGridModel': models.FourierGridModel,
        'DirectVoxGO': models.DirectVoxGO,
        'DirectContractedVoxGO': models.DirectContractedVoxGO,
        'DirectMPIGO': models.DirectMPIGO,
        'MaskedAdam': masked_adam.MaskedAdam,
        'create_optimizer_or_freeze_model': masked_adam.create_optimizer_or_freeze_model,
    }


class ModelPatch:
    """What install_models / install_metrics / install_arf changed: ``restore()`` (or leaving the ``with`` block) puts every
    original name back."""

    def __init__(self, saved):
        self.saved = saved          # [(module, name, original object)]

    def restore(self):
        for module, name, original in reversed(self.saved):
            setattr(module, name, original)
        self.saved = []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.restore()
        return False


def install_models(*reference_modules):
    """In each given reference module (run_train, dvgo, dcvgo, dmpigo, FourierGrid_ckpt_manager, load_everything, utils,
    masked_adam ...), rebind every name of model_names() the module defines to this package's class or function.  Callers
    that look the names up at call time -- create_new_model, load_existing_model, the isinstance checks of run_train.py:191-196
    -- then build, load and rescale the fused models with no edit.  Returns a ModelPatch that restores the originals."""
    return _rebind(reference_modules, model_names())


def install_metrics(*reference_modules):
    """In each given reference module that defines ``rgb_ssim`` (utils.py:79-125), rebind it to metrics.rgb_ssim: same arguments,
    same result types, computed on the GPU.  run_render.render_viewpoints looks it up as ``utils.rgb_ssim`` at call time, so with
    install_metrics(utils) its ``eval_ssim`` scores on the GPU with no edit.  Returns a ModelPatch that restores the originals."""
    from .. import metrics
    return _rebind(reference_modules, {'rgb_ssim': metrics.rgb_ssim})


def install_arf(*reference_modules):
    """In each given reference module that defines ``ARF`` (arf.py:9-89; run_render.py imports it by name), rebind it to
    arf.ARF: same constructor and attributes, match_colors_for_image_set with the same result types, computed on the GPU.
    run_render.run_render builds ``ARF(cfg, data_dict, device)`` at call time, so with install_arf(run_render) its block render
    stylizes on the colour kernels with no edit.  Returns a ModelPatch that restores the originals."""
    from .. import arf
    return _rebind(reference_modules, {'ARF': arf.ARF})


def _rebind(reference_modules, table):
    saved = []
    for module in reference_modules:
        for name, ours in table.items():
            if hasattr(module, name):
                saved.append((module, name, getattr(module, name)))
                setattr(module, name, ours)
    return ModelPatch(saved)
