"""Benchmark of FourierGridModel at the k0 widths of the reference's Waymo and Tanks&Temples configs, on one GPU.  Prints one JSON
line per shape:

* waymo -- configs/waymo/waymo_no_block.py: 300^3 density and k0, fourier_freq_num 3 (P = 7), rgbnet_dim 3, viewbase_pe 2,
           contracted_norm l2, 2048 rays; loss weights main 3, entropy_last 1e-3, rgbper 1e-2, TV density 1e-6 / k0 1e-7;
* train -- configs/tankstemple_unbounded/train_single.py: 250^3, P = 7, rgbnet_dim 15, viewbase_pe 4, contracted_norm inf,
           4096 rays; loss weights main 1, entropy_last 1e-3, rgbper 1e-2, TV density 1e-6 / k0 1e-7.

Both use alpha_init 1e-4, stepsize 0.5 and fast_color_thres 5e-6 (the configs' schedule at step 0).  The Fourier-space MSE term
(weight_freq, Waymo only) and the distortion loss are not part of the timed step.  Per shape:

* train_step_ms -- one run_train.py step (forward, loss, backward, dense TV, MaskedAdam) for three legs from the same parameters:
                   ``fused`` (forward), ``forward_ops`` and ``reference_gpu`` (the reference's unmodified FourierGrid_model.py and
                   masked_adam.py, staged under oracle/_ref/py, over its own CUDA extension in oracle/_ref; an ``unavailable``
                   record when that was not built);
* kernels_ms    -- per-launch times of the fused step (CUDA events around the C-ABI calls, ``_cabi.timed``) and the rgbnet's
                   share of the step;
* outputs       -- fused vs forward_ops before the first step: survivor sets equal, max error over scale;
* gpu / power_limit_w -- where it ran, read in the same run.

    python scripts/bench_fg_widths.py [--steps 10] [--warmup 3] [--only waymo|train]
"""
import argparse
import contextlib
import importlib.util
import io
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_mpi import _gpu_info, _time  # noqa: E402

SHAPES = {
    'waymo': dict(world=300, rgbnet_dim=3, viewbase_pe=2, norm='l2', rays=2048, w_main=3.0),
    'train': dict(world=250, rgbnet_dim=15, viewbase_pe=4, norm='inf', rays=4096, w_main=1.0),
}
RK = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False)


def _kwargs(s):
    w = s['world'] ** 3
    return dict(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=w, num_voxels_base_density=w, num_voxels_rgb=w,
                num_voxels_base_rgb=w, num_voxels_viewdir=-1, alpha_init=1e-4, fast_color_thres=5e-6, rgbnet_dim=s['rgbnet_dim'],
                fourier_freq_num=3, viewbase_pe=s['viewbase_pe'], contracted_norm=s['norm'], bg_len=0.2)


def _train_step(m, opt, fwd, ro, rd, vd, target, it, w_main):
    N = len(ro)
    out = fwd(ro, rd, vd, global_step=it, is_train=True, **RK)
    opt.zero_grad(set_to_none=True)
    loss = w_main * F.mse_loss(out['rgb_marched'], target)
    pout = out['alphainv_last'].clamp(1e-6, 1 - 1e-6)
    loss = loss + 1e-3 * (-(pout * torch.log(pout) + (1 - pout) * torch.log(1 - pout)).mean())
    rgbper = (out['raw_rgb'] - target[out['ray_id']]).pow(2).sum(-1)
    loss = loss + 1e-2 * (rgbper * out['weights'].detach()).sum() / N
    loss.backward()
    m.density_total_variation_add_grad(1e-6 / N, True)
    m.k0_total_variation_add_grad(1e-7 / N, True)
    opt.step()
    return loss


def _reference():
    """The reference's FourierGrid package (oracle/_ref/py) bound to its own CUDA extension (oracle/_ref/*.so), or None."""
    from oracle import ref_gpu_py
    py = os.path.join(ROOT, 'oracle', '_ref', 'py')
    if ref_gpu_py.missing() is not None or not os.path.exists(os.path.join(py, 'FourierGrid', 'FourierGrid_model.py')):
        return None
    import types
    mods = {}
    for n in ref_gpu_py.EXTENSIONS:
        spec = importlib.util.spec_from_file_location(n, os.path.join(ROOT, 'oracle', '_ref', f'{n}.so'))
        mods[n] = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mods[n])
    ts = types.ModuleType('torch_scatter')
    ts.segment_coo, ts.scatter_add = ref_gpu_py._segment_coo, ref_gpu_py._scatter_add
    td = types.ModuleType('torch_efficient_distloss')
    td.flatten_eff_distloss = ref_gpu_py.flatten_eff_distloss
    sys.modules.update(mods, torch_scatter=ts, torch_efficient_distloss=td)
    sys.path.insert(0, py)
    from FourierGrid import FourierGrid_model, masked_adam
    return FourierGrid_model, masked_adam


def bench(name, s, args):
    import numpy as np
    from unboundednerfpytorch_b200 import _cabi, models
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    gpu, power = _gpu_info()
    res = dict(metric=f'FourierGridModel {name}: one training step', shape=dict(s, P=7), gpu=gpu, power_limit_w=power)
    g = torch.Generator().manual_seed(0)
    torch.manual_seed(0)
    m = models.FourierGridModel(**_kwargs(s))
    with torch.no_grad():
        m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=g) * 4 + 5)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
    state0 = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}
    m = m.cuda()
    n = s['rays']
    ro = (torch.rand(n, 3, generator=g) - 0.5).cuda()
    rd = torch.randn(n, 3, generator=g).cuda()
    vd = rd / rd.norm(dim=-1, keepdim=True)
    target = torch.rand(n, 3, generator=g).cuda()
    cfg = dict(lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])

    with torch.no_grad():
        a, b = m(ro, rd, vd, **RK), m.forward_ops(ro, rd, vd, **RK)
    same = torch.equal(a['ray_id'], b['ray_id']) and torch.equal(a['step_id'], b['step_id'])
    res['outputs'] = dict(survivors=int(a['ray_id'].numel()), same_survivors=bool(same),
                          **{k: ((a[k] - b[k]).abs().max() / b[k].abs().max().clamp_min(1e-30)).item()
                             for k in ('rgb_marched', 'alphainv_last') + (('weights', 'raw_rgb') if same else ())})
    del a, b

    res['train_step_ms'] = {}
    for leg in ('fused', 'forward_ops'):
        m.load_state_dict(state0)
        opt = create_optimizer_or_freeze_model(m, cfg, global_step=0)
        fwd = m.forward if leg == 'fused' else m.forward_ops
        res['train_step_ms'][leg] = _time(lambda i: _train_step(m, opt, fwd, ro, rd, vd, target, i + 1, s['w_main']),
                                          args.steps, args.warmup)
        del opt
        torch.cuda.empty_cache()

    # per-launch times of the fused step and the rgbnet's share
    m.load_state_dict(state0)
    opt = create_optimizer_or_freeze_model(m, cfg, global_step=0)
    _cabi.TIMER = _cabi.KernelTimer()
    try:
        step_ms = _time(lambda i: _train_step(m, opt, m.forward, ro, rd, vd, target, i + 1, s['w_main']), args.steps, 1)
        k = {n_: v[0] for n_, v in _cabi.TIMER.summary().items()}
    finally:
        _cabi.TIMER = None
    res['kernels_ms'] = k
    res['instrumented_step_ms'] = step_ms
    res['rgbnet_share_of_step'] = (k.get('rgbnet_fwd', 0.0) + k.get('rgbnet_bwd', 0.0)) / step_ms
    del opt
    m.cpu()
    torch.cuda.empty_cache()

    ref = _reference()
    if ref is None:
        res['train_step_ms']['reference_gpu'] = {'unavailable': 'oracle/_ref not built (needs the reference checkout at build time)'}
    else:
        fgm, madam = ref
        from oracle import ref_gpu_py
        kw = dict(_kwargs(s), xyz_min=np.array([-1.] * 3, dtype=np.float32), xyz_max=np.array([1.] * 3, dtype=np.float32))
        ref_gpu_py.default_cuda(True)           # run_FourierGrid.py:87: the reference allocates with the default tensor type
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                rm = fgm.FourierGridModel(**kw)
            rm.load_state_dict(state0, strict=False)
            rm = rm.cuda()
            ropt = madam.MaskedAdam([{'params': [rm.density.grid], 'lr': 0.1, 'skip_zero_grad': True},
                                     {'params': [rm.k0.grid], 'lr': 0.1, 'skip_zero_grad': True},
                                     {'params': list(rm.rgbnet.parameters()), 'lr': 1e-3, 'skip_zero_grad': False}])
            res['train_step_ms']['reference_gpu'] = _time(
                lambda i: _train_step(rm, ropt, rm.forward, ro, rd, vd, target, i + 1, s['w_main']), args.steps, args.warmup)
        finally:
            ref_gpu_py.default_cuda(False)
        res['speedup_vs_reference_gpu'] = res['train_step_ms']['reference_gpu'] / res['train_step_ms']['fused']
    res['speedup_vs_forward_ops'] = res['train_step_ms']['forward_ops'] / res['train_step_ms']['fused']
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--only', choices=list(SHAPES), default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_fg_widths.py needs a GPU'
    for name, s in SHAPES.items():
        if args.only in (None, name):
            print(json.dumps(bench(name, s, args)), flush=True)
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
