"""Benchmark of the forward-facing model DirectMPIGO at llff_default sizes (configs/llff/llff_default.py: 256^3-voxel budget,
mpi_depth 128, stepsize 0.5 -> 255 samples per ray, rgbnet_dim 9 / width 64, fast_color_thres 1e-3) on one GPU.  Prints one JSON
line:

* train_step_ms   -- one run_train.py:251-288 step with LLFF's fine-stage weights (forward, mse + entropy_last + distortion +
                     rgbper, backward, TV, MaskedAdam) on 4096 rays: the fused march (``fused``), the op-by-op composition
                     (``forward_ops``) and the reference's GPU path (``reference_gpu``: the reference's unmodified dmpigo.py and
                     masked_adam.py over its own CUDA extension, oracle/ref_gpu_py.py; an ``unavailable`` record when oracle/_ref
                     was not built); every leg starts from the same parameters;
* render_frame_ms -- one 1008x756 frame (762,048 rays) in 8192-ray chunks through the fused forward;
* kernels_ms      -- per-launch times of the march kernels, and the rgbnet's forward and backward time and share of the fused
                     step (CUDA events around the C-ABI calls -- ``rgbnet_fwd`` / ``rgbnet_bwd`` of the tensor-core rgbnet, the
                     per-ray bias GEMM outside them -- or, on the torch rgbnet, module hooks around it; a separate pass);
* legs            -- with ``--rgbnet kernel,torch``: the fused step, the rgbnet times and share and the frame time of each rgbnet
                     path (``torch``: shade.supported patched to False, so DirectMPIGO runs its nn.Sequential on cuBLAS), the
                     legs alternating --runs times in this one process after the top-level figures, which are always
                     those of the shipped path;
* march_hbm       -- algorithmic bytes of the march kernels (32 B density + 8 B act_shift + 1 B mask per queried sample in pass A,
                     8 x 36 B per survivor in pass B, doubled for the scatter) over their time, against 3.35 TB/s;
* outputs         -- fused vs forward_ops at the timed size (max error over scale, survivor sets equal);
* gpu / power_limit_w -- where it ran, read in the same run.

    python scripts/bench_mpi.py [--steps 20] [--warmup 5] [--rays 4096] [--rgbnet kernel,torch] [--runs 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12          # H100 SXM data sheet


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def _scene(n_rays, seed=0):
    from unboundednerfpytorch_b200 import models
    g = torch.Generator().manual_seed(seed)
    m = models.DirectMPIGO(xyz_min=[-1.4, -1.1, -1.], xyz_max=[1.4, 1.1, 1.], num_voxels=256 ** 3, mpi_depth=128,
                           rgbnet_dim=9, rgbnet_width=64, fast_color_thres=1e-3)
    with torch.no_grad():
        m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=g) * 3 - 1)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
        m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=g) < 0.9)

    def rays(n):
        ro = torch.cat([(torch.rand(n, 2, generator=g) - 0.5) * 2.6, -torch.ones(n, 1)], -1)
        rd = torch.cat([torch.randn(n, 2, generator=g) * 0.3, 2.0 + torch.randn(n, 1, generator=g) * 0.02], -1)
        return ro.cuda(), rd.cuda(), (rd / rd.norm(dim=-1, keepdim=True)).cuda()
    return m.cuda(), rays


RK = dict(near=0., far=1., bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False)


def _train_step(m, opt, fwd, ro, rd, vd, target, it, distloss=None):
    """run_train.py:251-288 with configs/llff/llff_default.py over configs/default.py (fine stage): weight_entropy_last 1e-3,
    weight_distortion 1e-2, weight_rgbper 1e-2, weight_tv_density 1e-5, weight_tv_k0 1e-6 (dense TV)."""
    if distloss is None:
        from unboundednerfpytorch_b200.functional import flatten_eff_distloss as distloss
    N = len(ro)
    out = fwd(ro, rd, vd, global_step=it, **RK)
    opt.zero_grad(set_to_none=True)
    loss = F.mse_loss(out['rgb_marched'], target)
    pout = out['alphainv_last'].clamp(1e-6, 1 - 1e-6)
    loss = loss + 1e-3 * (-(pout * torch.log(pout) + (1 - pout) * torch.log(1 - pout)).mean())      # weight_entropy_last
    loss = loss + 1e-2 * distloss(out['weights'], out['s'], 1 / out['n_max'], out['ray_id'])   # weight_distortion
    rgbper = (out['raw_rgb'] - target[out['ray_id']]).pow(2).sum(-1)
    loss = loss + 1e-2 * (rgbper * out['weights'].detach()).sum() / N                                    # weight_rgbper
    loss.backward()
    m.density_total_variation_add_grad(1e-5 / N, True)          # llff weight_tv_density (fine stage)
    m.k0_total_variation_add_grad(1e-6 / N, True)
    opt.step()
    return loss


def _time(fn, steps, warmup):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        fn(warmup + i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def _reference_gpu_leg(m, state0, ro, rd, vd, target, args):
    """The same step on the reference's GPU path, from the same parameters; ms per step, or an unavailable record."""
    from oracle import ref_gpu_py
    why = ref_gpu_py.missing()
    if why is not None:
        return {'unavailable': f'{why} not built (needs the reference checkout at build time)'}
    ns = ref_gpu_py.load()
    kw = {k: v for k, v in m.get_kwargs().items() if k != 'voxel_size_ratio'}
    ref_gpu_py.default_cuda(True)            # run_FourierGrid.py:87: the reference allocates with the default tensor type
    try:
        import contextlib
        import io
        with contextlib.redirect_stdout(io.StringIO()):
            ref = ns.dmpigo.DirectMPIGO(**kw)
        ref.load_state_dict(state0, strict=True)
        ref = ref.cuda()
        opt = ns.masked_adam.MaskedAdam([{'params': [ref.density.grid], 'lr': 0.1, 'skip_zero_grad': True},
                                         {'params': [ref.k0.grid], 'lr': 0.1, 'skip_zero_grad': True},
                                         {'params': list(ref.rgbnet.parameters()), 'lr': 1e-3, 'skip_zero_grad': False}])
        ms = _time(lambda i: _train_step(ref, opt, ref.forward, ro, rd, vd, target, i + 1, ns.flatten_eff_distloss),
                   args.steps, args.warmup)
    finally:
        ref_gpu_py.default_cuda(False)
    del ref, opt
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rays', type=int, default=4096)
    ap.add_argument('--rgbnet', default='kernel', help="comma-separated rgbnet paths to time in alternation: kernel, torch")
    ap.add_argument('--runs', type=int, default=2, help='alternating runs of each --rgbnet path')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_mpi.py needs a GPU'
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    name, power = _gpu_info()
    res = dict(metric='llff_default DirectMPIGO', gpu=name, power_limit_w=power, rays=args.rays)
    cfg = dict(lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])

    m, rays = _scene(args.rays)
    ro, rd, vd = rays(args.rays)
    target = torch.rand(args.rays, 3, device='cuda')
    state0 = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}

    # outputs: fused vs forward_ops at the timed size (before any step changes the grids)
    with torch.no_grad():
        a = m(ro, rd, vd, **RK, render_depth=True)
        b = m.forward_ops(ro, rd, vd, **RK, render_depth=True)
    same = torch.equal(a['ray_id'], b['ray_id'])
    res['outputs'] = dict(survivors=int(a['ray_id'].numel()), same_survivors=bool(same),
                          **{k: ((a[k] - b[k]).abs().max() / b[k].abs().max().clamp_min(1e-30)).item() if same or k != 'raw_rgb'
                             else None for k in ('rgb_marched', 'alphainv_last', 'depth', 'raw_rgb')})

    res['train_step_ms'] = {}
    for leg in ('fused', 'forward_ops'):
        m.load_state_dict(state0)
        opt = create_optimizer_or_freeze_model(m, cfg, global_step=0)
        fwd = m.forward if leg == 'fused' else m.forward_ops
        res['train_step_ms'][leg] = _time(lambda i: _train_step(m, opt, fwd, ro, rd, vd, target, i + 1), args.steps, args.warmup)
    res['train_step_ms']['reference_gpu'] = _reference_gpu_leg(m, state0, ro, rd, vd, target, args)
    if isinstance(res['train_step_ms']['reference_gpu'], float):
        res['speedup_vs_reference_gpu'] = res['train_step_ms']['reference_gpu'] / res['train_step_ms']['fused']

    # per-launch times (CUDA events around the C-ABI calls) and the rgbnet's forward / backward, in a pass of its own
    k, step_ms, rg = _instrumented(m, state0, cfg, ro, rd, vd, target, args)
    res['kernels_ms'] = k
    res.update(rg)
    res['rgbnet_share_of_step'] = (res['rgbnet_fwd_ms'] + res['rgbnet_bwd_ms']) / step_ms
    res['instrumented_step_ms'] = step_ms
    # algorithmic bytes of the march kernels at the timed size
    with torch.no_grad():
        out = m(ro, rd, vd, **RK)
        from unboundednerfpytorch_b200 import ops
        S = m._n_samples(0.5)
        pts, outb = ops.sample_ndc_pts_on_rays(ro, rd, m.xyz_min, m.xyz_max, S)
        queried = int(m.mask_cache(pts[~outb]).sum())
    M = int(out['ray_id'].numel())
    bytes_a = queried * (32 + 8 + 1)
    bytes_b = M * 8 * 36
    t_a = k.get('march_ndc_density_fwd', float('nan'))
    t_b = k.get('march_ndc_feature_fwd', float('nan'))
    t_bb = k.get('march_ndc_feature_bwd', float('nan'))
    res['march_hbm'] = dict(queried=queried, survivors=M, bytes_pass_a=bytes_a, bytes_pass_b=bytes_b,
                            density_fwd_frac_of_peak=bytes_a / (t_a * 1e-3) / HBM_PEAK,
                            feature_fwd_frac_of_peak=bytes_b / (t_b * 1e-3) / HBM_PEAK,
                            feature_bwd_frac_of_peak=2 * bytes_b / (t_bb * 1e-3) / HBM_PEAK)

    # one 1008x756 frame in 8192-ray chunks
    fro, frd, fvd = rays(1008 * 756)
    res['render_frame_ms'] = _frame(m, fro, frd, fvd, args)
    res['render_rays'] = 1008 * 756

    # the rgbnet paths, alternating: fused step, rgbnet times and share, frame
    legs = [leg.strip() for leg in args.rgbnet.split(',') if leg.strip()]
    if legs != ['kernel']:
        res['legs'] = {leg: [] for leg in legs}
        for _ in range(args.runs):
            for leg in legs:
                with _rgbnet_path(leg):
                    m.load_state_dict(state0)
                    opt = create_optimizer_or_freeze_model(m, cfg, global_step=0)
                    step = _time(lambda i: _train_step(m, opt, m.forward, ro, rd, vd, target, i + 1), args.steps, args.warmup)
                    _, ist, rg = _instrumented(m, state0, cfg, ro, rd, vd, target, args)
                    res['legs'][leg].append(dict(train_step_ms=step, **rg, rgbnet_share_of_step=(rg['rgbnet_fwd_ms'] + rg['rgbnet_bwd_ms']) / ist,
                                                 instrumented_step_ms=ist, render_frame_ms=_frame(m, fro, frd, fvd, args)))
    print(json.dumps(res))


def _rgbnet_path(leg):
    """'kernel': as shipped; 'torch': shade.supported patched to False, so the model runs its nn.Sequential rgbnet"""
    import contextlib
    from unboundednerfpytorch_b200 import shade
    assert leg in ('kernel', 'torch'), leg

    @contextlib.contextmanager
    def ctx():
        orig = shade.supported
        if leg == 'torch':
            shade.supported = lambda *a, **k: False
        try:
            yield
        finally:
            shade.supported = orig
    return ctx()


def _frame(m, fro, frd, fvd, args):
    from unboundednerfpytorch_b200 import render
    return _time(lambda i: render.render_rays(m, fro, frd, fvd, dict(RK), chunk=8192), max(2, args.steps // 5), 1)


def _instrumented(m, state0, cfg, ro, rd, vd, target, args):
    """One timed pass with CUDA events around the C-ABI calls and module hooks around the rgbnet: per-launch times, the step
    time of this pass, and the rgbnet's forward / backward ms (the tensor-core rgbnet's ``rgbnet_fwd`` / ``rgbnet_bwd`` ranges,
    or the hooks when the model ran the torch rgbnet)."""
    from unboundednerfpytorch_b200 import _cabi
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    m.load_state_dict(state0)
    opt = create_optimizer_or_freeze_model(m, cfg, global_step=0)
    timer = _cabi.KernelTimer()
    _cabi.TIMER = timer
    marks = {'fwd': [], 'bwd': []}

    def _mark(kind, end):
        def hook(*a):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            if end:
                marks[kind][-1].append(e)
            else:
                marks[kind].append([e])
        return hook
    hooks = [m.rgbnet.register_forward_pre_hook(_mark('fwd', False)), m.rgbnet.register_forward_hook(_mark('fwd', True)),
             m.rgbnet.register_full_backward_pre_hook(_mark('bwd', False)), m.rgbnet.register_full_backward_hook(_mark('bwd', True))]
    try:
        step_ms = _time(lambda i: _train_step(m, opt, m.forward, ro, rd, vd, target, i + 1), args.steps, 1)
    finally:
        _cabi.TIMER = None
        for h in hooks:
            h.remove()
    k = {n: v[0] for n, v in timer.summary().items()}
    rg = {}
    for kind in ('fwd', 'bwd'):
        if f'rgbnet_{kind}' in k:
            rg[f'rgbnet_{kind}_ms'] = k[f'rgbnet_{kind}']
        else:
            rg[f'rgbnet_{kind}_ms'] = sum(s.elapsed_time(e) for s, e in marks[kind][-args.steps:]) / args.steps
    rg['rgbnet_path'] = 'kernel' if 'rgbnet_fwd' in k else 'torch'
    return k, step_ms, rg


if __name__ == '__main__':
    main()
