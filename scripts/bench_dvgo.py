"""Time DirectVoxGO (bounded scenes, dvgo.py) on the GPU and print one JSON line.

    python scripts/bench_dvgo.py [--steps 20] [--warmup 5] [--shape default|lab] [--rounds 3]

Legs of the default shape, each from the same parameters:
* fine-stage training step (run_train.py:251-288 with configs/default.py's fine weights: entropy_last 1e-3, rgbper 1e-2, no TV,
  MaskedAdam skipping zero gradients on density and k0) at 160^3 voxels, 12-channel k0, 8192 rays: the fused march
  (``forward``), the op-by-op composition (``forward_ops``) and the reference's GPU path (its unmodified dvgo.py and
  masked_adam.py over its own CUDA build in oracle/_ref), or an "unavailable" record when oracle/_ref is absent;
* coarse-stage step at 1 024 000 voxels with configs/default.py's coarse settings (rgbnet_dim 0, alpha_init 1e-6,
  fast_color_thres 1e-7) and per-voxel lr;
* one 800x800 frame in 8192-ray chunks.
Per launch: the march kernels' CUDA-event times and their algorithmic HBM share against 3.35 TB/s, and the rgbnet's share of the
fused step.  Output check: fused against forward_ops (and against the reference's GPU path) at the timed size.  The GPU name and
power limit are read in the same run.

--shape lab: configs/free_dataset/lab.py's fine stage -- a 250^3 voxel budget, 9-channel k0, rgbnet width 64, fast_color_thres
1e-3, 4096 rays -- with the same training step for the fused, forward_ops and reference_gpu legs alternated for --rounds rounds,
the per-launch times and the rgbnet's share of the fused step, and the output check at the timed size."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

LO, HI = [-1.5, -1.5, -1.5], [1.5, 1.5, 1.5]
RK = dict(near=2.0, far=6.0, bg=1., rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False)
HBM = 3.35e12


def _gpu():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(',')]
        return name, pl
    except Exception as e:          # the bench still reports the device name torch sees
        return torch.cuda.get_device_name(0), f'unknown ({type(e).__name__})'


def _scene(nv, C, n, seed, cls=None, width=128, thres=None):
    """C = 12: the fine stage of configs/default.py (alpha_init 1e-2, fast_color_thres 1e-4); C = 3: its coarse stage
    (rgbnet_dim 0, alpha_init 1e-6, fast_color_thres 1e-7); C = 9: lab.py's fine stage (rgbnet width 64, fast_color_thres 1e-3)."""
    from unboundednerfpytorch_b200 import models
    cls = cls or models.DirectVoxGO
    g = torch.Generator().manual_seed(seed)
    if thres is None:
        thres = 1e-7 if C == 3 else 1e-4
    m = cls(xyz_min=LO, xyz_max=HI, num_voxels=nv, num_voxels_base=nv, alpha_init=1e-6 if C == 3 else 1e-2,
            fast_color_thres=thres, rgbnet_dim=0 if C == 3 else C, rgbnet_direct=True, rgbnet_width=width)
    with torch.no_grad():
        X, Y, Z = [int(v) for v in m.world_size]
        ax = [torch.linspace(-1, 1, k) for k in (X, Y, Z)]
        r2 = sum(a ** 2 for a in torch.meshgrid(*ax, indexing='ij'))
        m.density.grid.copy_((8.0 * (0.35 - r2) + torch.randn(X, Y, Z, generator=g))[None, None])
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g) * 0.5)
    o = torch.randn(n, 3, generator=g)
    o = o / o.norm(dim=-1, keepdim=True) * 4.0
    d = (torch.rand(n, 3, generator=g) - 0.5) * 2.0 - o
    d = d / d.norm(dim=-1, keepdim=True)             # unit directions: near = 2 is 2 units from the camera (NeRF-synthetic)
    return m.cuda(), o.cuda(), d.cuda(), (d / d.norm(dim=-1, keepdim=True)).cuda()


def _opt(m, pervoxel=None):
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    cfg = dict(lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])
    opt = create_optimizer_or_freeze_model(m, cfg, global_step=0)
    if pervoxel is not None:
        opt.set_pervoxel_lr(pervoxel)
    return opt


def _step(m, fn, opt, ro, rd, vd, target, it):
    ret = fn(ro, rd, vd, global_step=it, **RK)
    opt.zero_grad(set_to_none=True)
    loss = F.mse_loss(ret['rgb_marched'], target)
    pout = ret['alphainv_last'].clamp(1e-6, 1 - 1e-6)
    loss = loss + 1e-3 * -(pout * torch.log(pout) + (1 - pout) * torch.log(1 - pout)).mean()       # entropy_last
    rgbper = (ret['raw_rgb'] - target[ret['ray_id']]).pow(2).sum(-1)
    loss = loss + 1e-2 * (rgbper * ret['weights'].detach()).sum() / len(ro)
    loss.backward()
    opt.step()
    return ret


def _time(fn, steps, warmup):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(steps):
        fn(warmup + i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def _reference_leg(state, ours, ro, rd, vd, target, args):
    """The same step through the reference's GPU path: its unmodified dvgo.py and masked_adam.py over its own CUDA extension
    (oracle/_ref, staged by __graft_entry__.build()), run as run_train.py runs it, with CUDA as the default tensor type."""
    import contextlib
    import io
    from oracle import ref_gpu_py
    why = ref_gpu_py.missing()
    if why is not None:
        return {'unavailable': f'{why} not built'}
    ns = ref_gpu_py.load()
    ref_dvgo = sys.modules[ref_gpu_py.PKG + '.dvgo']
    kw = {k: v for k, v in ours.get_kwargs().items() if k != 'voxel_size_ratio'}
    with contextlib.redirect_stdout(io.StringIO()):        # built on the host like ours: the same voxel_size cube root
        ref = ref_dvgo.DirectVoxGO(**kw)
    ref.load_state_dict({k: v.contiguous() for k, v in state.items()}, strict=True)
    ref = ref.cuda()
    ours.load_state_dict(state)                            # the timed legs before this one trained ours: compare from the start
    ref_gpu_py.default_cuda(True)
    try:
        with torch.no_grad():
            a, b = ref(ro, rd, vd, **RK), ours(ro, rd, vd, **RK)
        same = torch.equal(a['ray_id'], b['ray_id'])
        check = {'ray_id_equal': same, 'weights_bit_identical': same and torch.equal(a['weights'], b['weights']),
                 'raw_alpha_bit_identical': same and torch.equal(a['raw_alpha'], b['raw_alpha']),
                 'alphainv_last_bit_identical': torch.equal(a['alphainv_last'], b['alphainv_last'])}
        opt = ns.masked_adam.MaskedAdam([{'params': [ref.density.grid], 'lr': 0.1, 'skip_zero_grad': True},
                                         {'params': [ref.k0.grid], 'lr': 0.1, 'skip_zero_grad': True},
                                         {'params': list(ref.rgbnet.parameters()), 'lr': 1e-3, 'skip_zero_grad': False}])
        ms = _time(lambda i: _step(ref, ref.forward, opt, ro, rd, vd, target, i + 1), args.steps, args.warmup)
    finally:
        ref_gpu_py.default_cuda(False)
    return {'ms': round(ms, 3), 'check_vs_fused': check}


def _check(a, b):
    same = torch.equal(a['ray_id'], b['ray_id'])
    return {'ray_id_equal': same, 'samples': int(len(a['ray_id'])),
            'weights_bit_identical': same and torch.equal(a['weights'], b['weights']),
            'raw_alpha_bit_identical': same and torch.equal(a['raw_alpha'], b['raw_alpha']),
            'alphainv_last_bit_identical': torch.equal(a['alphainv_last'], b['alphainv_last']),
            'rgb_marched_max_abs_diff': float((a['rgb_marched'] - b['rgb_marched']).abs().max())}


def lab(args):
    """lab.py's fine stage: the three legs alternated round by round, per-launch times of the fused step."""
    from unboundednerfpytorch_b200 import _cabi
    name, power = _gpu()
    out = {'bench': 'dvgo lab', 'gpu': name, 'power_limit': power, 'steps': args.steps, 'warmup': args.warmup,
           'shape': dict(num_voxels=250 ** 3, k0_channels=9, rgbnet_width=64, fast_color_thres=1e-3, rays=4096)}
    base, ro, rd, vd = _scene(250 ** 3, 9, 4096, 0, width=64, thres=1e-3)
    state = {k: v.clone() for k, v in base.state_dict().items()}
    with torch.no_grad():
        target = torch.rand(len(ro), 3, device='cuda', generator=torch.Generator('cuda').manual_seed(1))
        out['check'] = _check(base(ro, rd, vd, **RK), base.forward_ops(ro, rd, vd, **RK))
    legs = {'fused': [], 'forward_ops': [], 'reference_gpu': []}
    for _ in range(args.rounds):
        for leg in ('fused', 'forward_ops'):
            base.load_state_dict(state)
            opt = _opt(base)
            fn = base.forward if leg == 'fused' else base.forward_ops
            legs[leg].append(round(_time(lambda i: _step(base, fn, opt, ro, rd, vd, target, i + 1), args.steps, args.warmup), 3))
        ref = _reference_leg(state, base, ro, rd, vd, target, args)
        if 'ms' not in ref:
            legs['reference_gpu'] = ref
            break
        legs['reference_gpu'].append(ref['ms'])
        out['check_vs_reference_gpu'] = ref['check_vs_fused']
    out['step_ms_rounds'] = legs
    base.load_state_dict(state)
    opt = _opt(base)
    _cabi.TIMER = _cabi.KernelTimer()
    try:
        ms = _time(lambda i: _step(base, base.forward, opt, ro, rd, vd, target, i + 1), args.steps, 1)
        summ = _cabi.TIMER.summary()
    finally:
        _cabi.TIMER = None
    out['launches'] = {k: {'ms': round(v, 4), 'calls': c} for k, (v, c) in summ.items()}
    out['instrumented_step_ms'] = round(ms, 3)
    out['rgbnet_share_of_fused_step'] = round(sum(v for k, (v, _) in summ.items() if 'rgbnet' in k) / ms, 3)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--shape', choices=('default', 'lab'), default='default')
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_dvgo needs a CUDA device')
    if args.shape == 'lab':
        return lab(args)
    import unboundednerfpytorch_b200 as U
    from unboundednerfpytorch_b200 import _cabi, render
    name, power = _gpu()
    out = {'bench': 'dvgo', 'gpu': name, 'power_limit': power, 'steps': args.steps, 'warmup': args.warmup}

    # ---- fine stage: 160^3, C = 12, 8192 rays ----
    base, ro, rd, vd = _scene(160 ** 3, 12, 8192, 0)
    state = {k: v.clone() for k, v in base.state_dict().items()}
    with torch.no_grad():
        target = torch.rand(len(ro), 3, device='cuda', generator=torch.Generator('cuda').manual_seed(1))
        a = base(ro, rd, vd, **RK)
        b = base.forward_ops(ro, rd, vd, **RK)
    same = torch.equal(a['ray_id'], b['ray_id'])
    out['check'] = {'ray_id_equal': same, 'samples': int(len(a['ray_id'])),
                    'weights_bit_identical': same and torch.equal(a['weights'], b['weights']),
                    'raw_alpha_bit_identical': same and torch.equal(a['raw_alpha'], b['raw_alpha']),
                    'alphainv_last_bit_identical': torch.equal(a['alphainv_last'], b['alphainv_last']),
                    'rgb_marched_max_abs_diff': float((a['rgb_marched'] - b['rgb_marched']).abs().max())}
    legs = {}
    for leg in ('fused', 'forward_ops', 'fused', 'forward_ops'):          # alternated, each from the same parameters
        base.load_state_dict(state)
        opt = _opt(base)
        fn = base.forward if leg == 'fused' else base.forward_ops
        legs.setdefault(leg, []).append(_time(lambda i: _step(base, fn, opt, ro, rd, vd, target, i + 1), args.steps, args.warmup))
    out['fine_step_ms'] = {k: [round(x, 3) for x in v] for k, v in legs.items()}
    out['fine_step_ms']['reference_gpu'] = _reference_leg(state, base, ro, rd, vd, target, args)

    # per launch: march kernels and the rgbnet inside the fused step
    base.load_state_dict(state)
    opt = _opt(base)
    _cabi.TIMER = _cabi.KernelTimer()
    for i in range(args.steps):
        _step(base, base.forward, opt, ro, rd, vd, target, i + 1)
    summ = _cabi.TIMER.summary()
    _cabi.TIMER = None
    N, S = len(ro), int(U.march.box_s_max(LO, HI, base._stepdist(0.5)))
    M = out['check']['samples']
    nv = int(np.prod([int(v) for v in base.world_size]))
    # algorithmic bytes: pass A reads rays and writes 17 B per record of the rays' own n_steps (bounded by S), pass B writes
    # 48 B features + 24 B records per survivor and reads 8 corners x 48 B; density bwd reads the records; feature bwd 8 x 48 B of reds
    alg = {'march_box_density_fwd': N * S * 17, 'march_box_feature_fwd': M * (48 + 24 + 8 * 48),
           'march_box_density_bwd': N * S * 17, 'march_box_feature_bwd': M * (48 + 8 * 48)}
    launches = {}
    for k, (ms, cnt) in summ.items():
        launches[k] = {'ms': round(ms, 4), 'calls': cnt}
        if k in alg:
            launches[k]['hbm_share_upper_bound'] = round(alg[k] / HBM / (ms * 1e-3), 3)
    out['launches'] = launches
    fused_ms = float(np.mean(legs['fused']))
    rgb_ms = sum(v['ms'] for k, v in launches.items() if 'rgbnet' in k or 'shade' in k)
    out['rgbnet_share_of_fused_step'] = round(rgb_ms / fused_ms, 3) if rgb_ms else 'not measured'
    out['density_grid_voxels'] = nv

    # ---- coarse stage: 1 024 000 voxels, rgbnet_dim 0, per-voxel lr ----
    coarse, ro2, rd2, vd2 = _scene(1024000, 3, 8192, 2)
    cnt = coarse.voxel_count_views(ro2.reshape(8, 1024, 3), rd2.reshape(8, 1024, 3), [1] * 8, 2.0, 6.0, 0.5)
    opt2 = _opt(coarse, cnt)
    out['coarse_step_ms'] = round(_time(lambda i: _step(coarse, coarse.forward, opt2, ro2, rd2, vd2, target, i + 1),
                                        args.steps, args.warmup), 3)

    # ---- one 800x800 frame in 8192-ray chunks ----
    K = np.array([[1111., 0., 400.], [0., 1111., 400.], [0., 0., 1.]])
    c2w = np.array([[1, 0, 0, 0.], [0, 1, 0, 0.], [0, 0, 1, 4.0]], dtype=np.float32)          # 4 units out, looking at the box
    fn = lambda i: render.render_viewpoints(None, base, [c2w], [[800, 800]], [K], False, dict(RK, render_depth=True), chunk=8192,
                                            verbose=False)
    out['frame_800_ms'] = round(_time(fn, 3, 1), 2)
    rgbs, _, bg = fn(0)
    out['frame_800_covered'] = round(float((bg[0] < 0.999).mean()), 3)       # share of pixels that hit the object
    print(json.dumps(out))


if __name__ == '__main__':
    main()
