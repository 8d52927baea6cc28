"""Time one training step of DirectVoxGO with TensoRF grids at configs/nerf/ship.tensorf.py's fine shape and print one JSON line.

    python scripts/bench_tensorf.py [--steps 10] [--warmup 3] [--rounds 3]

The step is run_train.py:251-288 with bench_dvgo.py's loss weights (entropy_last 1e-3, rgbper 1e-2) and MaskedAdam skipping zero gradients on density and k0, on bench_dvgo.py's object-in-box scene: 384^3 voxel
budget, density n_comp 8, 12-channel k0 with n_comp 24, width-128 rgbnet, 8192 rays, stepsize 0.5, fast_color_thres 1e-4.
Legs, alternated in --rounds rounds in this one process: this library's step (forward on the fused box march), the same step
through the op-by-op composition (DirectVoxGO._compose with the same shading), and the reference's GPU path (its unmodified
dvgo.py / grid.py / masked_adam.py over its own CUDA build in oracle/_ref; an "unavailable" record when that is absent).
Reported: step times, CUDA-event times of the march and tensorf kernels, the algorithmic bytes and FLOPs of tensorf_fwd /
tensorf_bwd (from shapes, below), the survivor counts, the backward's time at each replicated vector-gradient copy count, and
the card's name and power limit read in the same run."""
import argparse
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_dvgo import HI, LO, RK, _gpu, _step, _time  # noqa: E402

KW = dict(xyz_min=LO, xyz_max=HI, num_voxels=384 ** 3, num_voxels_base=384 ** 3, alpha_init=1e-2, fast_color_thres=1e-4,
          density_type='TensoRFGrid', density_config=dict(n_comp=8), k0_type='TensoRFGrid', k0_config=dict(n_comp=24),
          rgbnet_dim=12, rgbnet_direct=True, rgbnet_width=128, rgbnet_depth=3, viewbase_pe=4)
COPIES = (1, 4, 8, 16, 32)


def _scene(n, seed):
    """bench_dvgo.py's object in the box, in factor form: each vector peaks mid-axis, so the products leave free space around a
    central object; noisy planes and k0 factors."""
    from unboundednerfpytorch_b200 import models
    torch.manual_seed(seed)
    g = torch.Generator().manual_seed(seed)
    with contextlib.redirect_stdout(io.StringIO()):
        m = models.DirectVoxGO(**KW)
    with torch.no_grad():
        for name in ('x_vec', 'y_vec', 'z_vec'):
            v = getattr(m.density, name)
            L = v.shape[2]
            prof = 0.6 - 2.5 * torch.linspace(-1, 1, L) ** 2
            v.copy_(prof[None, None, :, None] + 0.1 * torch.randn(v.shape, generator=g))
        for name in ('xy_plane', 'xz_plane', 'yz_plane'):
            getattr(m.density, name).copy_(0.8 + 0.2 * torch.randn(getattr(m.density, name).shape, generator=g))
    o = torch.randn(n, 3, generator=g)
    o = o / o.norm(dim=-1, keepdim=True) * 4.0
    d = (torch.rand(n, 3, generator=g) - 0.5) * 2.0 - o
    d = d / d.norm(dim=-1, keepdim=True)
    state = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}
    return m.cuda(), state, o.cuda(), d.cuda(), d.cuda()


def _opt(m):
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    cfg = dict(lrate_density=0.02, lrate_k0=0.02, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])
    return create_optimizer_or_freeze_model(m, cfg, global_step=0)


def _traffic(grid, M):
    """Algorithmic bytes and FLOPs of one tensorf_fwd / tensorf_bwd over M samples (every factor value counted once per use, no
    cache reuse).  Per sample and feature k (nfeat = 2R + Rxy of them): 4 plane corners + 2 vector nodes read (24 B), the
    bilinear and linear blends (6 FMA), the product (1 mul) and its projection onto C outputs (C FMA); plus xyz (12 B) and the
    C outputs (4C B).  Backward: the same reads and blends, grad_out (4C B), g_feat (C FMA), two gradient products, 4 + 2
    weighted reductions (24 B of atomics) and feat . grad_out into grad_f_vec (C FMA when C > 1)."""
    R, Rxy, C = grid.config['n_comp'], grid.config.get('n_comp_xy', grid.config['n_comp']), grid.channels
    nf = 2 * R + Rxy
    proj = C if C > 1 else 1
    fwd_b = M * (24 * nf + 12 + 4 * C)
    fwd_f = M * nf * (2 * 6 + 1 + 2 * proj)
    bwd_b = M * (24 * nf + 12 + 4 * C + 24 * nf)
    bwd_f = M * nf * (2 * 6 + 1 + 2 * proj + 2 + 6 + (2 * C if C > 1 else 0))
    return dict(fwd_bytes=fwd_b, fwd_flops=fwd_f, bwd_bytes=bwd_b, bwd_flops=bwd_f)


def _reference_leg(state, ro, rd, vd, target, args):
    from oracle import ref_gpu_py
    why = ref_gpu_py.missing()
    if why is not None:
        return None, {'unavailable': f'{why} not built'}
    ns = ref_gpu_py.load()
    ref_dvgo = sys.modules[ref_gpu_py.PKG + '.dvgo']
    kw = dict(KW, xyz_min=np.array(LO, dtype=np.float32), xyz_max=np.array(HI, dtype=np.float32))
    with contextlib.redirect_stdout(io.StringIO()):
        ref = ref_dvgo.DirectVoxGO(**kw)
    ref.load_state_dict(state, strict=True)
    ref = ref.cuda()
    opt = ns.masked_adam.MaskedAdam([{'params': list(ref.density.parameters()), 'lr': 0.02, 'skip_zero_grad': True},
                                     {'params': list(ref.k0.parameters()), 'lr': 0.02, 'skip_zero_grad': True},
                                     {'params': list(ref.rgbnet.parameters()), 'lr': 1e-3, 'skip_zero_grad': False}])

    def run():
        ref_gpu_py.default_cuda(True)
        try:
            return _time(lambda i: _step(ref, ref.forward, opt, ro, rd, vd, target, i + 1), args.steps, args.warmup)
        finally:
            ref_gpu_py.default_cuda(False)
    return run, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--rays', type=int, default=8192)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_tensorf.py needs a CUDA device')
    from unboundednerfpytorch_b200 import _cabi
    from unboundednerfpytorch_b200 import grid as G
    name, power = _gpu()
    out = {'bench': 'tensorf', 'gpu': name, 'power_limit': power, 'steps': args.steps, 'warmup': args.warmup,
           'rays': args.rays, 'config': 'ship.tensorf fine (384^3, n_comp 8 / 24, k0 C 12, rgbnet width 128)'}
    m, state, ro, rd, vd = _scene(args.rays, 0)
    target = torch.rand(args.rays, 3, generator=torch.Generator().manual_seed(1)).cuda()
    out['world_size'] = [int(v) for v in m.world_size]
    opt = _opt(m)

    # survivor counts of one forward
    with torch.no_grad():
        pts, ray_id, _ = m.sample_ray(ro, rd, **RK)
        n_dens = int(m.mask_cache(pts).sum())
        ret = m(ro, rd, vd, **RK)
    out['survivors'] = {'density_samples': n_dens, 'k0_samples': int(ret['ray_id'].numel())}

    ours = lambda: _time(lambda i: _step(m, m.forward, opt, ro, rd, vd, target, i), args.steps, args.warmup)  # noqa: E731
    compose_fwd = lambda a, b, c, global_step=None, **rk: m._compose(a, b, c, m._shade_k0, rk)  # noqa: E731
    compose = lambda: _time(lambda i: _step(m, compose_fwd, opt, ro, rd, vd, target, i), args.steps, args.warmup)  # noqa: E731
    ref_run, why = _reference_leg(state, ro, rd, vd, target, args)
    legs = {'ours': [], 'compose': [], 'reference_gpu': []}
    for _ in range(args.rounds):
        legs['ours'].append(round(ours(), 3))
        legs['compose'].append(round(compose(), 3))
        if ref_run is not None:
            legs['reference_gpu'].append(round(ref_run(), 3))
    out['step_ms'] = {k: (v if v else why) for k, v in legs.items()}
    if ref_run is not None:
        out['speedup_median'] = round(float(np.median(legs['reference_gpu']) / np.median(legs['ours'])), 2)
    out['fused_over_compose_median'] = round(float(np.median(legs['compose']) / np.median(legs['ours'])), 3)

    # per-kernel CUDA-event times at each replicated vector-gradient copy count
    per_k = {}
    for K in COPIES + COPIES[::-1]:          # each count twice, in both orders, so clock drift does not rank them
        G.TENSORF_VEC_COPIES = K
        _cabi.TIMER = _cabi.KernelTimer()
        _time(lambda i: _step(m, m.forward, opt, ro, rd, vd, target, i), args.steps, args.warmup)
        s = _cabi.TIMER.summary()
        _cabi.TIMER = None
        per_k.setdefault(K, []).append({k: round(v[0], 4) for k, v in s.items() if k.startswith(('tensorf_', 'march_box'))})
    out['kernel_ms_by_vec_copies'] = per_k
    traffic = {'density (c1)': _traffic(m.density, n_dens), 'k0 (c12)': _traffic(m.k0, out['survivors']['k0_samples'])}
    out['algorithmic'] = traffic
    out['note'] = ('density tensorf_fwd runs on every in-mask sample; its backward on the samples that pass the alpha threshold '
                   '(not counted separately: its bytes / FLOPs above are an upper bound)')
    print(json.dumps(out))


if __name__ == '__main__':
    main()
