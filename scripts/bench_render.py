"""Time the fused whole-frame render (render_fused of the contracted models, csrc/render.cu, and of DirectVoxGO / DirectMPIGO,
csrc/render_bounded.cu) against the chunk loop (``model(...)`` per 8192 rays, what render.render_rays runs without it) and print one
JSON line per workload.

    python scripts/bench_render.py [--rounds 3] [--warmup 1] [--workloads garden-dense,lego-opaque,...]

Workloads, each in a 'dense' scene (random density as in bench.py: rays rarely stop) and an 'opaque' one (the same plus a solid
sphere of high density, radius half the scene: most rays stop early):
  garden: bench.py --workload garden's model (DirectContractedVoxGO 320^3, l2 norm, 12-channel k0, rgbnet 128, viewbase_pe 4,
          fast_color_thres 0) and its 1600 x 1067 frame;
  truck:  a truck-shaped FourierGridModel (153^3, fourier_freq_num 4 -> 9 slabs, 12 channels, stepsize 0.5) on the same frame;
  fg7:    the shape of the reference's *_single FourierGrid configs: FourierGridModel 200^3, fourier_freq_num 3 -> 7 slabs,
          12 channels, stepsize 0.5, on the same frame.
          The Fourier-slab models take the fused render (csrc/render_fourier.cu) only with render_kwargs['fused_slabs'], which
          this script sets unless --fused-slabs 0 is given; then only their chunk loop is timed;
  lego:   DirectVoxGO at the NeRF-synthetic fine shape as scripts/bench_dvgo.py builds it (160^3, 12-channel k0, rgbnet 128,
          viewbase_pe 4, stepsize 0.5, fast_color_thres 1e-4, bg 1, its object-in-box scene: 'dense'; 'opaque' adds a solid ball of
          high density, radius half the box) and its 800 x 800 frame;
  fern:   DirectMPIGO at llff_default as scripts/bench_mpi.py builds it (256^3 voxel budget, mpi_depth 128, stepsize 0.5, 9-channel
          k0, rgbnet 64, viewbase_pe 0, fast_color_thres 1e-3, seeded grids: 'dense'; 'opaque' adds four planes of high density
          half way through) and one 1008 x 756 NDC frame.
The two paths alternate in one process (fused, loop, fused, loop ...).  Per workload: CUDA-event ms per frame of each (median and
all rounds), samples nominal (rays x samples per ray), marched (the 32-sample chunks the fused march walked before each ray
stopped) and shaded (its kept samples), peak device memory of each
call above what was allocated before it, max |delta| of rgb_marched / depth / alphainv_last against the chunk loop, and the card's
name and power limit, read in the same run."""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_dvgo import _gpu  # noqa: E402

SEED = 777
RK_GARDEN = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=1.045, render_depth=True, coherent_rays=False)
RK_TRUCK = dict(RK_GARDEN, stepsize=0.5)          # truck and fg7
RK_LEGO = dict(near=2.0, far=6.0, bg=1., rand_bkgd=False, stepsize=0.5, render_depth=True)
RK_FERN = dict(near=0., far=1., bg=1, rand_bkgd=False, stepsize=0.5, render_depth=True)


def _frame(dev, name):
    import numpy as np
    from unboundednerfpytorch_b200 import rays as R
    ndc = name == 'fern'
    if name == 'lego':          # scripts/bench_dvgo.py's frame: 4 units out, looking at the box
        H, W = 800, 800
        K = np.array([[1111., 0., 400.], [0., 1111., 400.], [0., 0., 1.]])
        c2w = torch.tensor([[1., 0., 0., 0.], [0., 1., 0., 0.], [0., 0., 1., 4.0]])
    elif ndc:
        H, W = 756, 1008
        K = np.array([[815., 0., 504.], [0., 815., 378.], [0., 0., 1.]])
        c2w = torch.tensor([[1., 0., 0., 0.], [0., 1., 0., 0.], [0., 0., 1., 0.]])
    else:
        H, W = 1067, 1600
        K = np.array([[float(W), 0, W / 2], [0, float(W), H / 2], [0, 0, 1]], dtype=np.float64)
        c2w = torch.tensor([[1., 0., 0., 0.15], [0., 1., 0., -0.10], [0., 0., 1., 0.35]])
    ro, rd, vd = R._rays_of_a_view(H, W, K, c2w, ndc, False, False, False, 'center', device=dev)
    return ro.reshape(-1, 3), rd.reshape(-1, 3), vd.reshape(-1, 3)


def _model(name, scene, dev):
    from unboundednerfpytorch_b200 import models
    torch.manual_seed(SEED)
    if name == 'lego':
        from bench_dvgo import _scene
        m = _scene(160 ** 3, 12, 1, 0)[0]
        if scene == 'opaque':
            X, Y, Z = m.density.grid.shape[2:]
            ax = [torch.linspace(-1, 1, n, device=dev) for n in (X, Y, Z)]
            r = (ax[0][:, None, None] ** 2 + ax[1][None, :, None] ** 2 + ax[2][None, None, :] ** 2).sqrt()
            with torch.no_grad():
                m.density.grid.add_(torch.where(r < 0.5, 40.0, 0.0))
        return m
    if name == 'fern':
        from bench_mpi import _scene
        m = _scene(1)[0]
        if scene == 'opaque':
            Z = m.density.grid.shape[-1]
            with torch.no_grad():
                m.density.grid[..., Z // 2:Z // 2 + 4] += 40.0
        return m
    if name == 'garden':
        w = 320
        m = models.DirectContractedVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=w ** 3, num_voxels_base=w ** 3,
                                         alpha_init=1e-4, fast_color_thres=0, rgbnet_dim=12, contracted_norm='l2').to(dev)
    else:
        w, F_ = (153, 4) if name == 'truck' else (200, 3)
        m = models.FourierGridModel(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=w ** 3, num_voxels_base_density=w ** 3,
                                    num_voxels_rgb=w ** 3, num_voxels_base_rgb=w ** 3, num_voxels_viewdir=-1, alpha_init=1e-4,
                                    fast_color_thres=0, rgbnet_dim=12, fourier_freq_num=F_).to(dev)
    g = torch.Generator(device=dev).manual_seed(SEED)
    with torch.no_grad():
        m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=g, device=dev))
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g, device=dev))
        if scene == 'opaque':
            X, Y, Z = m.density.grid.shape[2:]
            ax = [torch.linspace(-1, 1, n, device=dev) for n in (X, Y, Z)]
            r = (ax[0][:, None, None] ** 2 + ax[1][None, :, None] ** 2 + ax[2][None, None, :] ** 2).sqrt()
            m.density.grid.add_(torch.where(r < 0.5, 40.0, 0.0))
    return m


def _chunk_loop(m, ro, rd, vd, rk):
    outs = {k: [] for k in ('rgb_marched', 'depth', 'alphainv_last')}
    with torch.no_grad():
        for a, b, c in zip(ro.split(8192), rd.split(8192), vd.split(8192)):
            ret = m(a, b, c, **rk)
            for k in outs:
                outs[k].append(ret[k].reshape(a.shape[0], -1))
    return {k: torch.cat(v) for k, v in outs.items()}


def _fused(m, ro, rd, vd, rk, ns=None, nm=None):
    out = m.render_fused(ro, rd, vd, n_shaded=ns, n_marched=nm, **rk)
    return {k: out[k].reshape(ro.shape[0], -1) for k in out}


def _timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return out, s.elapsed_time(e), torch.cuda.max_memory_allocated() - base


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--workloads', default='garden-dense,garden-opaque,truck-dense,truck-opaque')
    ap.add_argument('--fused-slabs', type=int, default=1, help="set render_kwargs['fused_slabs'] for the Fourier-slab models")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_render.py needs a CUDA device')
    from unboundednerfpytorch_b200 import build
    build.build()
    dev = torch.device('cuda', 0)
    gpu, power = _gpu()
    for wl in args.workloads.split(','):
        name, scene = wl.split('-')
        ro, rd, vd = _frame(dev, name)
        n = ro.shape[0]
        m = _model(name, scene, dev)
        rk = {'garden': RK_GARDEN, 'truck': RK_TRUCK, 'fg7': RK_TRUCK, 'lego': RK_LEGO, 'fern': RK_FERN}[name]
        if name in ('truck', 'fg7') and args.fused_slabs:
            rk = dict(rk, fused_slabs=True)
        covered = m.render_fused_ok(ro, rk)
        if name == 'lego':
            S = int(m._box_cfg(rk).s_max)          # the bound of a ray's steps; its own n_steps may be fewer
        elif name == 'fern':
            S = int(m._ndc_cfg(rk)[1])
        else:
            S = int(m._march_inputs(rk['stepsize'], dev)[0].numel())
        ns = torch.empty(n, dtype=torch.int32, device=dev)
        nm = torch.empty(n, dtype=torch.int32, device=dev)
        if not covered:                       # Fourier slabs without fused_slabs: render_rays keeps the chunk loop
            _chunk_loop(m, ro, rd, vd, rk)
            t_l = [_timed(lambda: _chunk_loop(m, ro, rd, vd, rk))[1] for _ in range(args.rounds)]
            print(json.dumps({'workload': wl, 'rays': n, 'samples_per_ray': S, 'gpu': gpu, 'power_limit': power, 'fused': None,
                              'chunk_loop_ms': sorted(t_l)[len(t_l) // 2], 'chunk_loop_ms_rounds': t_l}), flush=True)
            del m
            torch.cuda.empty_cache()
            continue
        for _ in range(args.warmup):
            _fused(m, ro, rd, vd, rk)
            _chunk_loop(m, ro, rd, vd, rk)
        t_f, t_l, mem_f, mem_l = [], [], 0, 0
        for _ in range(args.rounds):
            fo, ms, mem = _timed(lambda: _fused(m, ro, rd, vd, rk))
            t_f.append(ms)
            mem_f = max(mem_f, mem)
            lo, ms, mem = _timed(lambda: _chunk_loop(m, ro, rd, vd, rk))
            t_l.append(ms)
            mem_l = max(mem_l, mem)
        _fused(m, ro, rd, vd, rk, ns, nm)
        delta = {k: float((fo[k] - lo[k]).abs().max()) for k in fo}
        med = lambda v: sorted(v)[len(v) // 2]
        print(json.dumps({
            'workload': wl, 'rays': n, 'samples_per_ray': S, 'gpu': gpu, 'power_limit': power,
            'fused_ms': med(t_f), 'chunk_loop_ms': med(t_l), 'speedup': med(t_l) / med(t_f),
            'fused_ms_rounds': t_f, 'chunk_loop_ms_rounds': t_l,
            'samples_nominal': n * S, 'samples_marched': int(nm.sum()), 'samples_shaded': int(ns.sum()),
            'fused_peak_mem_bytes': mem_f, 'chunk_loop_peak_mem_bytes': mem_l,
            'max_abs_delta_vs_chunk_loop': delta}), flush=True)
        del m
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
