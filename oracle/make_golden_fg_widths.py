"""oracle/make_golden_fg_widths.py -- TEST INFRASTRUCTURE ONLY.  Generates tests/golden/l2_fg_widths/*.pt.

Runs the reference's own FourierGrid_model.py / dcvgo.py, imported unmodified from /root/reference, on the CPU over the stand-ins of
oracle/stubs.py (as oracle/make_golden.py does) at the k0 widths of the reference's other FourierGrid configs:

* waymo -- FourierGridModel, rgbnet_dim 3, viewbase_pe 2, contracted_norm l2, fourier_freq_num 3 (configs/waymo/waymo_no_block.py);
* mega  -- the same with viewbase_pe 8 (configs/mega/building_no_block.py);
* train -- FourierGridModel, rgbnet_dim 15, viewbase_pe 4 (configs/tankstemple_unbounded/train_single.py);
* fg_rgb0 / dcvgo_rgb0 -- the rgbnet_dim = 0 colour grid (rgb = sigmoid(k0), C = 3) of FourierGridModel and DirectContractedVoxGO;

each at fast_color_thres 0 and 1e-4.  A record holds the constructor kwargs, the state dict WITHOUT the two grids (they are
regenerated from `grid_seed` by tests.test_gpu_fg_widths.golden_grids, which keeps every file well under 1 MB), the rays, the
forward outputs, and the gradients of the density grid, the k0 grid and the rgbnet for a seeded scalar functional of them.

    python -m oracle.make_golden_fg_widths       # from the repo root, where /root/reference exists
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, 'tests', 'golden', 'l2_fg_widths')
sys.path.insert(0, ROOT)

from oracle import stubs  # noqa: E402

stubs.install('/root/reference')
from FourierGrid import dcvgo as ref_dcvgo  # noqa: E402
from FourierGrid import FourierGrid_model as ref_fgmodel  # noqa: E402

from oracle.make_golden import _c, _grab, _rays  # noqa: E402
from tests.test_gpu_fg_widths import GOLDEN, golden_grids  # noqa: E402

SEED = 777


def record(name, spec, thres):
    torch.manual_seed(SEED)
    kw = dict(spec['kw'], fast_color_thres=thres)
    if spec['cls'] == 'FourierGridModel':
        m = ref_fgmodel.FourierGridModel(**kw)
    else:
        m = ref_dcvgo.DirectContractedVoxGO(**kw)
    grid_seed = SEED + 10 * list(GOLDEN).index(name) + (1 if thres > 0 else 0)
    dens, k0 = golden_grids(m.density.grid.shape, m.k0.grid.shape, grid_seed, thres)
    with torch.no_grad():
        m.density.grid.copy_(dens)
        m.k0.grid.copy_(k0)
    gen = torch.Generator().manual_seed(SEED + 1)
    N = spec['rays']
    ro, rd, vd = _rays(N, gen)
    # the reference's depth (FourierGrid_model.py:665-668) multiplies the per-sample weights by the unmasked [S] t-table when no
    # threshold compacts the samples, so depth is only recorded at fast_color_thres > 0
    rk = dict(near=0.0, far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False,
              render_depth=thres > 0)
    ret = m(ro, rd, vd, global_step=None, is_train=False, **rk)
    lw = dict(rgb=torch.randn(N, 3, generator=gen), last=torch.randn(N, generator=gen))
    rec = _grab(m, ret, lw)
    # without a threshold the reference returns raw_alpha / raw_density / t / s as [N, S] (nothing indexes them with a mask); the
    # per-sample records are stored flat, in the (ray, step) order of ray_id / step_id
    M = rec['ray_id'].numel()
    for k, v in rec.items():
        if torch.is_tensor(v) and v.dim() == 2 and v.numel() == M:
            rec[k] = v.reshape(-1)
    state = {k: _c(v) for k, v in m.state_dict().items() if k not in ('density.grid', 'k0.grid')}
    out = dict(cls=spec['cls'], kwargs=kw, state=state, grid_seed=grid_seed, rays_o=ro, rays_d=rd, viewdirs=vd, render_kwargs=rk,
               loss_w=lw, ret=rec)
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f'{name}_t{thres:g}.pt')
    torch.save(out, path)
    print(f'{os.path.relpath(path, ROOT)}: {os.path.getsize(path) / 1024:.1f} KiB, {int(ret["ray_id"].numel())} survivors')


if __name__ == '__main__':
    torch.set_num_threads(4)
    for name, spec in GOLDEN.items():
        for thres in (0.0, 1e-4):
            record(name, spec, thres)
