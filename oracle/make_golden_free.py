"""oracle/make_golden_free.py -- TEST INFRASTRUCTURE ONLY.  Generates tests/golden/l2_free/*.pt.

Runs the reference's own FourierGrid_model.py and dvgo.py, imported unmodified from /root/reference, on the CPU over the stand-ins
of oracle/stubs.py (as oracle/make_golden.py does) at reduced shapes of the free-dataset configs, both with a 9-channel k0 and the
width-64 rgbnet:

* grass -- FourierGridModel, rgbnet_dim 9, fourier_freq_num 3 (P = 7), viewbase_pe 4 (configs/free_dataset/grass.py);
* lab   -- DirectVoxGO (bounded), rgbnet_dim 9, rgbnet_direct, on a non-cubic box with a mask cache with holes
           (configs/free_dataset/lab.py);

each at fast_color_thres 0 and 1e-3 (the configs' value).  A record holds the constructor kwargs, the state dict (for grass
without the two grids, which tests.test_gpu_k0_c9.golden_grids regenerates from `grid_seed`), the rays, the forward outputs, and
the gradients of the density grid, the k0 grid and the rgbnet for a seeded scalar functional of them.  Every file stays under
about 1 MB.

    python -m oracle.make_golden_free       # from the repo root, where /root/reference exists
"""
import contextlib
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, 'tests', 'golden', 'l2_free')
sys.path.insert(0, ROOT)

from oracle.make_golden import _c, _grab, _rays  # noqa: E402  (installs the stand-ins and the reference path)
from oracle.make_golden_dvgo import _model as _dvgo_model, _rays as _box_rays  # noqa: E402
from FourierGrid import FourierGrid_model as ref_fgmodel  # noqa: E402

from tests.test_gpu_k0_c9 import GOLDEN, GOLDEN_THRES, golden_grids  # noqa: E402

SEED = 999


def _flat(rec):
    """Without a threshold the reference returns the per-sample records as [N, S]; store them flat, in ray_id / step_id order."""
    M = rec['ray_id'].numel()
    for k, v in rec.items():
        if torch.is_tensor(v) and v.dim() == 2 and v.numel() == M:
            rec[k] = v.reshape(-1)
    return rec


def record(name, spec, thres):
    torch.manual_seed(SEED)
    kw = dict(spec['kw'], fast_color_thres=thres)
    gen = torch.Generator().manual_seed(SEED + 1)
    N = spec['rays']
    out = dict(cls=spec['cls'], kwargs=kw)
    if spec['cls'] == 'FourierGridModel':
        m = ref_fgmodel.FourierGridModel(**kw)
        grid_seed = SEED + 10 * list(GOLDEN).index(name) + (1 if thres > 0 else 0)
        dens, k0 = golden_grids(m.density.grid.shape, m.k0.grid.shape, grid_seed)
        with torch.no_grad():
            m.density.grid.copy_(dens)
            m.k0.grid.copy_(k0)
        ro, rd, vd = _rays(N, gen)
        # the reference's depth multiplies the weights by the unmasked t-table when no threshold compacts the samples
        rk = dict(near=0.0, far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False,
                  render_depth=thres > 0)
        out['grid_seed'] = grid_seed
    else:
        with contextlib.redirect_stdout(io.StringIO()):
            m = _dvgo_model(kw, gen)
        ro, rd, vd = _box_rays(N, gen)
        rk = dict(near=0.2, far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=True, flip_x=False, flip_y=False,
                  render_depth=True)
    ret = m(ro, rd, vd, global_step=None, is_train=False, **rk)
    lw = dict(rgb=torch.randn(N, 3, generator=gen), last=torch.randn(N, generator=gen))
    rec = _flat(_grab(m, ret, lw))
    skip = ('density.grid', 'k0.grid') if 'grid_seed' in out else ()
    out.update(state={k: _c(v) for k, v in m.state_dict().items() if k not in skip}, rays_o=ro, rays_d=rd, viewdirs=vd,
               render_kwargs=rk, loss_w=lw, ret=rec)
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f'{name}_t{thres:g}.pt')
    torch.save(out, path)
    print(f'{os.path.relpath(path, ROOT)}: {os.path.getsize(path) / 1024:.1f} KiB, {int(rec["ray_id"].numel())} survivors')


if __name__ == '__main__':
    torch.set_num_threads(4)
    for name, spec in GOLDEN.items():
        for thres in GOLDEN_THRES:
            record(name, spec, thres)
