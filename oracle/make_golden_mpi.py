"""oracle/make_golden_mpi.py -- TEST INFRASTRUCTURE ONLY.  Generates tests/golden/l2_mpi/*.pt.

Runs the reference's UNMODIFIED FourierGrid/dmpigo.py (DirectMPIGO, the forward-facing NDC model) on CPU over the oracle
stand-ins of oracle/stubs.py, like oracle/make_golden.py does for the other models, and records seeded inputs and the
reference's outputs.  Runs on its own, so the existing fixtures are not regenerated:

    python -m oracle.make_golden_mpi      # from the repo root, where the reference checkout exists
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden import SEED, _c, _grab, _save  # noqa: E402  (installs the stand-ins and the reference path)
from FourierGrid import dmpigo as ref_dmpigo  # noqa: E402

RK = dict(near=0., far=1., bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False, render_depth=True)


def _quiet(fn, *a, **k):
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def _kwargs_rec(kw):
    return {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in kw.items()}


def _ndc_rays(n, gen, xy_spread):
    """Forward-facing NDC rays: origins on the z = -1 plane, z-component of the direction ~2 (ndc_rays, dvgo.py:532-550); some
    rays leave the box sideways and some end beyond z = 1, so the bbox drop is exercised."""
    ro = torch.cat([(torch.rand(n, 2, generator=gen) - 0.5) * 2 * xy_spread, -torch.ones(n, 1)], -1)
    rd = torch.cat([torch.randn(n, 2, generator=gen) * 0.3, 2.0 + torch.randn(n, 1, generator=gen) * 0.05], -1)
    vd = rd / rd.norm(dim=-1, keepdim=True)
    return ro.contiguous(), rd.contiguous(), vd.contiguous()


def golden_mpi_models():
    cases = {
        'mpi_rgb9': dict(kw=dict(xyz_min=[-1.2, -1.0, -1.0], xyz_max=[1.2, 1.0, 1.0], num_voxels=8000, mpi_depth=16,
                                 fast_color_thres=1e-3, rgbnet_dim=9, rgbnet_width=64), dstd=2.0, dmean=1.0, mask=True),
        'mpi_rgb0': dict(kw=dict(xyz_min=[-1.2, -1.0, -1.0], xyz_max=[1.2, 1.0, 1.0], num_voxels=8000, mpi_depth=16,
                                 fast_color_thres=0, rgbnet_dim=0), dstd=2.0, dmean=0.0, mask=False),
    }
    for tag, c in cases.items():
        gen = torch.Generator().manual_seed(SEED + 20)
        torch.manual_seed(SEED + 20)
        m = _quiet(ref_dmpigo.DirectMPIGO, **c['kw'])
        with torch.no_grad():
            m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=gen) * c['dstd'] + c['dmean'])
            m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=gen))
            if c['mask']:
                m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=gen) > 0.15)
        N = 40
        ro, rd, vd = _ndc_rays(N, gen, 1.2)
        ret = m(ro, rd, vd, global_step=None, **RK)
        lw = dict(rgb=torch.randn(N, 3, generator=gen), last=torch.randn(N, generator=gen))
        rec = _grab(m, ret, lw)
        _save(os.path.join('l2_mpi', tag + '.pt'),
              dict(kwargs=c['kw'], state=m.state_dict(), rays_o=ro, rays_d=rd, viewdirs=vd, render_kwargs=RK, loss_w=lw, ret=rec))


def golden_mpi_constructor():
    """What the reference's constructor computes for a few bboxes / mpi_depths / rgbnet widths, and its TV weights."""
    cases = []
    for xyz_min, xyz_max, nv, depth, dim in (([-1.2, -1.0, -1.0], [1.2, 1.0, 1.0], 13500, 16, 9),
                                             ([-1.5, -0.9, -1.0], [1.4, 0.8, 1.0], 64 ** 3, 32, 9),
                                             ([-1.37, -1.05, -1.0], [1.29, 1.11, 1.0], 96 ** 3, 48, 0),
                                             ([-1.0, -1.0, -1.0], [1.0, 1.0, 1.0], 100 ** 3, 64, 0)):
        kw = dict(xyz_min=np.array(xyz_min, dtype=np.float32), xyz_max=np.array(xyz_max, dtype=np.float32), num_voxels=nv,
                  mpi_depth=depth, fast_color_thres=1e-3, rgbnet_dim=dim, rgbnet_width=64)
        m = _quiet(ref_dmpigo.DirectMPIGO, **kw)
        tv = {}
        for name in ('density', 'k0'):
            calls = []
            grid = getattr(m, name)
            grid.total_variation_add_grad = lambda wx, wy, wz, dense, calls=calls: calls.append((float(wx), float(wy), float(wz)))
            getattr(m, f'{name}_total_variation_add_grad')(1e-6 / 4096, True)
            tv[name] = calls[0]
        cases.append(dict(kwargs=_kwargs_rec(kw), world_size=_c(m.world_size), voxel_size_ratio=m.voxel_size_ratio,
                          act_shift=_c(m.act_shift.grid), get_kwargs=_kwargs_rec(m.get_kwargs()),
                          state_shapes={k: tuple(v.shape) for k, v in m.state_dict().items()}, tv=tv, tv_weight=1e-6 / 4096))
    _save(os.path.join('l2_mpi', 'constructor.pt'), cases)


if __name__ == '__main__':
    torch.set_num_threads(4)
    golden_mpi_models()
    golden_mpi_constructor()
