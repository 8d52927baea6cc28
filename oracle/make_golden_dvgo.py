"""oracle/make_golden_dvgo.py -- TEST INFRASTRUCTURE ONLY.  Generates tests/golden/l2_dvgo/.

Runs the reference's UNMODIFIED FourierGrid/dvgo.py (DirectVoxGO, the bounded-scene model) on CPU over the oracle stand-ins of
oracle/stubs.py, like oracle/make_golden.py does for the other models, and records seeded inputs and the reference's outputs:

* ``coarse.pt`` / ``fine.pt``: the coarse-stage model (rgbnet_dim 0, k0 C = 3) and the fine-stage model (C = 12, rgbnet_direct)
  on a non-cubic box with a mask cache with holes: forward outputs and the gradients of a fixed functional;
* ``maint.pt``: maskout_near_cam_vox, voxel_count_views, scale_volume_grid (grids and the rebuilt mask) and
  update_occupancy_cache, each from a recorded state;
* ``coarse_last.tar``: a coarse checkpoint written the way run_train.py:313-331 writes it; ``fine_mask.pt``: the mask_cache.mask of
  a fine model the reference builds from that file with mask_cache_path; ``fine_last.tar``: that fine model's checkpoint, whose
  model_kwargs carry the (relative) path.

The reference's MaskGrid(path) calls plain torch.load, which since torch 2.6 loads with weights_only=True and refuses the NumPy
arrays in model_kwargs; the NumPy globals those files need are allow-listed here (the reference file stays as it is).  Runs on its
own, so no other fixture is regenerated:

    python -m oracle.make_golden_dvgo      # from the repo root, where the reference checkout exists
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden import OUT, SEED, _c, _grab, _save  # noqa: E402  (installs the stand-ins and the reference path)
from FourierGrid import dvgo as ref_dvgo  # noqa: E402

DIR = os.path.join(OUT, 'l2_dvgo')
LO, HI = [-1.0, -1.3, -0.6], [1.1, 1.2, 0.8]          # non-cubic
RK = dict(near=0.2, far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False, render_depth=True)


def _quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def _allow_numpy():
    g = [np.ndarray, np.dtype, type(np.dtype(np.float32))]
    try:
        g.append(np._core.multiarray._reconstruct)
    except AttributeError:
        g.append(np.core.multiarray._reconstruct)
    torch.serialization.add_safe_globals(g)


def _rays(n, gen):
    """Cameras on a shell around the box looking at points inside it, plus rays that miss, start inside and have a zero
    direction component."""
    lo, hi = torch.tensor(LO), torch.tensor(HI)
    c = (lo + hi) / 2
    o = torch.randn(n, 3, generator=gen)
    o = c + o / o.norm(dim=-1, keepdim=True) * 3.0
    d = c + (torch.rand(n, 3, generator=gen) - 0.5) * (hi - lo) - o
    o[0], d[0] = torch.tensor([5., 5., 5.]), torch.tensor([1., 0.2, 0.1])          # misses
    o[1], d[1] = c, torch.tensor([0.3, -0.2, 0.9])                                  # starts inside
    o[2], d[2] = torch.tensor([-3., 0.1, 0.2]), torch.tensor([1., 0., 0.])          # zero components
    return o.contiguous(), d.contiguous(), (d / d.norm(dim=-1, keepdim=True)).contiguous()


def _model(kw, gen, mask_p=0.85):
    m = _quiet(ref_dvgo.DirectVoxGO, **kw)
    with torch.no_grad():
        X, Y, Z = [int(v) for v in m.world_size]
        ax = [torch.linspace(-1, 1, k) for k in (X, Y, Z)]
        r2 = sum(a ** 2 for a in torch.meshgrid(*ax, indexing='ij'))
        m.density.grid.copy_((6.0 * (0.5 - r2) + torch.randn(X, Y, Z, generator=gen))[None, None])
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=gen))
        m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=gen) < mask_p)
    return m


KW_COARSE = dict(xyz_min=LO, xyz_max=HI, num_voxels=16 ** 3, num_voxels_base=16 ** 3, alpha_init=1e-6, fast_color_thres=1e-7,
                 rgbnet_dim=0)
KW_FINE = dict(xyz_min=LO, xyz_max=HI, num_voxels=14 ** 3, num_voxels_base=16 ** 3, alpha_init=1e-2, fast_color_thres=1e-4,
               rgbnet_dim=12, rgbnet_direct=True, rgbnet_width=128, rgbnet_depth=3, viewbase_pe=4)


def golden_models():
    for tag, kw in (('coarse', KW_COARSE), ('fine', KW_FINE)):
        gen = torch.Generator().manual_seed(SEED + 30)
        torch.manual_seed(SEED + 30)
        m = _model(kw, gen)
        N = 48
        ro, rd, vd = _rays(N, gen)
        ret = m(ro, rd, vd, global_step=None, **RK)
        lw = dict(rgb=torch.randn(N, 3, generator=gen), last=torch.randn(N, generator=gen))
        rec = _grab(m, ret, lw)
        _save(os.path.join('l2_dvgo', tag + '.pt'),
              dict(kwargs=kw, get_kwargs=m.get_kwargs(), state=m.state_dict(), state_shapes={k: tuple(v.shape) for k, v in
                                                                                              m.state_dict().items()},
                   rays_o=ro, rays_d=rd, viewdirs=vd, render_kwargs=RK, loss_w=lw, ret=rec))


def golden_maint():
    gen = torch.Generator().manual_seed(SEED + 31)
    torch.manual_seed(SEED + 31)
    m = _model(KW_COARSE, gen, mask_p=1.0)
    rec = dict(kwargs=KW_COARSE, state=m.state_dict())
    with torch.no_grad():
        cams = torch.tensor([[0.9, 1.1, 0.7], [-0.9, -1.2, -0.5], [3., 3., 3.]])
        m.maskout_near_cam_vox(cams, 0.4)
        rec['maskout'] = dict(cam_o=cams, near_clip=0.4, density=_c(m.density.grid))
    n_views, H, W = 2, 6, 8
    ro, rd, _ = _rays(n_views * H * W, gen)
    ro, rd = ro.reshape(n_views * H, W, 3), rd.reshape(n_views * H, W, 3)
    cnt = _quiet(m.voxel_count_views, ro, rd, [H] * n_views, 0.2, 1e9, 0.5)
    rec['count_views'] = dict(rays_o=ro, rays_d=rd, imsz=[H] * n_views, near=0.2, far=1e9, stepsize=0.5, count=_c(cnt))
    with torch.no_grad():
        m.update_occupancy_cache()
        rec['occupancy'] = dict(mask=_c(m.mask_cache.mask))
        _quiet(m.scale_volume_grid, 21 ** 3)
        rec['scale'] = dict(num_voxels=21 ** 3, world_size=_c(m.world_size), density=_c(m.density.grid), k0=_c(m.k0.grid),
                            mask=_c(m.mask_cache.mask))
    _save(os.path.join('l2_dvgo', 'maint.pt'), rec)


def golden_coarse_to_fine():
    """coarse_last.tar as run_train.py:313-331 writes it, the fine mask the reference builds from it (dvgo.py:138-152), and the
    fine checkpoint whose model_kwargs carry the path.  The path is relative to tests/golden/l2_dvgo/."""
    gen = torch.Generator().manual_seed(SEED + 32)
    torch.manual_seed(SEED + 32)
    coarse = _model(dict(KW_COARSE, xyz_min=np.array(LO, dtype=np.float32), xyz_max=np.array(HI, dtype=np.float32)), gen)
    with torch.no_grad():
        coarse.density.grid.add_(8.0)          # alpha_init 1e-6: a trained coarse object clears mask_cache_thres inside only
    os.makedirs(DIR, exist_ok=True)
    cwd = os.getcwd()
    os.chdir(DIR)
    try:
        torch.save({'global_step': 5000, 'model_kwargs': coarse.get_kwargs(), 'model_state_dict': coarse.state_dict(),
                    'optimizer_state_dict': {}}, 'coarse_last.tar')
        _allow_numpy()
        fine_kw = dict(KW_FINE, xyz_min=np.array(LO, dtype=np.float32), xyz_max=np.array(HI, dtype=np.float32),
                       mask_cache_path='coarse_last.tar', mask_cache_thres=1e-3,
                       mask_cache_world_size=[int(v) for v in coarse.world_size])
        fine = _quiet(ref_dvgo.DirectVoxGO, **fine_kw)
        with torch.no_grad():
            fine.density.grid.copy_(torch.randn(fine.density.grid.shape, generator=gen))
            fine.k0.grid.copy_(torch.randn(fine.k0.grid.shape, generator=gen))
        torch.save({'global_step': 20000, 'model_kwargs': fine.get_kwargs(), 'model_state_dict': fine.state_dict(),
                    'optimizer_state_dict': {}}, 'fine_last.tar')
    finally:
        os.chdir(cwd)
    for f in ('coarse_last.tar', 'fine_last.tar'):
        print(f'{f}: {os.path.getsize(os.path.join(DIR, f)) / 1024:.1f} KiB')
    _save(os.path.join('l2_dvgo', 'fine_mask.pt'), dict(mask=_c(fine.mask_cache.mask), mask_cache_thres=1e-3,
                                                      mask_cache_world_size=[int(v) for v in coarse.world_size]))


if __name__ == '__main__':
    torch.set_num_threads(4)
    golden_models()
    golden_maint()
    golden_coarse_to_fine()
