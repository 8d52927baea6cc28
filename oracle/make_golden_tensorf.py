"""oracle/make_golden_tensorf.py -- TEST INFRASTRUCTURE ONLY.  Generates tests/golden/l2_tensorf/.

Runs the reference's UNMODIFIED FourierGrid/grid.py (TensoRFGrid) and dvgo.py (DirectVoxGO with TensoRF grids) on CPU over the
oracle stand-ins of oracle/stubs.py, seeded, and records:

* ``grid_<tag>.pt``: a TensoRFGrid built under a recorded seed (its parameters), a fixed point set with points on faces, edges
  and outside the box, the forward, the gradients of every factor for a fixed functional, get_dense_grid, scale_volume_grid and
  total_variation_add_grad, at non-cubic sizes, R != Rxy and C = 1 / 3 / 12;
* ``model.pt``: a TensoRF DirectVoxGO (density R = 2, 12-channel k0 with R = 3) forward and the gradients of a fixed functional,
  update_occupancy_cache and scale_volume_grid from the recorded state; ``model_last.tar``: its checkpoint as run_train.py writes it.

    python -m oracle.make_golden_tensorf      # from the repo root, where the reference checkout exists
"""
import contextlib
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden import OUT, SEED, _c, _grab, _save  # noqa: E402  (installs the stand-ins and the reference path)
from oracle.make_golden_dvgo import RK, _rays  # noqa: E402
from FourierGrid import dvgo as ref_dvgo  # noqa: E402
from FourierGrid import grid as ref_grid  # noqa: E402

DIR = os.path.join(OUT, 'l2_tensorf')
LO, HI = [-1.0, -1.3, -0.6], [1.1, 1.2, 0.8]          # non-cubic

# tag: (world_size, config, channels)
GRIDS = {
    'r3xy2_c1': ([23, 17, 11], dict(n_comp=3, n_comp_xy=2), 1),
    'r3xy2_c3': ([23, 17, 11], dict(n_comp=3, n_comp_xy=2), 3),
    'r3xy2_c12': ([19, 13, 9], dict(n_comp=3, n_comp_xy=2), 12),
    'r8_c1': ([12, 9, 2], dict(n_comp=8), 1),
    'r24_c12': ([9, 7, 5], dict(n_comp=24), 12),
}


def _quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def _points(gen, n=400):
    """Uniform points over a box 10% larger than the grid's (some outside), plus points on faces, edges and corners."""
    lo, hi = torch.tensor(LO), torch.tensor(HI)
    ext = (hi - lo) * 0.1
    p = lo - ext + torch.rand(n, 3, generator=gen) * (hi - lo + 2 * ext)
    special = []
    for i in range(8):
        corner = torch.where(torch.tensor([(i >> a) & 1 for a in range(3)]).bool(), hi, lo)
        special.append(corner)
    for a in range(3):
        for v in (lo[a], hi[a]):
            q = lo + torch.rand(3, generator=gen) * (hi - lo)
            q[a] = v
            special.append(q)
            e = q.clone()
            e[(a + 1) % 3] = lo[(a + 1) % 3]
            special.append(e)
    return torch.cat([p, torch.stack(special)]).contiguous()


def golden_grids():
    for i, (tag, (ws, cfg, C)) in enumerate(GRIDS.items()):
        seed = SEED + 40 + i
        torch.manual_seed(seed)
        g = ref_grid.TensoRFGrid(C, torch.tensor(ws), torch.tensor(LO), torch.tensor(HI), cfg)
        init = {k: _c(v) for k, v in g.state_dict().items()}
        gen = torch.Generator().manual_seed(seed)
        xyz = _points(gen)
        w = torch.randn(xyz.shape[0], C, generator=gen).squeeze(-1)
        out = g(xyz)
        (out * w).sum().backward()
        grads = {k: _c(p.grad) for k, p in g.named_parameters()}
        dense = _c(g.get_dense_grid())
        for p in g.parameters():
            p.grad = None
        wx, wy, wz = 0.7, 1.3, 0.4
        _quiet(g.total_variation_add_grad, wx, wy, wz, True)
        tv = {k: _c(p.grad) for k, p in g.named_parameters() if p.grad is not None}
        new_ws = [int(v * 1.4) + 1 for v in ws]
        g.scale_volume_grid(new_ws)
        scaled = {k: _c(v) for k, v in g.state_dict().items()}
        _save(os.path.join('l2_tensorf', f'grid_{tag}.pt'),
              dict(seed=seed, channels=C, world_size=ws, config=cfg, xyz_min=LO, xyz_max=HI, state=init, xyz=xyz, loss_w=w, out=_c(out),
                   grads=grads, dense=dense, tv_w=(wx, wy, wz), tv=tv, new_world_size=new_ws, scaled=scaled))


KW = dict(xyz_min=LO, xyz_max=HI, num_voxels=14 ** 3, num_voxels_base=14 ** 3, alpha_init=1e-2, fast_color_thres=1e-4,
          density_type='TensoRFGrid', density_config=dict(n_comp=2), k0_type='TensoRFGrid', k0_config=dict(n_comp=3),
          rgbnet_dim=12, rgbnet_direct=True, rgbnet_width=128, rgbnet_depth=3, viewbase_pe=4)


def golden_model():
    seed = SEED + 50
    torch.manual_seed(seed)
    m = _quiet(ref_dvgo.DirectVoxGO, **KW)
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        # an object in the box: the density's vectors peak mid-axis, so the products leave free space around it
        for name in ('x_vec', 'y_vec', 'z_vec'):
            v = getattr(m.density, name)
            L = v.shape[2]
            prof = 1.5 - 6.0 * torch.linspace(-1, 1, L) ** 2
            v.copy_(prof[None, None, :, None] + 0.3 * torch.randn(v.shape, generator=gen))
        for name in ('xy_plane', 'xz_plane', 'yz_plane'):
            p = getattr(m.density, name)
            p.copy_(1.0 + 0.3 * torch.randn(p.shape, generator=gen))
        m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=gen) < 0.9)
    state = {k: _c(v) for k, v in m.state_dict().items()}
    N = 64
    ro, rd, vd = _rays(N, gen)
    ret = m(ro, rd, vd, global_step=None, **RK)
    lw = dict(rgb=torch.randn(N, 3, generator=gen), last=torch.randn(N, generator=gen))
    rec = _grab(m, ret, lw)
    with torch.no_grad():
        m.update_occupancy_cache()
        occ = _c(m.mask_cache.mask)
        _quiet(m.scale_volume_grid, 17 ** 3)
        scaled = {k: _c(v) for k, v in m.state_dict().items() if not k.startswith('rgbnet')}
    os.makedirs(DIR, exist_ok=True)
    torch.save({'global_step': 3, 'model_kwargs': m.get_kwargs(), 'model_state_dict': m.state_dict(), 'optimizer_state_dict': {}},
               os.path.join(DIR, 'model_last.tar'))
    print(f'model_last.tar: {os.path.getsize(os.path.join(DIR, "model_last.tar")) / 1024:.1f} KiB')
    _save(os.path.join('l2_tensorf', 'model.pt'),
          dict(seed=seed, kwargs=KW, get_kwargs=m.get_kwargs(), state=state,
               state_shapes={k: tuple(v.shape) for k, v in state.items()}, rays_o=ro, rays_d=rd, viewdirs=vd, render_kwargs=RK,
               loss_w=lw, ret=rec, occupancy=occ, scale_num_voxels=17 ** 3, scaled=scaled))


if __name__ == '__main__':
    torch.set_num_threads(4)
    golden_grids()
    golden_model()
