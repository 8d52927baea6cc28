"""GPU: the fused marches at C = 9, the k0 width of the reference's free-dataset configs -- grass (FourierGridModel, rgbnet_dim 9,
width 64, fourier_freq_num 3: P = 7 slabs) and lab (DirectVoxGO, bounded, rgbnet_dim 9, width 64) -- and of DirectContractedVoxGO
with rgbnet_dim 9.

* contracted: fused forward vs forward_ops (identical survivors, bit-identical raw_density / raw_alpha / weights / alphainv_last,
  k0 bit-identical to F.grid_sample(...).mean(0)); the k0 scatter element by element against the fp64 adjoint of
  tests/test_gpu_march_scatter.py under every feature-kernel selection and at every 4-byte phase of the grid's base address;
* box (DirectVoxGO): fused vs forward_ops, ray geometries, the k0 scatter against the fp64 adjoint, rand_bkgd;
* the reference's own code: fixtures of oracle/make_golden_free.py, and its GPU path at a C = 9 size;
* the reference's unmodified run_train.scene_rep_reconstruction on grass- and lab-like configs;
* grass's 250^3, P = 7 grids with 4096 rays.
"""
import os

import numpy as np
import pytest
import torch

from tests.test_gpu_march_scatter import (Contracted, _ragged_structure, as_pxyzc, cells, judge as judge_scatter, ref_gather,
                                          ref_scatter, selections, slab_coords)  # noqa: F401 (fixture)
from tests.test_gpu_train_driver import ref  # noqa: F401 (fixture)
from tests.util import assert_close, assert_equal, seeded_rays

DEV = 'cuda:0'
C9 = 9
RK = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, render_depth=True)


def _timed_keys(fn):
    """The _cabi.timed launch names a call records."""
    from unboundednerfpytorch_b200 import _cabi
    timer, _cabi.TIMER = _cabi.TIMER, _cabi.KernelTimer()
    try:
        out = fn()
        return out, set(_cabi.TIMER.records)
    finally:
        _cabi.TIMER = timer


# ---- contracted: FourierGridModel (F > 0, P = 2 F + 1) and DirectContractedVoxGO (F = 0, P = 1) ----------------------------
def contracted_model(F_, norm='inf', thres=0.0, world=24, seed=0, viewbase_pe=4, dens_mean=0.0, dens_std=1.0):
    from unboundednerfpytorch_b200 import models
    torch.manual_seed(seed)
    common = dict(alpha_init=1e-4, fast_color_thres=thres, rgbnet_dim=C9, rgbnet_width=64, contracted_norm=norm,
                  viewbase_pe=viewbase_pe)
    if F_ > 0:
        m = models.FourierGridModel(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=world ** 3,
                                    num_voxels_base_density=world ** 3, num_voxels_rgb=world ** 3, num_voxels_base_rgb=world ** 3,
                                    num_voxels_viewdir=-1, fourier_freq_num=F_, **common)
    else:
        m = models.DirectContractedVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=world ** 3, num_voxels_base=world ** 3,
                                         **common)
    assert tuple(m.k0.grid.shape[:2]) == (2 * F_ + 1, C9)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=g) * dens_std + dens_mean)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
    return m.to(DEV)


FWD_CASES = [(F_, norm, thres) for F_ in (0, 1, 3, 4, 5) for norm in ('inf', 'l2') for thres in (0.0, 1e-3)]


def _fused_vs_ops(m, F_, ro, rd, vd, min_survivors):
    from oracle import cpu_ref
    assert m._fused_ok()
    with torch.no_grad():
        fused, keys = _timed_keys(lambda: m(ro, rd, vd, **RK))
    # forward reached the fused march and the tensor-core (9, 64) rgbnet, not the op-by-op path
    assert {'march_density_fwd', 'march_feature_fwd', 'rgbnet_fwd'} <= keys, keys
    with torch.no_grad():
        ops_ = m.forward_ops(ro, rd, vd, **RK)
        (w, last, alpha, dens, k0, ray_id, step_id, t, inner), _ = m._march(ro, rd, RK['stepsize'])
        pts, _, _ = m._sample_dense(ro, rd, RK['stepsize'])
        want = cpu_ref.fourier_grid_forward(m.k0.grid.detach().contiguous(), pts[ray_id, step_id], m.xyz_min, m.xyz_max, F_)
    assert fused['ray_id'].numel() > min_survivors
    assert_equal(fused['ray_id'], ops_['ray_id'], 'ray_id')
    assert_equal(fused['step_id'], ops_['step_id'], 'step_id')
    for k in ('raw_density', 'raw_alpha', 'weights', 'alphainv_last'):
        assert_equal(fused[k], ops_[k], k)
    assert_equal(k0, want, f'k0 C=9 P={2 * F_ + 1} vs F.grid_sample(...).mean(0)')
    assert_close(fused['rgb_marched'], ops_['rgb_marched'], rtol=1e-4, atol=1e-5, what='rgb_marched fused vs forward_ops')
    return fused, k0


@pytest.mark.gpu
@pytest.mark.parametrize('F_,norm,thres', FWD_CASES, ids=[f'P{2 * f + 1}-{n}-t{t:g}' for f, n, t in FWD_CASES])
def test_contracted_fused_vs_ops_and_grid_sample(F_, norm, thres):
    m = contracted_model(F_, norm, thres, dens_mean=5.0 if thres else 0.0, dens_std=3.0 if thres else 1.0, seed=9 + F_)
    ro, rd, vd = seeded_rays(300, 14 + F_, DEV)
    _fused_vs_ops(m, F_, ro, rd, vd, 500)


@pytest.mark.gpu
def test_coherent_rays_take_the_gather():
    """The TMA-staged render read is 12-channel only: a render forward with coherent_rays on a C = 9 model runs the gather and
    gives its result bit for bit."""
    from unboundednerfpytorch_b200 import march
    m = contracted_model(3, 'inf', 1e-3, dens_mean=5.0, dens_std=3.0, seed=4)
    assert not march.tma_supported(m.k0.grid)
    ro, rd, vd = seeded_rays(256, 21, DEV)
    with torch.no_grad():
        a, keys = _timed_keys(lambda: m(ro, rd, vd, coherent_rays=True, **RK))
        b = m(ro, rd, vd, **RK)
    assert 'march_feature_fwd' in keys and 'march_feature_fwd_tma' not in keys, keys
    for k in ('ray_id', 'weights', 'rgb_marched', 'raw_rgb'):
        assert_equal(a[k], b[k], k)


# ---- the contracted k0 scatter against the fp64 adjoint -------------------------------------------------------------------
class Wide9(Contracted):
    """The scatter test's contracted scene with a 9-channel k0 grid."""

    def __init__(self, **kw):
        super().__init__(**kw)
        X, Y, Z = self.shape
        self.kvals = torch.randn(self.P, X, Y, Z, C9, generator=torch.Generator().manual_seed(7 * C9 + self.P)).to(DEV)

    def run_at_phase(self, phase, g_feat=None, g_dens=None):
        """march.March with the k0 grid and its gradient buffer both starting `phase` floats past a 16-byte boundary."""
        from unboundednerfpytorch_b200 import grid as G
        from unboundednerfpytorch_b200 import march
        dg = self.dgrid.clone().requires_grad_(True)
        kg = at_phase(self.kvals, phase).requires_grad_(True)
        kbuf = at_phase(torch.zeros_like(self.kvals), phase)
        kg._ubn_grad_buffer = kbuf
        kdesc = G.grid_desc(kg, self.mn, self.mx, self.n_freqs)
        out = march.March.apply(dg, kg, self.ro, self.rd, self.t_table, None, self.cfg, self.ddesc, kdesc, self.thres <= 0, False)
        feat, dens, ray_id, step_id = out[4], out[3], out[5], out[6]
        if g_feat is not None:
            ((feat * g_feat).sum() + (dens * g_dens).sum()).backward()
            assert kg.grad is kbuf
        return dict(feat=feat.detach(), ray_id=ray_id, step_id=step_id, gk=kbuf)


def at_phase(vals, phase):
    """[P, X, Y, Z, C] values copied into storage that starts `phase` floats (4 * phase bytes) past a 16-byte boundary, as the
    channels-last [P, C, X, Y, Z] view the models use."""
    n = vals.numel()
    store = torch.zeros(n + 4, device=vals.device)
    assert store.data_ptr() % 16 == 0
    v = store[phase:phase + n].view(vals.shape)
    v.copy_(vals)
    return v.permute(0, 4, 1, 2, 3)


SHAPE = (23, 37, 41)            # odd X * Y * Z, X - 1 = 22 not divisible by 4
SHAPE4 = (41, 23, 37)           # X - 1 = 40 divisible by 4
SCATTER = {
    'P1': dict(P=1, shape=SHAPE), 'P3': dict(P=3, shape=SHAPE4), 'P5': dict(P=5, shape=SHAPE), 'P7': dict(P=7, shape=SHAPE4),
    'P7-l2': dict(P=7, shape=SHAPE, norm='l2'), 'P9': dict(P=9, shape=SHAPE4, n_far=32), 'P11': dict(P=11, shape=SHAPE),
    'P7-X2': dict(P=7, shape=(2, 37, 41)), 'P5-X5': dict(P=5, shape=(5, 37, 41)), 'P11-X3': dict(P=11, shape=(3, 23, 37)),
    'P7-ragged': dict(P=7, shape=SHAPE4, thres=1e-4, world_len=41, stepsize=0.5, n_x=768, n_rand=64, n_far=16),
    'P1-ragged': dict(P=1, shape=SHAPE4, thres=1e-4, world_len=41, stepsize=0.5, n_x=768, n_rand=64, n_far=16),
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(SCATTER))
def test_contracted_k0_scatter_vs_fp64(case, selections):
    """Every feature-kernel selection (0 .. 6: x-range splits 1 / 2 / 4) and every 4-byte phase of the grid's base address against
    the fp64 adjoint, the forward against the fp64 gather of the same cells.  Structural claims (record phases, runs of samples in
    one cell, chunks with 1 and with 32 survivors) are asserted from the data."""
    ops = selections
    sc = Wide9(**SCATTER[case])
    P, shape = sc.P, sc.shape
    ops.set_feature_kernel(5)
    base = sc.run_at_phase(0)
    ray_id, step_id = base['ray_id'], base['step_id']
    M = ray_id.numel()
    assert M > 1000, f'{case}: only {M} survivors'
    cs = slab_coords(sc.points(ray_id, step_id), sc.mn, sc.mx, sc.n_freqs)
    x0, f = cells(cs, shape)
    X, Y, Z = shape
    v = (x0[..., 0] * Y + x0[..., 1]) * Z + x0[..., 2]
    # every 4-byte phase of a 36-byte record's start occurs among the corners (before the base offset moves them all)
    phases = {int(p) for p in torch.unique(((v[..., None] + torch.tensor([0, 1, Z, Y * Z], device=DEV)) * C9) % 4)}
    assert phases == {0, 1, 2, 3}, f'{case}: record phases {phases}'
    # consecutive survivors of a ray in one slab-0 cell: the run scatter sums them in registers
    assert bool(((ray_id[1:] == ray_id[:-1]) & (v[0, 1:] == v[0, :-1])).any())
    if sc.thres > 0:                # chunks with one survivor (also on lane 31), full chunks, empty chunks, rays without survivors
        _ragged_structure(f'C=9 {case}', sc, ray_id, step_id, x0[0, :, 0])
    gen = torch.Generator(DEV).manual_seed(M)
    g_feat = torch.randn(M, C9, device=DEV, generator=gen)
    g_dens = torch.randn(M, device=DEV, generator=gen)
    want_k, bound_k = ref_scatter(x0, f, g_feat, shape)
    fk_want, fk_bound = ref_gather(x0, f, sc.kvals)
    fails = []
    for fk in range(7):
        ops.set_feature_kernel(fk)
        for phase in range(4):
            got = sc.run_at_phase(phase, g_feat, g_dens)
            what = f'C=9 {case} fk={fk} phase={phase}'
            try:
                assert torch.equal(got['ray_id'], ray_id) and torch.equal(got['step_id'], step_id), f'{what}: survivors differ'
                assert torch.equal(got['feat'], base['feat']), f'{what}: forward differs across selections / phases'
                judge_scatter(got['feat'][:, :, None], fk_want[:, :, None], fk_bound[:, :, None], what + ' k0 forward self-check',
                              'forward self-check', tau=1e-6)
                judge_scatter(as_pxyzc(got['gk']), want_k, bound_k, what + ' k0 scatter', f'k0 C=9 P={P}')
            except AssertionError as e:
                fails.append(str(e))
    assert not fails, '\n'.join(fails)


# ---- grass's size -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_grass_size():
    """configs/free_dataset/grass.py: 250^3, fourier_freq_num 3 (P = 7), rgbnet_dim 9 at width 64, fast_color_thres 1e-3, 4096 rays:
    fused vs forward_ops without a membership flip, bit-identical march outputs and k0."""
    m = contracted_model(3, 'inf', 1e-3, world=250, seed=5, dens_mean=5.0, dens_std=3.0)
    ro, rd, vd = seeded_rays(4096, 9, DEV)
    _fused_vs_ops(m, 3, ro, rd, vd, 10_000)


# ---- box: DirectVoxGO -------------------------------------------------------------------------------------------------------
def box_scene(nv=40 ** 3, n=2048, seed=3, thres=1e-4, mask_p=0.85):
    """tests/test_gpu_dvgo.py's object-in-a-non-cubic-box scene with a 9-channel k0 and the width-64 rgbnet of lab.py."""
    from tests.test_gpu_dvgo import HI, LO, _shell_rays
    from unboundednerfpytorch_b200 import models
    g = torch.Generator().manual_seed(seed)
    m = models.DirectVoxGO(xyz_min=LO, xyz_max=HI, num_voxels=nv, num_voxels_base=nv, alpha_init=1e-2, fast_color_thres=thres,
                           rgbnet_dim=C9, rgbnet_direct=True, rgbnet_width=64, rgbnet_depth=3)
    with torch.no_grad():
        X, Y, Z = [int(v) for v in m.world_size]
        ax = [torch.linspace(-1, 1, k) for k in (X, Y, Z)]
        r2 = sum(a ** 2 for a in torch.meshgrid(*ax, indexing='ij'))
        m.density.grid.copy_((6.0 * (0.5 - r2) + torch.randn(X, Y, Z, generator=g))[None, None])
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
        m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=g) < mask_p)
    ro, rd = _shell_rays(n, g)
    return m.to(DEV), ro, rd


def _box_compare(m, ro, rd, monkeypatch):
    """test_gpu_dvgo._compare (same ray_id, bit-identical raw_alpha / weights / alphainv_last / depth, colours and gradients as
    there), after checking that forward takes the fused box march and the tensor-core rgbnet."""
    from tests.test_gpu_dvgo import RK as BOX_RK, _compare, _vd
    with torch.no_grad():
        _, keys = _timed_keys(lambda: m(ro, rd, _vd(rd), **BOX_RK))
    assert {'march_box_density_fwd', 'march_box_feature_fwd', 'rgbnet_fwd'} <= keys, keys
    return _compare(m, ro, rd, C9, monkeypatch=monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize('thres', [0.0, 1e-4])
def test_box_fused_vs_forward_ops(thres, monkeypatch):
    m, ro, rd = box_scene(thres=thres)
    assert not bool(m.mask_cache.mask.all())
    ret = _box_compare(m, ro, rd, monkeypatch)
    assert len(ret['ray_id']) > 10 * len(ro)


@pytest.mark.gpu
def test_box_ray_geometry(monkeypatch):
    """Rays that miss the box, start inside it, have zero direction components, graze a face or an edge, or run the diagonal."""
    from tests.test_gpu_dvgo import HI, LO
    m, _, _ = box_scene(thres=1e-4)
    lo, hi = torch.tensor(LO), torch.tensor(HI)
    c = (lo + hi) / 2
    o = [torch.tensor([5., 5., 5.]), torch.tensor([-4., 0., 0.]), c, c + 0.1, torch.tensor([-3., 0.1, 0.2]),
         torch.tensor([0.1, -3., 0.2]), torch.tensor([-3., float(HI[1]), 0.1]), torch.tensor([-3., float(HI[1]), float(LO[2])]),
         lo - (hi - lo) * 0.5, hi]
    d = [torch.tensor([1., 0.2, 0.1]), torch.tensor([0., 1., 0.]), torch.tensor([0.3, -0.2, 0.9]), torch.tensor([-1., 0.5, 0.]),
         torch.tensor([1., 0., 0.]), torch.tensor([0., 1., 0.]), torch.tensor([1., 0., 0.]), torch.tensor([1., 0., 0.]), hi - lo,
         lo - hi]
    ro, rd = torch.stack(o).to(DEV), torch.stack(d).to(DEV)
    ret = _box_compare(m, ro, rd, monkeypatch)
    n_miss = 2
    assert not bool((ret['ray_id'] < n_miss).any())
    assert torch.equal(ret['alphainv_last'][:n_miss].cpu(), torch.ones(n_miss))
    hit = torch.bincount(ret['ray_id'], minlength=len(ro)).cpu()
    assert bool((hit[2:6] > 0).all()), hit          # the rays from inside and with zero components do march


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['C9', 'C9-longS'])
def test_box_k0_scatter_vs_fp64(case, selections, monkeypatch):
    """tests/test_gpu_march_scatter.py's box check at C = 9: BoxMarch's k0 scatter of 36-byte records (red.v4 / v2 / scalar by
    address) and the density scatter, on either side of the run scatter's limit."""
    from tests import test_gpu_march_scatter as scatter
    monkeypatch.setitem(scatter.BOX, case, dict(C=C9, stepdist=0.02 if case == 'C9' else 0.0013))
    scatter.test_box_scatter_vs_fp64(case, selections)


@pytest.mark.gpu
def test_box_rand_bkgd_uses_bg():
    """dvgo.py:406 adds alphainv_last * bg whatever rand_bkgd says (lab.py trains with rand_bkgd=True): a training forward with
    rand_bkgd is bit-identical to one without, and bg enters as alphainv_last * bg."""
    from tests.test_gpu_dvgo import RK as BOX_RK, _vd
    m, ro, rd = box_scene(thres=1e-3)
    rk = dict(BOX_RK, inverse_y=True)
    a = m(ro, rd, _vd(rd), global_step=1, is_train=True, **dict(rk, rand_bkgd=True))
    b = m(ro, rd, _vd(rd), global_step=1, is_train=True, **dict(rk, rand_bkgd=False))
    for k in ('rgb_marched', 'weights', 'alphainv_last', 'ray_id'):
        assert_equal(a[k], b[k], k)
    with torch.no_grad():
        c = m(ro, rd, _vd(rd), **dict(rk, bg=0.))
    assert_close(b['rgb_marched'] - c['rgb_marched'], b['alphainv_last'][:, None].expand(-1, 3), rtol=1e-6, atol=1e-6,
                 what='alphainv_last * bg')


@pytest.mark.gpu
def test_batch_without_survivors():
    """A training batch in which no sample survives (rays that miss DirectVoxGO's box; a FourierGridModel whose density keeps every
    alpha under fast_color_thres) runs forward and backward on the fused path and the width-64 rgbnet, whose backward then gets
    zero-sized buffers: the colour is the background term alone (DirectVoxGO adds alphainv_last * bg, FourierGridModel no background
    without rand_bkgd, FourierGrid_model.py:646) and every gradient is zero."""
    from tests.test_gpu_dvgo import RK as BOX_RK
    box, _, _ = box_scene(thres=1e-3)
    ro_box = torch.tensor([[5., 5., 5.]] * 4, device=DEV)
    rd_box = torch.tensor([[1., 0.2, 0.1]] * 4, device=DEV)
    fg = contracted_model(3, 'inf', 1e-3, dens_mean=-40.0, dens_std=1.0, seed=6)
    ro_fg, rd_fg, _ = seeded_rays(64, 8, DEV)
    for m, ro, rd, rk, bg in ((box, ro_box, rd_box, BOX_RK, 1.0), (fg, ro_fg, rd_fg, RK, 0.0)):
        for p in m.parameters():
            p.grad = None
        ret, keys = _timed_keys(lambda: m(ro, rd, rd / rd.norm(dim=-1, keepdim=True), global_step=1, is_train=True, **rk))
        assert ret['ray_id'].numel() == 0 and 'rgbnet_fwd' in keys, keys
        ret['rgb_marched'].pow(2).sum().backward()
        assert_equal(ret['rgb_marched'].detach(), ret['alphainv_last'].detach()[:, None].expand(-1, 3) * bg, 'background term')
        for name, p in m.named_parameters():
            assert p.grad is None or not bool(p.grad.any()), name


# ---- the reference's own code on the CPU: fixtures of oracle/make_golden_free.py ----------------------------------------------
LAB_LO, LAB_HI = [-1.0, -1.3, -0.6], [1.1, 1.2, 0.8]        # non-cubic, as a camera-frustum bbox is
GOLDEN = {
    # grass.py: FourierGrid, rgbnet_dim 9, width 64, fourier_freq_num 3 (default.py), viewbase_pe 4
    'grass': dict(cls='FourierGridModel', rays=96,
                  kw=dict(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=16 ** 3, num_voxels_base_density=16 ** 3,
                          num_voxels_rgb=10 ** 3, num_voxels_base_rgb=10 ** 3, num_voxels_viewdir=-1, alpha_init=1e-2, rgbnet_dim=9,
                          rgbnet_width=64, fourier_freq_num=3, viewbase_pe=4)),
    # lab.py: DVGO (bounded), rgbnet_dim 9, width 64, rgbnet_direct (default.py)
    'lab': dict(cls='DirectVoxGO', rays=128,
                kw=dict(xyz_min=LAB_LO, xyz_max=LAB_HI, num_voxels=16 ** 3, num_voxels_base=16 ** 3, alpha_init=1e-2, rgbnet_dim=9,
                        rgbnet_direct=True, rgbnet_width=64, rgbnet_depth=3, viewbase_pe=4)),
}
GOLDEN_THRES = (0.0, 1e-3)
GOLDEN_CASES = [(n, t, path) for n in GOLDEN for t in GOLDEN_THRES for path in ('fused', 'ops')]


def golden_grids(dens_shape, k0_shape, seed):
    """grass fixtures' density and k0 grids, regenerated from their seed (density centred at 4, see
    tests/test_gpu_fg_widths.golden_grids)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(dens_shape, generator=g) * 3 + 4.0, torch.randn(k0_shape, generator=g)


@pytest.mark.gpu
@pytest.mark.parametrize('name,thres,path', GOLDEN_CASES, ids=[f'{n}-t{t:g}-{p}' for n, t, p in GOLDEN_CASES])
def test_reference_fixtures(name, thres, path):
    """forward and forward_ops against the reference's FourierGrid_model.py / dvgo.py run on the CPU, at the golden tolerances of
    tests/test_gpu_models.py: sample ids bit-exact, outputs within 2e-5, gradients of the density grid, the k0 grid and the rgbnet
    within 5e-5 (+ 1e-5 of scale)."""
    from tests.test_gpu_models import _check_against_golden
    from tests.util import load_golden
    from unboundednerfpytorch_b200 import models
    rec = load_golden('l2_free.pt')[f'{name}_t{thres:g}']
    m = getattr(models, rec['cls'])(**rec['kwargs'])
    if 'grid_seed' in rec:
        dens, k0 = golden_grids(m.density.grid.shape, m.k0.grid.shape, rec['grid_seed'])
        missing, unexpected = m.load_state_dict(rec['state'], strict=False)
        assert not unexpected and sorted(missing) == ['density.grid', 'k0.grid'], (missing, unexpected)
        with torch.no_grad():
            m.density.grid.copy_(dens)
            m.k0.grid.copy_(k0)
    else:
        m.load_state_dict(rec['state'])
    m = m.to(DEV)
    assert m.k0.grid.shape[1] == C9
    if rec['cls'] == 'DirectVoxGO':
        assert m._fused_ok(rec['render_kwargs']['stepsize']) and not bool(m.mask_cache.mask.all())
    else:
        assert m._fused_ok()
    assert rec['ret']['ray_id'].numel() > 500
    _check_against_golden(m, rec, m.forward if path == 'fused' else m.forward_ops, f'{name} t={thres:g} {path}')
    assert set(rec['ret']['grads']) >= {'density.grid', 'k0.grid', 'rgbnet.0.weight'}


# ---- the reference's GPU path -------------------------------------------------------------------------------------------------
def _stat(a, b):
    return ((a.detach().float() - b.detach().float()).abs().max() / b.detach().float().abs().max().clamp_min(1e-30)).item()


@pytest.mark.gpu
def test_fouriergrid_vs_reference_gpu_path():
    """FourierGridModel at 96^3, P = 7, C = 9, width 64, 4096 rays, fast_color_thres 1e-3 against the reference's GPU path op for op
    (oracle.cpu_ref.model_forward on CUDA tensors with the reference's own CUDA extension from oracle/_ref: ATen grid_sample,
    cuBLAS rgbnet, its kernels): zero membership flips, bit-identical raw_alpha / weights / alphainv_last, colours within 1e-5."""
    from oracle import cpu_ref
    from tests.util import ref_ext
    ext = ref_ext()
    m = contracted_model(3, 'inf', 1e-3, world=96, seed=12, dens_mean=5.0, dens_std=3.0)
    ro, rd, vd = seeded_rays(4096, 31, DEV)
    kw = dict(num_voxels_density=96 ** 3, num_voxels_base_density=96 ** 3, fourier_freq_num=3, contracted_norm='inf',
              fast_color_thres=1e-3, bg_len=0.2)
    state = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}
    p = cpu_ref.params_from_state('fouriergrid', kw, state)
    p = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in p.items()}
    p['rgbnet'] = {k: v.to(DEV) for k, v in p['rgbnet'].items()}
    with torch.no_grad():
        a = cpu_ref.model_forward('fouriergrid', p, ro, rd, vd, RK['stepsize'], bg=1, render_depth=False, ext=ext)
        b = m(ro, rd, vd, **RK)
    assert_equal(b['ray_id'], a['ray_id'], 'ray_id (membership)')
    assert b['ray_id'].numel() > 10_000
    for k in ('raw_alpha', 'weights', 'alphainv_last'):
        assert_equal(b[k], a[k].reshape(b[k].shape), k)
    for k in ('rgb_marched', 'raw_rgb'):
        assert _stat(b[k], a[k]) <= 1e-5, k


@pytest.mark.gpu
def test_dvgo_vs_reference_gpu_path():
    """DirectVoxGO at 96^3, C = 9, width 64, 4096 rays, fast_color_thres 1e-3 against the reference's own dvgo.py over its own CUDA
    build (oracle/ref_gpu_py.py): zero membership flips, bit-identical raw_alpha / weights / alphainv_last, colours and depth
    within 1e-5 of scale, gradients as tests/test_gpu_dvgo_reference.py judges them."""
    from tests.test_gpu_dvgo import _vd
    from tests.test_gpu_dvgo_reference import _quiet, _ref_gpu_dvgo
    ref_gpu_py, _, ref_dvgo = _ref_gpu_dvgo()
    m, ro, rd = box_scene(nv=96 ** 3, n=4096, seed=13, thres=1e-3)
    vd = _vd(rd)
    rk = dict(near=0.2, far=1e9, bg=1., stepsize=0.5, render_depth=True)
    state = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}
    kw = {k: v for k, v in m.get_kwargs().items() if k != 'voxel_size_ratio'}
    ref = _quiet(ref_dvgo.DirectVoxGO, **kw)
    ref.load_state_dict(state, strict=True)
    ref = ref.to(DEV)
    assert float(ref.voxel_size) == float(m.voxel_size)
    ref_gpu_py.default_cuda(True)
    try:
        a = ref(ro, rd, vd, **rk)
        (a['rgb_marched'].pow(2).sum() + a['alphainv_last'].sum()).backward()
    finally:
        ref_gpu_py.default_cuda(False)
    b = m(ro, rd, vd, **rk)
    (b['rgb_marched'].pow(2).sum() + b['alphainv_last'].sum()).backward()
    assert_equal(b['ray_id'], a['ray_id'], 'ray_id (membership)')
    assert b['ray_id'].numel() > 50_000
    for k in ('raw_alpha', 'weights', 'alphainv_last'):
        assert_equal(b[k], a[k], k)
    for k in ('rgb_marched', 'raw_rgb', 'depth'):
        assert _stat(b[k], a[k]) <= 1e-5, k
    gr, go = dict(ref.named_parameters()), dict(m.named_parameters())
    assert _stat(go['density.grid'].grad, gr['density.grid'].grad) <= 2e-5
    gk, gkr = go['k0.grid'].grad, gr['k0.grid'].grad
    assert ((gk - gkr).abs() > 1e-5 * gkr.abs().max()).float().mean().item() <= 1e-3


# ---- the reference's training driver ---------------------------------------------------------------------------------------
GRASS_MODEL = dict(num_voxels_density=32 ** 3, num_voxels_rgb=32 ** 3, num_voxels_base_density=32 ** 3, num_voxels_base_rgb=32 ** 3,
                   num_voxels_viewdir=-1, alpha_init=1e-2, fast_color_thres=1e-3, rgbnet_dim=9, rgbnet_width=64, fourier_freq_num=3,
                   bg_len=0.2, stepsize=0.5, world_bound_scale=1, maskout_near_cam_vox=False)
LAB_MODEL = dict(num_voxels_density=32 ** 3, num_voxels_rgb=32 ** 3, num_voxels_base_density=32 ** 3, num_voxels_base_rgb=32 ** 3,
                 alpha_init=1e-2, fast_color_thres=1e-3, rgbnet_dim=9, rgbnet_width=64, rgbnet_direct=True, stepsize=0.5,
                 world_bound_scale=1, maskout_near_cam_vox=False)


@torch.no_grad()
def _lab_teacher_images(poses, HW, Ks):
    """Targets of the lab-like run: a seeded DirectVoxGO teacher in [-1, 1]^3 rendered with inverse_y, white background."""
    from unboundednerfpytorch_b200 import models, rays
    torch.manual_seed(4321)
    t = models.DirectVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=40 ** 3, num_voxels_base=40 ** 3, alpha_init=1e-2,
                           fast_color_thres=1e-3, rgbnet_dim=9, rgbnet_width=64, rgbnet_direct=True).to(DEV)
    ax = [torch.linspace(-1, 1, int(k), device=DEV) for k in t.world_size]
    t.density.grid.copy_((8.0 * (0.5 - sum(a ** 2 for a in torch.meshgrid(*ax, indexing='ij'))))[None, None])
    t.k0.grid.normal_(0., 1.)
    images = []
    for c2w, (H, W), K in zip(poses, HW, Ks):
        o, d, v = rays.get_rays_of_a_view(H, W, K, c2w.to(DEV), False, True, False, False)
        out = t(o.reshape(-1, 3), d.reshape(-1, 3), v.reshape(-1, 3), near=0.1, far=1e9, bg=1, stepsize=0.5)
        images.append(out['rgb_marched'].clamp(0, 1).reshape(H, W, 3).cpu())
    return torch.stack(images)


@torch.no_grad()
def _psnr(model, data_dict, inverse_y):
    from unboundednerfpytorch_b200 import rays
    model = model.to(DEV)
    err = []
    for c2w, (H, W), K, img in zip(data_dict['poses'], data_dict['HW'], data_dict['Ks'], data_dict['images']):
        o, d, v = rays.get_rays_of_a_view(H, W, K, c2w.to(DEV), False, inverse_y, False, False)
        out = model(o.reshape(-1, 3), d.reshape(-1, 3), v.reshape(-1, 3), near=0.1, far=1e9, bg=1, stepsize=0.5)
        err.append((out['rgb_marched'] - img.reshape(-1, 3).to(DEV)).pow(2).mean())
    return (-10 * torch.log10(torch.stack(err).mean())).item()


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['grass', 'lab'])
def test_driver_trains_free_configs(ref, tmp_path, kind):
    """The unmodified run_train.scene_rep_reconstruction under legacy.install_models, with a grass-like config (FourierGrid,
    dataset_type 'free', flatten sampler, one pg_scale step) and a lab-like one (DVGO bounded, rand_bkgd, inverse_y): every step on
    the fused march (launch names), PSNR rises, fine_last.tar loads into this package's class and the reference's."""
    from tests import test_gpu_train_driver as drv
    from unboundednerfpytorch_b200 import _cabi, ckpt, models
    poses, HW, Ks = drv._cameras(6)
    if kind == 'lab':           # inverse_y: OpenCV camera axes (y down, looking along +z)
        poses = poses.clone()
        poses[:, :, 1:3] *= -1
    if kind == 'grass':
        images = drv._teacher_images(poses, HW, Ks, 'fg')
        cfg = drv._cfg(tmp_path, 'FourierGrid', 'free', GRASS_MODEL, maskout_lt_nviews=0)
        ours_cls, ref_cls, inverse_y = models.FourierGridModel, ref.fg.FourierGridModel, False
        march_key = 'march_feature_fwd'
    else:
        images = _lab_teacher_images(poses, HW, Ks)
        cfg = drv._cfg(tmp_path, 'DVGO', 'free', LAB_MODEL, maskout_lt_nviews=0)
        cfg.data.update(unbounded_inward=False, rand_bkgd=True, inverse_y=True)
        ours_cls, ref_cls, inverse_y = models.DirectVoxGO, ref.dvgo.DirectVoxGO, True
        march_key = 'march_box_feature_fwd'
    assert float((images < 0.99).float().mean()) > 0.05          # the views see the object
    data_dict = {'HW': HW, 'Ks': Ks, 'near': 0.1, 'far': 6.0, 'near_clip': 0.1, 'i_train': np.arange(6), 'i_val': np.arange(0),
                 'i_test': np.arange(0), 'poses': poses, 'images': images, 'irregular_shape': False}
    os.makedirs(os.path.join(cfg.basedir, cfg.expname), exist_ok=True)
    args = drv._args(cfg, ref)
    np.random.seed(0)
    torch.manual_seed(0)
    timer, _cabi.TIMER = _cabi.TIMER, _cabi.KernelTimer()
    try:
        with drv._install(ref):
            psnr_last_step = ref.run_train.scene_rep_reconstruction(
                args=args, cfg=cfg, cfg_model=cfg.fine_model_and_render, cfg_train=cfg.fine_train,
                xyz_min=torch.tensor([-1.] * 3, device=DEV), xyz_max=torch.tensor([1.] * 3, device=DEV), data_dict=data_dict,
                stage='fine')
        records = dict(_cabi.TIMER.records)
    finally:
        _cabi.TIMER = timer
    assert np.isfinite(psnr_last_step)
    n_iters = cfg.fine_train.N_iters
    n_fused = len(records.get(march_key, []))
    assert n_fused >= n_iters, (march_key, n_fused, sorted(records))       # every training step marched fused
    assert 'rgbnet_fwd' in records
    first = os.path.join(cfg.basedir, cfg.expname, 'fine_000001.tar')
    last = os.path.join(cfg.basedir, cfg.expname, 'fine_last.tar')
    m_first = ckpt.load_model(ours_cls, first, DEV)
    m_last = ckpt.load_model(ours_cls, last, DEV)
    assert isinstance(m_last, ours_cls) and m_last.k0.grid.shape[1] == C9
    assert list(m_last.world_size.tolist()) != list(m_first.world_size.tolist())          # the pg_scale step ran
    p0, p1 = _psnr(m_first, data_dict, inverse_y), _psnr(m_last, data_dict, inverse_y)
    print(f'{kind}: PSNR after step 1 {p0:.2f} dB, after step {n_iters} {p1:.2f} dB')
    assert p1 > p0 + 0.5, (p0, p1)
    saved = ckpt._load(last)
    ref_model = ref_cls(**saved['model_kwargs'])
    ref_model.load_state_dict(saved['model_state_dict'])
    for k, v in ref_model.state_dict().items():
        assert torch.equal(v.cpu(), saved['model_state_dict'][k].cpu()), k
