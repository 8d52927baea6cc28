"""GPU: the fused march and the tensor-core rgbnet at the k0 widths of the reference's other FourierGrid configs -- C = 3
(rgbnet_dim = 3: Waymo / Mega-NeRF, and every rgbnet_dim <= 0 colour grid) and C = 15 (Tanks&Temples Train).

* fused forward vs forward_ops: identical survivors, bit-identical raw_density / raw_alpha / weights / alphainv_last, and k0
  features bit-identical to F.grid_sample(...).mean(0) on the same points (oracle.cpu_ref.fourier_grid_forward);
* the k0 scatter element by element against the fp64 adjoint of tests/test_gpu_march_scatter.py;
* the rgbnet at K = 3 / 15 against fp64 with the criterion of tests/test_gpu_rgbnet_layouts.py;
* a few training steps with TV + MaskedAdam and a ckpt round trip;
* the Waymo no-block size (300^3, P = 7, C = 3, 2048 rays).
"""
import math
import os
import tempfile

import pytest
import torch

from tests.test_gpu_march_scatter import (Contracted, as_pxyzc, cells, channels_last, judge as judge_scatter, part_bounds,
                                          ref_gather, ref_scatter, selections, slab_coords)  # noqa: F401 (fixture)
from tests.test_gpu_callers_unchanged import ref_modules  # noqa: F401 (fixture)
from tests.test_gpu_rgbnet_layouts import LAYOUTS, TAU, TINY, UNIT
from tests.util import assert_close, assert_equal, seeded_rays

DEV = 'cuda:0'


def _model(C, F_, norm='inf', thres=0.0, world=24, seed=0, viewbase_pe=4, dens_mean=0.0, dens_std=1.0, rgbnet=True):
    """FourierGridModel (F_ > 0, P = 2 F_ + 1) or DirectContractedVoxGO (F_ = 0, P = 1) with a C-channel k0 grid: rgbnet_dim = C,
    or the rgbnet_dim = 0 colour grid (C = 3)."""
    from unboundednerfpytorch_b200 import models
    torch.manual_seed(seed)
    dim = C if rgbnet else 0
    if F_ > 0:
        m = models.FourierGridModel(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=world ** 3,
                                    num_voxels_base_density=world ** 3, num_voxels_rgb=world ** 3, num_voxels_base_rgb=world ** 3,
                                    num_voxels_viewdir=-1, alpha_init=1e-4, fast_color_thres=thres, rgbnet_dim=dim,
                                    fourier_freq_num=F_, contracted_norm=norm, viewbase_pe=viewbase_pe)
    else:
        m = models.DirectContractedVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=world ** 3, num_voxels_base=world ** 3,
                                         alpha_init=1e-4, fast_color_thres=thres, rgbnet_dim=dim, contracted_norm=norm,
                                         viewbase_pe=viewbase_pe)
    assert m.k0.grid.shape[1] == C
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=g) * dens_std + dens_mean)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
    return m.to(DEV)


RK = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, render_depth=True)
FWD_CASES = [(C, F_, norm, thres) for C in (3, 15) for F_ in (0, 1, 3, 4, 5) for norm in ('inf', 'l2') for thres in (0.0, 1e-4)]


@pytest.mark.gpu
@pytest.mark.parametrize('C,F_,norm,thres', FWD_CASES, ids=[f'C{c}-P{2 * f + 1}-{n}-t{t:g}' for c, f, n, t in FWD_CASES])
def test_fused_vs_ops_and_grid_sample(C, F_, norm, thres):
    from oracle import cpu_ref
    from unboundednerfpytorch_b200 import _cabi
    m = _model(C, F_, norm, thres, dens_mean=5.0 if thres else 0.0, dens_std=3.0 if thres else 1.0, seed=C + F_)
    assert m._fused_ok()
    ro, rd, vd = seeded_rays(300, 5 + C, DEV)
    timer, _cabi.TIMER = _cabi.TIMER, _cabi.KernelTimer()
    try:
        with torch.no_grad():
            fused = m(ro, rd, vd, **RK)
        keys = set(_cabi.TIMER.records)
    finally:
        _cabi.TIMER = timer
    # forward reached the fused march and the tensor-core rgbnet.  forward_ops shades with the same tensor-core rgbnet (shade.supported
    # admits K = 3 / 15), so rgb_marched below checks the march; test_rgbnet_k_vs_fp64 and the fixtures check the rgbnet itself
    assert {'march_density_fwd', 'march_feature_fwd', 'rgbnet_fwd'} <= keys, keys
    with torch.no_grad():
        ops_ = m.forward_ops(ro, rd, vd, **RK)
        (w, last, alpha, dens, k0, ray_id, step_id, t, inner), _ = m._march(ro, rd, RK['stepsize'])
        pts, _, _ = m._sample_dense(ro, rd, RK['stepsize'])
        want = cpu_ref.fourier_grid_forward(m.k0.grid.detach().contiguous(), pts[ray_id, step_id], m.xyz_min, m.xyz_max, F_)
    assert fused['ray_id'].numel() > 500
    assert_equal(fused['ray_id'], ops_['ray_id'], 'ray_id')
    assert_equal(fused['step_id'], ops_['step_id'], 'step_id')
    for k in ('raw_density', 'raw_alpha', 'weights', 'alphainv_last'):
        assert_equal(fused[k], ops_[k], k)
    assert_equal(k0, want, f'k0 C={C} P={2 * F_ + 1} vs F.grid_sample(...).mean(0)')
    assert_close(fused['rgb_marched'], ops_['rgb_marched'], rtol=1e-4, atol=1e-5, what='rgb_marched fused vs forward_ops')


@pytest.mark.gpu
def test_colour_grid_stage_is_fused():
    """rgbnet_dim = 0: rgb = sigmoid(k0) of the fused 3-channel gather, on both contracted models."""
    for F_ in (0, 3):
        m = _model(3, F_, rgbnet=False, seed=11)
        assert m.rgbnet is None and m._fused_ok()
        ro, rd, vd = seeded_rays(256, 17, DEV)
        with torch.no_grad():
            a, b = m(ro, rd, vd, **RK), m.forward_ops(ro, rd, vd, **RK)
        assert_equal(a['ray_id'], b['ray_id'], 'ray_id')
        assert_equal(a['weights'], b['weights'], 'weights')
        assert_close(a['rgb_marched'], b['rgb_marched'], rtol=1e-5, atol=1e-6, what='rgb_marched')


# ---- the reference's own code: fixtures of oracle/make_golden_fg_widths.py ----------------------------------------------------
def _fg_kw(C, pe, norm, dens_world, k0_world):
    return dict(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=dens_world ** 3, num_voxels_base_density=dens_world ** 3,
                num_voxels_rgb=k0_world ** 3, num_voxels_base_rgb=k0_world ** 3, num_voxels_viewdir=-1, alpha_init=1e-2,
                rgbnet_dim=C, fourier_freq_num=3, viewbase_pe=pe, contracted_norm=norm)


# grid sizes keep every fixture file (outputs + the full density / k0 / rgbnet gradients) under about 1 MB
GOLDEN = {
    'waymo': dict(cls='FourierGridModel', kw=_fg_kw(3, 2, 'l2', 20, 16), rays=80),
    'mega': dict(cls='FourierGridModel', kw=_fg_kw(3, 8, 'l2', 20, 16), rays=80),
    'train': dict(cls='FourierGridModel', kw=_fg_kw(15, 4, 'inf', 16, 10), rays=96),
    'fg_rgb0': dict(cls='FourierGridModel', kw=_fg_kw(0, 4, 'inf', 20, 16), rays=96),
    'dcvgo_rgb0': dict(cls='DirectContractedVoxGO', kw=dict(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=20 ** 3,
                                                             num_voxels_base=20 ** 3, alpha_init=1e-2, rgbnet_dim=0,
                                                             contracted_norm='l2'), rays=96),
}


def golden_grids(dens_shape, k0_shape, seed, thres):
    """The fixtures' density and k0 grids, regenerated from their seed.  The density is centred at 4, away from 0: the
    reference's CPU run computes its contracted sample points with torch-CPU reductions, which differ from torch-CUDA's in the last
    bit, and near a zero crossing of the density that difference alone exceeds the relative golden tolerance."""
    g = torch.Generator().manual_seed(seed)
    dens = torch.randn(dens_shape, generator=g) * 3 + 4.0
    return dens, torch.randn(k0_shape, generator=g)


GOLDEN_CASES = [(n, t, path) for n in GOLDEN for t in (0.0, 1e-4) for path in ('fused', 'ops')]


@pytest.mark.gpu
@pytest.mark.parametrize('name,thres,path', GOLDEN_CASES, ids=[f'{n}-t{t:g}-{p}' for n, t, p in GOLDEN_CASES])
def test_reference_fixtures(name, thres, path):
    """forward and forward_ops against the reference's FourierGrid_model.py / dcvgo.py run on the CPU, at the golden tolerances of
    tests/test_gpu_models.py: sample ids bit-exact, outputs within 2e-5, gradients of the density grid, the k0 grid and the rgbnet
    within 5e-5 (+ 1e-5 of scale)."""
    from tests.test_gpu_models import _check_against_golden
    from tests.util import load_golden
    from unboundednerfpytorch_b200 import models
    rec = load_golden('l2_fg_widths.pt')[f'{name}_t{thres:g}']
    m = getattr(models, rec['cls'])(**rec['kwargs'])
    dens, k0 = golden_grids(m.density.grid.shape, m.k0.grid.shape, rec['grid_seed'], thres)
    missing, unexpected = m.load_state_dict(rec['state'], strict=False)
    assert not unexpected and sorted(missing) == ['density.grid', 'k0.grid'], (missing, unexpected)
    with torch.no_grad():
        m.density.grid.copy_(dens)
        m.k0.grid.copy_(k0)
    m = m.to(DEV)
    assert m._fused_ok()
    assert rec['ret']['ray_id'].numel() > 1000
    _check_against_golden(m, rec, m.forward if path == 'fused' else m.forward_ops, f'{name} t={thres:g} {path}')
    assert set(rec['ret']['grads']) >= {'density.grid', 'k0.grid'}


# ---- the reference's unmodified FourierGrid_model.py on the GPU over legacy.install() ----------------------------------------
CALLER_CASES = {
    # configs/waymo/waymo_no_block.py: rgbnet_dim 3, viewbase_pe 2, l2; configs/tankstemple_unbounded/train_single.py: rgbnet_dim 15
    'waymo': dict(rgbnet_dim=3, viewbase_pe=2, contracted_norm='l2'),
    'train': dict(rgbnet_dim=15, viewbase_pe=4, contracted_norm='inf'),
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(CALLER_CASES))
def test_unmodified_reference_fouriergrid_at_width(case, ref_modules, monkeypatch):
    """tests/test_gpu_callers_unchanged.py's check, run on a FourierGridModel of this width: the reference's FourierGrid_model.py
    and masked_adam.py, staged unmodified under oracle/_ref/py, over legacy.install(); forward plus one training iteration with
    TV; sample ids bit-exact, outputs within 1e-5 of scale, gradients as there, and MaskedAdam bit for bit on equal gradients."""
    from tests import test_gpu_callers_unchanged as callers
    base = callers.CASES['fouriergrid']
    monkeypatch.setitem(callers.CASES, 'fouriergrid', dict(base, kw=dict(base['kw'], **CALLER_CASES[case])))
    callers.test_unmodified_reference_callers_run_on_this_library(ref_modules, 'fouriergrid')


# ---- k0 scatter against the fp64 adjoint -----------------------------------------------------------------------------------
class Wide(Contracted):
    """The scatter test's contracted scene with a C-channel k0 grid."""

    def __init__(self, C, **kw):
        from unboundednerfpytorch_b200 import grid as G
        super().__init__(**kw)
        X, Y, Z = self.shape
        self.kvals = torch.randn(self.P, X, Y, Z, C, generator=torch.Generator().manual_seed(7 * C + self.P)).to(DEV)
        self.kdesc = G.grid_desc(channels_last(self.kvals), self.mn, self.mx, self.n_freqs)


SHAPE = (23, 37, 41)            # odd X * Y * Z, X - 1 = 22 not divisible by 4
SHAPE4 = (41, 23, 37)           # X - 1 = 40 divisible by 4
SCATTER = {f'C{C}-{k}': dict(C=C, **v) for C in (3, 15) for k, v in {
    'P1': dict(P=1, shape=SHAPE), 'P3': dict(P=3, shape=SHAPE4), 'P5': dict(P=5, shape=SHAPE), 'P7': dict(P=7, shape=SHAPE4),
    'P7-l2': dict(P=7, shape=SHAPE, norm='l2'), 'P9': dict(P=9, shape=SHAPE4, n_far=32), 'P11': dict(P=11, shape=SHAPE),
    'P9-X2': dict(P=9, shape=(2, 37, 41)), 'P5-X5': dict(P=5, shape=(5, 37, 41)),
    'P9-ragged': dict(P=9, shape=SHAPE4, thres=1e-4, world_len=41, stepsize=0.5, n_x=768, n_rand=64, n_far=16),
    'P1-ragged': dict(P=1, shape=SHAPE4, thres=1e-4, world_len=41, stepsize=0.5, n_x=768, n_rand=64, n_far=16),
}.items()}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(SCATTER))
def test_k0_scatter_vs_fp64(case, selections):
    """Every x-range split (feature kernels 0 / 4 / 5 -> 1 / 2 / 4 ranges) against the fp64 adjoint; the forward against the fp64
    gather of the same cells.  Structural claims (record phases, boundary planes, equal-cell runs) are asserted from the data."""
    ops = selections
    spec = dict(SCATTER[case])
    C = spec.pop('C')
    sc = Wide(C, **spec)
    P, shape = sc.P, sc.shape
    ops.set_feature_kernel(5)
    base = sc.run()
    ray_id, step_id = base['ray_id'], base['step_id']
    M = ray_id.numel()
    assert M > 1000, f'{case}: only {M} survivors'
    cs = slab_coords(sc.points(ray_id, step_id), sc.mn, sc.mx, sc.n_freqs)
    x0, f = cells(cs, shape)
    X, Y, Z = shape
    v = (x0[..., 0] * Y + x0[..., 1]) * Z + x0[..., 2]                    # base voxel of every (slab, sample)
    # every 16-byte phase of the record addresses occurs (C * 4 bytes per voxel, 8 corners)
    phases = {int(p) for p in torch.unique(((v[..., None] + torch.tensor([0, 1, Z, Y * Z], device=DEV)) * C) % 4)}
    assert phases == {0, 1, 2, 3}, f'{case}: record phases {phases}'
    # survivors on both sides of the x-range boundary planes of the 2- and 4-way splits (dense scenes with X > 4)
    if 'ragged' not in case and X > 4:
        for n_split in (2, 4):
            for b in part_bounds(X, n_split):
                assert bool((x0[..., 0] == b).any()) and bool((x0[..., 0] == b - 1).any()), f'{case}: nothing at plane {b}'
    # consecutive survivors of a ray sharing a slab-0 cell (the register merge has work)
    assert bool(((ray_id[1:] == ray_id[:-1]) & (v[0, 1:] == v[0, :-1])).any())
    gen = torch.Generator(DEV).manual_seed(M)
    g_feat = torch.randn(M, C, device=DEV, generator=gen)
    g_dens = torch.randn(M, device=DEV, generator=gen)
    want_k, bound_k = ref_scatter(x0, f, g_feat, shape)
    fk_want, fk_bound = ref_gather(x0, f, sc.kvals)
    fails = []
    for fk in (0, 3, 4, 5):
        ops.set_feature_kernel(fk)
        got = sc.run(g_feat, g_dens)
        what = f'C={C} {case} fk={fk}'
        try:
            assert torch.equal(got['ray_id'], ray_id) and torch.equal(got['step_id'], step_id), f'{what}: survivors differ'
            assert torch.equal(got['feat'], base['feat']), f'{what}: forward differs across selections'
            judge_scatter(got['feat'][:, :, None], fk_want[:, :, None], fk_bound[:, :, None], what + ' k0 forward self-check',
                          'forward self-check', tau=1e-6)
            judge_scatter(as_pxyzc(got['gk']), want_k, bound_k, what + ' k0 scatter', f'k0 C={C} P={P}')
        except AssertionError as e:
            fails.append(str(e))
    assert not fails, '\n'.join(fails)


# ---- rgbnet at K = 3 / 15 against fp64 --------------------------------------------------------------------------------------
def ref64_k(feat, vb, ray_id, W1k, W2, b2, W3, b3, g_rgb):
    """fp64 rgb and gradients of the K-feature rgbnet with the bound B of tests/test_gpu_rgbnet_layouts.py::ref64."""
    d = lambda x: x.double()
    x, v, g = d(feat), d(vb[ray_id]), d(g_rgb)
    W1k, W2, b2, W3, b3 = map(d, (W1k, W2, b2, W3, b3))
    aW1, aW2, ab2, aW3, ab3 = (t.abs() for t in (W1k, W2, b2, W3, b3))
    z1 = x @ W1k.t() + v
    m1 = (z1 > 0).double()
    h1 = z1 * m1
    z2 = h1 @ W2.t() + b2
    m2 = (z2 > 0).double()
    h2 = z2 * m2
    y = torch.sigmoid(h2 @ W3.t() + b3)
    dz3 = g * y * (1 - y)
    dZ2 = (dz3 @ W3) * m2
    dZ1 = (dZ2 @ W2) * m1
    Bh1 = (x.abs() @ aW1.t() + v.abs()) * m1
    Bh2 = (Bh1 @ aW2.t() + ab2) * m2
    By = y * (1 - y) * (Bh2 @ aW3.t() + ab3) + y
    Bdz3 = g.abs() * (y * (1 - y) + (1 - 2 * y).abs() * By)
    BdZ2 = (Bdz3 @ aW3) * m2
    BdZ1 = (BdZ2 @ aW2) * m1
    N = vb.shape[0]
    gvb = torch.zeros(N, 128, dtype=torch.float64, device=feat.device).index_add_(0, ray_id, dZ1)
    Bgvb = torch.zeros_like(gvb).index_add_(0, ray_id, BdZ1)
    want = dict(rgb=y, g_feat=dZ1 @ W1k, g_vb=gvb, dW1k=dZ1.t() @ x, dW2=dZ2.t() @ h1, db2=dZ2.sum(0), dW3=dz3.t() @ h2,
                db3=dz3.sum(0))
    bound = dict(rgb=By, g_feat=BdZ1 @ aW1, g_vb=Bgvb, dW1k=BdZ1.t() @ x.abs(), dW2=BdZ2.t() @ Bh1, db2=BdZ2.sum(0),
                 dW3=Bdz3.t() @ Bh2, db3=Bdz3.sum(0))
    return want, bound


def _inputs_k(K, ray_id, N, seed):
    g = torch.Generator().manual_seed(seed)
    M = ray_id.numel()
    u = lambda *s, a: ((torch.rand(*s, generator=g) * 2 - 1) * a)
    p = dict(W1k=u(128, K, a=1 / math.sqrt(K + 27)), W2=u(128, 128, a=1 / math.sqrt(128)), b2=u(128, a=1 / math.sqrt(128)),
             W3=u(3, 128, a=1 / math.sqrt(128)), b3=torch.randn(3, generator=g) * 0.1)
    inp = dict(feat=torch.randn(M, K, generator=g), vb=torch.randn(N, 128, generator=g) * 0.5, ray_id=ray_id,
               g_rgb=torch.randn(M, 3, generator=g), **p)
    inp = {k: v.to(DEV) for k, v in inp.items()}
    # ReLU-ambiguous samples (an fp64 pre-activation within 1e-5 of zero) get their features redrawn
    for _ in range(8):
        x = inp['feat'].double()
        z1 = x @ inp['W1k'].double().t() + inp['vb'][inp['ray_id']].double()
        z2 = torch.relu(z1) @ inp['W2'].double().t() + inp['b2'].double()
        amb = torch.minimum(z1.abs().amin(1), z2.abs().amin(1)) <= 1e-5
        if not bool(amb.any()):
            return inp
        inp['feat'][amb] = torch.randn(int(amb.sum()), K, generator=g).to(DEV)
    raise AssertionError('ReLU-ambiguous samples remain')


RGB_CASES = [(K, lay, M) for K in (3, 15) for lay, M in
             (('aligned16', 1), ('offset16', 17), ('len4_o1', 129), ('alternating', 4099), ('one_ray_first', 4099),
              ('sparse_odd', 16 * 528 + 1), ('bounds4_m1', 16 * 528 - 1), ('bounds4_p1', 16 * 528 + 1), ('bounds8_0', 16 * 1056),
              ('geometric250', 16 * 1056 + 1), ('randint', 1_200_007))]


@pytest.mark.gpu
@pytest.mark.parametrize('K,layout,M', RGB_CASES, ids=[f'K{k}-{lay}-{m}' for k, lay, m in RGB_CASES])
def test_rgbnet_k_vs_fp64(K, layout, M):
    """rgb, g_feat, g_vb and the six parameter gradients within TAU * B of fp64 (tc3), the no_grad forward bit-identical to the
    grad-enabled one, rays without samples exactly zero.  'alternating' has units with more than 4 ray segments, the bounds*
    layouts put a ray boundary next to every warp-range boundary of the 4- / 8-warp partition."""
    from unboundednerfpytorch_b200 import shade as shade_mod
    ray_id, N = LAYOUTS[layout](M)
    inp = _inputs_k(K, ray_id, N, seed=M + K)
    want, bound = ref64_k(*(inp[k] for k in ('feat', 'vb', 'ray_id', 'W1k', 'W2', 'b2', 'W3', 'b3', 'g_rgb')))
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(shade_mod, 'MODE', 'tc3')
        leaves = {k: inp[k].clone().requires_grad_(True) for k in ('feat', 'vb', 'W1k', 'W2', 'b2', 'W3', 'b3')}
        args = [leaves['feat'], leaves['vb'], inp['ray_id']] + [leaves[k] for k in ('W1k', 'W2', 'b2', 'W3', 'b3')]
        rgb = shade_mod._ShadeFn.apply(*args, True)
        rgb.backward(inp['g_rgb'])
        with torch.no_grad():
            rgb_ng = shade_mod._ShadeFn.apply(*args, False)
    got = dict(rgb=rgb.detach(), g_feat=leaves['feat'].grad, g_vb=leaves['vb'].grad)
    got.update({'d' + k: leaves[k].grad for k in ('W1k', 'W2', 'b2', 'W3', 'b3')})
    assert torch.equal(rgb_ng, got['rgb'])
    empty = torch.bincount(inp['ray_id'], minlength=N) == 0
    assert not bool(got['g_vb'][empty].any())
    bad = {}
    for k in want:
        r = float(((got[k].double() - want[k]).abs() / (bound[k] + TINY / TAU)).max())
        if not r <= TAU:
            bad[k] = f'{r:.2e}'
    assert not bad, f'K={K} {layout} M={M}: |got - want| / B above {TAU:.0e}: {bad}'
    if layout == 'alternating':      # more than 4 segments in some unit: the per-sample path is taken
        starts = torch.ones(M, dtype=torch.bool)
        starts[1:] = ray_id[1:] != ray_id[:-1]
        per_unit = torch.zeros(-(-M // UNIT), dtype=torch.long).index_add_(0, torch.arange(M) // UNIT, starts.long())
        assert int(per_unit.max()) > 4


# ---- training end to end ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('C', [3, 15])
def test_training_and_checkpoint(C):
    from unboundednerfpytorch_b200 import ckpt, models
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    teacher = _model(C, 3, 'l2', 1e-4, world=32, seed=1, viewbase_pe=2, dens_mean=4.0, dens_std=3.0)
    student = _model(C, 3, 'l2', 0.0, world=32, seed=2, viewbase_pe=2, dens_mean=0.0, dens_std=0.1)
    cfg = dict(lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])
    opt = create_optimizer_or_freeze_model(student, cfg, global_step=0)
    rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5)
    ro, rd, vd = seeded_rays(2048, 3, DEV)
    with torch.no_grad():
        target = teacher(ro, rd, vd, **rk)['rgb_marched']
    losses = []
    for it in range(1, 21):
        ret = student(ro, rd, vd, global_step=it, is_train=True, **rk)
        opt.zero_grad(set_to_none=True)
        loss = torch.nn.functional.mse_loss(ret['rgb_marched'], target)
        loss.backward()
        student.density_total_variation_add_grad(1e-6 / len(ro), it < 10)
        student.k0_total_variation_add_grad(1e-7 / len(ro), it < 10)
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.95 * losses[0] and all(b < a for a, b in zip(losses, losses[1:])), losses
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'last.tar')
        ckpt.save_checkpoint(20, student, opt, path)
        back = ckpt.load_model(models.FourierGridModel, path, DEV)
    with torch.no_grad():
        a, b = student(ro, rd, vd, **rk), back(ro, rd, vd, **rk)
    for k in ('ray_id', 'weights', 'rgb_marched', 'raw_rgb'):
        assert_equal(a[k], b[k], f'{k} after save / load')


# ---- the Waymo no-block size --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_waymo_no_block_size():
    """300^3, fourier_freq_num 3 (P = 7), rgbnet_dim 3, l2 contraction, 2048 rays: fused vs forward_ops without a membership
    flip and with bit-identical alpha / weights."""
    m = _model(3, 3, 'l2', 1e-4, world=300, seed=5, viewbase_pe=2, dens_mean=5.0, dens_std=3.0)
    ro, rd, vd = seeded_rays(2048, 9, DEV)
    with torch.no_grad():
        a = m(ro, rd, vd, **RK)
        b = m.forward_ops(ro, rd, vd, **RK)
    assert a['ray_id'].numel() > 10_000
    assert_equal(a['ray_id'], b['ray_id'], 'ray_id')
    assert_equal(a['step_id'], b['step_id'], 'step_id')
    for k in ('raw_alpha', 'weights', 'alphainv_last'):
        assert_equal(a[k], b[k], k)
