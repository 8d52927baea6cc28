"""GPU: DirectVoxGO.forward with TensoRF grids on the fused box march (march.BoxTensorfMarch).  Its outputs must equal, bit for
bit, the op-by-op composition it replaces (_compose with _shade_k0: sample_pts_on_rays, the mask cache, the TensoRF kernels,
Raw2Alpha, Alphas2Weights) for all three grid pairings; its gradients equal the composition's up to fp32 reduction order, and
the density-factor gradients match an fp64 adjoint element by element."""
import numpy as np
import pytest
import torch

from unboundednerfpytorch_b200 import _cabi, march, models
from unboundednerfpytorch_b200 import grid as G

pytestmark = pytest.mark.gpu
DEV = 'cuda'
RK = dict(near=0.2, far=1e9, bg=1., rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False, render_depth=True)
LO, HI = [-1.0, -1.3, -0.6], [1.1, 1.2, 0.8]          # a non-cubic box
KEYS = ('ray_id', 'weights', 'alphainv_last', 'raw_alpha', 'raw_rgb', 'rgb_marched', 'depth')
PAIRINGS = [('TensoRFGrid', 'TensoRFGrid'), ('TensoRFGrid', 'DenseGrid'), ('DenseGrid', 'TensoRFGrid')]


def _model(dtype, ktype, nv=40 ** 3, R=8, Rxy=None, kR=12, rgbnet_dim=12, thres=1e-4, holes=True, seed=0):
    torch.manual_seed(seed)
    m = models.DirectVoxGO(xyz_min=LO, xyz_max=HI, num_voxels=nv, num_voxels_base=nv, alpha_init=1e-2, fast_color_thres=thres,
                           density_type=dtype, density_config=dict(n_comp=R, n_comp_xy=Rxy or R), k0_type=ktype,
                           k0_config=dict(n_comp=kR), rgbnet_dim=rgbnet_dim, rgbnet_direct=True, rgbnet_width=128,
                           rgbnet_depth=3, viewbase_pe=4).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    with torch.no_grad():
        if dtype == 'TensoRFGrid':         # products of O(1) factors: densities of both signs, a few units wide
            for p in m.density.factors():
                p.copy_(torch.randn(p.shape, generator=g, device=DEV) * (0.6 if p.shape[3] > 1 else 1.0))
        else:
            m.density.grid.normal_(0, 3, generator=g)
        if ktype == 'TensoRFGrid':
            for p in m.k0.factors():
                p.mul_(5)
        else:
            m.k0.grid.normal_(0, 1, generator=g)
        if holes:
            m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=g, device=DEV) > 0.3)
    return m


def _rays(n, seed=0):
    """Rays from outside at random, rays starting inside the box, rays missing it, rays with zero direction components and rays
    running along the box's faces, edges and through its corners."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(LO), torch.tensor(HI)
    o = torch.randn(n, 3, generator=g)
    o = o / o.norm(dim=-1, keepdim=True) * 3.5
    tgt = lo + (hi - lo) * torch.rand(n, 3, generator=g)
    d = tgt - o
    k = n // 8
    o[:k] = lo + (hi - lo) * torch.rand(k, 3, generator=g)                 # start inside
    d[k:2 * k] = o[k:2 * k] / o[k:2 * k].norm(dim=-1, keepdim=True)          # point away: miss
    d[2 * k:3 * k, 0] = 0                                                    # zero components
    d[3 * k:3 * k + k // 2, 1:] = 0
    special = []
    for a in range(3):                                                       # along faces, edges and corners, axis-aligned
        for u in (lo, hi):
            for v in (lo, hi):
                b, c = (a + 1) % 3, (a + 2) % 3
                oo = torch.zeros(3)
                oo[a] = lo[a] - 1.0
                oo[b], oo[c] = u[b], v[c]
                dd = torch.zeros(3)
                dd[a] = 1.0
                special.append((oo.clone(), dd.clone()))
                oo[c] = 0.5 * (lo[c] + hi[c])                                # on a face
                special.append((oo.clone(), dd.clone()))
    corners = torch.tensor([[x, y, z] for x in (LO[0], HI[0]) for y in (LO[1], HI[1]) for z in (LO[2], HI[2])])
    ctr = (lo + hi) / 2
    for cc in corners:                                                       # diagonals through opposite corners
        special.append((ctr + 2 * (cc - ctr), ctr - cc))
    so, sd = torch.stack([s[0] for s in special]), torch.stack([s[1] for s in special])
    o, d = torch.cat([o, so]), torch.cat([d, sd])
    vd = d / d.norm(dim=-1, keepdim=True)
    return o.to(DEV), d.to(DEV), vd.to(DEV)


def _routed(m, ro, rd, vd, rk=RK):
    _cabi.TIMER = _cabi.KernelTimer()
    try:
        out = m(ro, rd, vd, **rk)
    finally:
        names, _cabi.TIMER = set(_cabi.TIMER.records), None
    return out, names


def _expect_route(m, names):
    want = set()
    if isinstance(m.density, G.TensoRFGrid):
        want.add('march_box_tensorf_density_fwd')
    else:
        want.add('march_box_density_fwd')
    want.add('march_box_points_fwd')              # the k0 reads the survivor points with its own forward
    assert want <= names, (want, names)
    assert 'tensorf_fwd_c1' not in names          # the density is never read op by op


def _assert_same(a, b):
    for k in KEYS:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert torch.equal(a[k], b[k]), (k, (a[k].double() - b[k].double()).abs().max().item())


@pytest.mark.parametrize('dtype,ktype', PAIRINGS)
@pytest.mark.parametrize('rgbnet_dim', [12, 0])
@pytest.mark.parametrize('thres', [0.0, 1e-4])
def test_fused_equals_compose_bitwise(dtype, ktype, rgbnet_dim, thres):
    m = _model(dtype, ktype, rgbnet_dim=rgbnet_dim, thres=thres)
    ro, rd, vd = _rays(2048)
    with torch.no_grad():
        a, names = _routed(m, ro, rd, vd)
        b = m._compose(ro, rd, vd, m._shade_k0, RK)
    _expect_route(m, names)
    assert a['ray_id'].numel() > 1000
    _assert_same(a, b)


@pytest.mark.parametrize('R,Rxy', [(6, 6), (8, 4), (5, 7), (3, 2)])     # R != Rxy; R not a multiple of 4 (the W = 1 read)
def test_fused_equals_compose_factor_shapes(R, Rxy):
    m = _model('TensoRFGrid', 'TensoRFGrid', R=R, Rxy=Rxy, kR=R)
    ro, rd, vd = _rays(1024, seed=3)
    with torch.no_grad():
        a, names = _routed(m, ro, rd, vd)
        b = m._compose(ro, rd, vd, m._shade_k0, RK)
    _expect_route(m, names)
    _assert_same(a, b)


def test_fused_equals_compose_at_size():
    m = _model('TensoRFGrid', 'TensoRFGrid', nv=160 ** 3, R=8, kR=24, holes=False)
    ro, rd, vd = _rays(8192, seed=5)
    with torch.no_grad():
        a, names = _routed(m, ro, rd, vd)
        b = m._compose(ro, rd, vd, m._shade_k0, RK)
    _expect_route(m, names)
    _assert_same(a, b)


def test_s_max_overflow_raises():
    m = _model('TensoRFGrid', 'TensoRFGrid')
    ro, rd, _ = _rays(256)
    mscale, mshift, lo, hi = m._mask_geometry()
    cfg = march.make_box_cfg(lo, hi, RK['near'], m._stepdist(RK['stepsize']), float(m.act_shift), 0.5, m.fast_color_thres,
                             m.mask_cache.mask, mscale, mshift)
    cfg.s_max = 4
    fs = m.density.factors()
    with pytest.raises(RuntimeError, match='s_max'):
        march.BoxTensorfMarch.apply(ro, rd, m.mask_cache.mask, cfg, G.tensorf_desc(fs, 1, *m.density._bounds()), True, 8, *fs)


def _box_cfg(m):
    """The box cfg DirectVoxGO.forward builds."""
    mscale, mshift, lo, hi = m._mask_geometry()
    return march.make_box_cfg(lo, hi, RK['near'], m._stepdist(RK['stepsize']), float(m.act_shift),
                              RK['stepsize'] * float(m.voxel_size_ratio), m.fast_color_thres, m.mask_cache.mask, mscale, mshift)


def _index32(pts, m):
    """Continuous factor indices [M, 3] in fp32, formed as the kernels form them: ((p - min) / len * 2 - 1 + 1) * 0.5 * (size - 1)."""
    mn, mx = (torch.tensor(v, dtype=torch.float32, device=DEV) for v in m.density._bounds())
    size = torch.tensor([float(v) for v in m.density.world_size], dtype=torch.float32, device=DEV)
    nrm = (pts - mn) / (mx - mn) * 2 - 1
    return ((nrm + 1) * 0.5) * (size - 1)


def _tf_density64(fs, c):
    """fp64 TensoRF density at continuous indices c [M, 3] (fp64): bilinear plane reads times linear vector reads with zero
    padding (F.grid_sample, align_corners=True), the 3R products summed.  Differentiable in the factors fs [1,R,A,B]."""
    def plane(P, a, b):
        P = P[0]
        A, B = P.shape[1:]
        a0, b0 = c[:, a].floor(), c[:, b].floor()
        out = 0
        for da in (0, 1):
            for db in (0, 1):
                ia, ib = a0 + da, b0 + db
                w = (1 - (c[:, a] - ia).abs()) * (1 - (c[:, b] - ib).abs()) * ((ia >= 0) & (ia < A) & (ib >= 0) & (ib < B))
                out = out + P[:, ia.clamp(0, A - 1).long(), ib.clamp(0, B - 1).long()] * w
        return out

    def line(V, l):
        V = V[0, :, :, 0]
        L = V.shape[1]
        l0 = c[:, l].floor()
        out = 0
        for dl in (0, 1):
            il = l0 + dl
            w = (1 - (c[:, l] - il).abs()) * ((il >= 0) & (il < L))
            out = out + V[:, il.clamp(0, L - 1).long()] * w
        return out
    xy, xz, yz, xv, yv, zv = fs
    return (plane(xy, 0, 1) * line(zv, 2)).sum(0) + (plane(xz, 0, 2) * line(yv, 1)).sum(0) + (plane(yz, 1, 2) * line(xv, 0)).sum(0)


@pytest.mark.parametrize('K', [1, 2, 4, 8, 16, 32, 64])
def test_density_factor_gradients_vs_fp64(K):
    """The six density-factor gradients through raw_alpha, element by element against an fp64 adjoint, at 1e-5 of each element's
    own bound (the same adjoint with |gradient| and |factors|), accumulated into pre-filled .grad; every vector-copy count K, rays
    of 31 to 65 steps and longer in one launch."""
    m = _model('TensoRFGrid', 'TensoRFGrid', thres=1e-4)
    ro, rd, _ = _rays(1024, seed=11)
    cfg = _box_cfg(m)
    fs = m.density.factors()
    pre = [torch.randn_like(p) for p in fs]
    for p, g in zip(fs, pre):
        p.grad = g.clone()
    w, last, alpha, pts, ray_id, step_id = march.BoxTensorfMarch.apply(
        ro, rd, m.mask_cache.mask, cfg, G.tensorf_desc(fs, 1, *m.density._bounds()), True, K, *fs)
    _, pid, sid = m.sample_ray(ro, rd, **RK)            # in-box steps of every ray
    n_steps = torch.zeros(ro.shape[0], dtype=torch.int64, device=DEV).scatter_reduce(0, pid, sid + 1, 'amax')
    assert ((n_steps >= 31) & (n_steps <= 65)).sum() > 20 and (n_steps > 65).sum() > 20
    c = torch.rand(alpha.shape, generator=torch.Generator(DEV).manual_seed(4), device=DEV) - 0.5
    (alpha * c).sum().backward()

    idx = _index32(pts.detach(), m).double()
    f64 = [p.detach().double().requires_grad_() for p in fs]
    d64 = _tf_density64(f64, idx)
    e = torch.exp(d64 + float(m.act_shift))
    a64 = 1 - (1 + e) ** (-cfg.interval)
    ref = torch.autograd.grad((a64 * c.double()).sum(), f64)
    g_abs = (c.double().abs() * cfg.interval * e * (1 + e) ** (-cfg.interval - 1)).detach()
    fabs = [p.detach().double().abs().requires_grad_() for p in fs]
    bound = torch.autograd.grad((g_abs * _tf_density64(fabs, idx)).sum(), fabs)
    for name, p, g0, r, b in zip(G.TENSORF_FACTORS, fs, pre, ref, bound):
        err = (p.grad.double() - (g0.double() + r)).abs()
        tol = 1e-5 * b + 2 ** -23 * g0.double().abs()
        assert (err <= tol).all(), (name, (err - tol).max().item(), int((err > tol).sum()))
        assert (b > 0).float().mean() > 0.05, name


def test_in_place_factor_change_before_backward_raises():
    m = _model('TensoRFGrid', 'TensoRFGrid')
    ro, rd, vd = _rays(256)
    out = m(ro, rd, vd, **RK)
    with torch.no_grad():
        m.density.xy_plane.mul_(2)
    with pytest.raises(RuntimeError, match='modified by an inplace operation'):
        out['rgb_marched'].sum().backward()


def _grads(m, fn, ro, rd, vd, target, prefill=None):
    m.zero_grad(set_to_none=True)
    if prefill is not None:
        for p, g in zip(m.parameters(), prefill):
            p.grad = g.clone()
    out = fn(ro, rd, vd)
    loss = ((out['rgb_marched'] - target) ** 2).mean() + out['alphainv_last'].mean() + 1e-2 * out['weights'].sum()
    loss.backward()
    return {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}


def _close(ga, gb, rtol, what):
    assert set(ga) == set(gb), (set(ga) ^ set(gb))
    for n in ga:
        bound = gb[n].abs().max().item() + 1e-12
        err = (ga[n] - gb[n]).abs().max().item()
        assert err <= rtol * bound, (what, n, err, bound)


@pytest.mark.parametrize('dtype,ktype', PAIRINGS)
@pytest.mark.parametrize('K', [1, 2, 4, 8, 16, 32, 64])
def test_gradients_match_compose(dtype, ktype, K, monkeypatch):
    """Every parameter's gradient (density factors or grid, k0 factors and f_vec or grid, rgbnet) against the composition's, for
    every replicated vector-copy count, also accumulated into pre-filled .grad."""
    monkeypatch.setattr(G, 'TENSORF_VEC_COPIES', K)
    m = _model(dtype, ktype, thres=1e-4)
    ro, rd, vd = _rays(1024, seed=7)
    target = torch.rand(ro.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    fused = lambda a, b, c: m(a, b, c, **RK)                                  # noqa: E731
    comp = lambda a, b, c: m._compose(a, b, c, m._shade_k0, RK)               # noqa: E731
    ga, gb = _grads(m, fused, ro, rd, vd, target), _grads(m, comp, ro, rd, vd, target)
    _close(ga, gb, 1e-5, 'fresh')
    pre = [torch.randn_like(p) for p in m.parameters()]
    ga, gb = _grads(m, fused, ro, rd, vd, target, pre), _grads(m, comp, ro, rd, vd, target, pre)
    _close(ga, gb, 1e-5, 'prefilled')


def test_training_rescale_and_checkpoint(tmp_path):
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    m = _model('TensoRFGrid', 'TensoRFGrid', nv=32 ** 3)
    ro, rd, vd = _rays(2048, seed=9)
    target = torch.rand(ro.shape[0], 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    cfg = dict(lrate_density=0.02, lrate_k0=0.02, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])
    for step in range(6):
        if step == 3:
            m.scale_volume_grid(48 ** 3)          # the box cfg follows the new voxel size
        opt = create_optimizer_or_freeze_model(m, cfg, global_step=0) if step in (0, 3) else opt
        opt.zero_grad(set_to_none=True)
        out, names = _routed(m, ro, rd, vd)
        _expect_route(m, names)
        loss = ((out['rgb_marched'] - target) ** 2).mean()
        assert torch.isfinite(loss)
        loss.backward()
        opt.step()
        if step == 1:
            m.update_occupancy_cache()
    with torch.no_grad():
        _assert_same(m(ro, rd, vd, **RK), m._compose(ro, rd, vd, m._shade_k0, RK))
    path = tmp_path / 'fine_last.tar'
    torch.save({'model_kwargs': m.get_kwargs(), 'model_state_dict': m.state_dict()}, path)
    st = torch.load(path, weights_only=False)
    m2 = models.DirectVoxGO(**st['model_kwargs']).to(DEV)
    m2.load_state_dict(st['model_state_dict'])
    with torch.no_grad():
        a, names = _routed(m2, ro, rd, vd)
        _expect_route(m2, names)
        _assert_same(a, m2._compose(ro, rd, vd, m2._shade_k0, RK))


def test_render_viewpoints_equals_compose():
    from unboundednerfpytorch_b200 import rays as R
    from unboundednerfpytorch_b200 import render
    m = _model('TensoRFGrid', 'TensoRFGrid')
    H, W = 48, 64
    K = np.array([[60., 0., 32.], [0., 60., 24.], [0., 0., 1.]])
    c2w = np.array([[1, 0, 0, 0.05], [0, 1, 0, -0.05], [0, 0, 1, 3.0]], dtype=np.float32)
    rgbs, depths, bgmaps = render.render_viewpoints(None, m, [c2w], [[H, W]], [K], False, dict(RK), chunk=1024, verbose=False)
    ro, rd, vd = R.get_rays_of_a_view(H, W, K, torch.as_tensor(c2w), False, False, False, False)
    ro, rd, vd = (t.reshape(-1, 3).to(DEV) for t in (ro, rd, vd))
    with torch.no_grad():
        outs = [m._compose(a, b, c, m._shade_k0, RK) for a, b, c in zip(ro.split(1024), rd.split(1024), vd.split(1024))]
    rgb = torch.cat([o['rgb_marched'] for o in outs]).reshape(H, W, 3).cpu().numpy()
    assert np.array_equal(rgbs[0], rgb)
    assert (bgmaps[0] < 0.999).mean() > 0.1
