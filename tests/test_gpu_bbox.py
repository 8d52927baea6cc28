"""H100: the scene bounds of bbox.py (csrc/bounds.cu) against the reference's torch compositions run through this library on the
same GPU -- bit for bit -- and against the reference's own results in tests/golden/l2_bbox/ (oracle/make_golden_bbox.py).

* frustum: rays.get_rays_of_a_view per view, then the near / far (or near_clip) points and amin / amax folded with
  torch.minimum / maximum from +-inf (bbox_compute.py:10-45, :96-110), in every branch, with per-view H, W and K;
* the coarse-geometry lattice: torch.meshgrid / linspace on the device (:144-149);
* coarse geometry: model.density + activate_density on that lattice, alpha > thres, amin / amax (:150-160) -- DenseGrid at 160^3
  and at a non-cubic world size, the no-active-voxel fallback, a TensoRF density;
* end to end: coarse checkpoint -> compute_bbox_by_coarse_geo -> the fine DirectVoxGO's world_size and voxel_size.
"""
import contextlib
import io
import os
import types

import numpy as np
import pytest
import torch

from tests.util import ROOT, assert_close, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda'
GOLDEN_RTOL = 2e-6        # CPU reference vs GPU: the ray arithmetic of test_rays_of_a_view_golden


def _cfg(dataset_type='blender', model='DVGO', ndc=False, inverse_y=False, flip_x=False, flip_y=False, unbounded_inward=False,
         unbounded_inner_r=1.0, boundary_ratio=0.0):
    ns = types.SimpleNamespace
    return ns(model=model, data=ns(dataset_type=dataset_type, ndc=ndc, inverse_y=inverse_y, flip_x=flip_x, flip_y=flip_y,
                                   unbounded_inward=unbounded_inward, unbounded_inner_r=unbounded_inner_r,
                                   boundary_ratio=boundary_ratio))


def _same(a, b, what):
    """Bit-identical, NaN where the other is NaN (torch.equal would call NaN unequal to itself)."""
    a, b = a.detach().cpu(), b.detach().cpu()
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert torch.equal(a.isnan(), b.isnan()), (what, a, b)
    ok = ~a.isnan()
    assert torch.equal(a[ok], b[ok]), (what, a.tolist(), b.tolist())


# ---- the reference's frustum composition, on this library's rays ----------------------------------------------------------------
def _torch_frustum(cfg, HW, Ks, poses, i_train, near, far, near_clip):
    from unboundednerfpytorch_b200 import rays
    branch = ('nerfpp' if cfg.data.dataset_type == 'nerfpp' or cfg.model == 'FourierGrid' else
              'unbounded' if cfg.data.unbounded_inward else 'bounded')
    xyz_min = torch.tensor([np.inf, np.inf, np.inf], device=DEV)
    xyz_max = -xyz_min
    for (H, W), K, c2w in zip(HW[i_train], Ks[i_train], poses[i_train]):
        rays_o, rays_d, viewdirs = rays.get_rays_of_a_view(H=H, W=W, K=K, c2w=c2w, ndc=cfg.data.ndc, inverse_y=cfg.data.inverse_y,
                                                           flip_x=cfg.data.flip_x, flip_y=cfg.data.flip_y)
        if branch == 'bounded':
            if cfg.data.ndc:
                pts = torch.stack([rays_o + rays_d * near, rays_o + rays_d * far])
            else:
                pts = torch.stack([rays_o + viewdirs * near, rays_o + viewdirs * far])
            xyz_min = torch.minimum(xyz_min, pts.amin((0, 1, 2)))
            xyz_max = torch.maximum(xyz_max, pts.amax((0, 1, 2)))
        else:
            pts = rays_o + rays_d * near_clip
            xyz_min = torch.minimum(xyz_min, pts.amin((0, 1)))
            xyz_max = torch.maximum(xyz_max, pts.amax((0, 1)))
    if branch != 'bounded':
        center = (xyz_min + xyz_max) * 0.5
        radius = (center - xyz_min).max() * cfg.data.unbounded_inner_r
        xyz_min, xyz_max = center - radius, center + radius
    return xyz_min, xyz_max


def _run(cfg, HW, Ks, poses, i_train, near, far, near_clip, block_num=2):
    from unboundednerfpytorch_b200 import bbox
    kw = {} if near_clip is None else dict(near_clip=near_clip)
    return bbox.compute_bbox_by_cam_frustrm(types.SimpleNamespace(block_num=block_num), cfg, HW, Ks, poses, i_train, near, far, **kw)


RAY_CASES = ('bounded', 'bounded_invy_flipx', 'bounded_ndc', 'unbounded', 'nerfpp', 'fouriergrid')


@pytest.mark.parametrize('tag', RAY_CASES)
def test_frustum_golden_cases(tag):
    g = load_golden('l2_bbox/frustum.pt')[tag]
    cfg = _cfg(**g['cfg'])
    lo, hi = _run(cfg, g['HW'], g['Ks'], g['poses'], g['i_train'], g['near'], g['far'], g['near_clip'])
    assert lo.is_cuda and hi.is_cuda and lo.dtype == torch.float32 and lo.shape == (3,)
    rlo, rhi = _torch_frustum(cfg, g['HW'], g['Ks'], g['poses'], g['i_train'], g['near'], g['far'], g['near_clip'])
    _same(lo, rlo, tag + ' xyz_min')
    _same(hi, rhi, tag + ' xyz_max')
    assert_close(lo, g['xyz_min'], rtol=GOLDEN_RTOL, what=tag + ' xyz_min vs reference')
    assert_close(hi, g['xyz_max'], rtol=GOLDEN_RTOL, what=tag + ' xyz_max vs reference')


def _cameras(gen, n, sizes):
    HW, Ks, poses = [], [], []
    for i in range(n):
        H, W = sizes[i % len(sizes)]
        f = float(0.8 * W + 40 * torch.rand(1, generator=gen))
        Ks.append(np.array([[f, 0, 0.5 * W + float(torch.rand(1, generator=gen))], [0, 1.02 * f, 0.5 * H - 0.3], [0, 0, 1]]))
        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=gen, dtype=torch.float64))
        t = torch.randn(3, 1, generator=gen, dtype=torch.float64) * 2
        poses.append(torch.cat([q, t], 1).numpy())
        HW.append((H, W))
    return np.array(HW), np.array(Ks), np.array(poses, dtype=np.float32)


@pytest.mark.parametrize('flags', [(False, False, False, False), (False, True, True, False), (True, False, False, True),
                                   (True, True, True, True)])
def test_frustum_per_view_sizes(flags):
    """Views of different H, W and K, sizes up to 801 x 799 (many blocks per view), every branch, each flag combination."""
    ndc, inverse_y, flip_x, flip_y = flags
    gen = torch.Generator().manual_seed(11 + sum(f << i for i, f in enumerate(flags)))
    HW, Ks, poses = _cameras(gen, 7, [(801, 799), (33, 1), (1, 65), (257, 129), (480, 641)])
    if ndc:   # forward-facing: keep the camera axes close to the identity so rays_d[2] stays away from zero
        poses[:, :, :3] = np.eye(3, dtype=np.float32) + 0.05 * poses[:, :, :3]
        poses[:, 2, 3] = 0.1 * poses[:, 2, 3]
    i_train = np.array([6, 0, 3, 1, 4, 2])
    for kw in (dict(), dict(unbounded_inward=True, unbounded_inner_r=0.7), dict(dataset_type='nerfpp'),
               dict(model='FourierGrid', unbounded_inner_r=1.3)):
        cfg = _cfg(ndc=ndc, inverse_y=inverse_y, flip_x=flip_x, flip_y=flip_y, **kw)
        near, far = (0.0, 1.0) if ndc else (0.2, 5.5)
        lo, hi = _run(cfg, HW, Ks, poses, i_train, near, far, 0.37)
        rlo, rhi = _torch_frustum(cfg, HW, Ks, poses, i_train, near, far, 0.37)
        _same(lo, rlo, f'{kw} {flags} xyz_min')
        _same(hi, rhi, f'{kw} {flags} xyz_max')


def test_frustum_nan_propagates():
    """A NaN camera translation makes that axis NaN, as torch.minimum / amin propagate it; an empty view set leaves +-inf."""
    from unboundednerfpytorch_b200 import bbox
    gen = torch.Generator().manual_seed(5)
    HW, Ks, poses = _cameras(gen, 3, [(9, 7)])
    poses[1, 1, 3] = np.nan
    cfg = _cfg()
    lo, hi = _run(cfg, HW, Ks, poses, np.arange(3), 0.1, 2.0, None)
    rlo, rhi = _torch_frustum(cfg, HW, Ks, poses, np.arange(3), 0.1, 2.0, None)
    assert bool(lo[1].isnan()) and bool(hi[1].isnan()) and not bool(lo[0].isnan())
    _same(lo, rlo, 'xyz_min')
    _same(hi, rhi, 'xyz_max')
    lo, hi = bbox.frustum_bounds(HW[:0], Ks[:0], poses[:0], False, False, False, False, 0.1, 2.0)
    assert torch.equal(lo.cpu(), torch.full((3,), np.inf)) and torch.equal(hi.cpu(), torch.full((3,), -np.inf))


def test_frustum_matches_ray_kernel_bits():
    """The frustum points come from the same per-pixel arithmetic as ubn_get_rays_of_a_view: a one-pixel view bounds exactly
    its ray's points."""
    from unboundednerfpytorch_b200 import bbox, rays
    gen = torch.Generator().manual_seed(9)
    HW, Ks, poses = _cameras(gen, 1, [(1, 1)])
    o, d, v = rays.get_rays_of_a_view(1, 1, Ks[0], poses[0], False, False, False, False)
    lo, hi = bbox.frustum_bounds(HW, Ks, poses, False, False, False, False, 0.75, 0.75)
    p = (o + v * 0.75).reshape(3)
    _same(lo, p, 'one-pixel min')
    _same(hi, p, 'one-pixel max')


# ---- coarse geometry ----------------------------------------------------------------------------------------------------------
def _torch_lattice(xyz_min, xyz_max, ws):
    interp = torch.stack(torch.meshgrid(*[torch.linspace(0, 1, int(n), device=DEV) for n in ws], indexing='ij'), -1)
    return xyz_min * (1 - interp) + xyz_max * interp


def _torch_coarse_geo(model, thres):
    dense_xyz = _torch_lattice(model.xyz_min, model.xyz_max, model.world_size)
    alpha = model.activate_density(model.density(dense_xyz))
    mask = alpha > thres
    if not mask.max() > 0:
        mask = alpha > -1
    active = dense_xyz[mask]
    return active.amin(0), active.amax(0), int(mask.sum())


@pytest.mark.parametrize('ws', [(160, 160, 160), (17, 20, 11), (1, 7, 2), (64, 3, 129)])
def test_lattice_points(ws):
    from unboundednerfpytorch_b200 import bbox
    lo = torch.tensor([-1.3, -0.7, -2.1], device=DEV)
    hi = torch.tensor([1.1, 2.05, 0.35], device=DEV)
    xyz = bbox.lattice_points(lo.tolist(), hi.tolist(), ws)
    ref = _torch_lattice(lo, hi, ws)
    assert xyz.shape == ref.shape
    assert torch.equal(xyz, ref)


def _dense_model(ws_target, lo, hi, seed, alpha_init=1e-2):
    from unboundednerfpytorch_b200 import models
    g = torch.Generator().manual_seed(seed)
    nv = int(np.prod(ws_target))
    with contextlib.redirect_stdout(io.StringIO()):
        m = models.DirectVoxGO(xyz_min=lo, xyz_max=hi, num_voxels=nv, num_voxels_base=nv, alpha_init=alpha_init, rgbnet_dim=0)
    X, Y, Z = [int(v) for v in m.world_size]
    with torch.no_grad():
        ax = [torch.linspace(-1, 1, k) for k in (X, Y, Z)]
        r2 = sum(a ** 2 for a in torch.meshgrid(*ax, indexing='ij'))
        m.density.grid.copy_((14.0 * (0.3 - r2) + 2.0 * torch.randn(X, Y, Z, generator=g))[None, None])
    return m.to(DEV)


@pytest.mark.parametrize('shape', ['cube160', 'noncubic'])
def test_coarse_geo_dense(shape):
    from unboundednerfpytorch_b200 import bbox
    if shape == 'cube160':
        m = _dense_model((160, 160, 160), [-1.0] * 3, [1.0] * 3, 3)
        assert [int(v) for v in m.world_size] == [160, 160, 160]
    else:
        m = _dense_model((40, 30, 20), [-1.0, -1.3, -0.6], [1.1, 1.2, 0.8], 4)
        assert len({int(v) for v in m.world_size}) == 3
    for thres in (1e-4, 1e-2, 0.3):
        lo, hi = bbox.coarse_geo_bounds(m, thres)
        rlo, rhi, n = _torch_coarse_geo(m, thres)
        assert 0 < n < int(np.prod([int(v) for v in m.world_size])), (thres, n)
        _same(lo, rlo, f'{shape} thres {thres} xyz_min')
        _same(hi, rhi, f'{shape} thres {thres} xyz_max')


def test_coarse_geo_fallback(capsys):
    """No lattice point above the threshold: the bounds of the whole lattice, with the reference's warning."""
    from unboundednerfpytorch_b200 import bbox
    m = _dense_model((23, 19, 29), [-1.0, -1.3, -0.6], [1.1, 1.2, 0.8], 6)
    lo, hi = bbox.coarse_geo_bounds(m, 1.0)
    assert 'No activated voxels' in capsys.readouterr().out
    rlo, rhi, _ = _torch_coarse_geo(m, 1.0)
    _same(lo, rlo, 'xyz_min')
    _same(hi, rhi, 'xyz_max')
    _same(lo, m.xyz_min, 'lattice corner')


def test_coarse_geo_tensorf():
    from unboundednerfpytorch_b200 import bbox, ckpt, models
    g = load_golden('l2_bbox/coarse_geo.pt')['tensorf']
    path = os.path.join(ROOT, 'tests', 'golden', g['path'])
    m = ckpt.load_model(models.DirectVoxGO, path, DEV)
    for thres in (g['thres'], 1e-3, 0.5):
        lo, hi = bbox.coarse_geo_bounds(m, thres)
        rlo, rhi, _ = _torch_coarse_geo(m, thres)
        _same(lo, rlo, f'tensorf {thres} xyz_min')
        _same(hi, rhi, f'tensorf {thres} xyz_max')
    with contextlib.redirect_stdout(io.StringIO()):
        lo, hi = bbox.compute_bbox_by_coarse_geo(models.DirectVoxGO, path, g['thres'], DEV)
    assert_close(lo, g['xyz_min'], rtol=GOLDEN_RTOL, what='tensorf xyz_min vs reference')
    assert_close(hi, g['xyz_max'], rtol=GOLDEN_RTOL, what='tensorf xyz_max vs reference')


@pytest.mark.parametrize('tag', ['dvgo_some', 'dvgo_none'])
def test_coarse_geo_golden(tag):
    from unboundednerfpytorch_b200 import bbox, ckpt, models
    g = load_golden('l2_bbox/coarse_geo.pt')[tag]
    path = os.path.join(ROOT, 'tests', 'golden', g['path'])
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        lo, hi = bbox.compute_bbox_by_coarse_geo(models.DirectVoxGO, path, g['thres'], DEV)
    assert lo.is_cuda and lo.dtype == torch.float32 and lo.shape == (3,)
    assert ('No activated voxels' in out.getvalue()) == (tag == 'dvgo_none')
    assert_close(lo, g['xyz_min'], rtol=GOLDEN_RTOL, what=tag + ' xyz_min vs reference')
    assert_close(hi, g['xyz_max'], rtol=GOLDEN_RTOL, what=tag + ' xyz_max vs reference')
    rlo, rhi, _ = _torch_coarse_geo(ckpt.load_model(models.DirectVoxGO, path, DEV), g['thres'])
    _same(lo, rlo, tag + ' xyz_min')
    _same(hi, rhi, tag + ' xyz_max')


def test_coarse_to_fine_end_to_end():
    """run_train.py:379-385: the coarse checkpoint's bounds build the fine DirectVoxGO (with the coarse mask cache) at the
    reference's world_size and voxel_size."""
    from unboundednerfpytorch_b200 import bbox, models
    rec = load_golden('l2_bbox/coarse_geo.pt')
    g, fine = rec['dvgo_some'], rec['fine']
    path = os.path.join(ROOT, 'tests', 'golden', g['path'])
    with contextlib.redirect_stdout(io.StringIO()):
        lo, hi = bbox.compute_bbox_by_coarse_geo(models.DirectVoxGO, path, g['thres'], DEV)
        m = models.DirectVoxGO(xyz_min=lo, xyz_max=hi, mask_cache_path=path, mask_cache_thres=1e-3, **fine['kwargs']).to(DEV)
    assert m.world_size.tolist() == fine['world_size'].tolist()
    assert_close(m.xyz_min, fine['xyz_min'], rtol=GOLDEN_RTOL, what='fine xyz_min')
    assert_close(m.xyz_max, fine['xyz_max'], rtol=GOLDEN_RTOL, what='fine xyz_max')
    assert abs(float(m.voxel_size) - fine['voxel_size']) <= 1e-6 * fine['voxel_size']
    assert abs(float(m.voxel_size_ratio) - fine['voxel_size_ratio']) <= 1e-6 * fine['voxel_size_ratio']
    assert m.mask_cache.mask.shape == tuple(fine['world_size'].tolist())
