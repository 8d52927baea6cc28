"""Scene bounding boxes with the reference's names and signatures (FourierGrid/bbox_compute.py), the ray and lattice passes on
device: one launch reduces the frustum points of every training view (``ubn_frustum_bounds``), one launch reduces the active
voxels of a coarse density (``ubn_lattice_bounds``), instead of ~20 torch ops and a full ray tensor per view, or a [X,Y,Z,3]
lattice plus its density and alpha tensors.

* ``compute_bbox_by_cam_frustrm`` -- bbox_compute.py:113-133, the same dispatch on ``cfg.data.dataset_type``, ``cfg.model`` and
  ``cfg.data.unbounded_inward``.  The Waymo and Mega-NeRF branches use camera centres only and run on the host, as there.
* ``compute_bbox_by_coarse_geo`` -- bbox_compute.py:136-165, loading through ``ckpt.load_model`` (the reference's commented-out
  path, :140) rather than load_everything.load_existing_model.
* ``coarse_geo_bounds`` -- the same bounds for a DirectVoxGO already in memory (DenseGrid or TensoRFGrid density).

The results are [3] float32 tensors on the device, equal to what the reference computes when run_FourierGrid.py:87 makes CUDA the
default tensor type.  Min and max do not depend on the reduction order, so they are exact: only a bound that is zero may differ in
the sign of that zero, which torch leaves to the order it visits the points in.
"""
import ctypes
import time

import numpy as np
import torch

from . import grid as G
from ._cabi import c_f, c_i64, c_int, check, ptr, stream_of
from .functional import host_scalar
from .ops import _Guard


def _device(poses, host_ok=False):
    """The device of the result: that of ``poses`` when it is a CUDA tensor, else the current CUDA device (or, for the branches
    that only read camera centres on the host, the CPU when there is no CUDA device)."""
    if torch.is_tensor(poses) and poses.is_cuda:
        return poses.device
    if host_ok and not torch.cuda.is_available():
        return torch.device('cpu')
    return torch.device('cuda', torch.cuda.current_device())


def _host(x):
    return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def _empty_bounds(device):
    return torch.tensor([np.inf] * 3 + [-np.inf] * 3, dtype=torch.float32, device=device)


def _f3(v):
    return (ctypes.c_float * 3)(*[float(a) for a in v])


# ---- camera frustum -----------------------------------------------------------------------------------------------------------
def frustum_bounds(HW, Ks, poses, ndc, inverse_y, flip_x, flip_y, near, far=None, inward=False, device=None):
    """(xyz_min, xyz_max) of the frustum points of every view (the 'center' rays of rays.get_rays_of_a_view, bit for bit):
    rays_o + rays_d * near when ``inward`` (bbox_compute.py:19, :38), else rays_o + dir * near and rays_o + dir * far with
    dir = rays_d under NDC and viewdirs otherwise (:104-107).  HW [n,2], Ks [n,3,3], poses [n,3|4,4]; views may differ in H, W
    and K.  One upload of the camera table and one reduction launch; no ray is written."""
    hw = np.ascontiguousarray(_host(HW).reshape(-1, 2).astype(np.int64))
    n = hw.shape[0]
    if (hw <= 0).any() or (hw > np.iinfo(np.int32).max).any():
        raise ValueError('image sizes must be positive')
    K = np.ascontiguousarray(_host(Ks).astype(np.float32).reshape(n, 9))
    c2w = np.ascontiguousarray(_host(poses).astype(np.float32)[:, :3, :4].reshape(n, 12))
    dev = torch.device(device) if device is not None else _device(poses)
    hw_d, K_d, c2w_d = (torch.from_numpy(a).to(dev) for a in (hw.astype(np.int32), K, c2w))
    bounds = _empty_bounds(dev)
    max_pixels = int((hw[:, 0] * hw[:, 1]).max()) if n else 0
    with _Guard(bounds) as lib:
        check(lib.ubn_frustum_bounds(ptr(hw_d), ptr(K_d), ptr(c2w_d), c_i64(n), c_i64(max_pixels), c_int(int(bool(ndc))),
                                     c_int(int(bool(inverse_y))), c_int(int(bool(flip_x))), c_int(int(bool(flip_y))),
                                     c_int(int(bool(inward))), c_f(float(near)), c_f(float(far) if far is not None else 0.),
                                     ptr(bounds), stream_of(bounds)))
    return bounds[:3], bounds[3:]


def _centre_radius(cfg, xyz_min, xyz_max):
    """The cube around the box's centre with the half-extent of its longest axis times unbounded_inner_r (:22-25)."""
    center = (xyz_min + xyz_max) * 0.5
    radius = (center - xyz_min).max() * cfg.data.unbounded_inner_r
    return center - radius, center + radius


def _camera_centres(poses, i_train):
    """[c2w[:, 3][a].item() for c2w in poses[i_train]] per axis a (:50-53, :77-80)."""
    xs, ys, zs = [], [], []
    for c2w in _host(poses)[np.asarray(i_train)]:
        xs.append(c2w[:, 3][0].item())
        ys.append(c2w[:, 3][1].item())
        zs.append(c2w[:, 3][2].item())
    return xs, ys, zs


def _selected(HW, Ks, poses, i_train):
    idx = np.asarray(i_train)
    return _host(HW)[idx], _host(Ks)[idx], _host(poses)[idx]


def _compute_bbox_by_cam_frustrm_unbounded(cfg, HW, Ks, poses, i_train, near_clip):
    """bbox_compute.py:10-26: the frustum points rays_o + rays_d * near_clip, then the cube around their box."""
    if near_clip is None:
        raise TypeError('the unbounded-inward branch needs near_clip')
    xyz_min, xyz_max = frustum_bounds(*_selected(HW, Ks, poses, i_train), cfg.data.ndc, cfg.data.inverse_y, cfg.data.flip_x,
                                      cfg.data.flip_y, near_clip, inward=True, device=_device(poses))
    return _centre_radius(cfg, xyz_min, xyz_max)


def FourierGrid_compute_bbox_by_cam_frustrm_nerfpp(cfg, HW, Ks, poses, i_train, near_clip):
    """bbox_compute.py:29-45, the same body as the unbounded-inward branch."""
    return _compute_bbox_by_cam_frustrm_unbounded(cfg, HW, Ks, poses, i_train, near_clip)


def FourierGrid_compute_bbox_by_cam_frustrm_waymo(cfg, HW, Ks, poses, i_train, near_clip):
    """bbox_compute.py:48-72: the camera centres' box extended by fixed margins, then the cube around it (host)."""
    xs, ys, zs = _camera_centres(poses, i_train)
    zmin, zmax = min(zs), max(zs)
    xmin, xmax = min(xs), max(xs)
    ymin, ymax = min(ys), max(ys)
    x_extend = 0.05
    y_extend = 0.01
    z_extend = 0.01
    xyz_min = torch.tensor([xmin - x_extend, ymin - y_extend, zmin - z_extend], dtype=torch.float32)
    xyz_max = torch.tensor([xmax + x_extend, ymax + y_extend, zmax + z_extend], dtype=torch.float32)
    dev = _device(poses, host_ok=True)
    return tuple(t.to(dev) for t in _centre_radius(cfg, xyz_min, xyz_max))


def FourierGrid_compute_bbox_by_cam_frustrm_mega(cfg, HW, Ks, poses, i_train, near_clip):
    """bbox_compute.py:75-93: the camera centres' box widened by boundary_ratio of its extent, then the cube around it (host).
    The reference defines it without dispatching to it (Mega-NeRF configs run cfg.model 'FourierGrid', the nerfpp branch)."""
    xs, ys, zs = _camera_centres(poses, i_train)
    zmin, zmax = min(zs), max(zs)
    xmin, xmax = min(xs), max(xs)
    ymin, ymax = min(ys), max(ys)
    x_distance, y_distance, z_distance = abs(xmax - xmin), abs(ymax - ymin), abs(zmax - zmin)
    boundary_ratio = cfg.data.boundary_ratio
    xyz_min = torch.tensor([xmin - boundary_ratio * x_distance, ymin - boundary_ratio * y_distance,
                            zmin - boundary_ratio * z_distance], dtype=torch.float32)
    xyz_max = torch.tensor([xmax + boundary_ratio * x_distance, ymax + boundary_ratio * y_distance,
                            zmax + boundary_ratio * z_distance], dtype=torch.float32)
    dev = _device(poses, host_ok=True)
    return tuple(t.to(dev) for t in _centre_radius(cfg, xyz_min, xyz_max))


def _compute_bbox_by_cam_frustrm_bounded(cfg, HW, Ks, poses, i_train, near, far):
    """bbox_compute.py:96-110: the near and far frustum points of every ray."""
    return frustum_bounds(*_selected(HW, Ks, poses, i_train), cfg.data.ndc, cfg.data.inverse_y, cfg.data.flip_x, cfg.data.flip_y,
                          near, far, inward=False, device=_device(poses))


def frustum_branch(cfg):
    """The branch compute_bbox_by_cam_frustrm takes (bbox_compute.py:117-128): 'waymo', 'nerfpp' (a nerfpp dataset or any
    FourierGrid model), 'unbounded' or 'bounded'."""
    if cfg.data.dataset_type == 'waymo':
        return 'waymo'
    if cfg.data.dataset_type == 'nerfpp' or cfg.model == 'FourierGrid':
        return 'nerfpp'
    if cfg.data.unbounded_inward:
        return 'unbounded'
    return 'bounded'


def compute_bbox_by_cam_frustrm(args, cfg, HW, Ks, poses, i_train, near, far, **kwargs):
    """bbox_compute.py:113-133 -> (xyz_min, xyz_max), [3] float32 tensors on the CUDA device."""
    verbose = args.block_num <= 1
    if verbose:
        print('compute_bbox_by_cam_frustrm: start')
    branch = frustum_branch(cfg)
    if branch == 'waymo':
        xyz_min, xyz_max = FourierGrid_compute_bbox_by_cam_frustrm_waymo(cfg, HW, Ks, poses, i_train, kwargs.get('near_clip', None))
    elif branch == 'nerfpp':
        xyz_min, xyz_max = FourierGrid_compute_bbox_by_cam_frustrm_nerfpp(cfg, HW, Ks, poses, i_train, kwargs.get('near_clip', None))
    elif branch == 'unbounded':
        xyz_min, xyz_max = _compute_bbox_by_cam_frustrm_unbounded(cfg, HW, Ks, poses, i_train, kwargs.get('near_clip', None))
    else:
        xyz_min, xyz_max = _compute_bbox_by_cam_frustrm_bounded(cfg, HW, Ks, poses, i_train, near, far)
    if verbose:
        print('compute_bbox_by_cam_frustrm: xyz_min', xyz_min)
        print('compute_bbox_by_cam_frustrm: xyz_max', xyz_max)
        print('compute_bbox_by_cam_frustrm: finish')
    return xyz_min, xyz_max


# ---- coarse geometry ----------------------------------------------------------------------------------------------------------
def lattice_points(xyz_min, xyz_max, world_size, device=None):
    """[X,Y,Z,3] = xyz_min * (1 - t) + xyz_max * t, t = torch.linspace(0, 1, n) per axis (bbox_compute.py:144-149), bit for bit."""
    X, Y, Z = [int(v) for v in world_size]
    dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    xyz = torch.empty(X, Y, Z, 3, dtype=torch.float32, device=dev)
    with _Guard(xyz) as lib:
        check(lib.ubn_lattice_points(_f3(xyz_min), _f3(xyz_max), c_i64(X), c_i64(Y), c_i64(Z), ptr(xyz), stream_of(xyz)))
    return xyz


@torch.no_grad()
def coarse_geo_bounds(model, thres):
    """bbox_compute.py:144-160 for a DirectVoxGO in memory -> (xyz_min, xyz_max), the bounds of the lattice points of
    model.world_size whose alpha exceeds ``thres`` (of every lattice point, with the reference's warning, when none does).
    A DenseGrid density is read, activated and reduced in one launch; a TensoRFGrid density is evaluated on the materialised
    lattice (model.density, as the reference's generic call does) and its alpha reduced by the same reduction."""
    if not model.xyz_min.is_cuda:
        raise RuntimeError('coarse_geo_bounds needs the model on a CUDA device')
    dev = model.xyz_min.device
    ws = [int(v) for v in model.world_size]
    lo, hi = model.xyz_min.tolist(), model.xyz_max.tolist()
    bounds = _empty_bounds(dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    if isinstance(model.density, G.TensoRFGrid):
        alpha = model.activate_density(model.density(lattice_points(lo, hi, ws, dev).reshape(-1, 3))).contiguous()

        def reduce(t):
            with _Guard(bounds) as lib:
                check(lib.ubn_lattice_bounds_alpha(ptr(alpha), _f3(lo), _f3(hi), c_i64(ws[0]), c_i64(ws[1]), c_i64(ws[2]),
                                                   c_f(float(t)), ptr(bounds), ptr(count), stream_of(bounds)))
    elif isinstance(model.density, G.DenseGrid):
        grid = model.density.grid.data
        mn, mx = model.density._bounds()
        desc = G.grid_desc(grid, mn, mx, model.density.num_freqs)
        shift, interval = host_scalar(model._density_shift()), host_scalar(model._voxel_size_ratio())

        def reduce(t):
            with _Guard(bounds) as lib:
                check(lib.ubn_lattice_bounds(ptr(grid), desc, _f3(lo), _f3(hi), c_i64(ws[0]), c_i64(ws[1]), c_i64(ws[2]),
                                             c_f(shift), c_f(interval), c_f(float(t)), ptr(bounds), ptr(count), stream_of(bounds)))
    else:
        raise NotImplementedError(f'coarse_geo_bounds: {type(model.density).__name__} density')
    reduce(thres)
    if int(count.item()) == 0:
        print('Warning! No activated voxels found.')
        reduce(-1)
        if int(count.item()) == 0:
            raise RuntimeError('compute_bbox_by_coarse_geo: no lattice point has a finite alpha')
    return bounds[:3], bounds[3:]


@torch.no_grad()
def compute_bbox_by_coarse_geo(model_class, model_path, thres, device, args=None, cfg=None):
    """bbox_compute.py:136-165 -> (xyz_min, xyz_max) of the coarse checkpoint's active voxels, [3] float32 tensors on
    ``device``.  ``args`` and ``cfg`` are accepted for the reference's signature; the checkpoint carries everything needed."""
    print('compute_bbox_by_coarse_geo: start')
    eps_time = time.time()
    from . import ckpt
    model = ckpt.load_model(model_class, model_path)
    model.to(device)
    xyz_min, xyz_max = coarse_geo_bounds(model, thres)
    print('compute_bbox_by_coarse_geo: xyz_min', xyz_min)
    print('compute_bbox_by_coarse_geo: xyz_max', xyz_max)
    eps_time = time.time() - eps_time
    print('compute_bbox_by_coarse_geo: finish (eps time:', eps_time, 'secs)')
    return xyz_min, xyz_max
