"""Host-side mirror of the reference's four extension modules, on top of the C ABI.

Same function names, argument order/meaning, return values and error behaviour as
``render_utils_cuda`` (FourierGrid/cuda/render_utils.cpp:170-184), ``total_variation_cuda``
(total_variation.cpp:22-24), ``adam_upd_cuda`` (adam_upd.cpp:79-86) and ``ub360_utils_cuda``
(ub360_utils.cpp:20-22): tensor arguments must be CUDA + contiguous (``RuntimeError`` otherwise, the
reference's CHECK_CUDA / CHECK_CONTIGUOUS, render_utils.cpp:46-48); outputs are freshly allocated.
Differences, all supersets: outputs live on the *input's* device (the reference hard-codes the current
device, SURVEY.md 2a), kernels run on torch's current stream, launch errors are checked, fp32 only.
"""
import ctypes

import torch

from . import _cabi
from ._cabi import c_f, c_i64, c_int, check, ptr, stream_of


def _chk(x, name, dtype=torch.float32, contiguous=True):
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise RuntimeError(f'{name} must be a CUDA tensor')
    if contiguous and not x.is_contiguous():
        raise RuntimeError(f'{name} must be contiguous')
    if dtype is not None and x.dtype != dtype:
        raise RuntimeError(f'{name} must be {dtype} (got {x.dtype})')
    return x


def _scalar(v):
    """Python number, 0-d / 1-element tensor -> float (the reference relies on pybind's float caster,
    i.e. Tensor.__float__, for `shift` / `interval`: dvgo.py:439, FourierGrid_model.py:493)."""
    return float(v)


class _Guard:
    """CUDAGuard equivalent: make the tensor's device current for the duration of the call."""

    def __init__(self, t):
        self.dev = torch.cuda.device(t.device)

    def __enter__(self):
        self.dev.__enter__()
        return _cabi.load()

    def __exit__(self, *a):
        return self.dev.__exit__(*a)


# --------------------------------------------------------------------------------------------------
# render_utils_cuda
# --------------------------------------------------------------------------------------------------
def infer_t_minmax(rays_o, rays_d, xyz_min, xyz_max, near, far):
    _chk(rays_o, 'rays_o'); _chk(rays_d, 'rays_d'); _chk(xyz_min, 'xyz_min'); _chk(xyz_max, 'xyz_max')
    n = rays_o.shape[0]
    t_min = torch.empty(n, dtype=torch.float32, device=rays_o.device)
    t_max = torch.empty_like(t_min)
    with _Guard(rays_o) as lib:
        check(lib.ubn_infer_t_minmax(ptr(rays_o), ptr(rays_d), ptr(xyz_min), ptr(xyz_max), c_f(near), c_f(far),
                                     c_i64(n), ptr(t_min), ptr(t_max), stream_of(rays_o)))
    return [t_min, t_max]


def infer_n_samples(rays_d, t_min, t_max, stepdist):
    _chk(rays_d, 'rays_d'); _chk(t_min, 't_min'); _chk(t_max, 't_max')
    n = t_min.shape[0]
    out = torch.empty(n, dtype=torch.int64, device=rays_d.device)
    with _Guard(rays_d) as lib:
        check(lib.ubn_infer_n_samples(ptr(rays_d), ptr(t_min), ptr(t_max), c_f(stepdist), c_i64(n), ptr(out),
                                      stream_of(rays_d)))
    return out


def infer_ray_start_dir(rays_o, rays_d, t_min):
    _chk(rays_o, 'rays_o'); _chk(rays_d, 'rays_d'); _chk(t_min, 't_min')
    n = rays_o.shape[0]
    start, dirs = torch.empty_like(rays_o), torch.empty_like(rays_o)
    with _Guard(rays_o) as lib:
        check(lib.ubn_infer_ray_start_dir(ptr(rays_o), ptr(rays_d), ptr(t_min), c_i64(n), ptr(start), ptr(dirs),
                                          stream_of(rays_o)))
    return [start, dirs]


def sample_pts_on_rays(rays_o, rays_d, xyz_min, xyz_max, near, far, stepdist):
    _chk(rays_o, 'rays_o'); _chk(rays_d, 'rays_d'); _chk(xyz_min, 'xyz_min'); _chk(xyz_max, 'xyz_max')
    dev = rays_o.device
    n = rays_o.shape[0]
    t_min = torch.empty(n, dtype=torch.float32, device=dev)
    t_max = torch.empty_like(t_min)
    n_steps = torch.empty(n, dtype=torch.int64, device=dev)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    scratch = torch.empty(n // 1024 + 4, dtype=torch.int64, device=dev)
    with _Guard(rays_o) as lib:
        st = stream_of(rays_o)
        check(lib.ubn_sample_pts_count(ptr(rays_o), ptr(rays_d), ptr(xyz_min), ptr(xyz_max), c_f(near), c_f(far),
                                       c_f(stepdist), c_i64(n), ptr(t_min), ptr(t_max), ptr(n_steps), ptr(offsets),
                                       ptr(scratch), st))
        total = int(offsets[n].item())   # the one host sync the return contract requires (ragged size)
        pts = torch.empty(total, 3, dtype=torch.float32, device=dev)
        mask = torch.empty(total, dtype=torch.bool, device=dev)
        ray_id = torch.empty(total, dtype=torch.int64, device=dev)
        step_id = torch.empty(total, dtype=torch.int64, device=dev)
        check(lib.ubn_sample_pts_emit(ptr(rays_o), ptr(rays_d), ptr(xyz_min), ptr(xyz_max), ptr(t_min), ptr(offsets),
                                      c_f(stepdist), c_i64(n), c_i64(total), ptr(pts), ptr(mask), ptr(ray_id),
                                      ptr(step_id), st))
    return [pts, mask, ray_id, step_id, n_steps, t_min, t_max]


def sample_ndc_pts_on_rays(rays_o, rays_d, xyz_min, xyz_max, N_samples):
    _chk(rays_o, 'rays_o'); _chk(rays_d, 'rays_d'); _chk(xyz_min, 'xyz_min'); _chk(xyz_max, 'xyz_max')
    n = rays_o.shape[0]
    pts = torch.empty(n, N_samples, 3, dtype=torch.float32, device=rays_o.device)
    mask = torch.empty(n, N_samples, dtype=torch.bool, device=rays_o.device)
    with _Guard(rays_o) as lib:
        check(lib.ubn_sample_ndc_pts_on_rays(ptr(rays_o), ptr(rays_d), ptr(xyz_min), ptr(xyz_max), c_i64(N_samples),
                                             c_i64(n), ptr(pts), ptr(mask), stream_of(rays_o)))
    return [pts, mask]


def sample_bg_pts_on_rays(rays_o, rays_d, t_max, bg_preserve, N_samples):
    _chk(rays_o, 'rays_o'); _chk(rays_d, 'rays_d'); _chk(t_max, 't_max')
    n = rays_o.shape[0]
    pts = torch.empty(n, N_samples, 3, dtype=torch.float32, device=rays_o.device)
    with _Guard(rays_o) as lib:
        check(lib.ubn_sample_bg_pts_on_rays(ptr(rays_o), ptr(rays_d), ptr(t_max), c_f(bg_preserve), c_i64(N_samples),
                                            c_i64(n), ptr(pts), stream_of(rays_o)))
    return pts


def maskcache_lookup(world, xyz, xyz2ijk_scale, xyz2ijk_shift):
    _chk(world, 'world', torch.bool); _chk(xyz, 'xyz')
    _chk(xyz2ijk_scale, 'xyz2ijk_scale'); _chk(xyz2ijk_shift, 'xyz2ijk_shift')
    n = xyz.shape[0]
    out = torch.empty(n, dtype=torch.bool, device=xyz.device)
    if n == 0:
        return out
    with _Guard(xyz) as lib:
        check(lib.ubn_maskcache_lookup(ptr(world), ptr(xyz), ptr(xyz2ijk_scale), ptr(xyz2ijk_shift),
                                       c_i64(world.shape[0]), c_i64(world.shape[1]), c_i64(world.shape[2]), c_i64(n),
                                       ptr(out), stream_of(xyz)))
    return out


def raw2alpha(density, shift, interval):
    _chk(density, 'density')
    exp_d, alpha = torch.empty_like(density), torch.empty_like(density)
    with _Guard(density) as lib:
        check(lib.ubn_raw2alpha(ptr(density), c_f(_scalar(shift)), c_f(_scalar(interval)), ptr(None),
                                c_i64(density.numel()), ptr(exp_d), ptr(alpha), stream_of(density)))
    return [exp_d, alpha]


def raw2alpha_nonuni(density, shift, interval):
    _chk(density, 'density'); _chk(interval, 'interval')
    exp_d, alpha = torch.empty_like(density), torch.empty_like(density)
    with _Guard(density) as lib:
        check(lib.ubn_raw2alpha(ptr(density), c_f(_scalar(shift)), c_f(0.0), ptr(interval), c_i64(density.numel()),
                                ptr(exp_d), ptr(alpha), stream_of(density)))
    return [exp_d, alpha]


def raw2alpha_backward(exp_d, grad_back, interval):
    _chk(exp_d, 'exp'); _chk(grad_back, 'grad_back')
    grad = torch.empty_like(exp_d)
    with _Guard(exp_d) as lib:
        check(lib.ubn_raw2alpha_backward(ptr(exp_d), ptr(grad_back), c_f(_scalar(interval)), ptr(None),
                                         c_i64(exp_d.numel()), ptr(grad), stream_of(exp_d)))
    return grad


def raw2alpha_nonuni_backward(exp_d, grad_back, interval):
    _chk(exp_d, 'exp'); _chk(grad_back, 'grad_back'); _chk(interval, 'interval')
    grad = torch.empty_like(exp_d)
    with _Guard(exp_d) as lib:
        check(lib.ubn_raw2alpha_backward(ptr(exp_d), ptr(grad_back), c_f(0.0), ptr(interval), c_i64(exp_d.numel()),
                                         ptr(grad), stream_of(exp_d)))
    return grad


def alpha2weight(alpha, ray_id, n_rays):
    _chk(alpha, 'alpha'); _chk(ray_id, 'ray_id', torch.int64)
    dev = alpha.device
    n = alpha.numel()
    weight, T = torch.empty_like(alpha), torch.empty_like(alpha)
    last = torch.empty(n_rays, dtype=torch.float32, device=dev)
    i_start = torch.empty(n_rays, dtype=torch.int64, device=dev)
    i_end = torch.empty(n_rays, dtype=torch.int64, device=dev)
    with _Guard(alpha) as lib:
        check(lib.ubn_alpha2weight(ptr(alpha), ptr(ray_id), c_i64(n), c_i64(n_rays), ptr(weight), ptr(T), ptr(last),
                                   ptr(i_start), ptr(i_end), stream_of(alpha)))
    return [weight, T, last, i_start, i_end]


def alpha2weight_backward(alpha, weight, T, alphainv_last, i_start, i_end, n_rays, grad_weights, grad_last):
    _chk(alpha, 'alpha'); _chk(weight, 'weight'); _chk(T, 'T'); _chk(alphainv_last, 'alphainv_last')
    _chk(i_start, 'i_start', torch.int64); _chk(i_end, 'i_end', torch.int64)
    _chk(grad_weights, 'grad_weights'); _chk(grad_last, 'grad_last')
    grad = torch.empty_like(alpha)
    with _Guard(alpha) as lib:
        check(lib.ubn_alpha2weight_backward(ptr(alpha), ptr(weight), ptr(T), ptr(alphainv_last), ptr(i_start),
                                            ptr(i_end), c_i64(alpha.numel()), c_i64(n_rays), ptr(grad_weights),
                                            ptr(grad_last), ptr(grad), stream_of(alpha)))
    return grad


# --------------------------------------------------------------------------------------------------
# total_variation_cuda / adam_upd_cuda / ub360_utils_cuda
# --------------------------------------------------------------------------------------------------
def _sweep_layout(param):
    """(lead, inner) of a 5-D [P,C,X,Y,Z] grid stored either contiguous or channels-last."""
    if param.dim() != 5:
        raise RuntimeError('param must be 5-D [P,C,X,Y,Z]')
    P, C = param.shape[0], param.shape[1]
    if param.is_contiguous():
        return P * C, 1
    if param.permute(0, 2, 3, 4, 1).is_contiguous():
        return P, C
    raise RuntimeError('param must be contiguous (or channels-last contiguous)')


def total_variation_add_grad(param, grad, wx, wy, wz, dense_mode):
    if not (isinstance(param, torch.Tensor) and param.is_cuda):
        raise RuntimeError('param must be a CUDA tensor')
    if not (isinstance(grad, torch.Tensor) and grad.is_cuda):
        raise RuntimeError('grad must be a CUDA tensor')
    lead, inner = _sweep_layout(param)
    if grad.shape != param.shape or grad.stride() != param.stride():
        raise RuntimeError('grad must be contiguous')   # same layout as param
    with _Guard(param) as lib:
        check(lib.ubn_total_variation_add_grad(ptr(param), ptr(grad), c_f(float(wx)), c_f(float(wy)), c_f(float(wz)),
                                               c_i64(lead), c_i64(param.shape[2]), c_i64(param.shape[3]),
                                               c_i64(param.shape[4]), c_i64(inner), c_int(int(bool(dense_mode))),
                                               stream_of(param)))


def _is_dense(t):
    """True when t covers its storage span exactly once (contiguous in SOME dimension order)."""
    if t.is_contiguous() or t.numel() == 0:
        return True
    order = sorted(range(t.dim()), key=lambda d: (-t.stride(d), d))
    return t.permute(order).is_contiguous()


def _dense_like(a, b, name):
    if not (isinstance(b, torch.Tensor) and b.is_cuda):
        raise RuntimeError(f'{name} must be a CUDA tensor')
    if b.shape != a.shape or b.stride() != a.stride() or b.dtype != torch.float32:
        raise RuntimeError(f'{name} must be contiguous')


def _adam(param, grad, exp_avg, exp_avg_sq, perlr, step, beta1, beta2, lr, eps, mode):
    if not (isinstance(param, torch.Tensor) and param.is_cuda):
        raise RuntimeError('param must be a CUDA tensor')
    # elementwise: any dense (non-overlapping) layout works as long as all operands share it
    if not _is_dense(param):
        raise RuntimeError('param must be contiguous')
    _dense_like(param, grad, 'grad'); _dense_like(param, exp_avg, 'exp_avg'); _dense_like(param, exp_avg_sq, 'exp_avg_sq')
    if perlr is not None:
        _dense_like(param, perlr, 'perlr')
    with _Guard(param) as lib:
        check(lib.ubn_adam_upd(ptr(param), ptr(grad), ptr(exp_avg), ptr(exp_avg_sq), ptr(perlr), c_i64(param.numel()),
                               c_int(int(step)), c_f(beta1), c_f(beta2), c_f(lr), c_f(eps), c_int(mode),
                               stream_of(param)))


def adam_upd(param, grad, exp_avg, exp_avg_sq, step, beta1, beta2, lr, eps):
    _adam(param, grad, exp_avg, exp_avg_sq, None, step, beta1, beta2, lr, eps, 0)


def masked_adam_upd(param, grad, exp_avg, exp_avg_sq, step, beta1, beta2, lr, eps):
    _adam(param, grad, exp_avg, exp_avg_sq, None, step, beta1, beta2, lr, eps, 1)


def adam_upd_with_perlr(param, grad, exp_avg, exp_avg_sq, perlr, step, beta1, beta2, lr, eps):
    _adam(param, grad, exp_avg, exp_avg_sq, perlr, step, beta1, beta2, lr, eps, 2)


def tv_adam_fused(param, grad, exp_avg, exp_avg_sq, wx, wy, wz, tv_mode, step, beta1, beta2, lr, eps,
                  skip_zero_grad=True, zero_grad=True):
    """Training-step tail in two sweeps instead of three (+ no grad memset): TV (tv_mode 0 none / 1 dense /
    2 sparse) then (masked) Adam that also clears the gradients it consumed."""
    lead, inner = _sweep_layout(param)
    _dense_like(param, grad, 'grad'); _dense_like(param, exp_avg, 'exp_avg'); _dense_like(param, exp_avg_sq, 'exp_avg_sq')
    with _Guard(param) as lib:
        check(lib.ubn_tv_adam_fused(ptr(param), ptr(grad), ptr(exp_avg), ptr(exp_avg_sq), c_f(float(wx)), c_f(float(wy)),
                                    c_f(float(wz)), c_i64(lead), c_i64(param.shape[2]), c_i64(param.shape[3]),
                                    c_i64(param.shape[4]), c_i64(inner), c_int(int(tv_mode)), c_int(int(step)),
                                    c_f(beta1), c_f(beta2), c_f(lr), c_f(eps), c_int(1 if skip_zero_grad else 0),
                                    c_int(1 if zero_grad else 0), stream_of(param)))


def tv_adam_pingpong_supported(param):
    """Channels-last 5-D grid whose (Z, C) row fits one CTA of the streaming kernel."""
    if param.dim() != 5 or param.is_contiguous() or not param.permute(0, 2, 3, 4, 1).is_contiguous():
        return False
    C, X, Z = param.shape[1], param.shape[2], param.shape[4]
    return C % 4 == 0 and X >= 8 and 32 <= Z * C // 4 <= 512


def tv_adam_pingpong(param, param_out, grad, exp_avg, exp_avg_sq, wx, wy, wz, dense_mode, step, beta1, beta2, lr, eps,
                     skip_zero_grad=True, write_grad=True):
    """TV + (masked) Adam in one sweep, updated parameters written to ``param_out`` (same layout; caller swaps)."""
    if not tv_adam_pingpong_supported(param):
        raise RuntimeError('tv_adam_pingpong needs a channels-last [P,C,X,Y,Z] grid with C % 4 == 0')
    lead, inner = _sweep_layout(param)
    for t, nm in ((param_out, 'param_out'), (grad, 'grad'), (exp_avg, 'exp_avg'), (exp_avg_sq, 'exp_avg_sq')):
        _dense_like(param, t, nm)
    if param_out.data_ptr() == param.data_ptr():
        raise RuntimeError('param_out must be a different buffer')
    with _Guard(param) as lib:
        check(lib.ubn_tv_adam_pingpong(ptr(param), ptr(param_out), ptr(grad), ptr(exp_avg), ptr(exp_avg_sq), c_f(float(wx)),
                                       c_f(float(wy)), c_f(float(wz)), c_i64(lead), c_i64(param.shape[2]), c_i64(param.shape[3]),
                                       c_i64(param.shape[4]), c_i64(inner), c_int(int(bool(dense_mode))), c_int(int(step)),
                                       c_f(beta1), c_f(beta2), c_f(lr), c_f(eps), c_int(1 if skip_zero_grad else 0),
                                       c_int(1 if write_grad else 0), stream_of(param)))


def tv_adam_peer(param, param_out_ptrs, grad_ptrs, exp_avg, exp_avg_sq, wx, wy, wz, dense_mode, plane_begin, plane_end, step,
                 beta1, beta2, lr, eps, skip_zero_grad=True):
    """Multi-GPU tail sweep (ubn_tv_adam_peer): mean of the ranks' gradients -> TV -> (masked) Adam -> updated parameters stored
    into every rank's ping-pong buffer, for the planes [plane_begin, plane_end) of the flattened (slab, X) axis this rank owns.
    ``param_out_ptrs`` / ``grad_ptrs``: device addresses (ints, rank order) of whole-grid buffers mapped into this process."""
    import ctypes
    if not tv_adam_pingpong_supported(param):
        raise RuntimeError('tv_adam_peer needs a channels-last [P,C,X,Y,Z] grid with C % 4 == 0')
    n = len(grad_ptrs)
    if n != len(param_out_ptrs) or n not in (1, 2, 4, 8):
        raise RuntimeError('tv_adam_peer needs 1, 2, 4 or 8 peers')
    lead, inner = _sweep_layout(param)
    _dense_like(param, exp_avg, 'exp_avg'); _dense_like(param, exp_avg_sq, 'exp_avg_sq')
    po = (ctypes.c_void_p * n)(*[int(a) for a in param_out_ptrs])
    gp = (ctypes.c_void_p * n)(*[int(a) for a in grad_ptrs])
    with _Guard(param) as lib:
        check(lib.ubn_tv_adam_peer(ptr(param), po, gp, c_int(n), ptr(exp_avg), ptr(exp_avg_sq), c_f(float(wx)), c_f(float(wy)),
                                   c_f(float(wz)), c_i64(lead), c_i64(param.shape[2]), c_i64(param.shape[3]), c_i64(param.shape[4]),
                                   c_i64(inner), c_int(int(bool(dense_mode))), c_i64(int(plane_begin)), c_i64(int(plane_end)),
                                   c_int(int(step)), c_f(beta1), c_f(beta2), c_f(lr), c_f(eps), c_int(1 if skip_zero_grad else 0),
                                   stream_of(param)))


# --------------------------------------------------------------------------------------------------
# grid-native occupancy / progressive-growing utilities (csrc/grid_utils.cu; SURVEY.md 8a row a13)
# --------------------------------------------------------------------------------------------------
def lattice_alpha(density_grid, xyz_min, xyz_max, num_freqs, lattice_min, lattice_max, lattice_shape, act_shift, interval):
    """alpha = Raw2Alpha(density(p)) on the [mX,mY,mZ] lattice of linspace(lattice_min, lattice_max) points -- steps 1-3 of
    update_occupancy_cache (FourierGrid_model.py:443-450) without the meshgrid / grid_sample / activation tensors."""
    import ctypes
    from .grid import grid_desc
    _chk(density_grid, 'density_grid', contiguous=False)
    d = grid_desc(density_grid, xyz_min, xyz_max, num_freqs)
    if d.C != 1:
        raise RuntimeError('lattice_alpha needs a single-channel (density) grid')
    mX, mY, mZ = [int(v) for v in lattice_shape]
    alpha = torch.empty(mX, mY, mZ, dtype=torch.float32, device=density_grid.device)
    lo = (ctypes.c_float * 3)(*[float(v) for v in lattice_min])
    hi = (ctypes.c_float * 3)(*[float(v) for v in lattice_max])
    with _Guard(density_grid) as lib:
        check(lib.ubn_lattice_alpha(ptr(density_grid), d, lo, hi, c_i64(mX), c_i64(mY), c_i64(mZ), c_f(float(act_shift)),
                                    c_f(float(interval)), ptr(alpha), stream_of(density_grid)))
    return alpha


def maxpool3_gt_and_(mask, alpha, thres):
    """mask &= F.max_pool3d(alpha, 3, stride 1, padding 1) > thres, in place (FourierGrid_model.py:451-452)."""
    if not (mask.is_cuda and mask.dtype == torch.bool and mask.is_contiguous() and mask.dim() == 3):
        raise RuntimeError('mask must be a contiguous CUDA bool [X,Y,Z] tensor')
    if alpha.shape != mask.shape or not alpha.is_contiguous() or alpha.dtype != torch.float32:
        raise RuntimeError('alpha must be a contiguous fp32 tensor of the mask shape')
    X, Y, Z = mask.shape
    with _Guard(mask) as lib:
        check(lib.ubn_maxpool3_gt_and(ptr(alpha), c_i64(X), c_i64(Y), c_i64(Z), c_f(float(thres)), ptr(mask), stream_of(mask)))
    return mask


def resample_grid(grid, new_world_size):
    """F.interpolate(grid, size, mode='trilinear', align_corners=True) for a [P,C,X,Y,Z] grid in its own layout (the result is
    channels-last when C > 1) -- scale_volume_grid (grid.py:63-68, FourierGrid_grid.py:80-85)."""
    from .grid import grid_desc, zeros_grid
    _chk(grid, 'grid', contiguous=False)
    P, C = grid.shape[0], grid.shape[1]
    ws = [int(v) for v in new_world_size]
    out = zeros_grid([P, C, *ws], device=grid.device)
    zero3 = [0.0, 0.0, 0.0]
    with _Guard(grid) as lib:
        check(lib.ubn_resample_grid(ptr(grid), grid_desc(grid, zero3, zero3, 0), ptr(out), grid_desc(out, zero3, zero3, 0),
                                    stream_of(grid)))
    return out


def view_scatter_ones(rays_o, rays_d, xyz_min, xyz_max, world_size, n_samples, near, far, step, grad):
    """grad [X,Y,Z] += adjoint of DenseGrid(1, world_size)(pts).sum() over the sample points of the rays
    (FourierGrid_model.py:405-417); ``step`` = stepsize * voxel_size."""
    from ._cabi import UbnGridDesc
    _chk(rays_o, 'rays_o'); _chk(rays_d, 'rays_d'); _chk(grad, 'grad')
    d = UbnGridDesc()
    d.P, d.C, d.num_freqs = 1, 1, 0
    d.X, d.Y, d.Z = [int(v) for v in world_size]
    d.stride_p, d.stride_c, d.stride_v = d.X * d.Y * d.Z, 1, 1
    for a in range(3):
        d.xyz_min[a], d.xyz_max[a] = float(xyz_min[a]), float(xyz_max[a])
    n = rays_o.shape[0]
    with _Guard(rays_o) as lib:
        check(lib.ubn_view_scatter_ones(ptr(rays_o), ptr(rays_d), c_i64(n), c_i64(int(n_samples)), c_f(float(near)), c_f(float(far)),
                                        c_f(float(step)), d, ptr(grad), stream_of(rays_o)))


def view_scatter_ones_contracted(rays_o, rays_d, t_table, scene_center, scene_radius, bg_len, contracted_norm, xyz_min, xyz_max,
                                 world_size, grad):
    """grad [X,Y,Z] += adjoint of DenseGrid(1, world_size, xyz_min, xyz_max)(pts).sum() over the contracted sample points of the
    rays: pts[r, s] = the point sample_ray (dcvgo.py:228-262, FourierGrid_model.py:509-552) puts at t_table[s], all of them
    (dcvgo.py:203-207).  ``scene_center`` / ``scene_radius`` / ``xyz_min`` / ``xyz_max`` are host 3-sequences."""
    from . import march
    from ._cabi import UbnGridDesc
    _chk(rays_o, 'rays_o'); _chk(rays_d, 'rays_d'); _chk(t_table, 't_table'); _chk(grad, 'grad')
    d = UbnGridDesc()
    d.P, d.C, d.num_freqs = 1, 1, 0
    d.X, d.Y, d.Z = [int(v) for v in world_size]
    if grad.numel() != d.X * d.Y * d.Z:
        raise RuntimeError('grad must have world_size elements')
    d.stride_p, d.stride_c, d.stride_v = d.X * d.Y * d.Z, 1, 1
    for a in range(3):
        d.xyz_min[a], d.xyz_max[a] = float(xyz_min[a]), float(xyz_max[a])
    cfg = march.make_cfg(scene_center, scene_radius, bg_len, contracted_norm, t_table.numel(), 0., 0., 0.)
    n = rays_o.shape[0]
    with _Guard(rays_o) as lib:
        check(lib.ubn_view_scatter_ones_contracted(ptr(rays_o), ptr(rays_d), c_i64(n), ptr(t_table), cfg, d, ptr(grad),
                                                   stream_of(rays_o)))
    return grad


def count_gt_(count, grad, thres=1.0):
    """count += (grad > thres), in place (FourierGrid_model.py:418-419)."""
    _chk(count, 'count', contiguous=False); _chk(grad, 'grad', contiguous=False)
    if count.numel() != grad.numel():
        raise RuntimeError('count / grad size mismatch')
    with _Guard(count) as lib:
        check(lib.ubn_count_gt(ptr(grad), c_f(float(thres)), c_i64(grad.numel()), ptr(count), stream_of(count)))
    return count


def maskout_near_cam_(slab, cams, near_clip, fill=-100.0, lattice=None):
    """slab [X,Y,Z] (a view of one grid slab; unit or channel stride) <- fill where the nearest of ``cams`` [n,3] is within
    near_clip of the lattice point: linspace(-1, 1) per axis (FourierGrid_model.py:383-388), or linspace(lo[a], hi[a]) for
    ``lattice = (lo, hi)`` host 3-sequences (DirectVoxGO's world lattice, dvgo.py:185-198)."""
    if slab.dim() != 3:
        raise RuntimeError('slab must be [X,Y,Z]')
    X, Y, Z = slab.shape
    sv = slab.stride(2)
    if slab.stride(1) != Z * sv or slab.stride(0) != Y * Z * sv:
        raise RuntimeError('slab must be a dense [X,Y,Z] view')
    cams = cams.contiguous().float()
    with _Guard(slab) as lib:
        if lattice is None:
            check(lib.ubn_maskout_near_cam(ptr(slab), c_i64(sv), c_i64(X), c_i64(Y), c_i64(Z), ptr(cams), c_i64(cams.shape[0]),
                                           c_f(float(near_clip)), c_f(float(fill)), stream_of(slab)))
        else:
            lo, hi = ((c_f * 3)(*[float(v) for v in b]) for b in lattice)
            check(lib.ubn_maskout_near_cam_lattice(ptr(slab), c_i64(sv), c_i64(X), c_i64(Y), c_i64(Z), lo, hi, ptr(cams),
                                                   c_i64(cams.shape[0]), c_f(float(near_clip)), c_f(float(fill)), stream_of(slab)))
    return slab


def set_feature_kernel(variant):
    """Pass-B kernel family for 12-channel channels-last feature grids: 0 = warp-cooperative, 1 = lane-per-sample forward,
    2 = lane-per-sample forward + backward, 3 / 4 / 5 = lane-per-sample forward + slab-major scatter with each slab swept in 1 / 2 / 4 x-ranges,
    6 = as 3 with the 8-samples-per-instruction gather (ubn_set_feature_kernel).
    Process-wide."""
    from ._cabi import load
    check(load().ubn_set_feature_kernel(c_int(int(variant))))


def get_feature_kernel():
    from ._cabi import load
    return int(load().ubn_get_feature_kernel())


def set_density_scatter(variant):
    """Density-grid scatter of the fused march backward: 1 = run-merging two-launch scatter (default), 0 = per-sample scatter
    (ubn_set_density_scatter).  Process-wide."""
    from ._cabi import load
    check(load().ubn_set_density_scatter(c_int(int(variant))))


def get_density_scatter():
    from ._cabi import load
    return int(load().ubn_get_density_scatter())


def set_dw2_engine(engine):
    """grad_W2 of the width-128 rgbnet backward with ReLU masks: 1 = warpgroup MMA (default), 0 = mma.sync
    (ubn_set_dw2_engine).  Process-wide."""
    from ._cabi import load
    check(load().ubn_set_dw2_engine(c_int(int(engine))))


def cumdist_thres(dist, thres):
    _chk(dist, 'dist')
    mask = torch.empty(dist.shape, dtype=torch.bool, device=dist.device)
    if dist.numel() == 0:
        return mask
    with _Guard(dist) as lib:
        check(lib.ubn_cumdist_thres(ptr(dist), c_f(float(thres)), c_i64(dist.shape[0]), c_i64(dist.shape[1]), ptr(mask),
                                    stream_of(dist)))
    return mask
