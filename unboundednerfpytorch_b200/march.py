"""Fused ray march (autograd.Function) over the C ABI: the hot path of FourierGridModel.forward
(FourierGrid_model.py:554-621) and DirectContractedVoxGO.forward (dcvgo.py:264-331) -- ``March`` -- and of
DirectMPIGO.forward (dmpigo.py:251-295) -- ``NdcMarch`` -- and of DirectVoxGO.forward (dvgo.py:330-366) -- ``BoxMarch``, and
``BoxTensorfMarch`` with TensoRF grids -- up to and including the feature-grid read, in 3 launches forward (pass A, scan, pass B)
and 2 backward.  All of them run the one forward body and the one backward body below (_forward / _backward); a geometry record
(_Contracted, _Ndc, _Box, _BoxTensorf) binds them to the C entries of its sampling policy and density.
"""
import functools
import os

import numpy as np
import torch

from . import _cabi, ops
from ._cabi import UbnMarchCfg, UbnNdcMarchCfg, c_i64, c_int, check, ptr, stream_of
from .grid import _factor_array, grid_desc


@functools.lru_cache(maxsize=64)
def _t_schedule_cpu(world_len, stepsize, bg_len, t_boundary):
    """t table exactly as the reference builds it (torch.linspace on fp32, midpoints):
    dcvgo.py:241-248 (t_boundary = 2) and FourierGrid_model.py:524-532 (t_boundary = 1.5)."""
    n_inner = int(2 / (2 + 2 * bg_len) * world_len / stepsize) + 1
    n_outer = n_inner
    b_inner = torch.linspace(0, t_boundary, n_inner + 1, dtype=torch.float32, device='cpu')
    b_outer = t_boundary / torch.linspace(1, 1 / 128, n_outer + 1, dtype=torch.float32, device='cpu')
    return torch.cat([(b_inner[1:] + b_inner[:-1]) * 0.5, (b_outer[1:] + b_outer[:-1]) * 0.5]).contiguous()


_t_dev_cache = {}


def t_schedule(world_len, stepsize, bg_len, t_boundary, device):
    key = (int(world_len), float(stepsize), float(bg_len), float(t_boundary), str(device))
    hit = _t_dev_cache.get(key)
    if hit is None:
        hit = _t_schedule_cpu(*key[:4]).to(device)
        _t_dev_cache[key] = hit
    return hit


TMA_STATS = None          # optional torch.int64[2] CUDA tensor: += {blocks served by TMA, blocks served by the fallback} (tests / bench)


def tma_supported(k0_grid):
    """Single-slab 12-channel channels-last feature grid (DenseGrid k0 of the DCVGO / DVGO family)."""
    return (k0_grid.is_cuda and k0_grid.dim() == 5 and k0_grid.shape[0] == 1 and k0_grid.shape[1] == 12 and k0_grid.stride(1) == 1
            and min(k0_grid.shape[2:]) >= 2)


def _set_mask_fields(c, mask, mask_scale, mask_shift):
    """The mask-cache fields every march cfg carries: the occupancy grid's size and its world -> index map."""
    c.use_maskcache = 1 if mask is not None else 0
    if mask is not None:
        for a in range(3):
            c.mask_sz[a] = int(mask.shape[a])
            c.mask_scale[a] = float(mask_scale[a])
            c.mask_shift[a] = float(mask_shift[a])
    return c


def make_cfg(scene_center, scene_radius, bg_len, contracted_norm, n_samples, act_shift, interval,
             fast_color_thres, cumdist_thres=None, mask=None, mask_scale=None, mask_shift=None):
    c = UbnMarchCfg()
    for a in range(3):
        c.scene_center[a] = float(scene_center[a])
        c.scene_radius[a] = float(scene_radius[a])
    # torch narrows the Python doubles (1+bg_len) and bg_len to fp32 when they meet an fp32 tensor
    c.contract_B = float(np.float32(1 + bg_len))
    c.contract_A = float(np.float32((1 + bg_len) * 1.0 - 1.0))
    if contracted_norm == 'inf':
        c.contracted_norm = 0
    elif contracted_norm == 'l2':
        c.contracted_norm = 1
    else:
        raise NotImplementedError(contracted_norm)
    c.n_samples = int(n_samples)
    c.act_shift = float(act_shift)
    c.interval = float(interval)
    c.fast_color_thres = float(fast_color_thres)
    c.use_cumdist = 1 if cumdist_thres is not None else 0
    c.cumdist_thres = float(cumdist_thres) if cumdist_thres is not None else 0.0
    return _set_mask_fields(c, mask, mask_scale, mask_shift)


def _pass_a_buffers(N, S, dev):
    """Dense per-sample records of pass A: density, alpha, weight, T [N*S], flags [N*S], alphainv_last [N], n_keep [N]."""
    f32 = dict(dtype=torch.float32, device=dev)
    return (torch.empty(N * S, **f32), torch.empty(N * S, **f32), torch.empty(N * S, **f32), torch.empty(N * S, **f32),
            torch.empty(N * S, dtype=torch.uint8, device=dev), torch.empty(N, **f32), torch.empty(N, dtype=torch.int32, device=dev))


def _grad_target(param, meta, want, dev):
    """(gradient buffer to scatter into, the parameter's persistent buffer or None).  Persistent gradient buffers
    (dist.PeerTail / grid.attach_grad_buffer): the scatter adds straight into a buffer the training loop owns (peer-mapped for
    the multi-GPU tail, zero at the start of a step) instead of a fresh zero-filled allocation per step."""
    if not want:
        return None, None
    buf = getattr(param, '_ubn_grad_buffer', None)
    return (buf if buf is not None else torch.empty_strided(*meta, dtype=torch.float32, device=dev).zero_()), buf


def _hand_over(param, grad, buf):
    """With a persistent buffer the parameter's .grad is pointed at it and autograd gets no gradient to accumulate."""
    if buf is not None:
        param.grad = buf
        return None
    return grad


class _Geometry:
    """Binds _forward / _backward to one sampling policy's C entries ubn_<entry>_{density,feature}_{fwd,bwd}, timed under the
    same names without the ubn_ prefix.  These defaults are the NDC march's; the contracted and box marches override what
    their entries add."""
    entry = 'march_ndc'
    lead = ()              # tensors every entry takes right after rays_o, rays_d
    shift = ()             # pass A's arguments right after the density grid's desc

    def steps(self, cfg):
        return cfg.n_samples

    def pass_a_tail(self, dev):
        return ()

    def survivors(self, offsets, tail, N, S):
        return int(offsets[N].item())         # the march's one device-to-host read

    def pass_b(self, lib, head, k0_grid, dens, alpha, weight, out, st):
        """Launch pass B into out = (feat, alpha, weight, ray_id, step_id).  Returns the further outputs: (those with a gradient,
        which the density backward takes right after g_alpha), (constants)."""
        with _cabi.timed(self.entry + '_feature_fwd'):
            check(getattr(lib, f'ubn_{self.entry}_feature_fwd')(*head, ptr(alpha), ptr(weight), *map(ptr, out), st))
        return (), ()

    def saved_density(self, density):
        """Density tensors the backward reads (saved with save_for_backward, so an in-place change before it raises): none."""
        return ()

    def density_fwd(self, lib, rays, density, ddesc, mask_world, cfg, N, records, tail, st):
        """Pass A on the density tensors (one grid here)."""
        with _cabi.timed(self.entry + '_density_fwd'):
            check(getattr(lib, f'ubn_{self.entry}_density_fwd')(*rays, ptr(density[0]), ddesc, *self.shift, ptr(mask_world), cfg,
                                                                  c_i64(N), *map(ptr, records), *map(ptr, tail), st))

    def density_bwd(self, lib, ctx, rays, N, args, grads, gd, st):
        """The density's reverse scan and scatter, adding into grads (one per density tensor); args = the pass A records, the
        offsets and the output gradients, in the C entry's order."""
        with _cabi.timed(self.entry + '_density_bwd'):
            check(getattr(lib, f'ubn_{self.entry}_density_bwd')(*rays, ctx.ddesc, ctx.cfg, c_i64(N), *map(ptr, (*args, grads[0], gd)),
                                                                  st))


class _Contracted(_Geometry):
    """Every entry takes the t table; pass B also writes raw_density, t and the inner-sphere flag, and on the render path may
    stage the feature grid by TMA."""
    entry = 'march'

    def __init__(self, t_table, dense_known, coherent):
        self.lead = (t_table,)
        self.dense_known, self.coherent = dense_known, coherent

    def survivors(self, offsets, tail, N, S):
        # known without a host sync when nothing can be masked out
        return N * S if self.dense_known else super().survivors(offsets, tail, N, S)

    def pass_b(self, lib, head, k0_grid, dens, alpha, weight, out, st):
        feat, o_alpha, o_weight, ray_id, step_id = out
        M, dev = o_alpha.shape[0], o_alpha.device
        o_dens = torch.empty(M, dtype=torch.float32, device=dev)
        o_t = torch.empty(M, dtype=torch.float32, device=dev)
        o_inner = torch.empty(M, dtype=torch.bool, device=dev)
        # render path: bricks of the feature grid staged by TMA for 32 adjacent rays x 4 steps
        use_tma = self.coherent and tma_supported(k0_grid) and not torch.is_grad_enabled()
        name = 'march_feature_fwd_tma' if use_tma else 'march_feature_fwd'
        with _cabi.timed(name):
            check(getattr(lib, 'ubn_' + name)(*head, *map(ptr, (dens, alpha, weight, feat, o_dens, o_alpha, o_weight, ray_id, step_id,
                                                                 o_t, o_inner)), *((ptr(TMA_STATS),) if use_tma else ()), st))
        return (o_dens,), (o_t, o_inner)


def _forward(ctx, geo, density, k0_grid, rays_o, rays_d, mask_world, cfg, ddesc, kdesc, d_at=(0,), k_at=1):
    """Pass A (dense per-sample records), the exclusive scan of the per-ray survivor counts, pass B (compacted records and the
    feature read).  density: the density tensors (a grid, or the six TensoRF factors), at the Function's inputs d_at; k0_grid at
    input k_at, or None (k_at None) when pass B writes the survivor points instead of reading a k0.  Returns (weights[M], alphainv_last[N],
    raw_alpha[M], *geometry outputs with a gradient, k0_feat[M,C] (or points[M,3]), ray_id[M] i64, step_id[M] i64, *constant
    geometry outputs)."""
    dev = rays_o.device
    rays_o = rays_o.contiguous().float()
    rays_d = rays_d.contiguous().float()
    N, S = rays_o.shape[0], geo.steps(cfg)
    f32 = dict(dtype=torch.float32, device=dev)
    records = _pass_a_buffers(N, S, dev)
    dens, alpha, weight, T, flags, last, nkeep = records
    tail = geo.pass_a_tail(dev)
    with ops._Guard(rays_o) as lib:
        st = stream_of(rays_o)
        rays = (ptr(rays_o), ptr(rays_d), *map(ptr, geo.lead))
        geo.density_fwd(lib, rays, density, ddesc, mask_world, cfg, N, records, tail, st)
        offsets = torch.empty(N + 1, dtype=torch.int64, device=dev)
        scratch = torch.empty(N // 1024 + 4, dtype=torch.int64, device=dev)
        check(lib.ubn_exclusive_scan_i32(ptr(nkeep), c_i64(N), ptr(offsets), ptr(scratch), st))
        M = geo.survivors(offsets, tail, N, S)
        out = (torch.empty(M, k0_grid.shape[1] if k0_grid is not None else 3, **f32), torch.empty(M, **f32), torch.empty(M, **f32),
               torch.empty(M, dtype=torch.int64, device=dev), torch.empty(M, dtype=torch.int64, device=dev))
        feat, o_alpha, o_weight, ray_id, step_id = out
        head = (*rays, ptr(k0_grid), kdesc, cfg, c_i64(N), ptr(flags), ptr(offsets))
        differentiable, constant = geo.pass_b(lib, head, k0_grid, dens, alpha, weight, out, st)
    ctx.save_for_backward(rays_o, rays_d, dens, alpha, weight, T, flags, last, offsets, *geo.saved_density(density))
    ctx.geo, ctx.cfg, ctx.ddesc, ctx.kdesc = geo, cfg, ddesc, kdesc
    ctx.n_extra = len(differentiable)
    ctx.dmeta = [(t.shape, t.stride()) for t in density]
    ctx.kmeta = (k0_grid.shape, k0_grid.stride()) if k0_grid is not None else None
    ctx.dparam, ctx.kparam = density, k0_grid      # for their persistent gradient buffers (_grad_target)
    ctx.d_at, ctx.k_at = d_at, k_at
    ctx.mark_non_differentiable(ray_id, step_id, *constant, *((feat,) if k0_grid is None else ()))
    return (o_weight, last, o_alpha, *differentiable, feat, ray_id, step_id, *constant)


@torch.autograd.function.once_differentiable
def _backward(ctx, g_weight, g_last, g_alpha, *rest):
    """The k0 scatter, then the density reverse scan and scatter.  Gradients for the density tensors and k0_grid, None for the
    rest."""
    rays_o, rays_d, dens, alpha, weight, T, flags, last, offsets = ctx.saved_tensors[:9]
    geo = ctx.geo
    dev = rays_o.device
    N = rays_o.shape[0]
    cont = lambda g: g.contiguous() if g is not None else None
    g_extra = [cont(g) for g in rest[:ctx.n_extra]]
    g_weight, g_last, g_alpha, g_feat = map(cont, (g_weight, g_last, g_alpha, rest[ctx.n_extra]))
    with ops._Guard(rays_o) as lib:
        st = stream_of(rays_o)
        rays = (ptr(rays_o), ptr(rays_d), *map(ptr, geo.lead))
        want_k = ctx.k_at is not None and ctx.needs_input_grad[ctx.k_at] and g_feat is not None
        want_d = any(ctx.needs_input_grad[i] for i in ctx.d_at)
        targets_d = [_grad_target(p, m, want_d, dev) for p, m in zip(ctx.dparam, ctx.dmeta)]
        grad_k, buf_k = _grad_target(ctx.kparam, ctx.kmeta, want_k, dev)
        if want_k:
            with _cabi.timed(geo.entry + '_feature_bwd'):
                check(getattr(lib, f'ubn_{geo.entry}_feature_bwd')(*rays, ctx.kdesc, ctx.cfg, c_i64(N), ptr(flags), ptr(offsets),
                                                                     ptr(g_feat), ptr(grad_k), st))
        if want_d:
            gd = torch.empty_like(dens)     # per-sample density gradients between the backward's two launches
            geo.density_bwd(lib, ctx, rays, N, (dens, alpha, weight, T, flags, last, offsets, g_weight, g_alpha, *g_extra, g_last),
                            [g for g, _ in targets_d], gd, st)
    grads = [None] * len(ctx.needs_input_grad)
    for i, p, (g, buf) in zip(ctx.d_at, ctx.dparam, targets_d):
        grads[i] = _hand_over(p, g, buf)
    if ctx.k_at is not None:
        grads[ctx.k_at] = _hand_over(ctx.kparam, grad_k, buf_k)
    return tuple(grads)


class March(torch.autograd.Function):
    """(density_grid, k0_grid, rays) -> compacted per-survivor records.

    Returns (weights[M], alphainv_last[N], raw_alpha[M], raw_density[M], k0_feat[M,C], ray_id[M] i64,
    step_id[M] i64, t[M], inner[M] bool).  Differentiable wrt density_grid and k0_grid through weights,
    alphainv_last, raw_alpha, raw_density and k0_feat.
    """

    @staticmethod
    def forward(ctx, density_grid, k0_grid, rays_o, rays_d, t_table, mask_world, cfg, ddesc, kdesc, dense_known, coherent=False):
        return _forward(ctx, _Contracted(t_table, dense_known, coherent), (density_grid,), k0_grid, rays_o, rays_d, mask_world, cfg,
                        ddesc, kdesc)

    backward = staticmethod(_backward)


def make_ndc_cfg(xyz_min, xyz_max, n_samples, interval, fast_color_thres, mask, mask_scale, mask_shift):
    c = UbnNdcMarchCfg()
    for a in range(3):
        c.xyz_min[a] = float(xyz_min[a])
        c.xyz_max[a] = float(xyz_max[a])
    c.n_samples = int(n_samples)
    c.interval = float(interval)
    c.fast_color_thres = float(fast_color_thres)
    return _set_mask_fields(c, mask, mask_scale, mask_shift)


def ndc_supported(k0_grid):
    """Grids the fused NDC feature read covers: single-slab channels-last k0 with 3 or 9 channels, >= 2 voxels per axis."""
    return (k0_grid.is_cuda and k0_grid.dim() == 5 and k0_grid.shape[0] == 1 and k0_grid.shape[1] in (3, 9)
            and k0_grid.stride(1) == 1 and min(k0_grid.shape[2:]) >= 2 and k0_grid[0, 0].numel() < 2 ** 31)


class _Ndc(_Geometry):
    def __init__(self, act_shift_grid, sdesc):
        self.shift = (ptr(act_shift_grid), sdesc)


class NdcMarch(torch.autograd.Function):
    """DirectMPIGO's march: (density_grid, k0_grid, rays) -> compacted per-survivor records.

    Returns (weights[M], alphainv_last[N], raw_alpha[M], k0_feat[M,C], ray_id[M] i64, step_id[M] i64).  Differentiable wrt
    density_grid and k0_grid; act_shift_grid is a constant (requires_grad=False in the reference, dmpigo.py:50)."""

    @staticmethod
    def forward(ctx, density_grid, k0_grid, act_shift_grid, rays_o, rays_d, mask_world, cfg, ddesc, kdesc, sdesc):
        return _forward(ctx, _Ndc(act_shift_grid, sdesc), (density_grid,), k0_grid, rays_o, rays_d, mask_world, cfg, ddesc, kdesc)

    backward = staticmethod(_backward)


def box_s_max(xyz_min, xyz_max, stepdist):
    """Record stride of the box march: a host bound on every ray's n_steps = max(ceil((t_max - t_min) * |d| / stepdist), 1).
    (t_max - t_min) * |d| is the length of the ray's chord through the box (a zero direction component is replaced by 1e-6,
    which only lengthens the direction the slabs see, so |d| under-measures that chord), and a chord through a box is at most
    its diagonal.  The margin of 4 steps covers the fp32 rounding of t_min, t_max and the product.  A ray beyond it (a camera
    ~1e7 box lengths away) is reported by pass A, never truncated."""
    diag = float(np.linalg.norm(np.asarray(xyz_max, dtype=np.float64) - np.asarray(xyz_min, dtype=np.float64)))
    return int(np.ceil(diag / float(np.float32(stepdist)))) + 4


BOX_S_MAX_LIMIT = 4096     # the backward's per-ray chunk table


def make_box_cfg(xyz_min, xyz_max, near, stepdist, act_shift, interval, fast_color_thres, mask, mask_scale, mask_shift):
    c = _cabi.UbnBoxMarchCfg()
    for a in range(3):
        c.xyz_min[a] = float(xyz_min[a])
        c.xyz_max[a] = float(xyz_max[a])
    c.near = float(near)
    c.stepdist = float(stepdist)
    c.s_max = box_s_max(xyz_min, xyz_max, stepdist)
    if c.s_max > BOX_S_MAX_LIMIT:
        raise ValueError(f'the box march bounds a ray at {BOX_S_MAX_LIMIT} steps; this bbox / stepsize needs {c.s_max}')
    c.act_shift = float(act_shift)
    c.interval = float(interval)
    c.fast_color_thres = float(fast_color_thres)
    return _set_mask_fields(c, mask, mask_scale, mask_shift)


def box_supported(density_grid, k0_grid):
    """Grids the fused box march covers: box_density_supported and box_k0_supported."""
    return box_density_supported(density_grid) and box_k0_supported(k0_grid)


class _Box(_Geometry):
    """Records of cfg.s_max steps per ray; pass A also sets an overflow word when a ray needs more."""
    entry = 'march_box'

    def steps(self, cfg):
        return cfg.s_max

    def pass_a_tail(self, dev):
        return (torch.zeros(1, dtype=torch.int32, device=dev),)

    def survivors(self, offsets, tail, N, S):
        # the march's one device-to-host read: the survivor count and the overflow word together
        M, over = torch.stack([offsets[N], tail[0][0].to(torch.int64)]).tolist() if N > 0 else (0, 0)
        if over:
            raise RuntimeError(f'box march: a ray needs more than s_max = {S} steps (bbox / stepsize / ray origin out of range)')
        return M


class BoxMarch(torch.autograd.Function):
    """DirectVoxGO's march: (density_grid, k0_grid, rays) -> compacted per-survivor records sorted by (ray, step).

    Returns (weights[M], alphainv_last[N], raw_alpha[M], k0_feat[M,C], ray_id[M] i64, step_id[M] i64); step_id is the ray's own
    step index.  Differentiable wrt density_grid and k0_grid.  A ray needing more than cfg.s_max steps raises."""

    @staticmethod
    def forward(ctx, density_grid, k0_grid, rays_o, rays_d, mask_world, cfg, ddesc, kdesc):
        return _forward(ctx, _Box(), (density_grid,), k0_grid, rays_o, rays_d, mask_world, cfg, ddesc, kdesc)

    backward = staticmethod(_backward)


def box_density_supported(density_grid):
    """Density grids the box march's pass A reads: contiguous single slab, one channel, >= 2 voxels per axis, 32-bit offsets."""
    return (density_grid.is_cuda and density_grid.dim() == 5 and density_grid.shape[:2] == (1, 1) and density_grid.is_contiguous()
            and min(density_grid.shape[2:]) >= 2 and density_grid.numel() < 2 ** 31)


def box_k0_supported(k0_grid):
    """k0 grids the box march's pass B reads: single slab, channels-last, 3, 9 or 12 channels (16-byte aligned records for 12),
    >= 2 voxels per axis, 32-bit voxel offsets."""
    return (k0_grid.is_cuda and k0_grid.dim() == 5 and k0_grid.shape[0] == 1 and k0_grid.shape[1] in (3, 9, 12)
            and k0_grid.stride(1) == 1 and k0_grid.stride(4) == k0_grid.shape[1] and min(k0_grid.shape[2:]) >= 2
            and k0_grid[0, 0].numel() < 2 ** 31 and (k0_grid.shape[1] != 12 or k0_grid.data_ptr() % 16 == 0))


def tensorf_supported(factors):
    """TensoRF grids the box march reads: CUDA factors with R + R + Rxy <= 96 (one grad_f_vec row per thread of the backward)."""
    return all(t.is_cuda for t in factors) and 2 * factors[1].shape[1] + factors[0].shape[1] <= 96


class _BoxTensorf(_Box):
    """The box march for TensoRF models: pass A reads the density -- the six TensoRF factors (its backward adds into their
    gradients through vec_copies replicated vector copies) or a dense grid -- and pass B writes the survivor points, which the
    model's own k0 reads."""

    def __init__(self, tensorf_density, vec_copies):
        self.tensorf_density, self.vec_copies = tensorf_density, vec_copies

    def saved_density(self, density):
        return tuple(density) if self.tensorf_density else ()      # the adjoint multiplies plane values by line values

    def density_fwd(self, lib, rays, density, ddesc, mask_world, cfg, N, records, tail, st):
        if not self.tensorf_density:
            return super().density_fwd(lib, rays, density, ddesc, mask_world, cfg, N, records, tail, st)
        with _cabi.timed('march_box_tensorf_density_fwd'):
            check(lib.ubn_march_box_tensorf_density_fwd(*rays, _factor_array(density), ddesc, ptr(mask_world), cfg, c_i64(N),
                                                        *map(ptr, records), *map(ptr, tail), st))

    def density_bwd(self, lib, ctx, rays, N, args, grads, gd, st):
        if not self.tensorf_density:
            return super().density_bwd(lib, ctx, rays, N, args, grads, gd, st)
        d, K = ctx.ddesc, self.vec_copies
        vec = torch.empty(K * (d.X * d.R + d.Y * d.R + d.Z * d.Rxy), dtype=torch.float32, device=gd.device)
        with _cabi.timed('march_box_tensorf_density_bwd'):
            check(lib.ubn_march_box_tensorf_density_bwd(*rays, _factor_array(ctx.saved_tensors[9:]), d, ctx.cfg, c_i64(N),
                                                        *map(ptr, args), _factor_array(grads), c_int(K), ptr(gd), ptr(vec), st))

    def pass_b(self, lib, head, k0_grid, dens, alpha, weight, out, st):
        rays_o, rays_d, _, _, cfg, N, flags, offsets = head
        with _cabi.timed('march_box_points_fwd'):
            check(lib.ubn_march_box_points_fwd(rays_o, rays_d, cfg, N, flags, offsets, ptr(alpha), ptr(weight), *map(ptr, out), st))
        return (), ()


class BoxTensorfMarch(torch.autograd.Function):
    """DirectVoxGO's march for TensoRF models: the inputs it differentiates are the density tensors -- the six TensoRF factors
    (tensorf_density) or the dense density grid.  Returns (weights[M], alphainv_last[N], raw_alpha[M], points[M, 3], ray_id[M]
    i64, step_id[M] i64): pass B writes each survivor's point (no gradient) where BoxMarch returns its k0 features, for the
    model's k0 -- TensoRFGrid or DenseGrid -- to read with its own forward.  A ray needing more than cfg.s_max steps raises."""

    @staticmethod
    def forward(ctx, rays_o, rays_d, mask_world, cfg, ddesc, tensorf_density, vec_copies, *density):
        return _forward(ctx, _BoxTensorf(tensorf_density, vec_copies), density, None, rays_o, rays_d, mask_world, cfg, ddesc, None,
                        d_at=tuple(range(7, 7 + len(density))), k_at=None)

    backward = staticmethod(_backward)
