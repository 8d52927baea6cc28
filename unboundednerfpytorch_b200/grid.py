"""Voxel-grid modules with the reference's class / method surface, backed by the sm_90a kernels.

* ``DenseGrid``   -- FourierGrid/grid.py:41-84  (trilinear read = F.grid_sample there, grid.py:57)
* ``FourierGrid`` -- FourierGrid/FourierGrid_grid.py:42-101 (P = 1+2F slabs sampled at gamma_n(x), mean)
* ``TensoRFGrid`` -- FourierGrid/grid.py:90-201 (vector-matrix factors; see the class)
* ``MaskGrid``    -- FourierGrid/grid.py:207-242 / FourierGrid_grid.py:138-171 (nearest-voxel occupancy)
* ``create_grid`` -- grid.py:30-36 / FourierGrid_grid.py:14-18

The logical parameter shape stays ``[P, C, X, Y, Z]`` with the reference's names (``.grid``, ``xyz_min``,
``xyz_max``) so state_dicts interchange, but the PHYSICAL layout is channels-last
(``torch.channels_last_3d``: memory order [P, X, Y, Z, C]) so that the 8 corner records of a sample are
8 contiguous C-float records (128-bit loads / vector reds) instead of 8*C scattered 4-byte words on C
separate planes.  Gradients are produced in the same layout (autograd's layout contract keeps them so).
"""
import ctypes

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _cabi, ops
from ._cabi import UbnGridDesc, c_f, c_i64, c_int, check, ptr, stream_of


def _as_cl3d(t):
    """[P,C,X,Y,Z] tensor -> same values, channels-last-3d strides (no copy when already so)."""
    P, C, X, Y, Z = t.shape
    want = (X * Y * Z * C, 1, Y * Z * C, Z * C, C)
    if C == 1 and t.is_contiguous():
        return t
    if tuple(t.stride()) == want:
        return t
    out = torch.empty_strided(t.shape, want, dtype=t.dtype, device=t.device)
    out.copy_(t)
    return out


def zeros_grid(shape, device=None, dtype=torch.float32):
    P, C, X, Y, Z = [int(v) for v in shape]
    if C <= 1:
        return torch.zeros([P, C, X, Y, Z], dtype=dtype, device=device)
    return torch.zeros([P, X, Y, Z, C], dtype=dtype, device=device).permute(0, 4, 1, 2, 3)


def grid_desc(grid, xyz_min, xyz_max, num_freqs):
    """Describe a [P,C,X,Y,Z] tensor (reference-contiguous or channels-last) for the C ABI."""
    if grid.dim() != 5:
        raise RuntimeError('grid must be 5-D [P,C,X,Y,Z]')
    P, C, X, Y, Z = grid.shape
    sp, sc, sx, sy, sz = grid.stride()
    if C == 1:
        sc = 1
    if not (sy == Z * sz and sx == Y * Z * sz):
        raise RuntimeError('grid must be contiguous or channels-last contiguous')
    d = UbnGridDesc()
    d.P, d.C, d.X, d.Y, d.Z = P, C, X, Y, Z
    d.num_freqs = int(num_freqs) if num_freqs and num_freqs > 0 else 0
    d.stride_p, d.stride_c, d.stride_v = sp, sc, sz
    mn = [float(v) for v in xyz_min]
    mx = [float(v) for v in xyz_max]
    for a in range(3):
        d.xyz_min[a] = mn[a]
        d.xyz_max[a] = mx[a]
    return d


class _GridSample(torch.autograd.Function):
    """out[M,C] = trilinear read of grid at xyz[M,3]; backward = scatter into a grid-shaped gradient
    (only dL/d(grid) exists in the reference: ray points never require grad, SURVEY.md 3.3)."""

    @staticmethod
    def forward(ctx, grid, xyz, xyz_min, xyz_max, num_freqs):
        if not grid.is_cuda:
            raise RuntimeError('grid must be a CUDA tensor')
        if not xyz.is_cuda:
            raise RuntimeError('xyz must be a CUDA tensor')
        xyz = xyz.contiguous().float()
        desc = grid_desc(grid, xyz_min, xyz_max, num_freqs)
        n = xyz.shape[0]
        out = torch.empty(n, grid.shape[1], dtype=torch.float32, device=grid.device)
        with ops._Guard(grid) as lib:
            check(lib.ubn_grid_sample_fwd(ptr(grid), desc, ptr(xyz), c_i64(n), ptr(out), stream_of(grid)))
        ctx.save_for_backward(xyz)
        ctx.desc = desc
        ctx.grid_meta = (grid.shape, grid.stride())
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        (xyz,) = ctx.saved_tensors
        shape, stride = ctx.grid_meta
        grad_grid = torch.empty_strided(shape, stride, dtype=torch.float32, device=xyz.device).zero_()
        grad_out = grad_out.contiguous()
        with ops._Guard(xyz) as lib:
            check(lib.ubn_grid_sample_bwd(ptr(grad_out), ctx.desc, ptr(xyz), c_i64(xyz.shape[0]), ptr(grad_grid),
                                          stream_of(xyz)))
        return grad_grid, None, None, None, None


def grid_sample(grid, xyz, xyz_min, xyz_max, num_freqs=0):
    """Functional form: xyz [...,3] -> [...,C] (squeezed when C == 1), reference shape rules (grid.py:54-61)."""
    shape = xyz.shape[:-1]
    C = grid.shape[1]
    out = _GridSample.apply(grid, xyz.reshape(-1, 3), xyz_min, xyz_max, num_freqs)
    out = out.reshape(*shape, C)
    if C == 1:
        out = out.squeeze(-1)
    return out


def create_grid(type, **kwargs):
    """grid.py:30-36 / FourierGrid_grid.py:14-18: 'DenseGrid' -> DenseGrid, or FourierGrid when the
    Fourier keyword set (use_nerf_pos / fourier_freq_num) is given; 'TensoRFGrid' -> TensoRFGrid."""
    if type == 'DenseGrid':
        if 'use_nerf_pos' in kwargs or 'fourier_freq_num' in kwargs:
            return FourierGrid(**kwargs)
        return DenseGrid(**kwargs)
    if type == 'TensoRFGrid':
        return TensoRFGrid(**kwargs)
    raise NotImplementedError(type)


class _Bounded(nn.Module):
    """The xyz_min / xyz_max buffers and their host copy, which the kernels take by value."""

    def _register_bounds(self, xyz_min, xyz_max):
        self.register_buffer('xyz_min', torch.as_tensor(np.asarray(xyz_min if not torch.is_tensor(xyz_min) else xyz_min.cpu()),
                                                        dtype=torch.float32).clone())
        self.register_buffer('xyz_max', torch.as_tensor(np.asarray(xyz_max if not torch.is_tensor(xyz_max) else xyz_max.cpu()),
                                                        dtype=torch.float32).clone())
        self._bounds_cache = None

    def _bounds(self):
        # host copies of the bbox (the kernels take them by value): one D2H read, cached
        if self._bounds_cache is None:
            self._bounds_cache = (self.xyz_min.detach().cpu().tolist(), self.xyz_max.detach().cpu().tolist())
        return self._bounds_cache

    def _apply(self, fn, *a, **k):
        self._bounds_cache = None
        return super()._apply(fn, *a, **k)

    def _load_from_state_dict(self, *a, **k):
        self._bounds_cache = None
        return super()._load_from_state_dict(*a, **k)


class _VoxelGridBase(_Bounded):
    def _init_common(self, channels, world_size, xyz_min, xyz_max, slabs):
        self.channels = channels
        self.world_size = world_size
        self._register_bounds(xyz_min, xyz_max)
        ws = [int(v) for v in world_size]
        self.grid = nn.Parameter(zeros_grid([slabs, channels, *ws]))

    def scale_volume_grid(self, new_world_size):
        """grid.py:63-68: trilinear resample (align_corners=True) to the new resolution."""
        ws = [int(v) for v in new_world_size]
        if self.channels == 0:
            self.grid = nn.Parameter(torch.zeros([1, self.channels, *ws], device=self.grid.device))
        else:
            # one kernel, layout-preserving (the reference: F.interpolate(..., mode='trilinear', align_corners=True) on a
            # contiguous copy; here no [P,C,X,Y,Z] <-> channels-last round trips)
            self.grid = nn.Parameter(ops.resample_grid(self.grid.data, ws))
        self.world_size = new_world_size

    def total_variation_add_grad(self, wx, wy, wz, dense_mode):
        """grid.py:70-73: add the TV gradient in place into ``self.grid.grad``."""
        ops.total_variation_add_grad(self.grid, self.grid.grad, wx, wy, wz, dense_mode)

    def get_dense_grid(self):
        return self.grid

    @torch.no_grad()
    def __isub__(self, val):
        self.grid.data -= val
        return self

    def extra_repr(self):
        ws = self.world_size.tolist() if torch.is_tensor(self.world_size) else list(self.world_size)
        return f'channels={self.channels}, world_size={ws}'


class DenseGrid(_VoxelGridBase):
    """Dense 3-D grid (FourierGrid/grid.py:41-84)."""

    def __init__(self, channels, world_size, xyz_min, xyz_max, **kwargs):
        super().__init__()
        self._init_common(channels, world_size, xyz_min, xyz_max, slabs=1)
        self.num_freqs = 0

    def forward(self, xyz):
        mn, mx = self._bounds()
        return grid_sample(self.grid, xyz, mn, mx, 0)


class FourierGrid(_VoxelGridBase):
    """FourierGrid (FourierGrid/FourierGrid_grid.py:42-101): grid [1+2F, C, X, Y, Z] when use_nerf_pos."""

    def __init__(self, channels, world_size, xyz_min, xyz_max, use_nerf_pos=False, fourier_freq_num=0, config=None,
                 **kwargs):
        super().__init__()
        if use_nerf_pos:
            self.nerf_pos_num_freq = int(fourier_freq_num)
            self.pos_embed_output_dim = 1 + 2 * self.nerf_pos_num_freq
            slabs = self.pos_embed_output_dim
        else:
            self.nerf_pos_num_freq = -1
            self.pos_embed_output_dim = -1
            slabs = 1
        self._init_common(channels, world_size, xyz_min, xyz_max, slabs=slabs)
        self.num_freqs = self.nerf_pos_num_freq if use_nerf_pos else 0

    def forward(self, xyz):
        mn, mx = self._bounds()
        return grid_sample(self.grid, xyz, mn, mx, self.num_freqs)


TENSORF_FACTORS = ('xy_plane', 'xz_plane', 'yz_plane', 'x_vec', 'y_vec', 'z_vec')
# replicated copies the backward reduces the vector gradients into (ubn_tensorf_bwd's vec_copies)
TENSORF_VEC_COPIES = 8


def _as_cl4(t):
    """[1,R,A,B] factor -> same values with strides (A*B*R, 1, B*R, R): a node's R components form one record.  Set explicitly:
    torch.channels_last leaves strides of unit dimensions (the vectors' last axis) up to the input."""
    _, R, A, B = t.shape
    want = (A * B * R, 1, B * R, R)
    if tuple(t.stride()) == want:
        return t
    out = torch.empty_strided(t.shape, want, dtype=t.dtype, device=t.device)
    out.copy_(t)
    return out


def _factor_array(ts):
    return (ctypes.c_void_p * 6)(*[t.data_ptr() for t in ts])


def tensorf_desc(factors, channels, xyz_min, xyz_max):
    """Describe the six [1,R,A,B] factors (any strides; channels-last is the fast path) for the C ABI."""
    if len(factors) != 6 or any(t.dim() != 4 or t.shape[0] != 1 or t.dtype != torch.float32 for t in factors):
        raise RuntimeError('TensoRF factors must be six fp32 [1,R,A,B] tensors')
    xy, xz, yz, xv, yv, zv = factors
    Rxy, X, Y = xy.shape[1:]
    R, Z = xz.shape[1], xz.shape[3]
    want = [(Rxy, X, Y), (R, X, Z), (R, Y, Z), (R, X, 1), (R, Y, 1), (Rxy, Z, 1)]
    if [tuple(t.shape[1:]) for t in factors] != want:
        raise RuntimeError(f'TensoRF factor shapes disagree: {[tuple(t.shape) for t in factors]}')
    d = _cabi.UbnTensorfDesc()
    d.X, d.Y, d.Z, d.R, d.Rxy, d.C = X, Y, Z, R, Rxy, int(channels)
    for f, t in enumerate(factors):
        d.stride_r[f], d.stride_a[f], d.stride_b[f] = t.stride(1), t.stride(2), (t.stride(3) if f < 3 else 0)
    for a in range(3):
        d.xyz_min[a] = float(xyz_min[a])
        d.xyz_max[a] = float(xyz_max[a])
    return d


class _TensorfSample(torch.autograd.Function):
    """out[M,C] = the TensoRF read of the factors at xyz[M,3] (ubn_tensorf_fwd); backward = ubn_tensorf_bwd into gradients laid
    out like their factors."""

    @staticmethod
    def forward(ctx, xyz, f_vec, channels, xyz_min, xyz_max, vec_copies, *factors):
        if not (xyz.is_cuda and all(t.is_cuda for t in factors)):
            raise RuntimeError('TensoRFGrid needs CUDA tensors')
        desc = tensorf_desc(factors, channels, xyz_min, xyz_max)
        n = xyz.shape[0]
        out = torch.empty(n, channels, dtype=torch.float32, device=xyz.device)
        with ops._Guard(xyz) as lib, _cabi.timed(f'tensorf_fwd_c{channels}'):
            check(lib.ubn_tensorf_fwd(_factor_array(factors), ptr(f_vec), desc, ptr(xyz), c_i64(n), ptr(out), stream_of(xyz)))
        ctx.save_for_backward(xyz, f_vec, *factors)
        ctx.desc, ctx.vec_copies = desc, vec_copies
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        xyz, f_vec, *factors = ctx.saved_tensors
        d = ctx.desc
        grads = [torch.zeros_like(t, memory_format=torch.preserve_format) for t in factors]
        grad_f = torch.zeros_like(f_vec) if f_vec is not None else None
        K = int(ctx.vec_copies)
        nfeat = 2 * d.R + d.Rxy
        n_scratch = K * (d.X * d.R + d.Y * d.R + d.Z * d.Rxy) + _cabi.TENSORF_BWD_MAX_CTAS * nfeat * d.C
        scratch = torch.empty(n_scratch, dtype=torch.float32, device=xyz.device)
        grad_out = grad_out.contiguous()
        gptrs = (ctypes.c_void_p * 6)(*[g.data_ptr() for g in grads])
        with ops._Guard(xyz) as lib, _cabi.timed(f'tensorf_bwd_c{d.C}'):
            check(lib.ubn_tensorf_bwd(_factor_array(factors), ptr(f_vec), d, ptr(xyz), c_i64(xyz.shape[0]), ptr(grad_out), gptrs,
                                      ptr(grad_f), c_int(K), ptr(scratch), stream_of(xyz)))
        return (None, grad_f, None, None, None, None, *grads)


def tensorf_sample(factors, f_vec, xyz, xyz_min, xyz_max, channels, vec_copies=None):
    """Functional TensoRFGrid read: xyz [...,3] -> [...,C] (squeezed when C == 1), grid.py:111-129."""
    shape = xyz.shape[:-1]
    out = _TensorfSample.apply(xyz.reshape(-1, 3).contiguous().float(), f_vec if channels > 1 else None, int(channels),
                               xyz_min, xyz_max, TENSORF_VEC_COPIES if vec_copies is None else vec_copies, *factors)
    out = out.reshape(*shape, channels)
    if channels == 1:
        out = out.squeeze(-1)
    return out


class TensoRFGrid(_Bounded):
    """Vector-matrix factorised grid (FourierGrid/grid.py:90-172, TensoRF arXiv 2203.09517).  Parameters keep the reference's
    names and logical shapes -- xy_plane [1,Rxy,X,Y], xz_plane [1,R,X,Z], yz_plane [1,R,Y,Z], x_vec [1,R,X,1], y_vec [1,R,Y,1],
    z_vec [1,Rxy,Z,1] and, for channels > 1, f_vec [R+R+Rxy, channels] -- so state dicts interchange; the factors are stored
    channels-last ([A,B,R] in memory) so that a node's R components are one record.  Reads, their adjoint, TV, the dense
    materialisation and the rescale run on the kernels of csrc/tensorf.cu and csrc/grid_utils.cu."""

    def __init__(self, channels, world_size, xyz_min, xyz_max, config):
        super().__init__()
        self.channels = channels
        self.world_size = world_size
        self.config = config
        self._register_bounds(xyz_min, xyz_max)
        X, Y, Z = [int(v) for v in world_size]
        R = config['n_comp']
        Rxy = config.get('n_comp_xy', R)
        # the reference's initialisation, in its order (seeded constructions give the reference's values)
        self.xy_plane = nn.Parameter(_as_cl4(torch.randn([1, Rxy, X, Y]) * 0.1))
        self.xz_plane = nn.Parameter(_as_cl4(torch.randn([1, R, X, Z]) * 0.1))
        self.yz_plane = nn.Parameter(_as_cl4(torch.randn([1, R, Y, Z]) * 0.1))
        self.x_vec = nn.Parameter(_as_cl4(torch.randn([1, R, X, 1]) * 0.1))
        self.y_vec = nn.Parameter(_as_cl4(torch.randn([1, R, Y, 1]) * 0.1))
        self.z_vec = nn.Parameter(_as_cl4(torch.randn([1, Rxy, Z, 1]) * 0.1))
        if self.channels > 1:
            self.f_vec = nn.Parameter(torch.ones([R + R + Rxy, channels]))
            nn.init.kaiming_uniform_(self.f_vec, a=np.sqrt(5))

    def factors(self):
        return [getattr(self, n) for n in TENSORF_FACTORS]

    def _f_vec(self):
        return self.f_vec if self.channels > 1 else None

    def forward(self, xyz):
        mn, mx = self._bounds()
        return tensorf_sample(self.factors(), self._f_vec(), xyz, mn, mx, self.channels)

    @torch.no_grad()
    def scale_volume_grid(self, new_world_size):
        """grid.py:131-140: every factor resampled with F.interpolate(bilinear, align_corners=True) arithmetic -- the trilinear
        resample kernel on the factor viewed as [1,R,A,B,1] (a unit axis resamples exactly)."""
        if self.channels == 0:
            return
        X, Y, Z = [int(v) for v in new_world_size]
        sizes = [(X, Y), (X, Z), (Y, Z), (X, 1), (Y, 1), (Z, 1)]
        for name, (A, B) in zip(TENSORF_FACTORS, sizes):
            t = getattr(self, name).data
            t5 = t.as_strided([*t.shape, 1], [*t.stride(), t.stride(3)])
            out = ops.resample_grid(t5, [A, B, 1])[..., 0]
            setattr(self, name, nn.Parameter(_as_cl4(out)))
        self.world_size = new_world_size

    @torch.no_grad()
    def total_variation_add_grad(self, wx, wy, wz, dense_mode):
        """grid.py:142-154: the gradient of the smooth-L1 TV sum / 6, added in place into the factors' .grad (dense_mode is
        ignored, as there)."""
        fs = self.factors()
        for p in fs:
            if p.grad is None:
                p.grad = torch.zeros_like(p, memory_format=torch.preserve_format)
            elif p.grad.stride() != p.stride():
                p.grad = torch.empty_like(p, memory_format=torch.preserve_format).copy_(p.grad)
        mn, mx = self._bounds()
        desc = tensorf_desc(fs, self.channels, mn, mx)
        gptrs = (ctypes.c_void_p * 6)(*[p.grad.data_ptr() for p in fs])
        with ops._Guard(fs[0]) as lib:
            check(lib.ubn_tensorf_tv_add_grad(_factor_array(fs), gptrs, desc, c_f(float(wx)), c_f(float(wy)), c_f(float(wz)),
                                              stream_of(fs[0])))

    @torch.no_grad()
    def get_dense_grid(self):
        """grid.py:156-169: [1, C, X, Y, Z] (contiguous) node products, projected by f_vec when C > 1.  Not differentiable (the
        model calls it under no_grad only)."""
        fs = self.factors()
        mn, mx = self._bounds()
        desc = tensorf_desc(fs, self.channels, mn, mx)
        out = torch.empty([1, self.channels, desc.X, desc.Y, desc.Z], dtype=torch.float32, device=fs[0].device)
        with ops._Guard(fs[0]) as lib:
            check(lib.ubn_tensorf_dense(_factor_array(fs), ptr(self._f_vec()), desc, ptr(out), stream_of(fs[0])))
        return out

    def extra_repr(self):
        ws = self.world_size.tolist() if torch.is_tensor(self.world_size) else list(self.world_size)
        return f'channels={self.channels}, world_size={ws}, n_comp={self.config["n_comp"]}'


class MaskGrid(nn.Module):
    """Occupancy mask (FourierGrid/grid.py:207-242).  ``path`` re-derives the mask from a coarse checkpoint
    with alpha = 1 - exp(-softplus(maxpool3(density) + act_shift) * voxel_size_ratio) (grid.py:210-220)."""

    def __init__(self, path=None, mask_cache_thres=None, mask=None, xyz_min=None, xyz_max=None):
        super().__init__()
        if path is not None:
            st = torch.load(path, map_location='cpu', weights_only=False)
            self.mask_cache_thres = mask_cache_thres
            density_grid = st['model_state_dict']['density.grid']
            if density_grid.shape[0] > 1 or density_grid.shape[1] > 1:
                density_grid = density_grid[0][0][None, None]
            density = F.max_pool3d(density_grid.contiguous(), kernel_size=3, padding=1, stride=1)
            ratio = st['model_kwargs'].get('voxel_size_ratio', st['model_kwargs'].get('voxel_size_ratio_density'))
            alpha = 1 - torch.exp(-F.softplus(density + st['model_state_dict']['act_shift']) * ratio)
            mask = (alpha >= self.mask_cache_thres).squeeze(0).squeeze(0)
            xyz_min = torch.as_tensor(st['model_kwargs']['xyz_min'], dtype=torch.float32)
            xyz_max = torch.as_tensor(st['model_kwargs']['xyz_max'], dtype=torch.float32)
        else:
            mask = mask.bool()
            xyz_min = torch.as_tensor(np.asarray(xyz_min.cpu() if torch.is_tensor(xyz_min) else xyz_min), dtype=torch.float32)
            xyz_max = torch.as_tensor(np.asarray(xyz_max.cpu() if torch.is_tensor(xyz_max) else xyz_max), dtype=torch.float32)
        self.register_buffer('mask', mask.contiguous())
        xyz_len = xyz_max - xyz_min
        self.register_buffer('xyz2ijk_scale', (torch.tensor(list(mask.shape), dtype=torch.float32) - 1) / xyz_len)
        self.register_buffer('xyz2ijk_shift', -xyz_min * self.xyz2ijk_scale)

    @torch.no_grad()
    def forward(self, xyz):
        shape = xyz.shape[:-1]
        xyz = xyz.reshape(-1, 3).contiguous()
        mask = ops.maskcache_lookup(self.mask, xyz, self.xyz2ijk_scale, self.xyz2ijk_shift)
        return mask.reshape(shape)

    def extra_repr(self):
        return f'mask.shape={list(self.mask.shape)}'
