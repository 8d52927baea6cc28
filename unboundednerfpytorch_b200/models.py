"""Voxel-grid radiance-field models with the reference's constructor / forward surface:

* ``FourierGridModel``       -- FourierGrid/FourierGrid_model.py:134-681
* ``DirectContractedVoxGO``  -- FourierGrid/dcvgo.py:28-384
* ``DirectVoxGO``            -- FourierGrid/dvgo.py:26-425 (bounded scenes)
* ``DirectMPIGO``            -- FourierGrid/dmpigo.py:18-340 (forward-facing scenes in NDC space)

Same constructor keywords, ``get_kwargs()`` keys, state-dict names (``density.grid``, ``k0.grid``,
``rgbnet.{0,2.0,3}.{weight,bias}``, ``mask_cache.mask`` ...), ``forward(rays_o, rays_d, viewdirs,
global_step=None, is_train=False, **render_kwargs)`` and ``ret_dict`` keys, so run_train.py /
run_render.py style callers work unchanged.  ``forward`` runs the fused march (march.py: 3 launches
instead of ~40 and no boolean-mask compaction syncs except the one ragged-size read); ``forward_ops``
composes the individual drop-in ops in the reference's order (used for cross-checks and for grids the
fused feature kernel does not cover, e.g. the 3-channel coarse-stage k0).
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import grid as G
from . import march
from . import shade as shade_mod
from .functional import Alphas2Weights, Raw2Alpha, composite_rgb, host_scalar, segment_sum


def _host_array(v):
    """A bbox argument as a host array: lists, NumPy arrays and tensors on any device (compute_bbox_by_cam_frustrm /
    compute_bbox_by_coarse_geo return CUDA tensors, which run_train.py passes straight to the model constructors)."""
    return np.asarray(v.detach().cpu() if torch.is_tensor(v) else v)


def _cube_root_size(xyz_min, xyz_max, num_voxels):
    return ((xyz_max - xyz_min).prod() / num_voxels).pow(1 / 3)


def _make_rgbnet(dim0, width, depth):
    # Linear-ReLU-(Sequential(Linear,ReLU))*-Linear: identical module tree => identical state-dict keys
    net = nn.Sequential(
        nn.Linear(dim0, width), nn.ReLU(inplace=True),
        *[nn.Sequential(nn.Linear(width, width), nn.ReLU(inplace=True)) for _ in range(depth - 2)],
        nn.Linear(width, 3))
    nn.init.constant_(net[-1].bias, 0)
    return net


def _view_embed(viewdirs, viewfreq):
    emb = (viewdirs.unsqueeze(-1) * viewfreq).flatten(-2)
    return torch.cat([viewdirs, emb.sin(), emb.cos()], -1)


class _GridModel(nn.Module):
    """What the four models share: the host copies of the geometry the march cfgs take by value, activate_density, the TV
    terms, the rgbnet and its shading, and the mask cache's lattice and rebuild."""

    _HOST_BUFFERS = ('xyz_min', 'xyz_max')        # the two bbox buffers the march cfg takes by value
    _host_cache = None          # (mask_cache it was read from, host bbox, host mask geometry)

    def _host_geometry(self):
        """The geometry the march cfgs take by value, read to the host once and again after _apply, a state-dict load or a
        new mask_cache."""
        if self._host_cache is None or self._host_cache[0] is not self.mask_cache:
            mc = self.mask_cache
            self._host_cache = (mc, tuple(getattr(self, name).detach().cpu().tolist() for name in self._HOST_BUFFERS),
                                (mc.xyz2ijk_scale.cpu().tolist(), mc.xyz2ijk_shift.cpu().tolist()))
        return self._host_cache

    def _host(self):
        """The two _HOST_BUFFERS as host lists."""
        return self._host_geometry()[1]

    def _mask_geometry(self):
        """(mask_scale, mask_shift): the mask cache's world -> index map as host lists."""
        return self._host_geometry()[2]

    def _apply(self, fn, *a, **k):
        self._host_cache = None
        return super()._apply(fn, *a, **k)

    def _load_from_state_dict(self, *a, **k):
        self._host_cache = None
        return super()._load_from_state_dict(*a, **k)

    def _voxel_size(self):
        return self.voxel_size

    def _voxel_size_ratio(self):
        return self.voxel_size_ratio

    def _density_shift(self):
        return self.act_shift

    def activate_density(self, density, interval=None):
        interval = interval if interval is not None else self._voxel_size_ratio()
        shape = density.shape
        return Raw2Alpha.apply(density.flatten().contiguous(), self._density_shift(), interval).reshape(shape)

    def density_total_variation_add_grad(self, weight, dense_mode):
        self.density.total_variation_add_grad(*self._tv_weights(self.density, weight, dense_mode))

    def k0_total_variation_add_grad(self, weight, dense_mode):
        self.k0.total_variation_add_grad(*self._tv_weights(self.k0, weight, dense_mode))

    def tv_terms(self, weight_density=0., weight_k0=0., dense_mode=True):
        """{grid parameter: (wx, wy, wz, dense_mode)} with the weights of the two methods above -- the form
        dist.reduce_tv_step consumes to pipeline all-reduce / TV / Adam slab by slab."""
        return {grid.grid: self._tv_weights(grid, weight, dense_mode)
                for grid, weight in ((self.density, weight_density), (self.k0, weight_k0)) if weight > 0}

    def _add_rgbnet(self, feat_dim, viewbase_pe, width, depth):
        """The view-frequency buffer, then the rgbnet on cat[feat_dim features, view embedding]."""
        self.register_buffer('viewfreq', torch.FloatTensor([(2 ** i) for i in range(viewbase_pe)]))
        self.rgbnet = _make_rgbnet(3 + 3 * viewbase_pe * 2 + feat_dim, width, depth)

    def _shade(self, k0, viewdirs, ray_id):
        if self.rgbnet is None:
            return torch.sigmoid(k0)
        emb = _view_embed(viewdirs, self.viewfreq).flatten(0, -2)
        if shade_mod.supported(self.rgbnet, k0.shape[-1]):
            return shade_mod.shade(self.rgbnet, k0, emb, ray_id)          # fused on-chip MLP (csrc/shade.cu)
        return torch.sigmoid(self.rgbnet(torch.cat([k0, emb[ray_id]], -1)))   # other widths / depths: torch (cuBLAS)

    # ---- the fused render of the bounded models (DirectVoxGO, DirectMPIGO) ------------------------------------------------
    FUSED_FRAME_BY_DEFAULT = True      # render.render_rays takes render_fused where it applies even without fused_frame=True

    def _render_net_ok(self, C, covered):
        """Whether the fused render kernels take this model's rgbnet on a C-channel k0: none with C = 3 (sigmoid(k0)), or a
        3-layer float32 CUDA rgbnet on cat[k0, view embedding] whose (C, viewbase_pe, width) is in ``covered``."""
        net = self.rgbnet
        if net is None:
            return C == 3
        try:
            l1, l2, l3 = net[0], net[2][0], net[3]
        except Exception:
            return False
        pe, W = self.viewfreq.numel(), l1.weight.shape[0]
        return (len(net) == 4 and (C, pe, W) in covered and tuple(l1.weight.shape) == (W, C + 3 + 6 * pe)
                and tuple(l2.weight.shape) == (W, W) and tuple(l3.weight.shape) == (3, W)
                and all(t.is_cuda and t.dtype == torch.float32 for t in (l1.weight, l2.weight, l3.weight)))

    def _render_net_args(self):
        """((W1, b1, W2, b2, W3, b3), width, viewbase_pe) for a render entry; NULL weights, 0, 0 without an rgbnet."""
        if self.rgbnet is None:
            return (None,) * 6, 0, 0
        l1, l2, l3 = self.rgbnet[0], self.rgbnet[2][0], self.rgbnet[3]
        net = tuple(t.detach().contiguous() for t in (l1.weight, l1.bias, l2.weight, l2.bias, l3.weight, l3.bias))
        return net, l1.weight.shape[0], self.viewfreq.numel()

    def _render_grids_ok(self, rays_o, render_kwargs):
        """What both bounded models' render_fused_ok require besides their own geometry: no gradient, CUDA rays, a contiguous
        float32 one-slab density, a float32 k0 and a numeric bg."""
        dg, kg = self.density.grid, self.k0.grid
        return (not torch.is_grad_enabled() and rays_o.is_cuda and isinstance(render_kwargs.get('bg'), (int, float))
                and march.box_density_supported(dg) and dg.dtype == torch.float32 and kg.dtype == torch.float32
                and kg.numel() < 2 ** 31)

    def _mask_lattice(self, world_size):
        """[X, Y, Z, 3]: linspace(xyz_min, xyz_max, world_size) per axis, the points a mask cache is built on."""
        ws = [int(v) for v in world_size]
        axes = [torch.linspace(float(self.xyz_min[a]), float(self.xyz_max[a]), ws[a], device=self.xyz_min.device) for a in range(3)]
        return torch.stack(torch.meshgrid(*axes, indexing='ij'), -1)

    def _set_mask_cache(self, mask):
        self.mask_cache = G.MaskGrid(path=None, mask=mask, xyz_min=self.xyz_min, xyz_max=self.xyz_max).to(mask.device)

    @torch.no_grad()
    def update_occupancy_cache(self):
        """mask_cache.mask &= max_pool3d(Raw2Alpha(density(mask lattice))) > fast_color_thres (FourierGrid_model.py:441-456,
        dcvgo.py:214-226, dvgo.py:236-246, dmpigo.py:174-187: DirectMPIGO's shift is 0, without its act_shift grid, as there).
        Two kernels: ops.lattice_alpha generates the lattice points in registers; ops.maxpool3_gt_and_ pools, thresholds and
        ANDs (4 B + 1 B per cell)."""
        from . import ops
        mn, mx = self.density._bounds()
        alpha = ops.lattice_alpha(self.density.grid.data, mn, mx, self.density.num_freqs, self.xyz_min.tolist(),
                                  self.xyz_max.tolist(), self.mask_cache.mask.shape, host_scalar(self._density_shift()),
                                  float(self._voxel_size_ratio()))
        ops.maxpool3_gt_and_(self.mask_cache.mask, alpha, self.fast_color_thres)

    @torch.no_grad()
    def _rebuild_mask_cache(self, world_size, density):
        """After a rescale: mask(lattice) & (max_pool3d(alpha(density)) > fast_color_thres) on the new lattice."""
        xyz = self._mask_lattice(world_size)
        alpha = F.max_pool3d(self.activate_density(density.contiguous()), kernel_size=3, padding=1, stride=1)[0, 0]
        self._set_mask_cache(self.mask_cache(xyz) & (alpha > self.fast_color_thres))


class _CoarseGeo:
    """hit_coarse_geo, for the models whose reference has it (FourierGridModel, DirectVoxGO)."""

    def hit_coarse_geo(self, rays_o, rays_d, near, far, stepsize, **render_kwargs):
        """FourierGrid_model.py:495-507, dvgo.py:292-304: does a ray hit the occupancy mask?"""
        from . import ops
        shape = rays_o.shape[:-1]
        rays_o = rays_o.reshape(-1, 3).contiguous()
        rays_d = rays_d.reshape(-1, 3).contiguous()
        ray_pts, mask_outbbox, ray_id = ops.sample_pts_on_rays(rays_o, rays_d, self.xyz_min, self.xyz_max, near, 1e9,
                                                               stepsize * float(self._voxel_size()))[:3]
        mask_inbbox = ~mask_outbbox
        hit = torch.zeros([len(rays_o)], dtype=torch.bool, device=rays_o.device)
        hit[ray_id[mask_inbbox][self.mask_cache(ray_pts[mask_inbbox])]] = 1
        return hit.reshape(shape)


class _ContractedBase(_GridModel):
    """Shared machinery of the two contracted-space models."""

    T_BOUNDARY = 2.0          # dcvgo.py:243-244; FourierGridModel overrides with 1.5
    USE_CUMDIST = False
    USE_MASKCACHE = False
    _HOST_BUFFERS = ('scene_center', 'scene_radius')

    # ---- helpers --------------------------------------------------------------------------------
    def _init_scene(self, xyz_min, xyz_max, bg_len, fast_color_thres, contracted_norm):
        xyz_min = torch.as_tensor(_host_array(xyz_min), dtype=torch.float32)
        xyz_max = torch.as_tensor(_host_array(xyz_max), dtype=torch.float32)
        assert len(((xyz_max - xyz_min) * 100000).long().unique()), 'scene bbox must be a cube'
        self.register_buffer('scene_center', (xyz_min + xyz_max) * 0.5)
        self.register_buffer('scene_radius', (xyz_max - xyz_min) * 0.5)
        self.register_buffer('xyz_min', torch.tensor([-1., -1., -1.]) - bg_len)
        self.register_buffer('xyz_max', torch.tensor([1., 1., 1.]) + bg_len)
        if isinstance(fast_color_thres, dict):
            self._fast_color_thres = fast_color_thres
            self.fast_color_thres = fast_color_thres[0]
        else:
            self._fast_color_thres = None
            self.fast_color_thres = fast_color_thres
        self.bg_len = bg_len
        self.contracted_norm = contracted_norm

    def _maybe_update_thres(self, global_step):
        if isinstance(self._fast_color_thres, dict) and global_step in self._fast_color_thres:
            self.fast_color_thres = self._fast_color_thres[global_step]

    def _sample_dense(self, ori_rays_o, ori_rays_d, stepsize):
        """Dense [N,S,3] contracted points with torch elementwise ops (dcvgo.py:239-262,
        FourierGrid_model.py:522-552) -- only the op-by-op path and API users need them materialised."""
        rays_o = (ori_rays_o - self.scene_center) / self.scene_radius
        rays_d = ori_rays_d / ori_rays_d.norm(dim=-1, keepdim=True)
        t = march.t_schedule(self._world_len(), stepsize, self.bg_len, self.T_BOUNDARY, ori_rays_o.device)
        ray_pts = rays_o[:, None, :] + rays_d[:, None, :] * t[None, :, None]
        if self.contracted_norm == 'inf':
            norm = ray_pts.abs().amax(dim=-1, keepdim=True)
        elif self.contracted_norm == 'l2':
            norm = ray_pts.norm(dim=-1, keepdim=True)
        else:
            raise NotImplementedError
        inner_mask = (norm <= 1)
        B = 1 + self.bg_len
        A = B * 1.0 - 1.0
        ray_pts = torch.where(inner_mask, ray_pts, ray_pts / norm * (B - A / norm))
        return ray_pts, inner_mask.squeeze(-1), t

    # ---- the fused forward --------------------------------------------------------------------------
    def _fused_ok(self):
        kg = self.k0.grid
        if kg.shape[1] in (3, 9, 15):      # march_feature.cu's scalar-channel kernels: odd slab counts up to 11
            return (kg.is_cuda and kg.shape[0] in (1, 3, 5, 7, 9, 11) and kg.stride(1) == 1 and min(kg.shape[2:]) >= 2
                    and kg[0].numel() < 2 ** 31)       # 32-bit offsets inside a slab
        return kg.is_cuda and kg.shape[1] in (4, 8, 12, 16) and kg.shape[0] <= 16

    def _march_inputs(self, stepsize, dev):
        """(t table, march cfg, mask cache or None, density desc, k0 desc) of the fused march and the fused render."""
        t_table = march.t_schedule(self._world_len(), stepsize, self.bg_len, self.T_BOUNDARY, dev)
        interval = stepsize * float(self._voxel_size_ratio())
        center, radius = self._host()
        mscale, mshift = self._mask_geometry()
        mask = self.mask_cache.mask if self.USE_MASKCACHE else None
        cum = None
        if self.USE_CUMDIST:
            cum = (2 + 2 * self.bg_len) / self._world_len() * stepsize * 0.95
        cfg = march.make_cfg(center, radius, self.bg_len, self.contracted_norm, t_table.numel(),
                             host_scalar(self.act_shift), interval, self.fast_color_thres,
                             cumdist_thres=cum, mask=mask, mask_scale=mscale, mask_shift=mshift)
        dmn, dmx = self.density._bounds()
        kmn, kmx = self.k0._bounds()
        ddesc = G.grid_desc(self.density.grid, dmn, dmx, self.density.num_freqs)
        kdesc = G.grid_desc(self.k0.grid, kmn, kmx, self.k0.num_freqs)
        return t_table, cfg, mask, ddesc, kdesc

    def _march(self, rays_o, rays_d, stepsize, coherent=False):
        t_table, cfg, mask, ddesc, kdesc = self._march_inputs(stepsize, rays_o.device)
        dense_known = (self.fast_color_thres <= 0) and not self.USE_CUMDIST and not self.USE_MASKCACHE
        out = march.March.apply(self.density.grid, self.k0.grid, rays_o, rays_d, t_table, mask, cfg, ddesc, kdesc,
                                dense_known, coherent)
        return out, t_table

    # ---- the fused render ---------------------------------------------------------------------------
    RENDER_USES_BG = False      # DirectContractedVoxGO adds alphainv_last * bg outside training

    def render_fused_ok(self, rays_o, render_kwargs):
        """Whether render_fused covers this model and call (render.render_rays takes it exactly then): one-slab density and k0
        grids (DirectContractedVoxGO; FourierGridModel at fourier_freq_num 0), a channels-last k0 of 12 or 3 channels, the
        reference's unbounded rgbnets ((rgbnet_dim, viewbase_pe) = (12, 4) or (3, 8), width 128, depth 3) or none (sigmoid(k0),
        3 channels), no gradient, CUDA rays, and a background the fused composite reproduces: none for FourierGridModel
        (rand_bkgd draws a random one), a number for DirectContractedVoxGO.
        With render_kwargs['fused_slabs'] = True also FourierGridModel with Fourier slabs: density and k0 of the same slab count
        7, 9 or 11 (fourier_freq_num 3, 4, 5), a 12-channel k0 and the (12, 4) rgbnet (csrc/render_fourier.cu).  Opt-in: on dense
        scenes the fused slab render is not always faster than the chunk loop (DESIGN.md §7), and its frames agree with the loop to
        about 1e-6, not bit for bit."""
        kg, dg = self.k0.grid, self.density.grid
        if torch.is_grad_enabled() or not (rays_o.is_cuda and kg.is_cuda and dg.is_cuda and self._fused_ok()):
            return False
        P, C = kg.shape[0], kg.shape[1]
        if P != 1 and not (render_kwargs.get('fused_slabs', False) and P in (7, 9, 11) and C == 12 and self.rgbnet is not None):
            return False
        if not (C in (3, 12) and kg.stride(1) == 1 and kg.dtype == torch.float32
                and tuple(dg.shape[:2]) == (P, 1) and dg.is_contiguous() and dg.dtype == torch.float32):
            return False
        if self.RENDER_USES_BG:
            if not isinstance(render_kwargs.get('bg', 0), (int, float)):
                return False
        elif render_kwargs.get('rand_bkgd', False):
            return False
        net = self.rgbnet
        if net is None:
            return C == 3
        try:
            l1, l2, l3 = net[0], net[2][0], net[3]
        except Exception:
            return False
        pe = self.viewfreq.numel()
        return (len(net) == 4 and (C, pe) in ((12, 4), (3, 8)) and tuple(l1.weight.shape) == (128, C + 3 + 6 * pe)
                and tuple(l2.weight.shape) == (128, 128) and tuple(l3.weight.shape) == (3, 128)
                and all(t.is_cuda and t.dtype == torch.float32 for t in (l1.weight, l2.weight, l3.weight)))

    @torch.no_grad()
    def render_fused(self, rays_o, rays_d, viewdirs, n_shaded=None, n_marched=None, **render_kwargs):
        """{'rgb_marched' [N,3], 'depth' [N], 'alphainv_last' [N]} of N rays in one launch (csrc/render.cu): the march, the k0
        read of the kept samples, the rgbnet and the composite with no per-sample buffers, so a whole frame is one call.  Same
        kept samples and alphainv_last (bit for bit) as forward; rgb_marched and depth as forward's composite, summed in step order.
        Fourier slabs (render_kwargs['fused_slabs']) run csrc/render_fourier.cu, the same kernel and contract instantiated on the
        slab count.  n_shaded / n_marched: optional int32 [N] that receive each ray's kept samples / the samples of the
        32-sample chunks marched before the ray stopped.  Only where render_fused_ok holds."""
        from . import _cabi
        from ._cabi import c_f, c_i64, c_int, check, ptr, stream_of
        N = rays_o.shape[0]
        dev = rays_o.device
        rays_o = rays_o.contiguous().float()
        rays_d = rays_d.contiguous().float()
        viewdirs = viewdirs.contiguous().float()
        rgb = torch.empty(N, 3, dtype=torch.float32, device=dev)
        depth = torch.empty(N, dtype=torch.float32, device=dev)
        last = torch.empty(N, dtype=torch.float32, device=dev)
        t_table, cfg, mask, ddesc, kdesc = self._march_inputs(render_kwargs['stepsize'], dev)
        if self.rgbnet is not None:
            l1, l2, l3 = self.rgbnet[0], self.rgbnet[2][0], self.rgbnet[3]
            net = tuple(t.detach().contiguous() for t in (l1.weight, l1.bias, l2.weight, l2.bias, l3.weight, l3.bias))
            pe = self.viewfreq.numel()
        else:
            net, pe = (None,) * 6, 0
        use_bg = 1 if self.RENDER_USES_BG else 0
        bg = float(render_kwargs.get('bg', 0)) if use_bg else 0.0
        name = 'render_fourier' if self.k0.grid.shape[0] > 1 else 'render_contracted'
        with _cabi.timed(name):
            check(getattr(_cabi.load(), 'ubn_' + name)(
                ptr(rays_o), ptr(rays_d), ptr(viewdirs), ptr(t_table), ptr(self.density.grid), ddesc, ptr(self.k0.grid), kdesc,
                ptr(mask), cfg, c_i64(N), *map(ptr, net), c_int(128), c_int(pe), c_int(use_bg), c_f(bg), ptr(rgb), ptr(depth),
                ptr(last), ptr(n_shaded), ptr(n_marched), stream_of(rgb)))
        return {'rgb_marched': rgb, 'depth': depth, 'alphainv_last': last}

    def _tv_weights(self, grid, weight, dense_mode):
        w = weight * float(max(grid.grid.shape[2:])) / 128         # each grid's own largest dimension
        return (w, w, w, dense_mode)

    @torch.no_grad()
    def update_occupancy_cache_lt_nviews(self, rays_o_tr, rays_d_tr, imsz, render_kwargs, maskout_lt_nviews):
        """dcvgo.py:195-213: mask_cache.mask &= (number of training views whose contracted samples put a trilinear weight > 1 on a
        voxel of a ones grid over [xyz_min, xyz_max] at world_size) >= maskout_lt_nviews.  Every one of a view's n_rays * S samples
        counts, as the reference scatters sample_ray's whole point tensor.  The reference materialises [8192, S, 3] points and runs
        grid_sample's backward per chunk; here one kernel per view (ops.view_scatter_ones_contracted) generates each sample in
        registers and scatters its eight weights into a per-view buffer, and ops.count_gt_ adds (buffer > 1) to the count."""
        from . import ops
        dev = self.density.grid.device
        ws = [int(v) for v in self.world_size]
        t_table = march.t_schedule(self._world_len(), render_kwargs['stepsize'], self.bg_len, self.T_BOUNDARY, dev)
        center, radius = self._host()
        lo, hi = self.xyz_min.tolist(), self.xyz_max.tolist()
        count = torch.zeros(ws, device=dev)
        buf = torch.empty(ws, device=dev)
        for rays_o, rays_d in zip(rays_o_tr.split(imsz), rays_d_tr.split(imsz)):
            rays_o = rays_o.to(dev, torch.float32).reshape(-1, 3).contiguous()
            rays_d = rays_d.to(dev, torch.float32).reshape(-1, 3).contiguous()
            buf.zero_()
            ops.view_scatter_ones_contracted(rays_o, rays_d, t_table, center, radius, self.bg_len, self.contracted_norm, lo, hi, ws,
                                             buf)
            ops.count_gt_(count, buf, 1.0)
        self.mask_cache.mask &= (count >= maskout_lt_nviews)


@torch.no_grad()
def _scale_dense_model(model, num_voxels):
    """scale_volume_grid of the DenseGrid models (dcvgo.py:196-212, dvgo.py:213-234): new resolution, both grids resampled, and
    -- up to 256^3 voxels -- the mask cache rebuilt on the new lattice as mask(lattice) & (max_pool3d(alpha(density)) > thres)."""
    model._set_grid_resolution(num_voxels)
    model.density.scale_volume_grid(model.world_size)
    model.k0.scale_volume_grid(model.world_size)
    if np.prod(model.world_size.tolist()) <= 256 ** 3:
        model._rebuild_mask_cache(model.world_size, model.density.get_dense_grid())


@torch.no_grad()
def _count_views(density, world_size, voxel_size, rays_o_tr, rays_d_tr, imsz, near, stepsize, downrate, irregular_shape):
    """voxel_count_views (FourierGrid_model.py:390-420, dvgo.py:238-277): per-voxel number of training views that see it.  The
    reference materialises the sample points of 10 000 rays at a time and runs DenseGrid(ones).sum().backward(); here one kernel
    per view scatters the trilinear weights of every (ray, sample) straight into a per-view buffer, a second adds (buffer > 1) to
    the count.  far is 1e9 as the reference sets it."""
    from . import ops
    far = 1e9
    dev = density.xyz_min.device
    ws = [int(v) for v in world_size]
    n_samples = int(np.linalg.norm(np.array(ws) + 1) / stepsize) + 1
    step = float(stepsize * voxel_size)
    mn, mx = density._bounds()
    count = torch.zeros(1, 1, *ws, device=dev)
    buf = torch.empty(*ws, device=dev)
    for rays_o_, rays_d_ in zip(rays_o_tr.split(imsz), rays_d_tr.split(imsz)):
        if not irregular_shape:
            rays_o_, rays_d_ = rays_o_[::downrate, ::downrate], rays_d_[::downrate, ::downrate]
        ro = rays_o_.to(dev).reshape(-1, 3).contiguous().float()
        rd = rays_d_.to(dev).reshape(-1, 3).contiguous().float()
        buf.zero_()
        ops.view_scatter_ones(ro, rd, mn, mx, ws, n_samples, near, far, step, buf)
        ops.count_gt_(count, buf, 1.0)
    return count


# ======================================================================================================
class FourierGridModel(_CoarseGeo, _ContractedBase):
    """FourierGrid/FourierGrid_model.py:134-681."""

    T_BOUNDARY = 1.5          # FourierGrid_model.py:526

    def __init__(self, xyz_min, xyz_max, num_voxels_density=0, num_voxels_base_density=0, num_voxels_rgb=0,
                 num_voxels_base_rgb=0, num_voxels_viewdir=0, alpha_init=None, mask_cache_world_size=None,
                 fast_color_thres=0, bg_len=0.2, contracted_norm='inf', density_type='DenseGrid', k0_type='DenseGrid',
                 density_config={}, k0_config={}, rgbnet_dim=0, rgbnet_depth=3, rgbnet_width=128, fourier_freq_num=5,
                 viewbase_pe=4, img_emb_dim=-1, verbose=False, **kwargs):
        super().__init__()
        self._init_scene(xyz_min, xyz_max, bg_len, fast_color_thres, contracted_norm)
        self.verbose = verbose
        self.fourier_freq_num = fourier_freq_num
        self.num_voxels_base_density = num_voxels_base_density
        self.voxel_size_base_density = _cube_root_size(self.xyz_min, self.xyz_max, num_voxels_base_density)
        self.num_voxels_base_rgb = num_voxels_base_rgb
        self.voxel_size_base_rgb = _cube_root_size(self.xyz_min, self.xyz_max, num_voxels_base_rgb)
        self.num_voxels_viewdir = num_voxels_viewdir
        self._set_grid_resolution(num_voxels_density, num_voxels_rgb)
        self.alpha_init = alpha_init
        self.register_buffer('act_shift', torch.FloatTensor([np.log(1 / (1 - alpha_init) - 1)]))
        self.density_type, self.density_config = density_type, density_config
        self.k0_type, self.k0_config = k0_type, k0_config
        self.world_size = self.world_size_density
        self.density = G.FourierGrid(channels=1, world_size=self.world_size_density, xyz_min=self.xyz_min,
                                     xyz_max=self.xyz_max, use_nerf_pos=True, fourier_freq_num=fourier_freq_num,
                                     config=density_config)
        self.rgbnet_kwargs = dict(rgbnet_dim=rgbnet_dim, rgbnet_depth=rgbnet_depth, rgbnet_width=rgbnet_width,
                                  viewbase_pe=viewbase_pe)
        self.sample_num = kwargs.get('sample_num', -1)
        self.img_embeddings, self.img_embed_dim, self.pos_emb = None, 0, None
        if rgbnet_dim <= 0:
            self.k0_dim = 3
            self.k0 = G.FourierGrid(channels=3, world_size=self.world_size_rgb, xyz_min=self.xyz_min,
                                    xyz_max=self.xyz_max, use_nerf_pos=False, fourier_freq_num=fourier_freq_num,
                                    config=k0_config)
            self.rgbnet = None
        else:
            self.k0_dim = rgbnet_dim
            self.k0 = G.FourierGrid(channels=rgbnet_dim, world_size=self.world_size_rgb, xyz_min=self.xyz_min,
                                    xyz_max=self.xyz_max, use_nerf_pos=True, fourier_freq_num=fourier_freq_num,
                                    config=k0_config)
            self._add_rgbnet(rgbnet_dim, viewbase_pe, rgbnet_width, rgbnet_depth)
        self.vd = None      # view-direction grid variant (num_voxels_viewdir > 0) is not on the benchmarked path
        if num_voxels_viewdir is not None and num_voxels_viewdir > 0:
            raise NotImplementedError('num_voxels_viewdir > 0 (view-direction grid) is outside the hot-path scope')
        if mask_cache_world_size is None:
            mask_cache_world_size = self.world_size_density
        self.mask_cache = G.MaskGrid(path=None, mask=torch.ones([int(v) for v in mask_cache_world_size], dtype=torch.bool),
                                     xyz_min=self.xyz_min, xyz_max=self.xyz_max)

    def _set_grid_resolution(self, num_voxels_density, num_voxels_rgb):
        self.num_voxels_density, self.num_voxels_rgb = num_voxels_density, num_voxels_rgb
        self.voxel_size_density = _cube_root_size(self.xyz_min, self.xyz_max, num_voxels_density)
        self.voxel_size_rgb = _cube_root_size(self.xyz_min, self.xyz_max, num_voxels_rgb)
        self.world_size_density = ((self.xyz_max - self.xyz_min) / self.voxel_size_density).long()
        self.world_size_rgb = ((self.xyz_max - self.xyz_min) / self.voxel_size_rgb).long()
        self.world_len_density = self.world_size_density[0].item()
        self.world_len_rgb = self.world_size_rgb[0].item()
        self.voxel_size_ratio_density = self.voxel_size_density / self.voxel_size_base_density
        self.voxel_size_ratio_rgb = self.voxel_size_rgb / self.voxel_size_base_rgb

    def _world_len(self):
        return self.world_len_density

    def _voxel_size(self):
        return self.voxel_size_density

    def _voxel_size_ratio(self):
        return self.voxel_size_ratio_density

    def get_kwargs(self):
        return {
            'xyz_min': self.xyz_min.cpu().numpy(), 'xyz_max': self.xyz_max.cpu().numpy(),
            'num_voxels_density': self.num_voxels_density, 'num_voxels_rgb': self.num_voxels_rgb,
            'num_voxels_viewdir': self.num_voxels_viewdir, 'fourier_freq_num': self.fourier_freq_num,
            'num_voxels_base_density': self.num_voxels_base_density, 'num_voxels_base_rgb': self.num_voxels_base_rgb,
            'alpha_init': self.alpha_init, 'voxel_size_ratio_density': self.voxel_size_ratio_density,
            'voxel_size_ratio_rgb': self.voxel_size_ratio_rgb,
            'mask_cache_world_size': list(self.mask_cache.mask.shape), 'fast_color_thres': self.fast_color_thres,
            'contracted_norm': self.contracted_norm, 'density_type': self.density_type, 'k0_type': self.k0_type,
            'density_config': self.density_config, 'k0_config': self.k0_config, 'sample_num': self.sample_num,
            **self.rgbnet_kwargs,
        }

    @torch.no_grad()
    def scale_volume_grid(self, num_voxels_density, num_voxels_rgb):
        self._set_grid_resolution(num_voxels_density, num_voxels_rgb)
        self.density.scale_volume_grid(self.world_size_density)
        self.k0.scale_volume_grid(self.world_size_rgb)
        self.world_size = self.world_size_density
        if np.prod(self.world_size_density.tolist()) <= 256 ** 3:
            self._rebuild_mask_cache(self.world_size_density, self.density.get_dense_grid())

    @torch.no_grad()
    def maskout_near_cam_vox(self, cam_o, near_clip):
        """FourierGrid_model.py:375-388: density of the grid points closer than near_clip to any camera position (taken in each
        slab's own embedded coordinates gamma_i) is set to -100.  One kernel per slab: every voxel scans the camera list."""
        from . import ops
        dev = self.density.grid.device
        ind_norm = ((cam_o.to(dev) - self.xyz_min) / (self.xyz_max - self.xyz_min)).flip((-1,)) * 2 - 1
        F_ = self.density.nerf_pos_num_freq
        freqs = 2 ** torch.linspace(0, F_ - 1, F_, device=dev)
        emb = [ind_norm] + [f(fr * ind_norm) for fr in freqs for f in (torch.sin, torch.cos)]      # gamma_i of FourierGrid_grid.py:32-36
        for i, cam in enumerate(emb):
            # the reference writes `self.density.grid[0][i][...] = -100` (:388), which for its own [P,1,X,Y,Z] density grid raises an
            # IndexError at i = 1; the evident intent -- slab i, masked in slab i's embedded coordinates -- is grid[i][0]
            ops.maskout_near_cam_(self.density.grid.data[i][0], cam.reshape(-1, 3), near_clip, -100.0)

    def voxel_count_views(self, rays_o_tr, rays_d_tr, imsz, near, far, stepsize, downrate=1, irregular_shape=False):
        """FourierGrid_model.py:390-420 (see _count_views)."""
        return _count_views(self.density, self.world_size_density, self.voxel_size_density, rays_o_tr, rays_d_tr, imsz, near,
                            stepsize, downrate, irregular_shape)

    def update_occupancy_cache_lt_nviews(self, rays_o_tr, rays_d_tr, imsz, render_kwargs, maskout_lt_nviews):
        """FourierGrid_model.py:458-480 (see _ContractedBase.update_occupancy_cache_lt_nviews).  The reference builds its ones grid
        as `FourierGrid_grid.FourierGrid(1, world_size_density, xyz_min, xyz_max)` (:466), which lacks three required arguments
        and raises a TypeError; the evident intent -- a single-slab ones grid over the density lattice -- is what runs here:
        DirectContractedVoxGO's semantics with this model's t schedule (T_BOUNDARY = 1.5)."""
        return super().update_occupancy_cache_lt_nviews(rays_o_tr, rays_d_tr, imsz, render_kwargs, maskout_lt_nviews)

    @torch.no_grad()
    def FourierGrid_get_training_rays(self, rgb_tr_ori, train_poses, HW, Ks, ndc, inverse_y, flip_x, flip_y):
        """FourierGrid_model.py:263-295 -> (rgb_tr, rays_o_tr, rays_d_tr, viewdirs_tr, indexs_tr, imsz): the flattened rays of
        rays.get_training_rays_flatten plus indexs_tr, a float [N, 3] tensor holding each ray's view ordinal in all three
        columns.  pos_emb is always None on this model (:209), so the poses are used as given."""
        from . import rays
        rgb_tr, rays_o_tr, rays_d_tr, viewdirs_tr, imsz = rays.get_training_rays_flatten(
            rgb_tr_ori, train_poses, HW, Ks, ndc, inverse_y, flip_x, flip_y)
        dev = rgb_tr.device
        view = torch.arange(len(imsz), dtype=torch.float32, device=dev).repeat_interleave(torch.tensor(imsz, device=dev))
        indexs_tr = view[:, None].expand(-1, 3).contiguous()
        return rgb_tr, rays_o_tr, rays_d_tr, viewdirs_tr, indexs_tr, imsz

    def gather_training_rays(self, data_dict, images, cfg, i_train, cfg_train, poses, HW, Ks, render_kwargs):
        """FourierGrid_model.py:297-333 -> (rgb_tr, rays_o_tr, rays_d_tr, viewdirs_tr, indexs_train, imsz, batch_index_sampler):
        the training rays of run_train.py's FourierGrid datasets, images kept on the host under load2gpu_on_the_fly."""
        from . import rays
        device = torch.device('cuda' if torch.cuda.is_available() else 'cpu')
        where = 'cpu' if cfg.data.load2gpu_on_the_fly else device
        if data_dict['irregular_shape']:
            rgb_tr_ori = [images[i].to(where) for i in i_train]
        else:
            rgb_tr_ori = images[i_train].to(where)
        views = dict(train_poses=poses[i_train], HW=HW[i_train], Ks=Ks[i_train], ndc=cfg.data.ndc, inverse_y=cfg.data.inverse_y,
                     flip_x=cfg.data.flip_x, flip_y=cfg.data.flip_y)
        indexs_train = None
        if cfg.data.dataset_type in ('waymo', 'mega', 'nerfpp') or cfg.model == 'FourierGrid':
            rgb_tr, rays_o_tr, rays_d_tr, viewdirs_tr, indexs_train, imsz = self.FourierGrid_get_training_rays(
                rgb_tr_ori=rgb_tr_ori, **views)
        elif cfg_train.ray_sampler == 'in_maskcache':
            rgb_tr, rays_o_tr, rays_d_tr, viewdirs_tr, imsz = rays.get_training_rays_in_maskcache_sampling(
                rgb_tr_ori=rgb_tr_ori, model=self, render_kwargs=render_kwargs, **views)
        elif cfg_train.ray_sampler == 'flatten':
            rgb_tr, rays_o_tr, rays_d_tr, viewdirs_tr, imsz = rays.get_training_rays_flatten(rgb_tr_ori=rgb_tr_ori, **views)
        else:
            rgb_tr, rays_o_tr, rays_d_tr, viewdirs_tr, imsz = rays.get_training_rays(rgb_tr=rgb_tr_ori, **views)
        index_generator = rays.batch_indices_generator(len(rgb_tr), cfg_train.N_rand)
        return rgb_tr, rays_o_tr, rays_d_tr, viewdirs_tr, indexs_train, imsz, lambda: next(index_generator)

    @torch.no_grad()
    def export_geometry_for_visualize(self, save_path):
        """FourierGrid_model.py:674-681: npz of alpha = activate_density(density grid) and rgb = sigmoid(k0 grid), slab and channel
        axes as the reference squeezes and permutes them."""
        alpha = self.activate_density(self.density.get_dense_grid()).squeeze().cpu().numpy()
        rgb = torch.sigmoid(self.k0.get_dense_grid()).squeeze().permute(1, 2, 3, 0).cpu().numpy()
        np.savez_compressed(save_path, alpha=alpha, rgb=rgb)

    def sample_ray(self, ori_rays_o, ori_rays_d, stepsize, is_train=False, **render_kwargs):
        """FourierGrid_model.py:509-552 return tuple (ray_pts, indexs, inner_mask, t, rays_d_extend)."""
        ray_pts, inner_mask, t = self._sample_dense(ori_rays_o, ori_rays_d, stepsize)
        return ray_pts, None, inner_mask, t, None

    def forward(self, rays_o, rays_d, viewdirs, global_step=None, is_train=False, **render_kwargs):
        assert len(rays_o.shape) == 2 and rays_o.shape[-1] == 3, 'Only support point queries in [N, 3] format'
        self._maybe_update_thres(global_step)
        if not self._fused_ok():
            return self.forward_ops(rays_o, rays_d, viewdirs, global_step=global_step, is_train=is_train, **render_kwargs)
        N = len(rays_o)
        (weights, alphainv_last, alpha, density, k0, ray_id, step_id, t, inner), t_table = self._march(
            rays_o, rays_d, render_kwargs['stepsize'])
        rgb = self._shade(k0, viewdirs, ray_id)
        return self._finish(N, weights, alphainv_last, density, alpha, rgb, ray_id, step_id, t, t_table.numel(), render_kwargs)

    def forward_ops(self, rays_o, rays_d, viewdirs, global_step=None, is_train=False, **render_kwargs):
        """Op-by-op composition in the reference's order (FourierGrid_model.py:566-672)."""
        N = len(rays_o)
        dev = rays_o.device
        ray_pts, _, inner_mask, t, _ = self.sample_ray(rays_o, rays_d, **render_kwargs)
        n_max = len(t)
        S = n_max
        interval = render_kwargs['stepsize'] * self.voxel_size_ratio_density
        ray_id = torch.arange(N, device=dev).view(-1, 1).expand(N, S).flatten()
        step_id = torch.arange(S, device=dev).view(1, -1).expand(N, S).flatten()
        t = t[None].repeat(N, 1)
        density = self.density(ray_pts)
        alpha = self.activate_density(density, interval)
        if self.fast_color_thres > 0:
            mask = (alpha > self.fast_color_thres)
            ray_pts, inner_mask, t = ray_pts[mask], inner_mask[mask], t[mask]
            ray_id, step_id = ray_id[mask.flatten()], step_id[mask.flatten()]
            density, alpha = density[mask], alpha[mask]
        weights, alphainv_last = Alphas2Weights.apply(alpha.flatten().contiguous(), ray_id.contiguous(), N)
        if self.fast_color_thres > 0:
            mask = (weights > self.fast_color_thres)
            ray_pts, inner_mask, t = ray_pts[mask], inner_mask[mask], t[mask]
            ray_id, step_id = ray_id[mask], step_id[mask]
            density, alpha, weights = density[mask], alpha[mask], weights[mask]
        else:
            ray_pts = ray_pts.reshape(-1, 3)
            inner_mask = inner_mask.reshape(-1)
            t, density, alpha = t.reshape(-1), density.reshape(-1), alpha.reshape(-1)
        k0 = self.k0(ray_pts)
        rgb = self._shade(k0, viewdirs, ray_id)
        return self._finish(N, weights, alphainv_last, density, alpha, rgb, ray_id, step_id, t, n_max, render_kwargs)

    def _finish(self, N, weights, alphainv_last, density, alpha, rgb, ray_id, step_id, t, n_max, render_kwargs):
        rgb_marched = composite_rgb(weights, rgb, ray_id, N)
        if render_kwargs.get('rand_bkgd', False):           # FourierGrid_model.py:646: a random background only, never bg
            rgb_marched = rgb_marched + alphainv_last.unsqueeze(-1) * torch.rand_like(rgb_marched)
        s = 1 - 1 / (1 + t)
        ret = {'alphainv_last': alphainv_last, 'weights': weights, 'rgb_marched': rgb_marched, 'raw_density': density,
               'raw_alpha': alpha, 'raw_rgb': rgb, 'ray_id': ray_id, 'step_id': step_id, 'n_max': n_max, 't': t, 's': s}
        if render_kwargs.get('render_depth', False):
            with torch.no_grad():
                ret['depth'] = segment_sum(weights * s, ray_id, N)
        return ret


# ======================================================================================================
class DirectContractedVoxGO(_ContractedBase):
    """FourierGrid/dcvgo.py:28-384 (DVGOv2 unbounded model): DenseGrid density/k0, cumdist_thres oversampling
    filter, mask cache, constant / random background term, wsum_mid."""

    T_BOUNDARY = 2.0
    USE_CUMDIST = True
    USE_MASKCACHE = True
    RENDER_USES_BG = True

    def __init__(self, xyz_min, xyz_max, num_voxels=0, num_voxels_base=0, alpha_init=None, mask_cache_world_size=None,
                 fast_color_thres=0, bg_len=0.2, contracted_norm='inf', density_type='DenseGrid', k0_type='DenseGrid',
                 density_config={}, k0_config={}, rgbnet_dim=0, rgbnet_depth=3, rgbnet_width=128, viewbase_pe=4, **kwargs):
        super().__init__()
        self._init_scene(xyz_min, xyz_max, bg_len, fast_color_thres, contracted_norm)
        self.num_voxels_base = num_voxels_base
        self.voxel_size_base = _cube_root_size(self.xyz_min, self.xyz_max, num_voxels_base)
        self._set_grid_resolution(num_voxels)
        self.alpha_init = alpha_init
        self.register_buffer('act_shift', torch.FloatTensor([np.log(1 / (1 - alpha_init) - 1)]))
        self.density_type, self.density_config = density_type, density_config
        self.k0_type, self.k0_config = k0_type, k0_config
        if density_type != 'DenseGrid' or k0_type != 'DenseGrid':
            raise NotImplementedError('only DenseGrid is on the hot path (TensoRFGrid is out of scope, SURVEY.md 2 #6)')
        self.density = G.DenseGrid(channels=1, world_size=self.world_size, xyz_min=self.xyz_min, xyz_max=self.xyz_max)
        self.rgbnet_kwargs = dict(rgbnet_dim=rgbnet_dim, rgbnet_depth=rgbnet_depth, rgbnet_width=rgbnet_width,
                                  viewbase_pe=viewbase_pe)
        if rgbnet_dim <= 0:
            self.k0_dim = 3
            self.rgbnet = None
        else:
            self.k0_dim = rgbnet_dim
            self._add_rgbnet(rgbnet_dim, viewbase_pe, rgbnet_width, rgbnet_depth)
        self.k0 = G.DenseGrid(channels=self.k0_dim, world_size=self.world_size, xyz_min=self.xyz_min, xyz_max=self.xyz_max)
        if mask_cache_world_size is None:
            mask_cache_world_size = self.world_size
        self.mask_cache = G.MaskGrid(path=None, mask=torch.ones([int(v) for v in mask_cache_world_size], dtype=torch.bool),
                                     xyz_min=self.xyz_min, xyz_max=self.xyz_max)

    def _set_grid_resolution(self, num_voxels):
        self.num_voxels = num_voxels
        self.voxel_size = _cube_root_size(self.xyz_min, self.xyz_max, num_voxels)
        self.world_size = ((self.xyz_max - self.xyz_min) / self.voxel_size).long()
        self.world_len = self.world_size[0].item()
        self.voxel_size_ratio = self.voxel_size / self.voxel_size_base

    def _world_len(self):
        return self.world_len

    def get_kwargs(self):
        return {
            'xyz_min': self.xyz_min.cpu().numpy(), 'xyz_max': self.xyz_max.cpu().numpy(),
            'num_voxels': self.num_voxels, 'num_voxels_base': self.num_voxels_base, 'alpha_init': self.alpha_init,
            'voxel_size_ratio': self.voxel_size_ratio, 'mask_cache_world_size': list(self.mask_cache.mask.shape),
            'fast_color_thres': self.fast_color_thres, 'contracted_norm': self.contracted_norm,
            'density_type': self.density_type, 'k0_type': self.k0_type, 'density_config': self.density_config,
            'k0_config': self.k0_config, **self.rgbnet_kwargs,
        }

    def scale_volume_grid(self, num_voxels):
        _scale_dense_model(self, num_voxels)

    def sample_ray(self, ori_rays_o, ori_rays_d, stepsize, is_train=False, **render_kwargs):
        """dcvgo.py:228-262 return tuple (ray_pts, inner_mask, t)."""
        return self._sample_dense(ori_rays_o, ori_rays_d, stepsize)

    def _finish(self, N, dev, weights, alphainv_last, density, alpha, rgb, ray_id, step_id, t, inner_mask, n_max,
                is_train, render_kwargs):
        rgb_marched = composite_rgb(weights, rgb, ray_id, N)
        if render_kwargs.get('rand_bkgd', False) and is_train:
            rgb_marched = rgb_marched + alphainv_last.unsqueeze(-1) * torch.rand_like(rgb_marched)
        else:
            rgb_marched = rgb_marched + alphainv_last.unsqueeze(-1) * render_kwargs['bg']
        wsum_mid = segment_sum(weights[inner_mask], ray_id[inner_mask], N)
        s = 1 - 1 / (1 + t)
        ret = {'alphainv_last': alphainv_last, 'weights': weights, 'wsum_mid': wsum_mid, 'rgb_marched': rgb_marched,
               'raw_density': density, 'raw_alpha': alpha, 'raw_rgb': rgb, 'ray_id': ray_id, 'step_id': step_id,
               'n_max': n_max, 't': t, 's': s}
        if render_kwargs.get('render_depth', False):
            with torch.no_grad():
                ret['depth'] = segment_sum(weights * s, ray_id, N)
        return ret

    def forward(self, rays_o, rays_d, viewdirs, global_step=None, is_train=False, **render_kwargs):
        assert len(rays_o.shape) == 2 and rays_o.shape[-1] == 3, 'Only support point queries in [N, 3] format'
        self._maybe_update_thres(global_step)
        if not self._fused_ok():
            return self.forward_ops(rays_o, rays_d, viewdirs, global_step=global_step, is_train=is_train, **render_kwargs)
        N = len(rays_o)
        # render_kwargs['coherent_rays'] (set by render.render_rays: a frame's image-ordered chunks) selects the TMA-staged
        # feature read; it is a hint, never a requirement -- any rays give the same result
        (weights, alphainv_last, alpha, density, k0, ray_id, step_id, t, inner), t_table = self._march(
            rays_o, rays_d, render_kwargs['stepsize'], coherent=bool(render_kwargs.get('coherent_rays', False)))
        rgb = self._shade(k0, viewdirs, ray_id)
        return self._finish(N, rays_o.device, weights, alphainv_last, density, alpha, rgb, ray_id, step_id, t, inner,
                            t_table.numel(), is_train, render_kwargs)

    def forward_ops(self, rays_o, rays_d, viewdirs, global_step=None, is_train=False, **render_kwargs):
        """Op-by-op composition in the reference's order (dcvgo.py:275-384)."""
        from . import ops
        N = len(rays_o)
        dev = rays_o.device
        ray_pts, inner_mask, t = self.sample_ray(rays_o, rays_d, is_train=global_step is not None, **render_kwargs)
        n_max = len(t)
        S = n_max
        interval = render_kwargs['stepsize'] * self.voxel_size_ratio
        ray_id = torch.arange(N, device=dev).view(-1, 1).expand(N, S).flatten()
        step_id = torch.arange(S, device=dev).view(1, -1).expand(N, S).flatten()
        mask = inner_mask.clone()
        dist_thres = (2 + 2 * self.bg_len) / self.world_len * render_kwargs['stepsize'] * 0.95
        dist = (ray_pts[:, 1:] - ray_pts[:, :-1]).norm(dim=-1)
        mask[:, 1:] |= ops.cumdist_thres(dist.contiguous(), dist_thres)
        ray_pts, inner_mask = ray_pts[mask], inner_mask[mask]
        t = t[None].repeat(N, 1)[mask]
        ray_id, step_id = ray_id[mask.flatten()], step_id[mask.flatten()]
        mask = self.mask_cache(ray_pts)
        ray_pts, inner_mask, t, ray_id, step_id = ray_pts[mask], inner_mask[mask], t[mask], ray_id[mask], step_id[mask]
        density = self.density(ray_pts)
        alpha = self.activate_density(density, interval)
        if self.fast_color_thres > 0:
            mask = (alpha > self.fast_color_thres)
            ray_pts, inner_mask, t, ray_id, step_id = ray_pts[mask], inner_mask[mask], t[mask], ray_id[mask], step_id[mask]
            density, alpha = density[mask], alpha[mask]
        weights, alphainv_last = Alphas2Weights.apply(alpha.contiguous(), ray_id.contiguous(), N)
        if self.fast_color_thres > 0:
            mask = (weights > self.fast_color_thres)
            ray_pts, inner_mask, t, ray_id, step_id = ray_pts[mask], inner_mask[mask], t[mask], ray_id[mask], step_id[mask]
            density, alpha, weights = density[mask], alpha[mask], weights[mask]
        k0 = self.k0(ray_pts)
        rgb = self._shade(k0, viewdirs, ray_id)
        return self._finish(N, dev, weights, alphainv_last, density, alpha, rgb, ray_id, step_id, t, inner_mask, n_max,
                            is_train, render_kwargs)


# ======================================================================================================
class DirectVoxGO(_CoarseGeo, _GridModel):
    """Bounded-scene model (FourierGrid/dvgo.py:26-425): ragged AABB sampling (sample_pts_on_rays) instead of the contracted
    schedule; depth = sum w * step_id.  ``forward`` runs the fused box march (march.BoxMarch: pass A, scan, pass B; one host read
    of the survivor count) with the rgb from ``_shade`` -- the tensor-core rgbnet when shade.supported (the default fine config:
    rgbnet_dim 12, rgbnet_direct, width 128) -- for a single-slab density and a 3- or 12-channel channels-last k0.  With
    rgbnet_direct=False the march is fused and the torch epilogue sigmoid(rgbnet(cat[k0[:, 3:], emb]) + k0[:, :3]) stays.
    ``forward_ops`` composes the drop-in ops in the reference's order (the cross-check and the path for other grids).  With a
    TensoRFGrid density or k0 (``density_type`` / ``k0_type``, built through ``grid.create_grid`` as dvgo.py does) ``forward`` runs
    the same fused box march (march.BoxTensorfMarch) in all three pairings: pass A reads a TensoRF density's factors (or the
    dense grid), pass B writes the survivor points, and the k0 reads them with its own forward.  Its outputs are bit-identical
    to that composition on the TensoRF kernels shaded with ``_shade``, which stays the route where the march does not apply
    (R + R + Rxy > 96, S_max beyond the march's bound, host tensors).

    The coarse-to-fine schedule of run_train.py works: maskout_near_cam_vox, voxel_count_views (per-voxel lr), scale_volume_grid,
    update_occupancy_cache, and ``mask_cache_path``.  The latter builds the fine mask as the reference does (dvgo.py:138-152):
    MaskGrid(path, mask_cache_thres) looked up on this model's linspace(xyz_min, xyz_max, mask_cache_world_size) lattice.  The
    lookup is a CUDA kernel, so a model built on the host (run_train.create_new_model constructs, then calls .to(device)) resolves
    it when it first moves to a CUDA device; a state dict that carries ``mask_cache.mask`` (a checkpoint of the fine model)
    supersedes it, so ckpt.load_model never reads the coarse file."""

    def __init__(self, xyz_min, xyz_max, num_voxels=0, num_voxels_base=0, alpha_init=None, mask_cache_path=None,
                 mask_cache_thres=1e-3, mask_cache_world_size=None, fast_color_thres=0, density_type='DenseGrid',
                 k0_type='DenseGrid', density_config={}, k0_config={}, rgbnet_dim=0, rgbnet_direct=False,
                 rgbnet_full_implicit=False, rgbnet_depth=3, rgbnet_width=128, viewbase_pe=4, **kwargs):
        super().__init__()
        if rgbnet_full_implicit:
            raise NotImplementedError('rgbnet_full_implicit is outside the hot-path scope')
        self.register_buffer('xyz_min', torch.as_tensor(_host_array(xyz_min), dtype=torch.float32))
        self.register_buffer('xyz_max', torch.as_tensor(_host_array(xyz_max), dtype=torch.float32))
        self.fast_color_thres = fast_color_thres
        self.num_voxels_base = num_voxels_base
        self.voxel_size_base = _cube_root_size(self.xyz_min, self.xyz_max, num_voxels_base)
        self.alpha_init = alpha_init
        self.register_buffer('act_shift', torch.FloatTensor([np.log(1 / (1 - alpha_init) - 1)]))
        self._set_grid_resolution(num_voxels)
        self.density_type, self.density_config, self.k0_type, self.k0_config = density_type, density_config, k0_type, k0_config
        self.density = G.create_grid(density_type, channels=1, world_size=self.world_size, xyz_min=self.xyz_min,
                                     xyz_max=self.xyz_max, config=self.density_config)
        self.rgbnet_kwargs = dict(rgbnet_dim=rgbnet_dim, rgbnet_direct=rgbnet_direct, rgbnet_full_implicit=rgbnet_full_implicit,
                                  rgbnet_depth=rgbnet_depth, rgbnet_width=rgbnet_width, viewbase_pe=viewbase_pe)
        self.rgbnet_direct = rgbnet_direct
        if rgbnet_dim <= 0:
            self.k0_dim, self.rgbnet = 3, None
        else:
            self.k0_dim = rgbnet_dim
            self._add_rgbnet(rgbnet_dim if rgbnet_direct else rgbnet_dim - 3, viewbase_pe, rgbnet_width, rgbnet_depth)
        self.k0 = G.create_grid(k0_type, channels=self.k0_dim, world_size=self.world_size, xyz_min=self.xyz_min,
                                xyz_max=self.xyz_max, config=self.k0_config)
        self.mask_cache_path, self.mask_cache_thres = mask_cache_path, mask_cache_thres
        if mask_cache_world_size is None:
            mask_cache_world_size = self.world_size
        self._pending_mask = None
        self.mask_cache = G.MaskGrid(path=None, mask=torch.ones([int(v) for v in mask_cache_world_size], dtype=torch.bool),
                                     xyz_min=self.xyz_min, xyz_max=self.xyz_max)
        if mask_cache_path:
            self._pending_mask = (mask_cache_path, mask_cache_thres, [int(v) for v in mask_cache_world_size])
            if self.xyz_min.is_cuda:
                self._resolve_mask_cache()

    # ---- the coarse-checkpoint mask cache (dvgo.py:138-152) ----------------------------------------------------------------
    @torch.no_grad()
    def _resolve_mask_cache(self):
        path, thres, ws = self._pending_mask
        coarse = G.MaskGrid(path=path, mask_cache_thres=thres).to(self.xyz_min.device)
        self._set_mask_cache(coarse(self._mask_lattice(ws)))
        self._pending_mask = None

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        if self._pending_mask is not None and self.xyz_min.is_cuda:
            self._resolve_mask_cache()
        return out

    def _load_from_state_dict(self, state_dict, prefix, *a, **k):
        if prefix + 'mask_cache.mask' in state_dict:
            self._pending_mask = None
        return super()._load_from_state_dict(state_dict, prefix, *a, **k)

    def _set_grid_resolution(self, num_voxels):
        self.num_voxels = num_voxels
        self.voxel_size = _cube_root_size(self.xyz_min, self.xyz_max, num_voxels)
        self.world_size = ((self.xyz_max - self.xyz_min) / self.voxel_size).long()
        self.voxel_size_ratio = self.voxel_size / self.voxel_size_base

    def get_kwargs(self):
        return {
            'xyz_min': self.xyz_min.cpu().numpy(), 'xyz_max': self.xyz_max.cpu().numpy(), 'num_voxels': self.num_voxels,
            'num_voxels_base': self.num_voxels_base, 'alpha_init': self.alpha_init, 'voxel_size_ratio': self.voxel_size_ratio,
            'mask_cache_path': self.mask_cache_path, 'mask_cache_thres': self.mask_cache_thres,
            'mask_cache_world_size': list(self.mask_cache.mask.shape), 'fast_color_thres': self.fast_color_thres,
            'density_type': self.density_type, 'k0_type': self.k0_type, 'density_config': self.density_config,
            'k0_config': self.k0_config, **self.rgbnet_kwargs,
        }

    # ---- grid maintenance (run_train.py's coarse and fine stages) -------------------------------------------------------------
    def scale_volume_grid(self, num_voxels):
        """dvgo.py:213-234 (the pg_scale steps of the fine stage)."""
        _scale_dense_model(self, num_voxels)

    def voxel_count_views(self, rays_o_tr, rays_d_tr, imsz, near, far, stepsize, downrate=1, irregular_shape=False):
        """dvgo.py:248-277 (see _count_views): feeds MaskedAdam.set_pervoxel_lr and the coarse stage's mask update."""
        return _count_views(self.density, self.world_size, self.voxel_size, rays_o_tr, rays_d_tr, imsz, near, stepsize, downrate,
                            irregular_shape)

    @torch.no_grad()
    def update_occupancy_cache(self):
        """dvgo.py:236-245.  A TensoRF density is read at the mask lattice through its own forward, then pooled and ANDed as for
        the dense grids."""
        if not self._tensorf():
            return super().update_occupancy_cache()
        from . import ops
        density = self.density(self._mask_lattice(self.mask_cache.mask.shape))
        alpha = self.activate_density(density).contiguous()
        ops.maxpool3_gt_and_(self.mask_cache.mask, alpha, self.fast_color_thres)

    @torch.no_grad()
    def maskout_near_cam_vox(self, cam_o, near_clip):
        """dvgo.py:185-198: density = -100 at the points of the world lattice linspace(xyz_min, xyz_max, world_size) that are
        within near_clip of a camera position (one kernel: every voxel scans the camera list)."""
        from . import ops
        if isinstance(self.density, G.TensoRFGrid):
            # dvgo.py:197 writes density.grid, which a TensoRFGrid does not have (the reference fails there as well); the
            # shipped TensoRF config runs it only in the DenseGrid coarse stage
            raise NotImplementedError('maskout_near_cam_vox needs a DenseGrid density (a TensoRFGrid has no voxel lattice)')
        lo, hi = self.xyz_min.cpu().tolist(), self.xyz_max.cpu().tolist()
        cams = cam_o.to(self.density.grid.device).reshape(-1, 3)
        ops.maskout_near_cam_(self.density.grid.data[0][0], cams, near_clip, -100.0, lattice=(lo, hi))

    def _tv_weights(self, grid, weight, dense_mode):
        w = weight * float(self.world_size.max()) / 128          # dvgo.py: the model's world size, for both grids
        return (w, w, w, dense_mode)

    def sample_ray(self, rays_o, rays_d, near, far, stepsize, **render_kwargs):
        """dvgo.py:306-328."""
        from . import ops
        far = 1e9
        stepdist = stepsize * float(self.voxel_size)
        ray_pts, mask_outbbox, ray_id, step_id, N_steps, t_min, t_max = ops.sample_pts_on_rays(
            rays_o.contiguous(), rays_d.contiguous(), self.xyz_min, self.xyz_max, near, far, stepdist)
        mask_inbbox = ~mask_outbbox
        return ray_pts[mask_inbbox], ray_id[mask_inbbox], step_id[mask_inbbox]

    # ---- rendering ------------------------------------------------------------------------------------------------------------
    def _stepdist(self, stepsize):
        # what sample_ray hands ubn_sample_pts_* (the same fp32 value reaches the march); host_scalar caches the read per tensor,
        # so a device-side voxel_size (after scale_volume_grid on a CUDA model) costs one sync per rescale, not per step
        return stepsize * host_scalar(self.voxel_size)

    def _tensorf(self):
        return isinstance(self.density, G.TensoRFGrid) or isinstance(self.k0, G.TensoRFGrid)

    def _fused_ok(self, stepsize):
        tf_d, tf_k = isinstance(self.density, G.TensoRFGrid), isinstance(self.k0, G.TensoRFGrid)
        d_ok = march.tensorf_supported(self.density.factors()) if tf_d else march.box_density_supported(self.density.grid)
        # a TensoRF model's k0 reads the survivor points with its own forward: any DenseGrid k0 will do next to a TensoRF density
        k_ok = march.tensorf_supported(self.k0.factors()) if tf_k else (tf_d or march.box_k0_supported(self.k0.grid))
        if not (d_ok and k_ok):
            return False
        lo, hi = self._host()
        return march.box_s_max(lo, hi, self._stepdist(stepsize)) <= march.BOX_S_MAX_LIMIT

    def _mask_geometry(self):
        """(mask_scale, mask_shift, xyz_min, xyz_max) as host lists: all the box march cfg takes by value."""
        return (*super()._mask_geometry(), *self._host())

    def forward(self, rays_o, rays_d, viewdirs, global_step=None, **render_kwargs):
        """dvgo.py:330-397 on the fused box march (see the class docstring); same keys as the reference's ret_dict."""
        assert len(rays_o.shape) == 2 and rays_o.shape[-1] == 3, 'Only suuport point queries in [N, 3] format'
        stepsize = render_kwargs['stepsize']
        if not (rays_o.is_cuda and self._fused_ok(stepsize)):
            if self._tensorf():     # the op-by-op composition on the TensoRF kernels, shaded as the march is
                return self._compose(rays_o, rays_d, viewdirs, self._shade_k0, render_kwargs)
            return self.forward_ops(rays_o, rays_d, viewdirs, global_step=global_step, **render_kwargs)
        N = len(rays_o)
        cfg = self._box_cfg(render_kwargs)
        if self._tensorf():
            weights, alphainv_last, alpha, k0, ray_id, step_id = self._march_tensorf(rays_o, rays_d, cfg)
        else:
            ddesc = G.grid_desc(self.density.grid, *self.density._bounds(), 0)
            kdesc = G.grid_desc(self.k0.grid, *self.k0._bounds(), 0)
            weights, alphainv_last, alpha, k0, ray_id, step_id = march.BoxMarch.apply(
                self.density.grid, self.k0.grid, rays_o, rays_d, self.mask_cache.mask, cfg, ddesc, kdesc)
        rgb = self._shade_k0(k0, viewdirs, ray_id)
        return self._finish(N, weights, alphainv_last, alpha, rgb, ray_id, step_id, render_kwargs)

    def _box_cfg(self, render_kwargs):
        """The box march cfg of forward and render_fused (a pending coarse mask cache resolved first): the bbox, near, the step
        length, act_shift, interval = stepsize * voxel_size_ratio, the threshold and the mask cache's geometry."""
        if self._pending_mask is not None:
            self._resolve_mask_cache()
        stepsize = render_kwargs['stepsize']
        mscale, mshift, lo, hi = self._mask_geometry()
        return march.make_box_cfg(lo, hi, render_kwargs['near'], self._stepdist(stepsize), host_scalar(self.act_shift),
                                  stepsize * host_scalar(self.voxel_size_ratio), self.fast_color_thres, self.mask_cache.mask,
                                  mscale, mshift)

    # ---- the fused render -----------------------------------------------------------------------------------------------------
    FUSED_FRAME_BY_DEFAULT = False     # render.render_rays takes render_fused only with fused_frame=True (DESIGN.md §7)
    RENDER_NETS = ((12, 4, 128), (9, 4, 64))      # (k0 channels, viewbase_pe, width) of csrc/render_bounded.cu's box kernels

    def render_fused_ok(self, rays_o, render_kwargs):
        """Whether render_fused covers this model and call (render.render_rays with fused_frame=True takes it exactly then): no
        gradient, CUDA rays, DenseGrid density and k0 where forward's fused box march applies (a contiguous one-slab density, a
        channels-last k0 of 12, 9 or 3 channels; no TensoRFGrid), an rgbnet_direct rgbnet with (rgbnet_dim, viewbase_pe, width) =
        (12, 4, 128) (the fine stage) or (9, 4, 64), or none with a 3-channel k0 (sigmoid(k0), the coarse stage), and a numeric
        bg."""
        if self._tensorf() or not self._render_grids_ok(rays_o, render_kwargs) or 'stepsize' not in render_kwargs:
            return False
        if not self._fused_ok(render_kwargs['stepsize']):
            return False
        if self.rgbnet is not None and not self.rgbnet_direct:
            return False
        return self._render_net_ok(self.k0.grid.shape[1], self.RENDER_NETS)

    @torch.no_grad()
    def render_fused(self, rays_o, rays_d, viewdirs, n_shaded=None, n_marched=None, **render_kwargs):
        """{'rgb_marched' [N,3], 'depth' [N], 'alphainv_last' [N]} of N rays in one launch (csrc/render_bounded.cu): the box
        march, the k0 read of the kept samples, the rgbnet and the composite with no per-sample buffers, so a whole frame is one
        call.  Same kept samples and alphainv_last (bit for bit) as forward; rgb_marched (+ alphainv_last * bg) and depth (sum of
        w * step_id) as forward's composite, summed in step order.  A ray needing more than the cfg's S_max steps raises as
        forward does.  n_shaded / n_marched: optional int32 [N] that receive each ray's kept samples / the samples of the
        32-sample chunks marched before the ray stopped.  Only where render_fused_ok holds."""
        from . import _cabi
        from ._cabi import c_f, c_i64, c_int, check, ptr, stream_of
        N = rays_o.shape[0]
        dev = rays_o.device
        rays_o = rays_o.contiguous().float()
        rays_d = rays_d.contiguous().float()
        viewdirs = viewdirs.contiguous().float()
        rgb = torch.empty(N, 3, dtype=torch.float32, device=dev)
        depth = torch.empty(N, dtype=torch.float32, device=dev)
        last = torch.empty(N, dtype=torch.float32, device=dev)
        over = torch.zeros(1, dtype=torch.int32, device=dev)
        cfg = self._box_cfg(render_kwargs)
        ddesc = G.grid_desc(self.density.grid, *self.density._bounds(), 0)
        kdesc = G.grid_desc(self.k0.grid, *self.k0._bounds(), 0)
        net, width, pe = self._render_net_args()
        with _cabi.timed('render_box'):
            check(_cabi.load().ubn_render_box(
                ptr(rays_o), ptr(rays_d), ptr(viewdirs), ptr(self.density.grid), ddesc, ptr(self.k0.grid), kdesc,
                ptr(self.mask_cache.mask), cfg, c_i64(N), *map(ptr, net), c_int(width), c_int(pe), c_f(float(render_kwargs['bg'])),
                ptr(rgb), ptr(depth), ptr(last), ptr(n_shaded), ptr(n_marched), ptr(over), stream_of(rgb)))
        if N > 0 and int(over.item()):
            raise RuntimeError(f'box march: a ray needs more than s_max = {cfg.s_max} steps (bbox / stepsize / ray origin out of '
                               'range)')
        return {'rgb_marched': rgb, 'depth': depth, 'alphainv_last': last}

    def _march_tensorf(self, rays_o, rays_d, cfg):
        """march.BoxTensorfMarch: a TensoRF density is read in pass A; the k0 (TensoRFGrid or DenseGrid) reads the survivor
        points pass B writes with its own forward and autograd -- the very read _compose runs on the same points."""
        if isinstance(self.density, G.TensoRFGrid):
            density = self.density.factors()
            ddesc = G.tensorf_desc(density, 1, *self.density._bounds())
        else:
            density = [self.density.grid]
            ddesc = G.grid_desc(self.density.grid, *self.density._bounds(), 0)
        weights, alphainv_last, alpha, points, ray_id, step_id = march.BoxTensorfMarch.apply(
            rays_o, rays_d, self.mask_cache.mask, cfg, ddesc, isinstance(self.density, G.TensoRFGrid), G.TENSORF_VEC_COPIES,
            *density)
        return weights, alphainv_last, alpha, self.k0(points), ray_id, step_id

    def _shade_k0(self, k0, viewdirs, ray_id):
        """rgb of the samples as forward computes it: _shade (the tensor-core rgbnet where shade.supported); with
        rgbnet_direct=False the torch epilogue sigmoid(rgbnet(cat[k0[:, 3:], emb]) + k0[:, :3])."""
        if self.rgbnet is None or self.rgbnet_direct:
            return self._shade(k0, viewdirs, ray_id)
        emb = _view_embed(viewdirs, self.viewfreq).flatten(0, -2)[ray_id]
        return torch.sigmoid(self.rgbnet(torch.cat([k0[:, 3:], emb], -1)) + k0[:, :3])

    def _shade_torch(self, k0, viewdirs, ray_id):
        """rgb of the samples with the rgbnet in torch, as dvgo.py:373-397 writes it."""
        if self.rgbnet is None:
            return torch.sigmoid(k0)
        k0_view = k0 if self.rgbnet_direct else k0[:, 3:]
        emb = _view_embed(viewdirs, self.viewfreq).flatten(0, -2)[ray_id]
        logit = self.rgbnet(torch.cat([k0_view, emb], -1))
        return torch.sigmoid(logit if self.rgbnet_direct else logit + k0[:, :3])

    def forward_ops(self, rays_o, rays_d, viewdirs, global_step=None, **render_kwargs):
        """Op-by-op composition in the reference's order (dvgo.py:330-397): ragged sample_pts_on_rays, boolean-mask compactions,
        grid reads with their autograd, the rgbnet in torch."""
        assert len(rays_o.shape) == 2 and rays_o.shape[-1] == 3, 'Only suuport point queries in [N, 3] format'
        return self._compose(rays_o, rays_d, viewdirs, self._shade_torch, render_kwargs)

    def _compose(self, rays_o, rays_d, viewdirs, shade, render_kwargs):
        """The body of forward_ops with the shading step ``shade(k0, viewdirs, ray_id) -> rgb`` as a parameter."""
        N, dev = len(rays_o), rays_o.device
        ray_pts, ray_id, step_id = self.sample_ray(rays_o=rays_o, rays_d=rays_d, **render_kwargs)
        interval = render_kwargs['stepsize'] * self.voxel_size_ratio
        if self.mask_cache is not None:
            mask = self.mask_cache(ray_pts)
            ray_pts, ray_id, step_id = ray_pts[mask], ray_id[mask], step_id[mask]
        density = self.density(ray_pts)
        alpha = self.activate_density(density, interval)
        if self.fast_color_thres > 0:
            mask = (alpha > self.fast_color_thres)
            ray_pts, ray_id, step_id, density, alpha = ray_pts[mask], ray_id[mask], step_id[mask], density[mask], alpha[mask]
        weights, alphainv_last = Alphas2Weights.apply(alpha.contiguous(), ray_id.contiguous(), N)
        if self.fast_color_thres > 0:
            mask = (weights > self.fast_color_thres)
            weights, alpha, ray_pts, ray_id, step_id = weights[mask], alpha[mask], ray_pts[mask], ray_id[mask], step_id[mask]
        k0 = self.k0(ray_pts)
        rgb = shade(k0, viewdirs, ray_id)
        return self._finish(N, weights, alphainv_last, alpha, rgb, ray_id, step_id, render_kwargs)

    def _finish(self, N, weights, alphainv_last, alpha, rgb, ray_id, step_id, render_kwargs):
        rgb_marched = composite_rgb(weights, rgb, ray_id, N)
        rgb_marched = rgb_marched + alphainv_last.unsqueeze(-1) * render_kwargs['bg']       # dvgo.py:406: always bg
        ret = {'alphainv_last': alphainv_last, 'weights': weights, 'rgb_marched': rgb_marched, 'raw_alpha': alpha,
               'raw_rgb': rgb, 'ray_id': ray_id}
        if render_kwargs.get('render_depth', False):
            with torch.no_grad():
                ret['depth'] = segment_sum(weights * step_id, ray_id, N)
        return ret


# ======================================================================================================
class DirectMPIGO(_GridModel):
    """Forward-facing model in NDC space (FourierGrid/dmpigo.py:18-340): a DenseGrid density with a frozen per-plane bias
    ``act_shift`` ([1,1,1,1,mpi_depth] DenseGrid), a DenseGrid k0 (3 channels, or rgbnet_dim features + rgbnet), a mask cache,
    NDC samples o + d * i/(S-1) inside the bbox.  ``forward`` runs the fused NDC march (march.NdcMarch); ``forward_ops``
    composes the drop-in ops in the reference's order."""

    def __init__(self, xyz_min, xyz_max, num_voxels=0, mpi_depth=0, mask_cache_path=None, mask_cache_thres=1e-3,
                 mask_cache_world_size=None, fast_color_thres=0, density_type='DenseGrid', k0_type='DenseGrid',
                 density_config={}, k0_config={}, rgbnet_dim=0, rgbnet_depth=3, rgbnet_width=128, viewbase_pe=0, **kwargs):
        super().__init__()
        if density_type != 'DenseGrid' or k0_type != 'DenseGrid':
            raise NotImplementedError('only DenseGrid is on the hot path (TensoRFGrid is out of scope)')
        self.register_buffer('xyz_min', torch.as_tensor(_host_array(xyz_min), dtype=torch.float32).clone())
        self.register_buffer('xyz_max', torch.as_tensor(_host_array(xyz_max), dtype=torch.float32).clone())
        self.fast_color_thres = fast_color_thres
        self._set_grid_resolution(num_voxels, mpi_depth)
        self.density_type, self.density_config = density_type, density_config
        self.density = G.DenseGrid(channels=1, world_size=self.world_size, xyz_min=self.xyz_min, xyz_max=self.xyz_max)
        # initial bias: every plane contributes the same alpha to a ray crossing all of them (dmpigo.py:45-57)
        self.act_shift = G.DenseGrid(channels=1, world_size=[1, 1, mpi_depth], xyz_min=xyz_min, xyz_max=xyz_max)
        self.act_shift.grid.requires_grad = False
        with torch.no_grad():
            g = np.full([mpi_depth], 1. / mpi_depth - 1e-6)
            p = [1 - g[0]]
            for i in range(1, len(g)):
                p.append((1 - g[:i + 1].sum()) / (1 - g[:i].sum()))
            for i in range(len(p)):
                self.act_shift.grid[..., i].fill_(np.log(p[i] ** (-1 / self.voxel_size_ratio) - 1))
        self.rgbnet_kwargs = dict(rgbnet_dim=rgbnet_dim, rgbnet_depth=rgbnet_depth, rgbnet_width=rgbnet_width,
                                  viewbase_pe=viewbase_pe)
        self.k0_type, self.k0_config = k0_type, k0_config
        if rgbnet_dim <= 0:
            self.k0_dim, self.rgbnet = 3, None
            self.k0 = G.DenseGrid(channels=3, world_size=self.world_size, xyz_min=self.xyz_min, xyz_max=self.xyz_max)
        else:
            self.k0_dim = rgbnet_dim
            self.k0 = G.DenseGrid(channels=rgbnet_dim, world_size=self.world_size, xyz_min=self.xyz_min, xyz_max=self.xyz_max)
            self._add_rgbnet(rgbnet_dim, viewbase_pe, rgbnet_width, rgbnet_depth)
        self.mask_cache_path, self.mask_cache_thres = mask_cache_path, mask_cache_thres
        if mask_cache_world_size is None:
            mask_cache_world_size = self.world_size
        if mask_cache_path:
            raise NotImplementedError('coarse-checkpoint mask cache needs a device at construction; build MaskGrid(path=...) '
                                      'and assign model.mask_cache instead')
        self.mask_cache = G.MaskGrid(path=None, mask=torch.ones([int(v) for v in mask_cache_world_size], dtype=torch.bool),
                                     xyz_min=self.xyz_min, xyz_max=self.xyz_max)

    def _set_grid_resolution(self, num_voxels, mpi_depth):
        """dmpigo.py:120-130: X, Y from the voxel budget per plane (fp32 sqrt, truncated to long), Z = mpi_depth."""
        self.num_voxels = num_voxels
        self.mpi_depth = mpi_depth
        mn, mx = self.xyz_min.cpu(), self.xyz_max.cpu()
        r = (num_voxels / self.mpi_depth / (mx - mn)[:2].prod()).sqrt()
        self.world_size = torch.zeros(3, dtype=torch.long)
        self.world_size[:2] = (mx - mn)[:2] * r
        self.world_size[2] = self.mpi_depth
        self.voxel_size_ratio = 256. / mpi_depth

    def get_kwargs(self):
        return {
            'xyz_min': self.xyz_min.cpu().numpy(), 'xyz_max': self.xyz_max.cpu().numpy(), 'num_voxels': self.num_voxels,
            'mpi_depth': self.mpi_depth, 'voxel_size_ratio': self.voxel_size_ratio, 'mask_cache_path': self.mask_cache_path,
            'mask_cache_thres': self.mask_cache_thres, 'mask_cache_world_size': list(self.mask_cache.mask.shape),
            'fast_color_thres': self.fast_color_thres, 'density_type': self.density_type, 'k0_type': self.k0_type,
            'density_config': self.density_config, 'k0_config': self.k0_config, **self.rgbnet_kwargs,
        }

    # ---- grid maintenance -----------------------------------------------------------------------------------------------
    @torch.no_grad()
    def scale_volume_grid(self, num_voxels, mpi_depth):
        """dmpigo.py:150-172.  The mask rebuild activates density + act_shift.grid (the per-sample path adds act_shift too)."""
        self._set_grid_resolution(num_voxels, mpi_depth)
        self.density.scale_volume_grid(self.world_size)
        self.k0.scale_volume_grid(self.world_size)
        if np.prod(self.world_size.tolist()) <= 256 ** 3:
            self._rebuild_mask_cache(self.world_size, self.density.get_dense_grid() + self.act_shift.grid)

    @torch.no_grad()
    def update_occupancy_cache_lt_nviews(self, rays_o_tr, rays_d_tr, imsz, render_kwargs, maskout_lt_nviews):
        """dmpigo.py:189-207: mask &= (number of training views whose samples reach a voxel's trilinear support with total weight
        > 1) >= maskout_lt_nviews.  Per view, the grid-sample adjoint of ones over the view's in-box NDC samples."""
        dev = self.density.grid.device
        mn, mx = self.density._bounds()
        count = torch.zeros_like(self.density.get_dense_grid(), dtype=torch.long)
        for rays_o_, rays_d_ in zip(rays_o_tr.split(imsz), rays_d_tr.split(imsz)):
            ones = torch.zeros_like(self.density.get_dense_grid()).requires_grad_(True)
            with torch.enable_grad():
                for rays_o, rays_d in zip(rays_o_.split(8192), rays_d_.split(8192)):
                    ray_pts = self.sample_ray(rays_o=rays_o.to(dev), rays_d=rays_d.to(dev), **render_kwargs)[0]
                    G.grid_sample(ones, ray_pts, mn, mx, 0).sum().backward()
            count += (ones.grad > 1)
        self.mask_cache.mask &= (count >= maskout_lt_nviews)[0, 0]

    def _tv_weights(self, grid, weight, dense_mode):
        """dmpigo.py:209-217: (wxy, wxy, wz) with wxy = weight * max(world_size[:2]) / 128 (an fp32 tensor expression there)
        and wz = weight * mpi_depth / 128, for both grids."""
        wxy = float(weight * self.world_size[:2].max() / 128)
        wz = weight * self.mpi_depth / 128
        return (wxy, wxy, wz, dense_mode)

    # ---- rendering ------------------------------------------------------------------------------------------------------
    def _density_shift(self):
        return 0.           # the act_shift grid is added to the density before the activation

    def _n_samples(self, stepsize):
        return int((self.mpi_depth - 1) / stepsize) + 1

    def sample_ray(self, rays_o, rays_d, near, far, stepsize, **render_kwargs):
        """dmpigo.py:224-249 -> (ray_pts [M,3], ray_id [M], step_id [M], N_samples) of the in-box NDC samples."""
        from . import ops
        assert near == 0 and far == 1
        N_samples = self._n_samples(stepsize)
        ray_pts, mask_outbbox = ops.sample_ndc_pts_on_rays(rays_o.contiguous(), rays_d.contiguous(), self.xyz_min, self.xyz_max,
                                                           N_samples)
        mask_inbbox = ~mask_outbbox
        dev = rays_o.device
        ray_id = torch.arange(mask_inbbox.shape[0], device=dev).view(-1, 1).expand_as(mask_inbbox)[mask_inbbox]
        step_id = torch.arange(mask_inbbox.shape[1], device=dev).view(1, -1).expand_as(mask_inbbox)[mask_inbbox]
        return ray_pts[mask_inbbox], ray_id, step_id, N_samples

    def _fused_ok(self):
        return march.ndc_supported(self.k0.grid) and self.density.grid.is_cuda

    def forward(self, rays_o, rays_d, viewdirs, global_step=None, **render_kwargs):
        assert len(rays_o.shape) == 2 and rays_o.shape[-1] == 3, 'Only suuport point queries in [N, 3] format'
        if not self._fused_ok():
            return self.forward_ops(rays_o, rays_d, viewdirs, global_step=global_step, **render_kwargs)
        assert render_kwargs['near'] == 0 and render_kwargs['far'] == 1
        N = len(rays_o)
        cfg, N_samples = self._ndc_cfg(render_kwargs)
        descs = [G.grid_desc(g.grid, *g._bounds(), 0) for g in (self.density, self.k0, self.act_shift)]
        weights, alphainv_last, alpha, k0, ray_id, step_id = march.NdcMarch.apply(
            self.density.grid, self.k0.grid, self.act_shift.grid, rays_o, rays_d, self.mask_cache.mask, cfg, *descs)
        rgb = self._shade(k0, viewdirs, ray_id)
        return self._finish(N, weights, alphainv_last, alpha, rgb, ray_id, step_id, N_samples, global_step, render_kwargs)

    def _ndc_cfg(self, render_kwargs):
        """(NDC march cfg, N_samples) of forward and render_fused: the bbox, N_samples = int((mpi_depth - 1) / stepsize) + 1,
        interval = stepsize * voxel_size_ratio, the threshold and the mask cache's geometry."""
        stepsize = render_kwargs['stepsize']
        N_samples = self._n_samples(stepsize)
        lo, hi = self._host()
        mscale, mshift = self._mask_geometry()
        cfg = march.make_ndc_cfg(lo, hi, N_samples, stepsize * self.voxel_size_ratio, self.fast_color_thres, self.mask_cache.mask,
                                 mscale, mshift)
        return cfg, N_samples

    # ---- the fused render -----------------------------------------------------------------------------------------------------
    FUSED_FRAME_BY_DEFAULT = False     # render.render_rays takes render_fused only with fused_frame=True (DESIGN.md §7)
    RENDER_NETS = ((9, 0, 64),)        # (k0 channels, viewbase_pe, width) of csrc/render_bounded.cu's NDC kernel: llff_default

    def render_fused_ok(self, rays_o, render_kwargs):
        """Whether render_fused covers this model and call (render.render_rays with fused_frame=True takes it exactly then): no
        gradient, CUDA rays, grids where forward's fused NDC march applies (a contiguous one-slab density, a channels-last k0 of
        9 or 3 channels, a one-slab act_shift grid), an rgbnet with (rgbnet_dim, viewbase_pe, width) = (9, 0, 64)
        (llff_default) or none with a 3-channel k0 (sigmoid(k0)), a numeric bg, and near = 0, far = 1."""
        sg = self.act_shift.grid
        if not (self._render_grids_ok(rays_o, render_kwargs) and self._fused_ok() and 'stepsize' in render_kwargs
                and render_kwargs.get('near') == 0 and render_kwargs.get('far') == 1):
            return False
        if not (sg.is_cuda and sg.dtype == torch.float32 and tuple(sg.shape[:2]) == (1, 1) and sg.is_contiguous()
                and self._n_samples(render_kwargs['stepsize']) >= 2):
            return False
        return self._render_net_ok(self.k0.grid.shape[1], self.RENDER_NETS)

    @torch.no_grad()
    def render_fused(self, rays_o, rays_d, viewdirs, n_shaded=None, n_marched=None, **render_kwargs):
        """{'rgb_marched' [N,3], 'depth' [N], 'alphainv_last' [N]} of N rays in one launch (csrc/render_bounded.cu): the NDC
        march, the k0 read of the kept samples, the rgbnet and the composite with no per-sample buffers, so a whole frame is one
        call.  Same kept samples and alphainv_last (bit for bit) as forward; rgb_marched (+ alphainv_last * bg; a render has no
        global_step, so never rand_bkgd) and depth (sum of w * (step_id + 0.5) / N_samples) as forward's composite, summed in step
        order.  n_shaded / n_marched: optional int32 [N] that receive each ray's kept samples / the samples of the 32-sample
        chunks marched before the ray stopped.  Only where render_fused_ok holds."""
        from . import _cabi
        from ._cabi import c_f, c_i64, c_int, check, ptr, stream_of
        N = rays_o.shape[0]
        dev = rays_o.device
        rays_o = rays_o.contiguous().float()
        rays_d = rays_d.contiguous().float()
        viewdirs = viewdirs.contiguous().float()
        rgb = torch.empty(N, 3, dtype=torch.float32, device=dev)
        depth = torch.empty(N, dtype=torch.float32, device=dev)
        last = torch.empty(N, dtype=torch.float32, device=dev)
        cfg, _ = self._ndc_cfg(render_kwargs)
        ddesc, sdesc, kdesc = (G.grid_desc(g.grid, *g._bounds(), 0) for g in (self.density, self.act_shift, self.k0))
        net, width, pe = self._render_net_args()
        with _cabi.timed('render_ndc'):
            check(_cabi.load().ubn_render_ndc(
                ptr(rays_o), ptr(rays_d), ptr(viewdirs), ptr(self.density.grid), ddesc, ptr(self.act_shift.grid), sdesc,
                ptr(self.k0.grid), kdesc, ptr(self.mask_cache.mask), cfg, c_i64(N), *map(ptr, net), c_int(width), c_int(pe),
                c_f(float(render_kwargs['bg'])), ptr(rgb), ptr(depth), ptr(last), ptr(n_shaded), ptr(n_marched), stream_of(rgb)))
        return {'rgb_marched': rgb, 'depth': depth, 'alphainv_last': last}

    def forward_ops(self, rays_o, rays_d, viewdirs, global_step=None, **render_kwargs):
        """Op-by-op composition in the reference's order (dmpigo.py:251-340)."""
        N = len(rays_o)
        ray_pts, ray_id, step_id, N_samples = self.sample_ray(rays_o=rays_o, rays_d=rays_d, **render_kwargs)
        interval = render_kwargs['stepsize'] * self.voxel_size_ratio
        mask = self.mask_cache(ray_pts)
        ray_pts, ray_id, step_id = ray_pts[mask], ray_id[mask], step_id[mask]
        density = self.density(ray_pts) + self.act_shift(ray_pts)
        alpha = self.activate_density(density, interval)
        if self.fast_color_thres > 0:
            mask = (alpha > self.fast_color_thres)
            ray_pts, ray_id, step_id, alpha = ray_pts[mask], ray_id[mask], step_id[mask], alpha[mask]
        weights, alphainv_last = Alphas2Weights.apply(alpha.contiguous(), ray_id.contiguous(), N)
        if self.fast_color_thres > 0:
            mask = (weights > self.fast_color_thres)
            ray_pts, ray_id, step_id, alpha, weights = ray_pts[mask], ray_id[mask], step_id[mask], alpha[mask], weights[mask]
        k0 = self.k0(ray_pts)
        rgb = self._shade(k0, viewdirs, ray_id)
        return self._finish(N, weights, alphainv_last, alpha, rgb, ray_id, step_id, N_samples, global_step, render_kwargs)

    def _finish(self, N, weights, alphainv_last, alpha, rgb, ray_id, step_id, N_samples, global_step, render_kwargs):
        rgb_marched = composite_rgb(weights, rgb, ray_id, N)
        if render_kwargs.get('rand_bkgd', False) and global_step is not None:
            rgb_marched = rgb_marched + alphainv_last.unsqueeze(-1) * torch.rand_like(rgb_marched)
        else:
            rgb_marched = rgb_marched + alphainv_last.unsqueeze(-1) * render_kwargs['bg']
        s = (step_id + 0.5) / N_samples
        ret = {'alphainv_last': alphainv_last, 'weights': weights, 'rgb_marched': rgb_marched, 'raw_alpha': alpha,
               'raw_rgb': rgb, 'ray_id': ray_id, 'n_max': N_samples, 's': s}
        if render_kwargs.get('render_depth', False):
            with torch.no_grad():
                ret['depth'] = segment_sum(weights * s, ray_id, N)
        return ret
