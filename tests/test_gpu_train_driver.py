"""The reference's own training driver on the fused models, and the model surface it needs.

* The unmodified ``run_train.scene_rep_reconstruction`` (staged by __graft_entry__.build() into git-ignored oracle/_ref/py/)
  trains ``models.FourierGridModel`` and ``models.DirectContractedVoxGO`` end to end with nothing but
  ``legacy.install_models`` applied: training rays from ``gather_training_rays``, the view-count mask
  (``update_occupancy_cache_lt_nviews``), a ``pg_scale`` rescale with the optimizer rebuilt, checkpoints that load into
  both this package's class and the reference's.
* ``ops.view_scatter_ones_contracted`` and ``update_occupancy_cache_lt_nviews`` against the reference's composition
  (dcvgo.py:195-213: sample_ray + grid.DenseGrid + autograd) on the same GPU, and against an fp64 adjoint.
* ``FourierGrid_get_training_rays`` / ``gather_training_rays`` / ``export_geometry_for_visualize`` against the reference's
  methods on the same inputs.

The dataset loaders load_everything.py imports (imageio, tkinter ...) are not needed by these runs and are stubbed."""
import contextlib
import copy
import os
import sys
import types
import warnings

import numpy as np
import pytest
import torch

from tests.util import ROOT, assert_close

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
PY = os.path.join(ROOT, 'oracle', '_ref', 'py')


class Cfg(dict):
    """The attribute-and-key access of the reference's mmengine Config."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None

    def __setattr__(self, k, v):
        self[k] = v


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


@pytest.fixture(scope='module')
def ref():
    if not os.path.exists(os.path.join(PY, 'FourierGrid', 'run_train.py')):
        if os.environ.get('UBN_ALLOW_NO_REF') == '1':
            pytest.skip('oracle/_ref/py not staged (UBN_ALLOW_NO_REF=1)')
        pytest.fail('oracle/_ref/py/FourierGrid/run_train.py is missing: run __graft_entry__.build() where the reference exists')
    from unboundednerfpytorch_b200 import functional as F_, legacy
    legacy.install()

    def unused(*a, **k):
        raise NotImplementedError('not on the path these tests drive')
    _stub('torch_scatter', segment_coo=F_.segment_coo, scatter_add=unused)
    _stub('torch_efficient_distloss', flatten_eff_distloss=F_.flatten_eff_distloss)
    try:
        import cv2  # noqa: F401       utils.py imports it at the top; nothing here calls it
    except ImportError:
        _stub('cv2')
    # dataset loaders of load_everything.py: the tests build their data in memory
    _stub('FourierGrid.common_data_loaders').__path__ = []
    _stub('FourierGrid.common_data_loaders.load_common_data', load_common_data=unused)
    _stub('FourierGrid.load_waymo', load_waymo_data=unused)
    _stub('FourierGrid.load_mega', load_mega_data=unused)
    sys.path.insert(0, PY)
    try:
        from FourierGrid import (FourierGrid_ckpt_manager, FourierGrid_model, dcvgo, dmpigo, dvgo, grid, load_everything,
                                 run_train, utils)
    finally:
        sys.path.remove(PY)
    return types.SimpleNamespace(run_train=run_train, ckpt=FourierGrid_ckpt_manager, fg=FourierGrid_model, dcvgo=dcvgo,
                                 dvgo=dvgo, dmpigo=dmpigo, grid=grid, load_everything=load_everything, utils=utils)


@contextlib.contextmanager
def _reference_defaults():
    """run_FourierGrid.py:87 `torch.set_default_tensor_type('torch.cuda.FloatTensor')`, which the reference's torch.Tensor(...)
    and torch.linspace(...) calls rely on to land on the GPU (deprecated in torch 2.x, still there; else set_default_device)."""
    def use(on):
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            try:
                torch.set_default_tensor_type('torch.cuda.FloatTensor' if on else 'torch.FloatTensor')
            except Exception:
                torch.set_default_device(DEV if on else 'cpu')
    use(True)
    try:
        yield
    finally:
        use(False)


def _install(ref):
    from unboundednerfpytorch_b200 import legacy
    return legacy.install_models(ref.run_train, ref.dvgo, ref.dcvgo, ref.dmpigo, ref.ckpt, ref.load_everything, ref.utils)


# ---------------------------------------------------------------------------------------------------------------------------
# a synthetic scene: views on a ring around the origin
# ---------------------------------------------------------------------------------------------------------------------------
def _look_at(cam):
    back = cam / np.linalg.norm(cam)
    right = np.cross([0., 0., 1.], back)
    right /= np.linalg.norm(right)
    up = np.cross(back, right)
    return np.stack([right, up, back, cam], 1).astype(np.float32)        # [3, 4] camera-to-world, OpenGL axes


def _cameras(n, radius=2.5, H=48, W=64, focal=50., seed=0):
    rng = np.random.default_rng(seed)
    poses = []
    for i in range(n):
        a = 2 * np.pi * i / n + rng.uniform(-0.1, 0.1)
        cam = np.array([radius * np.cos(a), radius * np.sin(a), rng.uniform(-0.4, 0.6)])
        poses.append(_look_at(cam))
    K = np.array([[focal, 0, W / 2], [0, focal, H / 2], [0, 0, 1]], dtype=np.float32)
    return torch.tensor(np.stack(poses)), np.array([[H, W]] * n), np.stack([K] * n)


FG_MODEL = dict(num_voxels_density=32 ** 3, num_voxels_rgb=32 ** 3, num_voxels_base_density=32 ** 3, num_voxels_base_rgb=32 ** 3,
                num_voxels_viewdir=-1, alpha_init=1e-2, fast_color_thres=1e-4, rgbnet_dim=12, fourier_freq_num=2, bg_len=0.2,
                contracted_norm='inf', stepsize=0.5, world_bound_scale=1, maskout_near_cam_vox=False)
DC_MODEL = dict(num_voxels_density=40 ** 3, num_voxels_rgb=40 ** 3, num_voxels_base_rgb=40 ** 3, alpha_init=1e-2,
                fast_color_thres=1e-4, rgbnet_dim=12, bg_len=0.2, contracted_norm='l2', stepsize=0.5, world_bound_scale=1,
                maskout_near_cam_vox=False)


@torch.no_grad()
def _teacher_images(poses, HW, Ks, kind):
    """Targets rendered by a seeded teacher of the same family (this package's fused forward)."""
    from unboundednerfpytorch_b200 import models, rays
    torch.manual_seed(1234)
    if kind == 'fg':
        kw = {k: v for k, v in FG_MODEL.items() if k not in ('stepsize', 'world_bound_scale', 'maskout_near_cam_vox')}
        t = models.FourierGridModel(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, **kw)
    else:
        kw = {k: v for k, v in DC_MODEL.items() if k not in ('stepsize', 'world_bound_scale', 'maskout_near_cam_vox',
                                                             'num_voxels_density', 'num_voxels_rgb', 'num_voxels_base_rgb')}
        t = models.DirectContractedVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=40 ** 3, num_voxels_base=40 ** 3, **kw)
    t = t.to(DEV)
    t.density.grid.normal_(0., 6.)
    t.k0.grid.normal_(0., 1.)
    images = []
    for c2w, (H, W), K in zip(poses, HW, Ks):
        o, d, v = rays.get_rays_of_a_view(H, W, K, c2w.to(DEV), False, False, False, False)
        out = t(o.reshape(-1, 3), d.reshape(-1, 3), v.reshape(-1, 3), near=0.1, far=1e9, bg=1, stepsize=0.5)
        images.append(out['rgb_marched'].clamp(0, 1).reshape(H, W, 3).cpu())
    return torch.stack(images)


def _data_dict(kind, n_views=6):
    poses, HW, Ks = _cameras(n_views)
    return {'HW': HW, 'Ks': Ks, 'near': 0.1, 'far': 6.0, 'near_clip': 0.1, 'i_train': np.arange(n_views),
            'i_val': np.arange(0), 'i_test': np.arange(0), 'poses': poses, 'images': _teacher_images(poses, HW, Ks, kind),
            'irregular_shape': False}


def _cfg(tmp_path, model, dataset_type, model_cfg, maskout_lt_nviews):
    data = Cfg(dataset_type=dataset_type, ndc=False, unbounded_inward=True, inverse_y=False, flip_x=False, flip_y=False,
               white_bkgd=True, rand_bkgd=False, load2gpu_on_the_fly=False)
    train = Cfg(N_iters=60, N_rand=1024, lrate_decay=20, lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, pg_scale=[20],
                ray_sampler='flatten', pervoxel_lr=False, pervoxel_lr_downrate=1, maskout_lt_nviews=maskout_lt_nviews,
                decay_after_scale=1.0, weight_main=1.0, weight_freq=0.0, weight_entropy_last=0.0, weight_nearclip=0.0,
                weight_distortion=0.0, weight_rgbper=0.0, tv_before=0, tv_after=0, tv_every=1, weight_tv_density=0.0,
                weight_tv_k0=0.0, tv_dense_before=0, skip_zero_grad_fields=[])
    return Cfg(model=model, basedir=str(tmp_path), expname='exp', data=data, fine_train=train,
               fine_model_and_render=Cfg(copy.deepcopy(model_cfg)))


def _args(cfg, ref):
    args = Cfg(no_reload=True, ft_path=None, sample_num=-1, block_num=1, i_print=10 ** 9, no_reload_optimizer=False,
               running_block_id=-1)
    args.ckpt_manager = ref.ckpt.FourierGridCheckpointManager(args, cfg)
    return args


@torch.no_grad()
def _psnr(model, data_dict):
    from unboundednerfpytorch_b200 import rays
    model = model.to(DEV)
    err = []
    for c2w, (H, W), K, img in zip(data_dict['poses'], data_dict['HW'], data_dict['Ks'], data_dict['images']):
        o, d, v = rays.get_rays_of_a_view(H, W, K, c2w.to(DEV), False, False, False, False)
        out = model(o.reshape(-1, 3), d.reshape(-1, 3), v.reshape(-1, 3), near=0.1, far=1e9, bg=1, stepsize=0.5)
        err.append((out['rgb_marched'] - img.reshape(-1, 3).to(DEV)).pow(2).mean())
    return (-10 * torch.log10(torch.stack(err).mean())).item()


def _run_driver(ref, tmp_path, monkeypatch, kind):
    from unboundednerfpytorch_b200 import _cabi, ckpt, models
    if kind == 'fg':
        cfg = _cfg(tmp_path, 'FourierGrid', 'mega', FG_MODEL, maskout_lt_nviews=1)
        ours_cls, ref_cls = models.FourierGridModel, ref.fg.FourierGridModel
    else:
        cfg = _cfg(tmp_path, 'DCVGO', 'nerf_unbounded', DC_MODEL, maskout_lt_nviews=2)
        ours_cls, ref_cls = models.DirectContractedVoxGO, ref.dcvgo.DirectContractedVoxGO
    data_dict = _data_dict(kind)
    os.makedirs(os.path.join(cfg.basedir, cfg.expname), exist_ok=True)
    args = _args(cfg, ref)
    calls = []
    orig = ours_cls.update_occupancy_cache_lt_nviews

    def spy(self, *a, **k):
        calls.append(type(self))
        return orig(self, *a, **k)
    np.random.seed(0)
    torch.manual_seed(0)
    monkeypatch.setattr(ours_cls, 'update_occupancy_cache_lt_nviews', spy)
    _cabi.reset_launch_count()
    with _install(ref):
        assert ref.run_train.FourierGridModel is models.FourierGridModel
        psnr_last_step = ref.run_train.scene_rep_reconstruction(
            args=args, cfg=cfg, cfg_model=cfg.fine_model_and_render, cfg_train=cfg.fine_train,
            xyz_min=torch.tensor([-1.] * 3, device=DEV), xyz_max=torch.tensor([1.] * 3, device=DEV), data_dict=data_dict,
            stage='fine')
    monkeypatch.undo()
    assert ref.run_train.FourierGridModel is ref.fg.FourierGridModel          # restored
    assert calls == [ours_cls]                        # the view-count mask ran, on this package's class
    assert _cabi.launch_count() > 0                   # and the training ran on this library's kernels
    assert np.isfinite(psnr_last_step)
    first = os.path.join(cfg.basedir, cfg.expname, 'fine_000001.tar')
    last = os.path.join(cfg.basedir, cfg.expname, 'fine_last.tar')
    m_first = ckpt.load_model(ours_cls, first, DEV)
    m_last = ckpt.load_model(ours_cls, last, DEV)
    assert isinstance(m_last, ours_cls)
    assert list(m_last.world_size.tolist()) != list(m_first.world_size.tolist())          # the pg_scale step ran
    p0, p1 = _psnr(m_first, data_dict), _psnr(m_last, data_dict)
    print(f'{kind}: PSNR after step 1 {p0:.2f} dB, after step {cfg.fine_train.N_iters} {p1:.2f} dB')
    assert p1 > p0 + 0.5, (p0, p1)
    # the final checkpoint loads into the reference's class with the same tensors
    saved = ckpt._load(last)
    ref_model = ref_cls(**saved['model_kwargs'])
    ref_model.load_state_dict(saved['model_state_dict'])
    for k, v in ref_model.state_dict().items():
        assert torch.equal(v.cpu(), saved['model_state_dict'][k].cpu()), k
    return m_last


def test_driver_trains_fouriergrid(ref, tmp_path, monkeypatch):
    _run_driver(ref, tmp_path, monkeypatch, 'fg')


def test_driver_trains_dcvgo(ref, tmp_path, monkeypatch):
    m = _run_driver(ref, tmp_path, monkeypatch, 'dcvgo')
    assert not bool(m.mask_cache.mask.all())             # maskout_lt_nviews = 2 removed voxels fewer than two views see


# ---------------------------------------------------------------------------------------------------------------------------
# the view-count kernel
# ---------------------------------------------------------------------------------------------------------------------------
def _fp64_adjoint(pts, xyz_min, xyz_max, ws):
    """sum over points of the eight trilinear weights (align_corners=True, zero padding), in fp64, as an [X, Y, Z] tensor."""
    p = pts.reshape(-1, 3).double()
    mn = torch.tensor(xyz_min, dtype=torch.float64, device=p.device)
    mx = torch.tensor(xyz_max, dtype=torch.float64, device=p.device)
    size = torch.tensor(ws, dtype=torch.float64, device=p.device)
    c = (p - mn) / (mx - mn) * (size - 1)
    f = c.floor()
    w1 = c - f
    out = torch.zeros(int(np.prod(ws)), dtype=torch.float64, device=p.device)
    for corner in range(8):
        b = torch.tensor([(corner >> 2) & 1, (corner >> 1) & 1, corner & 1], dtype=torch.float64, device=p.device)
        idx = f + b
        w = torch.where(b.bool(), w1, 1 - w1).prod(-1)
        ok = ((idx >= 0) & (idx < size)).all(-1)
        lin = (idx[:, 0] * ws[1] + idx[:, 1]) * ws[2] + idx[:, 2]
        out.index_add_(0, lin[ok].long(), w[ok])
    return out.reshape(ws)


def _probe_rays(n, seed, scene_radius=1.0):
    """Origins inside and outside the unit cube (normalised), some direction components exactly zero."""
    g = torch.Generator().manual_seed(seed)
    o = (torch.rand(n, 3, generator=g) - 0.5) * 5 * scene_radius
    d = torch.randn(n, 3, generator=g)
    d[::5, 0] = 0
    d[1::7, 1] = 0
    d[3::10, 1:] = 0                 # rows 3 mod 10 keep x != 0: no direction is the zero vector
    return o.to(DEV), d.to(DEV)


def _ref_view_grads(ref_model, ref_grid, ws, rays_o_tr, rays_d_tr, imsz, render_kwargs):
    """dcvgo.py:200-207 per view: ones = grid.DenseGrid(1, world_size, xyz_min, xyz_max); ones(sample_ray(...)[0]).sum().backward()
    per 8192 rays -> [ones.grid.grad] and the sample points."""
    grads, points = [], []
    with _reference_defaults():              # the reference builds its t table and ones grid on the default device
        for rays_o_, rays_d_ in zip(rays_o_tr.split(imsz), rays_d_tr.split(imsz)):
            ones = ref_grid.DenseGrid(1, ws, ref_model.xyz_min, ref_model.xyz_max).to(DEV)
            pts = []
            for rays_o, rays_d in zip(rays_o_.split(8192), rays_d_.split(8192)):
                out = ref_model.sample_ray(ori_rays_o=rays_o, ori_rays_d=rays_d, **render_kwargs)
                ray_pts = out[0]
                ones(ray_pts).sum().backward()
                pts.append(ray_pts.detach().reshape(-1, 3))
            grads.append(ones.grid.grad[0, 0].clone())
            points.append(torch.cat(pts))
    return grads, points


@pytest.mark.parametrize('kind,norm', [('dcvgo', 'inf'), ('dcvgo', 'l2'), ('fg', 'l2'), ('fg', 'inf')])
def test_lt_nviews_against_reference_composition(ref, kind, norm):
    from unboundednerfpytorch_b200 import march, models, ops
    torch.manual_seed(5)
    center, radius = [0.2, -0.1, 0.3], 1.3
    xyz_min = [c - radius for c in center]
    xyz_max = [c + radius for c in center]
    if kind == 'dcvgo':
        kw = dict(num_voxels=28 ** 3, num_voxels_base=28 ** 3, alpha_init=1e-2, fast_color_thres=1e-4, rgbnet_dim=12, bg_len=0.2,
                  contracted_norm=norm)
        ours = models.DirectContractedVoxGO(xyz_min, xyz_max, **kw).to(DEV)
        ref_model = ref.dcvgo.DirectContractedVoxGO(torch.tensor(xyz_min), torch.tensor(xyz_max), **kw).to(DEV)
    else:
        kw = dict(num_voxels_density=28 ** 3, num_voxels_base_density=28 ** 3, num_voxels_rgb=20 ** 3,
                  num_voxels_base_rgb=20 ** 3, num_voxels_viewdir=-1, alpha_init=1e-2, fast_color_thres=1e-4, rgbnet_dim=12,
                  fourier_freq_num=2, bg_len=0.3, contracted_norm=norm)
        ours = models.FourierGridModel(xyz_min, xyz_max, **kw).to(DEV)
        ref_model = ref.fg.FourierGridModel(torch.tensor(xyz_min), torch.tensor(xyz_max), **kw).to(DEV)
    ws = [int(v) for v in ours.world_size]
    imsz = [700, 1, 37, 300]                 # a one-ray view: fewer threads than one block
    rays_o_tr, rays_d_tr = _probe_rays(sum(imsz), seed=11)
    rays_o_tr = rays_o_tr * radius + torch.tensor(center, device=DEV)
    render_kwargs = dict(near=0.1, far=1e9, bg=1, stepsize=0.5)
    grads, points = _ref_view_grads(ref_model, ref.grid, ws, rays_o_tr, rays_d_tr, imsz, render_kwargs)

    # per-view buffers of the kernel: vs the reference's autograd sums and vs fp64
    t_table = march.t_schedule(ours._world_len(), 0.5, ours.bg_len, ours.T_BOUNDARY, DEV)
    c_host, r_host = ours._host()
    band_total, count_ours = 0, torch.zeros(ws, device=DEV)
    count_ref = torch.zeros(ws, device=DEV)
    for v, (ro, rd) in enumerate(zip(rays_o_tr.split(imsz), rays_d_tr.split(imsz))):
        buf = torch.zeros(ws, device=DEV)
        ops.view_scatter_ones_contracted(ro.contiguous(), rd.contiguous(), t_table, c_host, r_host, ours.bg_len, norm,
                                         ours.xyz_min.tolist(), ours.xyz_max.tolist(), ws, buf)
        exact = _fp64_adjoint(points[v], ours.xyz_min.tolist(), ours.xyz_max.tolist(), ws)
        scale = exact.abs().max().item()
        assert (buf.double() - exact).abs().max().item() <= 1e-5 * scale, f'view {v}: buffer vs fp64'
        assert (grads[v].double() - exact).abs().max().item() <= 1e-5 * scale
        band = (exact - 1).abs() <= 1e-5
        band_total += int(band.sum())
        mismatch = ((buf > 1) != (grads[v] > 1)) & ~band
        assert not bool(mismatch.any()), f'view {v}: {int(mismatch.sum())} count flips outside the band'
        count_ours += buf > 1
        count_ref += grads[v] > 1
    print(f'{kind}/{norm}: {band_total} voxel-views with an fp64 weight sum within 1e-5 of 1')

    # the model method: the counts of the per-view buffers above, and the reference's mask outside the band
    for n in (1, 2, 3):
        m = ours.mask_cache.mask
        m.fill_(True)
        m[0, :, :] = False                  # an existing hole stays a hole
        ours.update_occupancy_cache_lt_nviews(rays_o_tr, rays_d_tr, imsz, render_kwargs, n)
        expect_ours, expect_ref = count_ours >= n, count_ref >= n
        expect_ours[0] = expect_ref[0] = False
        assert torch.equal(ours.mask_cache.mask, expect_ours), n
        flips = int((ours.mask_cache.mask != expect_ref).sum())
        assert flips <= band_total, (n, flips, band_total)


def test_view_scatter_ones_contracted_non_cubic_world_vs_fp64():
    """The kernel alone on a non-cubic world (the models' worlds are cubes): against the fp64 adjoint of the points
    _sample_dense generates, which are the kernel's points bit for bit."""
    from unboundednerfpytorch_b200 import march, models, ops
    m = models.DirectContractedVoxGO([-1.] * 3, [1.] * 3, num_voxels=16 ** 3, num_voxels_base=16 ** 3, alpha_init=1e-2,
                                     bg_len=0.25, contracted_norm='inf').to(DEV)
    ws = [23, 9, 31]
    rays_o, rays_d = _probe_rays(513, seed=3)
    for norm in ('inf', 'l2'):
        m.contracted_norm = norm
        pts, _, t = m._sample_dense(rays_o, rays_d, 0.7)
        t_table = march.t_schedule(m._world_len(), 0.7, m.bg_len, m.T_BOUNDARY, DEV)
        assert torch.equal(t, t_table)
        buf = torch.zeros(ws, device=DEV)
        ops.view_scatter_ones_contracted(rays_o, rays_d, t_table, *m._host(), m.bg_len, norm, m.xyz_min.tolist(),
                                         m.xyz_max.tolist(), ws, buf)
        exact = _fp64_adjoint(pts, m.xyz_min.tolist(), m.xyz_max.tolist(), ws)
        assert (buf.double() - exact).abs().max().item() <= 1e-5 * exact.abs().max().item()
        assert abs(buf.double().sum().item() - pts.shape[0] * pts.shape[1]) <= 1e-4 * pts.shape[0] * pts.shape[1]
    with pytest.raises(RuntimeError):
        ops.view_scatter_ones_contracted(rays_o, rays_d, t_table, *m._host(), m.bg_len, 'inf', m.xyz_min.tolist(),
                                         m.xyz_max.tolist(), ws, torch.zeros(5, device=DEV))


# ---------------------------------------------------------------------------------------------------------------------------
# training rays and the geometry export
# ---------------------------------------------------------------------------------------------------------------------------
def _fg_pair(ref, rgbnet_dim=12):
    from unboundednerfpytorch_b200 import models
    kw = dict(num_voxels_density=24 ** 3, num_voxels_base_density=24 ** 3, num_voxels_rgb=24 ** 3, num_voxels_base_rgb=24 ** 3,
              num_voxels_viewdir=-1, alpha_init=1e-2, fast_color_thres=1e-4, rgbnet_dim=rgbnet_dim, fourier_freq_num=2)
    torch.manual_seed(3)
    ours = models.FourierGridModel([-1.] * 3, [1.] * 3, **kw).to(DEV)
    ours.density.grid.data.normal_(0, 4)
    ours.k0.grid.data.normal_()
    ref_model = ref.fg.FourierGridModel(torch.tensor([-1.] * 3), torch.tensor([1.] * 3), **kw)
    ref_model.load_state_dict({k: v.cpu() for k, v in ours.state_dict().items()})
    return ours, ref_model.to(DEV)


def _compare_rays(a, b):
    assert torch.equal(a[0], b[0]), 'rgb_tr'
    for i, name in ((1, 'rays_o'), (2, 'rays_d'), (3, 'viewdirs')):
        assert a[i].device == b[i].device
        assert_close(a[i], b[i], rtol=2e-6, what=name)


def test_fouriergrid_get_training_rays_matches_reference(ref):
    ours, ref_model = _fg_pair(ref)
    poses, HW, Ks = _cameras(4)
    HW = np.array([[48, 64], [31, 17], [48, 64], [1, 5]])
    Ks = Ks.copy()
    Ks[1, 0, 2], Ks[1, 1, 2], Ks[1, 0, 0] = 8.5, 15.5, 30.
    torch.manual_seed(9)
    imgs = [torch.rand(int(H), int(W), 3, device=DEV) for H, W in HW]
    args = dict(rgb_tr_ori=imgs, train_poses=poses, HW=HW, Ks=Ks, ndc=False, inverse_y=False, flip_x=False, flip_y=False)
    a = ours.FourierGrid_get_training_rays(**args)
    with _reference_defaults():
        b = ref_model.FourierGrid_get_training_rays(**copy.deepcopy(args))
    _compare_rays(a, b)
    assert a[4].dtype == b[4].dtype == torch.float32 and torch.equal(a[4], b[4]), 'indexs_tr'
    assert a[5] == b[5]
    assert torch.equal(poses, _cameras(4)[0])                 # the poses are not modified


@pytest.mark.parametrize('branch', ['FourierGrid', 'in_maskcache', 'flatten', 'random'])
@pytest.mark.parametrize('irregular', [False, True])
def test_gather_training_rays_matches_reference(ref, branch, irregular):
    if irregular and branch == 'random':
        pytest.skip('get_training_rays needs one image size (dvgo.py:562-563)')
    ours, ref_model = _fg_pair(ref)
    if branch == 'in_maskcache':                  # rays that miss the coarse geometry are dropped
        for m in (ours, ref_model):
            m.mask_cache.mask[:, :12] = False
    n = 5
    poses, HW, Ks = _cameras(n, H=24, W=32, focal=25.)
    poses = poses.to(DEV)           # run_FourierGrid.py loads them under CUDA as the default tensor type
    torch.manual_seed(2)
    images = torch.rand(n, 24, 32, 3)
    if irregular:
        HW = np.array([[24, 32], [24, 32], [20, 12], [24, 32], [7, 9]])
        images = [torch.rand(int(H), int(W), 3) for H, W in HW]
    data_dict = {'irregular_shape': irregular}
    cfg = Cfg(model='FourierGrid' if branch == 'FourierGrid' else 'DVGO',
              data=Cfg(dataset_type='llff', ndc=False, inverse_y=False, flip_x=False, flip_y=False, load2gpu_on_the_fly=False))
    cfg_train = Cfg(ray_sampler=branch if branch != 'FourierGrid' else 'flatten', N_rand=97)
    i_train = np.array([0, 2, 3, 4])
    render_kwargs = dict(near=0.1, far=1e9, bg=1, stepsize=0.5)
    a = ours.gather_training_rays(data_dict, images, cfg, i_train, cfg_train, poses, HW, Ks, render_kwargs)
    with _reference_defaults():
        b = ref_model.gather_training_rays(data_dict, images, cfg, i_train, cfg_train, poses, HW, Ks, render_kwargs)
    _compare_rays(a, b)
    if branch == 'FourierGrid':
        assert torch.equal(a[4], b[4]), 'indexs_train'
    else:
        assert a[4] is None and b[4] is None
    assert list(a[5]) == list(b[5])
    # the samplers draw np.random.permutation on their first call
    np.random.seed(6)
    batches = [a[6]() for _ in range(3)]
    np.random.seed(6)
    for x in batches:
        assert torch.equal(x, b[6]())


@pytest.mark.parametrize('load2gpu', [False, True])
def test_gather_training_rays_host_images(ref, load2gpu):
    """load2gpu_on_the_fly keeps images (and with them the flattened rays) on the host, as the reference does."""
    ours, ref_model = _fg_pair(ref)
    poses, HW, Ks = _cameras(3, H=16, W=20, focal=20.)
    images = torch.rand(3, 16, 20, 3)
    cfg = Cfg(model='FourierGrid', data=Cfg(dataset_type='mega', ndc=False, inverse_y=False, flip_x=False, flip_y=False,
                                            load2gpu_on_the_fly=load2gpu))
    cfg_train = Cfg(ray_sampler='flatten', N_rand=64)
    args = ({'irregular_shape': False}, images, cfg, np.arange(3), cfg_train, poses, HW, Ks, dict(stepsize=0.5))
    a = ours.gather_training_rays(*args)
    with _reference_defaults():
        b = ref_model.gather_training_rays(*args)
    assert a[0].device.type == ('cpu' if load2gpu else 'cuda')
    _compare_rays(a, b)
    assert torch.equal(a[4], b[4])


@pytest.mark.parametrize('rgbnet_dim', [0, 12])
def test_export_geometry_matches_reference(ref, tmp_path, rgbnet_dim):
    ours, ref_model = _fg_pair(ref, rgbnet_dim)
    pa, pb = str(tmp_path / 'ours.npz'), str(tmp_path / 'ref.npz')
    if rgbnet_dim > 0:
        # the fine model's k0 has 2F+1 slabs of rgbnet_dim channels: the reference's squeeze().permute(1, 2, 3, 0) of a 5-D grid
        # fails, and so does this one, in the same way
        with pytest.raises(RuntimeError):
            ref_model.export_geometry_for_visualize(pb)
        with pytest.raises(RuntimeError):
            ours.export_geometry_for_visualize(pa)
        return
    ours.export_geometry_for_visualize(pa)
    ref_model.export_geometry_for_visualize(pb)
    a, b = np.load(pa), np.load(pb)
    assert sorted(a.files) == sorted(b.files) == ['alpha', 'rgb']
    for k in ('alpha', 'rgb'):
        assert a[k].shape == b[k].shape and a[k].dtype == b[k].dtype, k
        np.testing.assert_array_equal(a[k], b[k])
