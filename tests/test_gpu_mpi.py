"""GPU tests of DirectMPIGO (forward-facing NDC model, dmpigo.py) and its fused NDC march (march.NdcMarch,
csrc/march.cu with NdcSampler + csrc/march_ndc.cu): the golden fixtures of the reference's own dmpigo.py through the fused path
and forward_ops, the C = 3 / 9 feature read against F.grid_sample, the unmodified staged dmpigo.py over legacy.install(), the
llff_default shape, grid maintenance, rendering, checkpoints and training."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_callers_unchanged import PY, _default_cuda, _stat, ref_modules  # noqa: F401  (module-scoped fixture)
from tests.test_gpu_models import _check_against_golden
from tests.util import assert_equal, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
RK = dict(near=0., far=1., bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False, render_depth=True)


def _build(rec):
    from unboundednerfpytorch_b200 import models
    m = models.DirectMPIGO(**rec['kwargs'])
    m.load_state_dict(rec['state'])
    return m.to(DEV)


@pytest.mark.parametrize('tag', ['mpi_rgb9', 'mpi_rgb0'])
@pytest.mark.parametrize('path', ['fused', 'ops'])
def test_mpi_golden(tag, path):
    rec = load_golden(f'l2_mpi/{tag}.pt')
    m = _build(rec)
    assert path == 'ops' or m._fused_ok()
    _check_against_golden(m, rec, m.forward if path == 'fused' else m.forward_ops, f'{tag}/{path}')
    ret = m(rec['rays_o'].to(DEV), rec['rays_d'].to(DEV), rec['viewdirs'].to(DEV), **rec['render_kwargs'])
    S = rec['ret']['n_max']
    assert ret['n_max'] == S
    # s = (step_id + 0.5) / N_samples: the fixture was recorded on the CPU, where torch divides by the scalar; on CUDA torch
    # multiplies by its reciprocal, so the last bit of s is the device's.  The step ids behind s are exact, and s is exactly
    # what the reference's expression gives on this device.
    step_ref = torch.round(rec['ret']['s'] * S - 0.5).long()
    assert_equal(torch.round(ret['s'].cpu() * S - 0.5).long(), step_ref, f'{tag} step ids behind s')
    assert_equal(ret['s'], (step_ref.to(DEV) + 0.5) / S, f'{tag} s')


def _ndc_scene(C, depth=32, nv=48 ** 3, n=4096, seed=5, thres=1e-3, mask_p=0.9, dmean=0.0, dstd=3.0):
    from unboundednerfpytorch_b200 import models
    g = torch.Generator().manual_seed(seed)
    m = models.DirectMPIGO(xyz_min=[-1.4, -1.1, -1.], xyz_max=[1.4, 1.1, 1.], num_voxels=nv, mpi_depth=depth,
                           rgbnet_dim=0 if C == 3 else C, rgbnet_width=64, fast_color_thres=thres)
    with torch.no_grad():
        m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=g) * dstd + dmean)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
        m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=g) < mask_p)
    ro = torch.cat([(torch.rand(n, 2, generator=g) - 0.5) * 3.0, -torch.ones(n, 1)], -1)
    rd = torch.cat([torch.randn(n, 2, generator=g) * 0.3, 2.0 + torch.randn(n, 1, generator=g) * 0.02], -1)
    vd = rd / rd.norm(dim=-1, keepdim=True)
    return m.to(DEV), ro.to(DEV), rd.to(DEV), vd.to(DEV)


def _torch_grid_sample(grid, xyz, mn, mx):
    """DenseGrid.forward of the reference (grid.py:50-61): F.grid_sample on the normalised, flipped coordinates."""
    ind = ((xyz - mn) / (mx - mn)).flip((-1,)) * 2 - 1
    out = F.grid_sample(grid, ind.reshape(1, 1, 1, -1, 3), mode='bilinear', align_corners=True)
    return out.reshape(grid.shape[1], -1).T


@pytest.mark.parametrize('C', [9, 3])
def test_ndc_feature_read_vs_grid_sample(C):
    """The fused C = 9 / C = 3 gather is bit-identical to F.grid_sample; its scatter equals autograd of F.grid_sample to fp32
    atomic-order tolerance."""
    from unboundednerfpytorch_b200 import march, ops
    from unboundednerfpytorch_b200 import grid as G
    m, ro, rd, vd = _ndc_scene(C, thres=0.0)
    S = m._n_samples(0.5)
    lo, hi = m._host()
    cfg = march.make_ndc_cfg(lo, hi, S, 0.5 * m.voxel_size_ratio, 0.0, m.mask_cache.mask, *m._mask_geometry())
    descs = [G.grid_desc(g.grid, *g._bounds(), 0) for g in (m.density, m.k0, m.act_shift)]
    k0 = m.k0.grid.detach().clone().requires_grad_(True)
    w, last, alpha, feat, ray_id, step_id = march.NdcMarch.apply(m.density.grid.detach(), k0, m.act_shift.grid, ro, rd,
                                                                 m.mask_cache.mask, cfg, *descs)
    assert feat.shape[0] > 10000
    pts = ops.sample_ndc_pts_on_rays(ro, rd, m.xyz_min, m.xyz_max, S)[0][ray_id, step_id]
    k0_ref = m.k0.grid.detach().contiguous().clone().requires_grad_(True)
    ref = _torch_grid_sample(k0_ref, pts, m.xyz_min, m.xyz_max)
    assert_equal(feat, ref, f'C={C} feature read vs F.grid_sample')
    gout = torch.randn(feat.shape, device=DEV)
    (feat * gout).sum().backward()
    (ref * gout).sum().backward()
    scale = k0_ref.grad.abs().max().item()
    err = (k0.grad - k0_ref.grad).abs().max().item()
    assert err <= 1e-5 * scale, f'C={C} scatter: {err:.3e} vs scale {scale:.3e}'


@pytest.mark.parametrize('C', [9, 3])
def test_llff_default_size_fused_vs_ops(C):
    """llff_default shape (mpi_depth 128, stepsize 0.5 -> S = 255, 4096 rays, fast_color_thres 1e-3): zero membership flips;
    the density read is bit-identical, so raw_alpha, weights and alphainv_last are too; colours within 1e-5 of scale; gradients
    within fp32 atomic-order tolerance."""
    m, ro, rd, vd = _ndc_scene(C, depth=128, nv=256 ** 3, seed=9, dmean=-1.0)
    a = m(ro, rd, vd, global_step=None, **RK)
    b = m.forward_ops(ro, rd, vd, global_step=None, **RK)
    assert a['n_max'] == 255
    assert_equal(a['ray_id'], b['ray_id'], 'ray_id')
    assert_equal(a['s'], b['s'], 's')
    assert a['ray_id'].numel() > 100000
    for k in ('raw_alpha', 'weights', 'alphainv_last'):
        assert_equal(a[k], b[k], k)
    for k in ('rgb_marched', 'raw_rgb', 'depth'):
        assert _stat(a[k], b[k]) <= 1e-5, k
    grads = []
    for ret in (a, b):
        m.zero_grad(set_to_none=True)
        (ret['rgb_marched'].pow(2).sum() + ret['alphainv_last'].sum()).backward()
        grads.append({k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None})
    assert 'act_shift.grid' not in grads[0]
    for k in grads[1]:
        assert _stat(grads[0][k], grads[1][k]) <= 2e-5, k


@pytest.mark.parametrize('C', [9, 3])
def test_llff_default_size_vs_reference_gpu(C):
    """llff_default shape against the reference's GPU path: its unmodified dmpigo.py over its own CUDA extension (oracle/_ref;
    oracle/ref_gpu_py.py), i.e. ATen grid_sample + cuBLAS + the reference's kernels, none of this library's.
    The fused density read IS bit-identical to the reference's `density(p) + act_shift(p)`: the density grid through the
    pre-clamped cell and the act_shift grid through the bounds-checked read both reproduce F.grid_sample's arithmetic (same
    corner order, same fma chain), and the two are added with one fp32 rounding.  With NDC points, the mask lookup, Raw2Alpha and
    the transmittance scan also bit-identical, the gates are: zero membership flips, raw_alpha / weights / alphainv_last
    bit-identical, colours within 1e-5 of scale."""
    from oracle import ref_gpu_py
    why = ref_gpu_py.missing()
    if why is not None:
        if os.environ.get('UBN_ALLOW_NO_REF') == '1':
            pytest.skip(f'{why} missing (UBN_ALLOW_NO_REF=1)')
        pytest.fail(f'{why} is missing: run __graft_entry__.build() where the reference checkout exists')
    ns = ref_gpu_py.load()
    m, ro, rd, vd = _ndc_scene(C, depth=128, nv=256 ** 3, seed=9, dmean=-1.0)
    state = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}
    kw = {k: v for k, v in m.get_kwargs().items() if k != 'voxel_size_ratio'}
    ref_gpu_py.default_cuda(True)
    try:
        ref = _quiet(ns.dmpigo.DirectMPIGO, **kw)
        ref.load_state_dict(state, strict=True)
        with torch.no_grad():
            a = ref.to(DEV)(ro, rd, vd, global_step=None, **RK)
    finally:
        ref_gpu_py.default_cuda(False)
    with torch.no_grad():
        b = m(ro, rd, vd, global_step=None, **RK)
    assert a['n_max'] == b['n_max'] == 255
    assert_equal(b['ray_id'], a['ray_id'], 'ray_id (membership)')
    assert_equal(b['s'], a['s'], 's')
    assert b['ray_id'].numel() > 100000
    for k in ('raw_alpha', 'weights', 'alphainv_last'):
        assert_equal(b[k], a[k], k)
    for k in ('rgb_marched', 'raw_rgb', 'depth'):
        assert _stat(b[k], a[k]) <= 1e-5, k


def _ref_mpi(ref_modules):
    sys.path.insert(0, PY)
    try:
        from FourierGrid import dmpigo
    finally:
        sys.path.remove(PY)
    return dmpigo.DirectMPIGO


def _quiet(fn, *a, **k):
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def _pair(ref_modules, C=9, **scene):
    """Ours and the staged reference class on the same state dict (the reference built like run_train.py: CUDA default type)."""
    ours, ro, rd, vd = _ndc_scene(C, **scene)
    state = {k: v.detach().clone().contiguous() for k, v in ours.state_dict().items()}
    kw = {k: v for k, v in ours.get_kwargs().items() if k != 'voxel_size_ratio'}
    _default_cuda(True)
    ref = _quiet(_ref_mpi(ref_modules), **kw)
    ref.load_state_dict(state, strict=True)
    return ours, ref.to(DEV), ro, rd, vd


def test_unmodified_dmpigo_runs_on_this_library(ref_modules):
    """The reference's own dmpigo.py over legacy.install(): forward (ray_id / s bit-exact, floats within 1e-5 of scale) and one
    run_train.py-style iteration (mse, entropy_last, distortion, rgbper; TV; MaskedAdam)."""
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200.functional import flatten_eff_distloss
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    try:
        ours, ref, ro, rd, vd = _pair(ref_modules, C=9, n=2048, depth=32, nv=64 ** 3, dmean=-1.0)
        N = len(ro)
        target = torch.rand(N, 3, generator=torch.Generator().manual_seed(3), device='cpu').to(DEV)
        a = ref(ro, rd, vd, global_step=None, **RK)
        b = ours(ro, rd, vd, global_step=None, **RK)
        assert_equal(b['ray_id'], a['ray_id'], 'ray_id')
        assert_equal(b['s'], a['s'], 's')
        assert a['ray_id'].numel() > 1000
        for k in ('rgb_marched', 'alphainv_last', 'weights', 'raw_alpha', 'raw_rgb', 'depth'):
            assert _stat(b[k], a[k]) <= 1e-5, k
        cfg = dict(lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])
        opt_ours = create_optimizer_or_freeze_model(ours, cfg, global_step=0)
        opt_ref = ref_modules.adam.MaskedAdam([{'params': [ref.density.grid], 'lr': 0.1, 'skip_zero_grad': True},
                                               {'params': [ref.k0.grid], 'lr': 0.1, 'skip_zero_grad': True},
                                               {'params': list(ref.rgbnet.parameters()), 'lr': 1e-3, 'skip_zero_grad': False}])
        for m, opt in ((ref, opt_ref), (ours, opt_ours)):
            out = m(ro, rd, vd, global_step=1, **RK)
            opt.zero_grad(set_to_none=True)
            loss = F.mse_loss(out['rgb_marched'], target)
            pout = out['alphainv_last'].clamp(1e-6, 1 - 1e-6)
            loss = loss + 1e-3 * (-(pout * torch.log(pout) + (1 - pout) * torch.log(1 - pout)).mean())
            loss = loss + 1e-2 * flatten_eff_distloss(out['weights'], out['s'], 1 / out['n_max'], out['ray_id'])
            rgbper = (out['raw_rgb'] - target[out['ray_id']]).pow(2).sum(-1)
            loss = loss + 1e-2 * (rgbper * out['weights'].detach()).sum() / N
            loss.backward()
            m.density_total_variation_add_grad(1e-6 / N, True)
            m.k0_total_variation_add_grad(1e-7 / N, True)
        ref_sd, ours_named = dict(ref.named_parameters()), dict(ours.named_parameters())
        assert _stat(ours_named['density.grid'].grad, ref_sd['density.grid'].grad) <= 2e-5
        gk, gr = ours_named['k0.grid'].grad, ref_sd['k0.grid'].grad
        assert ((gk - gr).abs() > 1e-5 * gr.abs().max()).float().mean().item() <= 1e-3
        for k, v in ours_named.items():
            if k.startswith('rgbnet'):
                assert _stat(v.grad, ref_sd[k].grad) <= 5e-4, k
        for k, v in ours_named.items():
            if v.grad is not None:
                g = ref_sd[k].grad.detach().clone()
                v.grad = G._as_cl3d(g) if g.dim() == 5 else g
        opt_ref.step()
        opt_ours.step()
        for k, v in ours.state_dict().items():
            if k in ('density.grid', 'k0.grid') or k.startswith('rgbnet'):
                assert torch.equal(v, ref.state_dict()[k]), f'{k} after MaskedAdam.step differs'
    finally:
        _default_cuda(False)


def test_grid_maintenance_matches_reference(ref_modules):
    """update_occupancy_cache, act_shift -= x, scale_volume_grid (+ mask rebuild) and update_occupancy_cache_lt_nviews against the
    staged reference class: masks element for element, grids within 1e-6."""
    try:
        ours, ref, ro, rd, vd = _pair(ref_modules, C=9, n=1024, depth=32, nv=40 ** 3, dmean=-2.0, mask_p=1.0)
        with torch.no_grad():
            for m in (ours, ref):
                _quiet(m.update_occupancy_cache)
            assert_equal(ours.mask_cache.mask, ref.mask_cache.mask, 'update_occupancy_cache')
            for m in (ours, ref):
                m.act_shift -= 0.25
            assert_equal(ours.act_shift.grid, ref.act_shift.grid, 'act_shift -= x')
            for m in (ours, ref):
                _quiet(m.scale_volume_grid, 48 ** 3, 32)
            assert torch.equal(ours.world_size.cpu(), ref.world_size.cpu())
            assert _stat(ours.density.grid, ref.density.grid) <= 1e-6 and _stat(ours.k0.grid, ref.k0.grid) <= 1e-6
            assert_equal(ours.mask_cache.mask, ref.mask_cache.mask, 'scale_volume_grid mask rebuild')
        rk = dict(RK, render_depth=False)
        imsz = [512, 512]
        for m in (ours, ref):
            _quiet(m.update_occupancy_cache_lt_nviews, ro, rd, imsz, rk, 2)
        assert_equal(ours.mask_cache.mask, ref.mask_cache.mask, 'update_occupancy_cache_lt_nviews')
    finally:
        _default_cuda(False)


def test_checkpoints_interchange(ref_modules, tmp_path):
    from unboundednerfpytorch_b200 import ckpt, models
    try:
        ours, ref, ro, rd, vd = _pair(ref_modules, C=9, n=256, depth=16, nv=32 ** 3)
        p_ours = str(tmp_path / 'ours.tar')
        ckpt.save_checkpoint(3, ours, None, p_ours)
        c = torch.load(p_ours, weights_only=False)
        kw = {k: v for k, v in c['model_kwargs'].items() if k != 'voxel_size_ratio'}
        r2 = _quiet(_ref_mpi(ref_modules), **kw)
        r2.load_state_dict(c['model_state_dict'], strict=True)
        p_ref = str(tmp_path / 'ref.tar')
        torch.save({'global_step': 3, 'model_kwargs': ref.get_kwargs(), 'model_state_dict': ref.state_dict(),
                    'optimizer_state_dict': {}}, p_ref)
    finally:
        _default_cuda(False)
    o2 = ckpt.load_model(models.DirectMPIGO, p_ref, DEV)
    a, b = o2(ro, rd, vd, **RK), ours(ro, rd, vd, **RK)
    assert_equal(a['rgb_marched'], b['rgb_marched'], 'reloaded reference checkpoint renders the same')


def test_render_viewpoints_ndc_equals_chunked_forward():
    from unboundednerfpytorch_b200 import rays as R
    from unboundednerfpytorch_b200 import render
    m, _, _, _ = _ndc_scene(9, depth=32, nv=48 ** 3)
    H, W = 60, 80
    K = np.array([[70., 0., 40.], [0., 70., 30.], [0., 0., 1.]])
    c2w = np.concatenate([np.eye(3), np.array([[0.], [0.], [0.]])], 1).astype(np.float32)
    rk = dict(RK)
    rgbs, depths, bgmaps = render.render_viewpoints(None, m, [c2w], [[H, W]], [K], True, rk, chunk=1024)
    ro, rd, vd = R.get_rays_of_a_view(H, W, K, torch.as_tensor(c2w), True, False, False, False)
    ro, rd, vd = (t.reshape(-1, 3).to(DEV) for t in (ro, rd, vd))
    with torch.no_grad():
        outs = [m(a, b, c, **rk) for a, b, c in zip(ro.split(1024), rd.split(1024), vd.split(1024))]
    rgb = torch.cat([o['rgb_marched'] for o in outs]).reshape(H, W, 3).cpu().numpy()
    dep = torch.cat([o['depth'] for o in outs]).reshape(H, W, 1).cpu().numpy()
    assert np.array_equal(rgbs[0], rgb) and np.array_equal(depths[0], dep)
    assert (bgmaps[0] < 0.999).mean() > 0.1          # the frame is not empty


def test_training_steps_reduce_loss():
    """100 steps of fwd + bwd + TV + MaskedAdam on a teacher / student pair of forward-facing scenes."""
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    teacher, ro, rd, vd = _ndc_scene(9, depth=32, nv=48 ** 3, seed=1, dmean=0.0)
    student, _, _, _ = _ndc_scene(9, depth=32, nv=48 ** 3, seed=2, dmean=-2.0, dstd=0.1, thres=1e-4)
    with torch.no_grad():
        student.mask_cache.mask.fill_(True)
        target = teacher(ro, rd, vd, **RK)['rgb_marched']
    cfg = dict(lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])
    opt = create_optimizer_or_freeze_model(student, cfg, global_step=0)
    losses = []
    for it in range(1, 101):
        ret = student(ro, rd, vd, global_step=it, **RK)
        opt.zero_grad(set_to_none=True)
        loss = F.mse_loss(ret['rgb_marched'], target)
        loss.backward()
        student.density_total_variation_add_grad(1e-6 / len(ro), it < 50)
        student.k0_total_variation_add_grad(1e-7 / len(ro), it < 50)
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.9 * losses[0], losses[::10]
    assert all(torch.isfinite(p).all() for p in student.parameters())
