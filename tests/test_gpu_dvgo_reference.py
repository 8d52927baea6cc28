"""DirectVoxGO against the reference itself: the fixtures its unmodified dvgo.py recorded (tests/golden/l2_dvgo/, written by
oracle/make_golden_dvgo.py) through ``forward`` and ``forward_ops``; the reference's GPU path (its dvgo.py over its own CUDA build
in oracle/_ref, oracle/ref_gpu_py.py) at the NeRF-synthetic fine shape; and its dvgo.py over legacy.install() (this library behind
the reference's extension names) for one training iteration with MaskedAdam, per-voxel lr included."""
import contextlib
import io
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_callers_unchanged import PY, _default_cuda, _stat, ref_modules  # noqa: F401  (module-scoped fixture)
from tests.test_gpu_models import _check_against_golden
from tests.util import ROOT, assert_equal, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GOLD = os.path.join(ROOT, 'tests', 'golden', 'l2_dvgo')


def _quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def _build(rec):
    from unboundednerfpytorch_b200 import models
    m = models.DirectVoxGO(**rec['kwargs'])
    m.load_state_dict(rec['state'])
    return m.to(DEV)


@pytest.mark.parametrize('tag', ['coarse', 'fine'])
@pytest.mark.parametrize('path', ['fused', 'ops'])
def test_dvgo_golden(tag, path):
    rec = load_golden(f'l2_dvgo/{tag}.pt')
    m = _build(rec)
    assert path == 'ops' or m._fused_ok(rec['render_kwargs']['stepsize'])
    assert rec['ret']['ray_id'].numel() > 200
    _check_against_golden(m, rec, m.forward if path == 'fused' else m.forward_ops, f'{tag}/{path}')


def test_dvgo_grid_maintenance_golden():
    """maskout_near_cam_vox, voxel_count_views, update_occupancy_cache and scale_volume_grid against the reference's dvgo.py."""
    rec = load_golden('l2_dvgo/maint.pt')
    m = _build(rec)
    mo = rec['maskout']
    m.maskout_near_cam_vox(mo['cam_o'].to(DEV), mo['near_clip'])
    assert_equal(m.density.grid.detach(), mo['density'], 'maskout_near_cam_vox')
    cv = rec['count_views']
    cnt = m.voxel_count_views(cv['rays_o'], cv['rays_d'], cv['imsz'], cv['near'], cv['far'], cv['stepsize'])
    want = cv['count'].to(DEV)
    assert want.sum() > 0
    # autograd's scatter order differs from the kernel's: a voxel whose weight sum is within rounding of 1 may count differently
    assert (cnt != want).float().mean().item() <= 1e-3
    m.update_occupancy_cache()
    assert_equal(m.mask_cache.mask, rec['occupancy']['mask'], 'update_occupancy_cache')
    sc = rec['scale']
    m.scale_volume_grid(sc['num_voxels'])
    assert torch.equal(m.world_size.cpu(), sc['world_size'])
    assert _stat(m.density.grid, sc['density'].to(DEV)) <= 1e-6 and _stat(m.k0.grid, sc['k0'].to(DEV)) <= 1e-6
    assert_equal(m.mask_cache.mask, sc['mask'], 'scale_volume_grid mask rebuild')


def test_mask_cache_path_and_reference_checkpoint_golden():
    """The fine model built from the reference's coarse_last.tar (on the host, then moved, as run_train.create_new_model does)
    has the reference's mask; the reference-written fine_last.tar, whose model_kwargs name that file, loads."""
    from unboundednerfpytorch_b200 import ckpt, models
    want = load_golden('l2_dvgo/fine_mask.pt')
    c = torch.load(os.path.join(GOLD, 'fine_last.tar'), map_location='cpu', weights_only=False)
    kw = dict(c['model_kwargs'], mask_cache_path=os.path.join(GOLD, 'coarse_last.tar'))
    m = models.DirectVoxGO(**kw).to(DEV)
    assert_equal(m.mask_cache.mask, want['mask'], 'mask from mask_cache_path')
    assert 0 < want['mask'].float().mean() < 1
    loaded = ckpt.load_model(models.DirectVoxGO, os.path.join(GOLD, 'fine_last.tar'), DEV)
    assert loaded.get_kwargs()['mask_cache_path'] == 'coarse_last.tar'
    assert_equal(loaded.mask_cache.mask, want['mask'], 'mask of the loaded checkpoint')
    for k, v in c['model_state_dict'].items():
        assert_equal(loaded.state_dict()[k], v, f'loaded {k}')


# ---- the reference's GPU path at the NeRF-synthetic fine shape --------------------------------------------------------------
def _ref_gpu_dvgo():
    from oracle import ref_gpu_py
    why = ref_gpu_py.missing()
    if why is not None:
        if os.environ.get('UBN_ALLOW_NO_REF') == '1':
            pytest.skip(f'{why} missing (UBN_ALLOW_NO_REF=1)')
        pytest.fail(f'{why} is missing: run __graft_entry__.build() where the reference checkout exists')
    ns = ref_gpu_py.load()
    return ref_gpu_py, ns, sys.modules[ref_gpu_py.PKG + '.dvgo']


def _fine_scene(nv=160 ** 3, n=8192, seed=11):
    from tests.test_gpu_dvgo import _scene, _vd
    m, ro, rd = _scene(12, nv=nv, n=n, seed=seed, mask_p=1.0)
    return m, ro, rd, _vd(rd)


def test_nerf_synthetic_fine_shape_vs_reference_gpu():
    """160^3, 12-channel k0, 8192 rays, stepsize 0.5, alpha_init 1e-2, fast_color_thres 1e-4 against the reference's own
    dvgo.py over its own CUDA extension (ATen grid_sample, cuBLAS, its kernels; none of this library's): zero membership flips,
    bit-identical raw_alpha / weights / alphainv_last, colours and depth within 1e-5 of scale; gradients as DESIGN.md §2 judges
    gradients through the ReLU MLP (density exact to atomic order, k0 elementwise with a 1e-3 share of ReLU-flip outliers)."""
    ref_gpu_py, ns, ref_dvgo = _ref_gpu_dvgo()
    m, ro, rd, vd = _fine_scene()
    rk = dict(near=0.2, far=1e9, bg=1., stepsize=0.5, render_depth=True)
    state = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}
    kw = {k: v for k, v in m.get_kwargs().items() if k != 'voxel_size_ratio'}
    # built on the host like ours, then moved: voxel_size is a cube root that the CPU and the GPU may round differently, and the
    # comparison is of the march on one geometry (the step length follows from voxel_size)
    ref = _quiet(ref_dvgo.DirectVoxGO, **kw)
    ref.load_state_dict(state, strict=True)
    ref = ref.to(DEV)
    assert float(ref.voxel_size) == float(m.voxel_size)
    ref_gpu_py.default_cuda(True)
    try:
        a = ref(ro, rd, vd, **rk)
        (a['rgb_marched'].pow(2).sum() + a['alphainv_last'].sum()).backward()
    finally:
        ref_gpu_py.default_cuda(False)
    b = m(ro, rd, vd, **rk)
    (b['rgb_marched'].pow(2).sum() + b['alphainv_last'].sum()).backward()
    assert_equal(b['ray_id'], a['ray_id'], 'ray_id (membership)')
    assert b['ray_id'].numel() > 100000
    for k in ('raw_alpha', 'weights', 'alphainv_last'):
        assert_equal(b[k], a[k], k)
    for k in ('rgb_marched', 'raw_rgb', 'depth'):
        assert _stat(b[k], a[k]) <= 1e-5, k
    gr, go = dict(ref.named_parameters()), dict(m.named_parameters())
    assert _stat(go['density.grid'].grad, gr['density.grid'].grad) <= 2e-5
    gk, gkr = go['k0.grid'].grad, gr['k0.grid'].grad
    assert ((gk - gkr).abs() > 1e-5 * gkr.abs().max()).float().mean().item() <= 1e-3
    for k in go:
        if k.startswith('rgbnet'):
            assert _stat(go[k].grad, gr[k].grad) <= 5e-4, k


# ---- the reference's dvgo.py over legacy.install() ----------------------------------------------------------------------------
def _ref_dvgo(ref_modules):
    sys.path.insert(0, PY)
    try:
        from FourierGrid import dvgo
    finally:
        sys.path.remove(PY)
    return dvgo.DirectVoxGO


@pytest.mark.parametrize('stage', ['coarse', 'fine'])
def test_unmodified_dvgo_runs_on_this_library(ref_modules, stage):
    """Forward and one run_train.py-style iteration of the reference's own dvgo.py over legacy.install() against
    models.DirectVoxGO on the same state: membership bit-exact, floats within 1e-5 of scale; then, on equal gradients, MaskedAdam
    bit for bit -- the coarse stage with per-voxel lr (voxel_count_views -> set_pervoxel_lr, the per-voxel-lr kernel)."""
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    from tests.test_gpu_dvgo import _scene, _vd
    C = 3 if stage == 'coarse' else 12
    ours, ro, rd = _scene(C, nv=48 ** 3, n=2048, seed=5, thres=1e-4 if C == 12 else 1e-7)
    vd = _vd(rd)
    rk = dict(near=0.2, far=1e9, bg=1., stepsize=0.5, render_depth=True)
    state = {k: v.detach().clone().contiguous() for k, v in ours.state_dict().items()}
    kw = {k: v for k, v in ours.get_kwargs().items() if k != 'voxel_size_ratio'}
    try:
        ref = _quiet(_ref_dvgo(ref_modules), **kw)          # on the host like ours (see the test above), then moved
        ref.load_state_dict(state, strict=True)
        ref = ref.to(DEV)
        assert float(ref.voxel_size) == float(ours.voxel_size)
        _default_cuda(True)
        N = len(ro)
        target = torch.rand(N, 3, generator=torch.Generator().manual_seed(3), device='cpu').to(DEV)
        a = ref(ro, rd, vd, global_step=None, **rk)
        b = ours(ro, rd, vd, global_step=None, **rk)
        assert_equal(b['ray_id'], a['ray_id'], 'ray_id')
        assert a['ray_id'].numel() > 1000
        for k in ('rgb_marched', 'alphainv_last', 'weights', 'raw_alpha', 'raw_rgb', 'depth'):
            assert _stat(b[k], a[k]) <= 1e-5, k
        cfg = dict(lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])
        opt_ours = create_optimizer_or_freeze_model(ours, cfg, global_step=0)
        groups = [{'params': [ref.density.grid], 'lr': 0.1, 'skip_zero_grad': True},
                  {'params': [ref.k0.grid], 'lr': 0.1, 'skip_zero_grad': True}]
        if ref.rgbnet is not None:
            groups.append({'params': list(ref.rgbnet.parameters()), 'lr': 1e-3, 'skip_zero_grad': False})
        opt_ref = ref_modules.adam.MaskedAdam(groups)
        if stage == 'coarse':
            ro_v, rd_v = ro[:1536].reshape(48, 32, 3), rd[:1536].reshape(48, 32, 3)
            cnt_ref = _quiet(ref.voxel_count_views, ro_v, rd_v, [16] * 3, 0.2, 1e9, 0.5)
            cnt = ours.voxel_count_views(ro_v, rd_v, [16] * 3, 0.2, 1e9, 0.5)
            assert (cnt != cnt_ref).float().mean().item() <= 1e-3
            opt_ref.set_pervoxel_lr(cnt_ref)
            opt_ours.set_pervoxel_lr(cnt_ref)
        for m, opt in ((ref, opt_ref), (ours, opt_ours)):
            out = m(ro, rd, vd, global_step=1, **rk)
            opt.zero_grad(set_to_none=True)
            loss = F.mse_loss(out['rgb_marched'], target)
            pout = out['alphainv_last'].clamp(1e-6, 1 - 1e-6)
            loss = loss + 1e-3 * (-(pout * torch.log(pout) + (1 - pout) * torch.log(1 - pout)).mean())
            rgbper = (out['raw_rgb'] - target[out['ray_id']]).pow(2).sum(-1)
            loss = loss + 1e-2 * (rgbper * out['weights'].detach()).sum() / N
            loss.backward()
        gr, go = dict(ref.named_parameters()), dict(ours.named_parameters())
        assert _stat(go['density.grid'].grad, gr['density.grid'].grad) <= 2e-5
        gk, gkr = go['k0.grid'].grad, gr['k0.grid'].grad
        assert ((gk - gkr).abs() > 1e-5 * gkr.abs().max()).float().mean().item() <= 1e-3
        for k, v in go.items():
            if v.grad is not None:
                g = gr[k].grad.detach().clone()
                v.grad = G._as_cl3d(g) if g.dim() == 5 else g
        opt_ref.step()
        opt_ours.step()
        for k, v in ours.state_dict().items():
            if k in ('density.grid', 'k0.grid') or k.startswith('rgbnet'):
                assert torch.equal(v, ref.state_dict()[k]), f'{k} after MaskedAdam.step differs'
    finally:
        _default_cuda(False)


def test_box_feature_adjoint_is_grid_sample_backward():
    """BoxMarch's k0 adjoint with a fixed random grad_feat against torch's grid_sampler_3d backward at the same points (no MLP in
    between): within 1e-5 of scale (atomic-add order only)."""
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import march, ops
    from tests.test_gpu_dvgo import RK, _scene
    for C in (12, 3):
        m, ro, rd = _scene(C, thres=1e-4)
        mscale, mshift, lo, hi = m._mask_geometry()
        stepdist = m._stepdist(RK['stepsize'])
        cfg = march.make_box_cfg(lo, hi, RK['near'], stepdist, float(m.act_shift), 0.5, 1e-4, m.mask_cache.mask, mscale, mshift)
        kg = m.k0.grid
        kg.grad = None
        _, _, _, k0, ray_id, step_id = march.BoxMarch.apply(
            m.density.grid.detach(), kg, ro, rd, m.mask_cache.mask, cfg, G.grid_desc(m.density.grid, *m.density._bounds(), 0),
            G.grid_desc(kg, *m.k0._bounds(), 0))
        gfeat = torch.randn(k0.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(7))
        (k0 * gfeat).sum().backward()
        with torch.no_grad():
            pts, _, rid = ops.sample_pts_on_rays(ro, rd, m.xyz_min, m.xyz_max, RK['near'], 1e9, stepdist)[:3]
            n_steps = torch.bincount(rid, minlength=len(ro))
            p = pts[(torch.cumsum(n_steps, 0) - n_steps)[ray_id] + step_id]
            ind = ((p - m.xyz_min) / (m.xyz_max - m.xyz_min)).flip((-1,)) * 2 - 1
        ref = kg.detach().contiguous().clone().requires_grad_(True)
        out = F.grid_sample(ref, ind.reshape(1, 1, 1, -1, 3), mode='bilinear', align_corners=True).reshape(C, -1).T
        (out * gfeat).sum().backward()
        assert len(k0) > 1000
        assert _stat(kg.grad, ref.grad) <= 1e-5, f'C={C}'
