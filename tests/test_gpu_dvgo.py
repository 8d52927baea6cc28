"""GPU tests of DirectVoxGO's fused box march (march.BoxMarch: csrc/march.cu with BoxSampler + the lane-per-sample feature read of
csrc/march_ndc.cu) against the op-by-op composition forward_ops, the ray geometries where the AABB sampling changes, and the
coarse-to-fine schedule of run_train.py (maskout, per-voxel lr, mask_cache_path, pg_scale rescaling, checkpoints)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.util import assert_equal

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
RK = dict(near=0.2, far=1e9, bg=1., rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False, render_depth=True)
LO, HI = [-1.0, -1.3, -0.6], [1.1, 1.2, 0.8]          # a non-cubic box


def _scene(C, nv=40 ** 3, n=2048, seed=3, thres=1e-4, mask_p=0.85, direct=True):
    """Seeded object-in-box scene: density peaked around the box centre, random k0, a mask cache with holes, cameras on a shell
    around the box looking at points inside it."""
    from unboundednerfpytorch_b200 import models
    g = torch.Generator().manual_seed(seed)
    m = models.DirectVoxGO(xyz_min=LO, xyz_max=HI, num_voxels=nv, num_voxels_base=nv, alpha_init=1e-2, fast_color_thres=thres,
                           rgbnet_dim=0 if C == 3 else C, rgbnet_direct=direct, rgbnet_width=128, rgbnet_depth=3)
    with torch.no_grad():
        X, Y, Z = [int(v) for v in m.world_size]
        ax = [torch.linspace(-1, 1, k) for k in (X, Y, Z)]
        r2 = sum(a ** 2 for a in torch.meshgrid(*ax, indexing='ij'))
        m.density.grid.copy_((6.0 * (0.5 - r2) + torch.randn(X, Y, Z, generator=g))[None, None])
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
        m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=g) < mask_p)
    ro, rd = _shell_rays(n, g)
    return m.to(DEV), ro, rd


def _shell_rays(n, g, radius=3.0):
    c = torch.tensor([(a + b) / 2 for a, b in zip(LO, HI)])
    o = torch.randn(n, 3, generator=g)
    o = c + o / o.norm(dim=-1, keepdim=True) * radius
    tgt = c + (torch.rand(n, 3, generator=g) - 0.5) * torch.tensor([b - a for a, b in zip(LO, HI)])
    d = tgt - o
    return o.to(DEV), d.to(DEV)


def _vd(rd):
    return rd / rd.norm(dim=-1, keepdim=True)


def _run(m, fn, ro, rd, loss_w, rk=RK):
    for p in m.parameters():
        p.grad = None
    ret = fn(ro, rd, _vd(rd), **rk)
    loss = (ret['rgb_marched'] * loss_w).sum() + 0.1 * ret['alphainv_last'].sum() + 1e-2 * ret['weights'].sum()
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    return {k: v.detach() for k, v in ret.items()}, grads


def _close(got, want, tau, what):
    scale = want.abs().max().item()
    err = (got - want).abs().max().item()
    assert err <= tau * max(scale, 1e-30), f'{what}: max |diff| {err:.3e} > {tau} * scale {scale:.3e}'


def _relu_close(got, want, what, tau=1e-5, share=1e-3):
    """Gradients through the ReLU MLP as DESIGN.md §2 judges them: elementwise within tau of scale except a share of voxels whose
    sum of per-sample terms is dominated by a ReLU that flips on last-bit different inputs.  The k0 adjoint itself is pinned at
    1e-5 without an MLP in between (test_gpu_dvgo_reference.test_box_feature_adjoint_is_grid_sample_backward)."""
    bad = ((got - want).abs() > tau * want.abs().max()).float().mean().item()
    assert bad <= share, f'{what}: {bad:.2e} of the elements beyond {tau} of scale'


def _compare(m, ro, rd, C, rk=RK, monkeypatch=None):
    """C = 3 (or a torch rgbnet on both paths): bit-identical colours.  C = 12: forward's rgbnet is the tensor-core one; the
    march's own gradients are then also checked with the torch rgbnet on both paths (``monkeypatch``), where only the scatter
    order differs."""
    from unboundednerfpytorch_b200 import models
    w = torch.rand(len(ro), 3, device=DEV, generator=torch.Generator(DEV).manual_seed(1))
    assert m._fused_ok(rk['stepsize'])
    fused, gf = _run(m, m.forward, ro, rd, w, rk)
    ops, go = _run(m, m.forward_ops, ro, rd, w, rk)
    assert set(fused) == set(ops) == {'alphainv_last', 'weights', 'rgb_marched', 'raw_alpha', 'raw_rgb', 'ray_id', 'depth'}
    assert_equal(fused['ray_id'], ops['ray_id'], 'ray_id')
    for k in ('raw_alpha', 'weights', 'alphainv_last', 'depth'):      # depth = sum w * step_id: equal step ids behind it
        assert_equal(fused[k], ops[k], k)
    if C == 3:
        assert_equal(fused['raw_rgb'], ops['raw_rgb'], 'raw_rgb')
        assert_equal(fused['rgb_marched'], ops['rgb_marched'], 'rgb_marched')
    else:          # the rgbnet moves from cuBLAS to 3xTF32 tensor cores
        _close(fused['raw_rgb'], ops['raw_rgb'], 1e-5, 'raw_rgb')
        _close(fused['rgb_marched'], ops['rgb_marched'], 1e-5, 'rgb_marched')
    _close(gf['density.grid'], go['density.grid'], 1e-5, 'grad density.grid')
    if C == 3:
        _close(gf['k0.grid'], go['k0.grid'], 1e-5, 'grad k0.grid')
    else:
        # through the 3xTF32 rgbnet a voxel's k0 gradient is a sum of many per-sample terms of both signs, each within ~1e-6 of
        # its own size: the sum's error is bounded by the terms, not by the (cancelled) sum, so the scale check is loose here ...
        _relu_close(gf['k0.grid'], go['k0.grid'], 'grad k0.grid (tensor-core rgbnet)')
        if monkeypatch is not None:       # ... and the march's adjoint itself is checked with the same torch rgbnet on both paths
            with monkeypatch.context() as mp:
                mp.setattr(models.shade_mod, 'supported', lambda *a, **k: False)
                _, gt = _run(m, m.forward, ro, rd, w, rk)
            _close(gt['density.grid'], go['density.grid'], 1e-5, 'grad density.grid (torch rgbnet on both paths)')
            # forward_ops reads k0 with ubn_grid_sample_fwd, whose 12-channel accumulation is not F.grid_sample's corner order
            # (the march's read is: test_box_feature_read_is_grid_sample), so the ReLU MLP sees last-bit different features on
            # the two paths and its backward amplifies them; the per-voxel sums cancel, as above
            _relu_close(gt['k0.grid'], go['k0.grid'], 'grad k0.grid (torch rgbnet on both paths)')
    return fused


@pytest.mark.parametrize('thres', [0.0, 1e-4])
@pytest.mark.parametrize('C', [12, 3])
def test_fused_vs_forward_ops(C, thres, monkeypatch):
    m, ro, rd = _scene(C, thres=thres)
    ret = _compare(m, ro, rd, C, monkeypatch=monkeypatch)
    assert len(ret['ray_id']) > 10 * len(ro)          # the rays do march through the object


def test_rgbnet_not_direct_keeps_torch_epilogue():
    m, ro, rd = _scene(12, direct=False)
    assert not m.rgbnet_direct
    _compare(m, ro, rd, 12)


@pytest.mark.parametrize('C', [12, 3])
def test_box_feature_read_is_grid_sample(C):
    """The box march's k0 features against torch's F.grid_sample (the reference's DenseGrid.forward, grid.py:57) at the same
    points: bit-identical."""
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import march, ops
    m, ro, rd = _scene(C, thres=1e-4)
    mscale, mshift, lo, hi = m._mask_geometry()
    stepdist = m._stepdist(RK['stepsize'])
    cfg = march.make_box_cfg(lo, hi, RK['near'], stepdist, float(m.act_shift), 0.5, 1e-4, m.mask_cache.mask, mscale, mshift)
    with torch.no_grad():
        _, _, _, k0, ray_id, step_id = march.BoxMarch.apply(
            m.density.grid, m.k0.grid, ro, rd, m.mask_cache.mask, cfg, G.grid_desc(m.density.grid, *m.density._bounds(), 0),
            G.grid_desc(m.k0.grid, *m.k0._bounds(), 0))
        pts, _, rid, sid = ops.sample_pts_on_rays(ro, rd, m.xyz_min, m.xyz_max, RK['near'], 1e9, stepdist)[:4]
        # the march's records are sorted by (ray, step): locate them in the ragged sample list
        n_steps = torch.bincount(rid, minlength=len(ro))
        start = torch.cumsum(n_steps, 0) - n_steps
        p = pts[start[ray_id] + step_id]
        grid = m.k0.grid.contiguous()
        ind = ((p - m.xyz_min) / (m.xyz_max - m.xyz_min)).flip((-1,)) * 2 - 1
        want = F.grid_sample(grid, ind.reshape(1, 1, 1, -1, 3), mode='bilinear', align_corners=True).reshape(C, -1).T
    assert len(k0) > 1000
    assert_equal(k0, want.contiguous(), f'k0 C={C} vs F.grid_sample')


def test_ray_geometry(monkeypatch):
    """Rays that miss the box, start inside it, have a zero direction component, graze a face or an edge, or run the longest
    diagonal (n_steps at its largest)."""
    m, _, _ = _scene(12, thres=1e-4)
    lo, hi = torch.tensor(LO), torch.tensor(HI)
    c = (lo + hi) / 2
    o, d = [], []
    o += [torch.tensor([5., 5., 5.]), torch.tensor([-4., 0., 0.])]; d += [torch.tensor([1., 0.2, 0.1]), torch.tensor([0., 1., 0.])]   # miss
    o += [c, c + 0.1]; d += [torch.tensor([0.3, -0.2, 0.9]), torch.tensor([-1., 0.5, 0.])]                                      # inside
    o += [torch.tensor([-3., 0.1, 0.2])]; d += [torch.tensor([1., 0., 0.])]                                                    # zero comps
    o += [torch.tensor([-3., float(HI[1]), 0.1])]; d += [torch.tensor([1., 0., 0.])]                                           # on a face
    o += [torch.tensor([-3., float(HI[1]), float(LO[2])])]; d += [torch.tensor([1., 0., 0.])]                                  # on an edge
    o += [lo - (hi - lo) * 0.5]; d += [hi - lo]                                                                                # diagonal
    o += [hi]; d += [lo - hi]                                                                                                  # corner in
    ro = torch.stack(o).to(DEV)
    rd = torch.stack(d).to(DEV)
    ret = _compare(m, ro, rd, 12, monkeypatch=monkeypatch)
    n_miss = 2
    assert not (ret['ray_id'] < n_miss).any()
    assert torch.equal(ret['alphainv_last'][:n_miss].cpu(), torch.ones(n_miss))
    assert torch.equal(ret['rgb_marched'][:n_miss].cpu(), torch.ones(n_miss, 3))
    # the diagonal ray's n_steps against the host bound
    from unboundednerfpytorch_b200 import march, ops
    stepdist = m._stepdist(RK['stepsize'])
    t_min, t_max = ops.infer_t_minmax(ro, rd, m.xyz_min, m.xyz_max, RK['near'], 1e9)
    n_steps = ops.infer_n_samples(rd, t_min, t_max, stepdist)
    assert int(n_steps.max()) <= march.box_s_max(LO, HI, stepdist)
    assert int(n_steps[-2]) >= march.box_s_max(LO, HI, stepdist) - 8          # the diagonal runs (almost) to the bound


def test_overflow_is_an_error():
    """A ray with more steps than the record stride fails the march instead of being cut short."""
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import march
    m, ro, rd = _scene(12)
    mscale, mshift, lo, hi = m._mask_geometry()
    cfg = march.make_box_cfg(lo, hi, RK['near'], m._stepdist(0.5), float(m.act_shift), 0.5, 1e-4, m.mask_cache.mask, mscale, mshift)
    cfg.s_max = 16
    ddesc = G.grid_desc(m.density.grid, *m.density._bounds(), 0)
    kdesc = G.grid_desc(m.k0.grid, *m.k0._bounds(), 0)
    with pytest.raises(RuntimeError, match='s_max'):
        march.BoxMarch.apply(m.density.grid, m.k0.grid, ro, rd, m.mask_cache.mask, cfg, ddesc, kdesc)


def test_nerf_synthetic_fine_shape_fused_vs_ops(monkeypatch):
    """160^3 voxels, 12-channel k0, 8192 rays, stepsize 0.5, alpha_init 1e-2, fast_color_thres 1e-4."""
    m, ro, rd = _scene(12, nv=160 ** 3, n=8192, seed=11, mask_p=1.0)
    _compare(m, ro, rd, 12, monkeypatch=monkeypatch)


def test_maskout_and_count_views_match_torch():
    m, ro, rd = _scene(3, nv=32 ** 3, thres=0.0)
    cams = torch.tensor([[0.9, 1.1, 0.7], [-0.9, -1.2, -0.5], [3., 3., 3.]], device=DEV)
    before = m.density.grid.detach().clone()
    m.maskout_near_cam_vox(cams, 0.4)
    X, Y, Z = [int(v) for v in m.world_size]
    xyz = torch.stack(torch.meshgrid(*[torch.linspace(LO[a], HI[a], s, device=DEV) for a, s in enumerate((X, Y, Z))],
                                     indexing='ij'), -1)
    near = (xyz.unsqueeze(-2) - cams).pow(2).sum(-1).sqrt().amin(-1) <= 0.4          # dvgo.py:190-197
    want = before.clone()
    want[near[None, None]] = -100
    assert near.any() and not near.all()
    assert_equal(m.density.grid.detach(), want, 'maskout_near_cam_vox')
    # voxel_count_views: the reference's autograd formulation (dvgo.py:248-277) on two "views"
    g = torch.Generator().manual_seed(4)
    ro2, rd2 = _shell_rays(2 * 24 * 32, g)
    ro2, rd2 = ro2.reshape(2 * 24, 32, 3), rd2.reshape(2 * 24, 32, 3)
    cnt = m.voxel_count_views(ro2, rd2, [24, 24], 0.2, 1e9, 0.5)
    N_samples = int(np.linalg.norm(np.array([X, Y, Z]) + 1) / 0.5) + 1
    rng = torch.arange(N_samples, device=DEV)[None].float()
    want = torch.zeros_like(cnt)
    lo, hi = m.xyz_min, m.xyz_max
    for o_, d_ in zip(ro2.split(24), rd2.split(24)):
        o_, d_ = o_.reshape(-1, 3), d_.reshape(-1, 3)
        ones = torch.zeros(1, 1, X, Y, Z, device=DEV, requires_grad=True)
        vec = torch.where(d_ == 0, torch.full_like(d_, 1e-6), d_)
        t_min = torch.minimum((hi - o_) / vec, (lo - o_) / vec).amax(-1).clamp(min=0.2, max=1e9)
        step = 0.5 * m.voxel_size.to(DEV) * rng
        pts = o_[..., None, :] + d_[..., None, :] * (t_min[..., None] + step / d_.norm(dim=-1, keepdim=True))[..., None]
        ind = ((pts - lo) / (hi - lo)).flip((-1,)) * 2 - 1
        F.grid_sample(ones, ind.reshape(1, 1, 1, -1, 3), mode='bilinear', align_corners=True).sum().backward()
        want += (ones.grad > 1)
    # the scatter order differs from autograd's, so a voxel whose weight sum is within rounding of 1 may count differently
    assert (cnt != want).float().mean().item() < 1e-3 and cnt.sum() > 0


def test_coarse_to_fine_end_to_end(tmp_path):
    """run_train.py's default bounded-scene schedule: coarse stage (maskout, count views, per-voxel lr, update of the mask from
    the counts), checkpoint, fine model from mask_cache_path built on the host then moved, pg_scale rescaling, 100 steps whose
    loss decreases, and load_model of the fine checkpoint."""
    from unboundednerfpytorch_b200 import ckpt, models
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    teacher, ro, rd = _scene(12, nv=48 ** 3, n=4096, seed=21, mask_p=1.0)
    vd = _vd(rd)
    with torch.no_grad():
        target = teacher(ro, rd, vd, **RK)['rgb_marched']
    # ---- coarse ----
    coarse = models.DirectVoxGO(xyz_min=LO, xyz_max=HI, num_voxels=32 ** 3, num_voxels_base=32 ** 3, alpha_init=1e-6,
                                fast_color_thres=1e-7).to(DEV)
    with torch.no_grad():          # a rough object in free space, as a coarse stage leaves it
        ax = [torch.linspace(-1, 1, int(k), device=DEV) for k in coarse.world_size]
        coarse.density.grid.copy_((30.0 * (0.4 - sum(a ** 2 for a in torch.meshgrid(*ax, indexing='ij'))))[None, None])
    coarse.maskout_near_cam_vox(ro[:64], 0.1)
    cnt = coarse.voxel_count_views(ro.reshape(64, 64, 3), rd.reshape(64, 64, 3), [16] * 4, 0.2, 1e9, 0.5)
    cfg = dict(lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])
    opt = create_optimizer_or_freeze_model(coarse, cfg, global_step=0)
    opt.set_pervoxel_lr(cnt)
    coarse.mask_cache.mask[cnt.squeeze() <= 2] = False
    for it in range(1, 31):
        ret = coarse(ro, rd, vd, global_step=it, **RK)
        opt.zero_grad(set_to_none=True)
        F.mse_loss(ret['rgb_marched'], target).backward()
        opt.step()
    coarse_path = str(tmp_path / 'coarse_last.tar')
    ckpt.save_checkpoint(30, coarse, opt, coarse_path)
    # ---- fine, from the coarse file (constructed on the host, then moved: run_train.create_new_model) ----
    fine = models.DirectVoxGO(xyz_min=LO, xyz_max=HI, num_voxels=24 ** 3, num_voxels_base=40 ** 3, alpha_init=1e-2,
                              fast_color_thres=1e-4, mask_cache_path=coarse_path, mask_cache_thres=1e-3, rgbnet_dim=12,
                              rgbnet_direct=True, mask_cache_world_size=[int(v) for v in coarse.world_size])
    fine = fine.to(DEV)
    ref = G.MaskGrid(path=coarse_path, mask_cache_thres=1e-3).to(DEV)
    ws = [int(v) for v in coarse.world_size]
    xyz = torch.stack(torch.meshgrid(*[torch.linspace(LO[a], HI[a], ws[a], device=DEV) for a in range(3)], indexing='ij'), -1)
    assert_equal(fine.mask_cache.mask, ref(xyz), 'fine mask from mask_cache_path')
    assert 0 < fine.mask_cache.mask.float().mean() < 1
    opt = create_optimizer_or_freeze_model(fine, cfg, global_step=0)
    losses = []
    for it in range(1, 101):
        if it in (20, 40, 60):        # pg_scale
            fine.scale_volume_grid(int(fine.num_voxels * 2))
            opt = create_optimizer_or_freeze_model(fine, cfg, global_step=it)
        ret = fine(ro, rd, vd, global_step=it, **RK)
        opt.zero_grad(set_to_none=True)
        loss = F.mse_loss(ret['rgb_marched'], target) + 1e-3 * ret['weights'].sum() / len(ro)
        loss.backward()
        opt.step()
        losses.append(F.mse_loss(ret['rgb_marched'], target).item())
    assert losses[-1] < 0.7 * losses[0], losses[::10]
    hit = fine.hit_coarse_geo(ro, rd, **RK)
    assert hit.any()
    fine.update_occupancy_cache()
    fine_path = str(tmp_path / 'fine_last.tar')
    ckpt.save_checkpoint(100, fine, opt, fine_path)
    import os
    os.remove(coarse_path)            # the fine checkpoint's own mask supersedes the coarse file it names
    loaded = ckpt.load_model(models.DirectVoxGO, fine_path, DEV)
    assert loaded.get_kwargs()['mask_cache_path'] == coarse_path
    sa, sb = fine.state_dict(), loaded.state_dict()
    assert set(sa) == set(sb)
    for k in sa:
        assert_equal(sa[k], sb[k], f'loaded {k}')
    # voxel_size is re-derived from num_voxels on the host at construction (on the device in scale_volume_grid), so the loaded
    # model's step length may differ in the last bit: the renders agree closely, not bit for bit
    with torch.no_grad():
        a = fine(ro[:512], rd[:512], vd[:512], **RK)
        b = loaded(ro[:512], rd[:512], vd[:512], **RK)
    assert (a['rgb_marched'] - b['rgb_marched']).abs().mean() < 1e-2


def test_render_viewpoints_equals_chunked_forward():
    from unboundednerfpytorch_b200 import rays as R
    from unboundednerfpytorch_b200 import render
    m, _, _ = _scene(12, nv=40 ** 3)
    H, W = 48, 64
    K = np.array([[60., 0., 32.], [0., 60., 24.], [0., 0., 1.]])
    c2w = np.array([[1, 0, 0, 0.05], [0, 1, 0, -0.05], [0, 0, 1, 3.0]], dtype=np.float32)      # looking down -z at the box
    rgbs, depths, bgmaps = render.render_viewpoints(None, m, [c2w], [[H, W]], [K], False, dict(RK), chunk=1024)
    ro, rd, vd = R.get_rays_of_a_view(H, W, K, torch.as_tensor(c2w), False, False, False, False)
    ro, rd, vd = (t.reshape(-1, 3).to(DEV) for t in (ro, rd, vd))
    with torch.no_grad():
        outs = [m(a, b, c, **RK) for a, b, c in zip(ro.split(1024), rd.split(1024), vd.split(1024))]
    rgb = torch.cat([o['rgb_marched'] for o in outs]).reshape(H, W, 3).cpu().numpy()
    assert np.array_equal(rgbs[0], rgb)
    assert (bgmaps[0] < 0.999).mean() > 0.1
