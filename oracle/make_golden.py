"""oracle/make_golden.py -- TEST INFRASTRUCTURE ONLY.  Generates tests/golden/*.pt.

Runs the REFERENCE'S OWN Python files (imported unmodified from /root/reference, which exists only in
the build container) on CPU -- grid.py, FourierGrid_grid.py, dvgo.py, dcvgo.py, FourierGrid_model.py,
masked_adam.py -- with the CUDA-only extension modules and the two missing third-party packages replaced
by the CPU oracle (oracle/stubs.py -> oracle/ref_ops.c / cpu_ref.py), and records seeded inputs and the
reference's outputs as small fixtures.  The fixtures travel to the GPU box; /root/reference does not.

    python -m oracle.make_golden          # from the repo root, in the build container

Seed 777 is the reference's default (run_FourierGrid.py:28).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, 'tests', 'golden')
sys.path.insert(0, ROOT)

from oracle import stubs  # noqa: E402

stubs.install('/root/reference')
from FourierGrid import grid as ref_grid  # noqa: E402
from FourierGrid import FourierGrid_grid as ref_fgrid  # noqa: E402
from FourierGrid import dvgo as ref_dvgo  # noqa: E402
from FourierGrid import dcvgo as ref_dcvgo  # noqa: E402
from FourierGrid import FourierGrid_model as ref_fgmodel  # noqa: E402
from FourierGrid import masked_adam as ref_adam  # noqa: E402

SEED = 777


def _save(name, obj):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    torch.save(obj, path)
    print(f'{name}: {os.path.getsize(path) / 1024:.1f} KiB')


def _c(t):
    return t.detach().clone().contiguous()


def _rays(n, gen, spread=0.5):
    ro = (torch.rand(n, 3, generator=gen) - 0.5) * 2 * spread
    rd = torch.randn(n, 3, generator=gen)
    vd = rd / rd.norm(dim=-1, keepdim=True)
    return ro, rd, vd


def golden_grids():
    gen = torch.Generator().manual_seed(SEED)
    out = {}
    xyz_min, xyz_max = [-1.2, -1.0, -0.8], [1.1, 1.3, 0.9]
    for C in (1, 3, 12):
        g = ref_grid.DenseGrid(channels=C, world_size=torch.tensor([5, 6, 7]), xyz_min=xyz_min, xyz_max=xyz_max)
        with torch.no_grad():
            g.grid.copy_(torch.randn(g.grid.shape, generator=gen))
        # points: mostly inside, a few outside the bbox (zero padding) and exactly on the faces
        xyz = torch.rand(61, 3, generator=gen) * (torch.tensor(xyz_max) - torch.tensor(xyz_min)) * 1.2 + torch.tensor(xyz_min) - 0.1 * (torch.tensor(xyz_max) - torch.tensor(xyz_min))
        xyz[0] = torch.tensor(xyz_min)
        xyz[1] = torch.tensor(xyz_max)
        y = g(xyz)
        w = torch.randn(y.shape, generator=gen)
        (y * w).sum().backward()
        out[f'dense_C{C}'] = dict(grid=_c(g.grid), xyz_min=xyz_min, xyz_max=xyz_max, xyz=_c(xyz), out=_c(y), w=_c(w),
                                  grad_grid=_c(g.grid.grad))
    for C, F_ in ((1, 2), (12, 4), (3, 1)):
        g = ref_fgrid.FourierGrid(channels=C, world_size=torch.tensor([6, 5, 7]), xyz_min=[-1.2] * 3, xyz_max=[1.2] * 3,
                                  use_nerf_pos=True, fourier_freq_num=F_, config={})
        with torch.no_grad():
            g.grid.copy_(torch.randn(g.grid.shape, generator=gen))
        xyz = (torch.rand(4, 13, 3, generator=gen) * 2 - 1) * 1.2
        y = g(xyz)
        w = torch.randn(y.shape, generator=gen)
        (y * w).sum().backward()
        out[f'fourier_C{C}_F{F_}'] = dict(grid=_c(g.grid), xyz_min=[-1.2] * 3, xyz_max=[1.2] * 3, num_freqs=F_, xyz=_c(xyz),
                                         out=_c(y), w=_c(w), grad_grid=_c(g.grid.grad))
    # MaskGrid
    mask = torch.rand(6, 7, 5, generator=gen) > 0.4
    mg = ref_grid.MaskGrid(path=None, mask=mask, xyz_min=xyz_min, xyz_max=xyz_max)
    xyz = torch.rand(200, 3, generator=gen) * 3 - 1.5
    out['maskgrid'] = dict(mask=_c(mask), xyz_min=xyz_min, xyz_max=xyz_max, xyz=_c(xyz), out=_c(mg(xyz)),
                           scale=_c(mg.xyz2ijk_scale), shift=_c(mg.xyz2ijk_shift))
    # TV through the module method
    g = ref_grid.DenseGrid(channels=2, world_size=torch.tensor([4, 5, 6]), xyz_min=xyz_min, xyz_max=xyz_max)
    with torch.no_grad():
        g.grid.copy_(torch.randn(g.grid.shape, generator=gen) * 2)
    tv = {}
    for dense in (True, False):
        g.grid.grad = torch.randn(g.grid.shape, generator=gen) * (torch.rand(g.grid.shape, generator=gen) > 0.5)
        g0 = _c(g.grid.grad)
        g.total_variation_add_grad(0.3, 0.2, 0.1, dense)
        tv[f'dense{int(dense)}'] = dict(grad_in=g0, grad_out=_c(g.grid.grad))
    out['tv'] = dict(param=_c(g.grid), wx=0.3, wy=0.2, wz=0.1, **tv)
    _save('l1_grids.pt', out)


def golden_autograd_fns():
    gen = torch.Generator().manual_seed(SEED + 1)
    out = {}
    # ragged rays incl. empty rays and one opaque ray that triggers the T < 1e-3 early stop
    counts = [5, 0, 9, 1, 0, 40, 3]
    ray_id = torch.cat([torch.full((c,), i, dtype=torch.int64) for i, c in enumerate(counts)])
    dens = torch.randn(len(ray_id), generator=gen) * 3
    dens[ray_id == 5] += 9.0                                   # opaque
    dens.requires_grad_(True)
    shift = torch.tensor([-2.0])
    alpha = ref_dvgo.Raw2Alpha.apply(dens, shift, 0.5)
    weights, last = ref_dvgo.Alphas2Weights.apply(alpha, ray_id, len(counts))
    gw = torch.randn(weights.shape, generator=gen)
    gl = torch.randn(last.shape, generator=gen)
    ((weights * gw).sum() + (last * gl).sum()).backward()
    out['chain'] = dict(density=_c(dens), shift=-2.0, interval=0.5, ray_id=_c(ray_id), n_rays=len(counts),
                        alpha=_c(alpha), weights=_c(weights), alphainv_last=_c(last), gw=_c(gw), gl=_c(gl),
                        grad_density=_c(dens.grad))
    d2 = (torch.randn(33, generator=gen) * 2).requires_grad_(True)
    itv = torch.rand(33, generator=gen) + 0.1
    a2 = ref_dvgo.Raw2Alpha_nonuni.apply(d2, 0.3, itv)
    g2 = torch.randn(33, generator=gen)
    (a2 * g2).sum().backward()
    out['nonuni'] = dict(density=_c(d2), shift=0.3, interval=_c(itv), alpha=_c(a2), g=_c(g2), grad_density=_c(d2.grad))
    _save('l1_autograd_fns.pt', out)


def golden_masked_adam():
    gen = torch.Generator().manual_seed(SEED + 2)
    out = {}
    for mode in ('plain', 'masked', 'perlr'):
        p = torch.nn.Parameter(torch.randn(1, 2, 3, 4, 5, generator=gen))
        q = torch.nn.Parameter(torch.randn(7, generator=gen))
        opt = ref_adam.MaskedAdam([{'params': [p], 'lr': 0.1, 'skip_zero_grad': mode == 'masked'},
                                   {'params': [q], 'lr': 1e-3, 'skip_zero_grad': False}])
        if mode == 'perlr':
            opt.set_pervoxel_lr(torch.randint(0, 9, p.shape, generator=gen))
        rec = dict(p0=_c(p), q0=_c(q), per_lr=_c(opt.per_lr) if opt.per_lr is not None else None, grads=[], ps=[], qs=[])
        for step in range(3):
            gp = torch.randn(p.shape, generator=gen) * (torch.rand(p.shape, generator=gen) > 0.5)
            gq = torch.randn(q.shape, generator=gen)
            p.grad, q.grad = gp.clone(), gq.clone()
            opt.step()
            rec['grads'].append((_c(gp), _c(gq)))
            rec['ps'].append(_c(p))
            rec['qs'].append(_c(q))
        out[mode] = rec
    _save('l1_masked_adam.pt', out)


def _grab(model, ret, loss_w):
    """ret_dict tensors + gradients of a fixed scalar functional wrt every parameter."""
    model.zero_grad()
    loss = (ret['rgb_marched'] * loss_w['rgb']).sum() + (ret['alphainv_last'] * loss_w['last']).sum()
    loss = loss + 0.01 * (ret['raw_rgb'].pow(2).sum(-1) * ret['weights'].detach()).sum() + 0.1 * ret['weights'].pow(2).sum()
    loss.backward()
    rec = {k: (_c(v) if torch.is_tensor(v) else v) for k, v in ret.items()}
    rec['grads'] = {n: _c(p.grad) for n, p in model.named_parameters() if p.grad is not None}
    rec['loss'] = float(loss)
    return rec


def golden_models():
    out = {}
    rk = dict(near=0.0, far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False,
              render_depth=True)
    # ---- FourierGridModel ------------------------------------------------------------------------
    for tag, thres, dstd, dmean in (('thres', 1e-4, 3.0, 0.0), ('opaque', 1e-3, 2.0, 7.0)):
        gen = torch.Generator().manual_seed(SEED + 3)
        torch.manual_seed(SEED + 3)
        kw = dict(xyz_min=[-1., -1., -1.], xyz_max=[1., 1., 1.], num_voxels_density=12 ** 3, num_voxels_base_density=12 ** 3,
                  num_voxels_rgb=10 ** 3, num_voxels_base_rgb=10 ** 3, num_voxels_viewdir=-1, alpha_init=1e-2,
                  fast_color_thres=thres, rgbnet_dim=12, fourier_freq_num=2)
        m = ref_fgmodel.FourierGridModel(**kw)
        with torch.no_grad():
            m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=gen) * dstd + dmean)
            m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=gen))
        N = 24
        ro, rd, vd = _rays(N, gen)
        ret = m(ro, rd, vd, global_step=None, is_train=False, **rk)
        lw = dict(rgb=torch.randn(N, 3, generator=gen), last=torch.randn(N, generator=gen))
        rec = _grab(m, ret, lw)
        out[f'fouriergrid_{tag}'] = dict(kwargs=kw, state=m.state_dict(), rays_o=ro, rays_d=rd, viewdirs=vd,
                                         render_kwargs=rk, loss_w=lw, ret=rec)
    # ---- DirectContractedVoxGO -----------------------------------------------------------------------
    for tag, norm, thres, dmean in (('inf', 'inf', 1e-4, 0.0), ('l2_opaque', 'l2', 1e-3, 6.0)):
        gen = torch.Generator().manual_seed(SEED + 4)
        torch.manual_seed(SEED + 4)
        kw = dict(xyz_min=[-1., -1., -1.], xyz_max=[1., 1., 1.], num_voxels=14 ** 3, num_voxels_base=14 ** 3, alpha_init=1e-2,
                  fast_color_thres=thres, contracted_norm=norm, rgbnet_dim=12)
        m = ref_dcvgo.DirectContractedVoxGO(**kw)
        with torch.no_grad():
            m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=gen) * 3 + dmean)
            m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=gen))
            m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=gen) > 0.15)
        N = 24
        ro, rd, vd = _rays(N, gen)
        ret = m(ro, rd, vd, global_step=None, is_train=False, **rk)
        lw = dict(rgb=torch.randn(N, 3, generator=gen), last=torch.randn(N, generator=gen))
        rec = _grab(m, ret, lw)
        out[f'dcvgo_{tag}'] = dict(kwargs=kw, state=m.state_dict(), rays_o=ro, rays_d=rd, viewdirs=vd, render_kwargs=rk,
                                   loss_w=lw, ret=rec)
    # ---- DirectVoxGO (bounded; BASELINE config 1 shape family): sampling + full forward -------------
    gen = torch.Generator().manual_seed(SEED + 5)
    torch.manual_seed(SEED + 5)
    kw = dict(xyz_min=[-1., -1., -1.], xyz_max=[1., 1., 1.], num_voxels=12 ** 3, num_voxels_base=12 ** 3, alpha_init=1e-2,
              fast_color_thres=1e-4, rgbnet_dim=12, rgbnet_direct=True, mask_cache_world_size=[12, 12, 12])
    m = ref_dvgo.DirectVoxGO(**kw)
    with torch.no_grad():
        m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=gen) * 3)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=gen))
    N = 32
    ro = torch.randn(N, 3, generator=gen) * 0.2 + torch.tensor([0., 0., -2.5])
    rd = torch.randn(N, 3, generator=gen) * 0.25 + torch.tensor([0., 0., 1.])
    rd[0, 0] = 0.0                                            # exercise the zero-direction-component branch
    vd = rd / rd.norm(dim=-1, keepdim=True)
    rk2 = dict(near=0.2, far=6.0, bg=1, stepsize=0.5, render_depth=True)
    samp = sys.modules['render_utils_cuda'].sample_pts_on_rays(ro.contiguous(), rd.contiguous(), m.xyz_min, m.xyz_max,
                                                             0.2, 1e9, 0.5 * float(m.voxel_size))
    ret = m(ro, rd, vd, **rk2)
    lw = dict(rgb=torch.randn(N, 3, generator=gen), last=torch.randn(N, generator=gen))
    rec = _grab(m, ret, lw)
    out['dvgo'] = dict(kwargs=kw, state=m.state_dict(), rays_o=ro, rays_d=rd, viewdirs=vd, render_kwargs=rk2, loss_w=lw,
                       ret=rec, stepdist=0.5 * float(m.voxel_size), sample=[_c(t) for t in samp])
    for k, rec in out.items():                 # one file per model record (tests.util.load_golden('l2_models.pt') reassembles them)
        _save(os.path.join('l2_models', k + '.pt'), rec)


from tests.util import cfg1_scene  # noqa: E402  (seeded scene shared with tests/test_gpu_models.py)


def golden_cfg1():
    """SURVEY.md 8c deliverable: the config-1 fixture (64^3, 1024 rays, reference python forward on CPU = torch F.grid_sample path)."""
    kw, dens, k0, net, ro, rd, vd = cfg1_scene()
    torch.manual_seed(SEED + 64)
    m = ref_dvgo.DirectVoxGO(**kw)
    with torch.no_grad():
        m.density.grid.copy_(dens)
        m.k0.grid.copy_(k0)
    m.load_state_dict(net, strict=False)
    rk = dict(near=0.2, far=6.0, bg=1, stepsize=0.5, render_depth=True)
    with torch.no_grad():
        ret = m(ro, rd, vd, **rk)
    ray_id = ret['ray_id']
    _save('l2_cfg1.pt', dict(seed=SEED + 64, render_kwargs=rk, n_survivors=int(ray_id.numel()),
                             per_ray_count=torch.bincount(ray_id, minlength=len(ro)).to(torch.int32),
                             rgb_marched=_c(ret['rgb_marched']), depth=_c(ret['depth']), alphainv_last=_c(ret['alphainv_last']),
                             weights_sum=torch.zeros(len(ro)).index_add_(0, ray_id, ret['weights'])))


def golden_checkpoint():
    """A reference-format checkpoint written by the reference's own classes: FourierGridModel + its MaskedAdam after two steps,
    saved exactly like FourierGridCheckpointManager.save_model (FourierGrid_ckpt_manager.py:44-51) -> tests/golden/ref_fine_last.tar."""
    torch.manual_seed(SEED + 9)
    gen = torch.Generator().manual_seed(SEED + 9)
    kw = dict(xyz_min=np.array([-1., -1., -1.], dtype=np.float32), xyz_max=np.array([1., 1., 1.], dtype=np.float32),
              num_voxels_density=8 ** 3, num_voxels_base_density=8 ** 3, num_voxels_rgb=8 ** 3, num_voxels_base_rgb=8 ** 3,
              num_voxels_viewdir=-1, alpha_init=1e-2, fast_color_thres=1e-4, rgbnet_dim=12, fourier_freq_num=2)
    m = ref_fgmodel.FourierGridModel(**kw)
    with torch.no_grad():
        m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=gen) * 3)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=gen))
    opt = ref_adam.MaskedAdam([{'params': [m.density.grid], 'lr': 0.1, 'skip_zero_grad': True},
                               {'params': [m.k0.grid], 'lr': 0.1, 'skip_zero_grad': True},
                               {'params': list(m.rgbnet.parameters()), 'lr': 1e-3, 'skip_zero_grad': False}])
    ro, rd, vd = _rays(16, gen)
    rk = dict(near=0.0, far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False)
    for it in range(2):
        opt.zero_grad(set_to_none=True)
        m(ro, rd, vd, global_step=it, is_train=True, **rk)['rgb_marched'].sum().backward()
        opt.step()
    path = os.path.join(OUT, 'ref_fine_last.tar')
    torch.save({'global_step': 2, 'model_kwargs': m.get_kwargs(), 'model_state_dict': m.state_dict(),
                'optimizer_state_dict': opt.state_dict()}, path)
    print(f'ref_fine_last.tar: {os.path.getsize(path) / 1024:.1f} KiB')


def golden_rays():
    """dvgo.get_rays_of_a_view / get_training_rays_flatten (dvgo.py:492-612) on small views, every flag combination."""
    g = torch.Generator().manual_seed(SEED + 5)
    rec = {'views': []}
    H, W = 5, 7
    K = np.array([[9.5, 0., 3.4], [0., 9.1, 2.6], [0., 0., 1.]])
    ang = 0.7
    R = torch.tensor([[np.cos(ang), -np.sin(ang), 0.], [np.sin(ang), np.cos(ang), 0.], [0., 0., 1.]], dtype=torch.float32)
    R = R @ torch.tensor([[1., 0., 0.], [0., 0.8, -0.6], [0., 0.6, 0.8]])
    c2w = torch.cat([R, torch.tensor([[0.3], [-0.2], [1.7]])], 1)
    for ndc in (False, True):
        for inverse_y in (False, True):
            for flip_x, flip_y in ((False, False), (True, False), (False, True), (True, True)):
                for mode in ('center', 'lefttop'):
                    o, d, v = ref_dvgo.get_rays_of_a_view(H, W, K, c2w, ndc, inverse_y, flip_x, flip_y, mode=mode)
                    rec['views'].append(dict(H=H, W=W, K=torch.tensor(K), c2w=c2w.clone(), ndc=ndc, inverse_y=inverse_y,
                                             flip_x=flip_x, flip_y=flip_y, mode=mode, rays_o=_c(o), rays_d=_c(d), viewdirs=_c(v)))
    # flattened training set of two views of different size
    imgs = [torch.rand(4, 6, 3, generator=g), torch.rand(5, 3, 3, generator=g)]
    poses = [c2w, torch.cat([R.t().contiguous(), torch.tensor([[-1.0], [0.4], [0.9]])], 1)]
    HW = np.array([[4, 6], [5, 3]])
    Ks = np.stack([K, K * np.array([[0.5], [0.5], [1.0]])])
    import contextlib, io
    with contextlib.redirect_stdout(io.StringIO()):
        out = ref_dvgo.get_training_rays_flatten(imgs, poses, HW, Ks, ndc=False, inverse_y=False, flip_x=False, flip_y=False)
    rec['flatten'] = dict(imgs=imgs, poses=poses, HW=torch.tensor(HW), Ks=torch.tensor(Ks), rgb_tr=_c(out[0]), rays_o_tr=_c(out[1]),
                          rays_d_tr=_c(out[2]), viewdirs_tr=_c(out[3]), imsz=list(out[4]))
    _save('l1_rays.pt', rec)


if __name__ == '__main__':
    torch.set_num_threads(4)
    golden_grids()
    golden_autograd_fns()
    golden_masked_adam()
    golden_models()
    golden_cfg1()
    golden_checkpoint()
    golden_rays()
