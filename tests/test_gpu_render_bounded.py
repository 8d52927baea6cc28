"""GPU: the fused whole-frame render of DirectVoxGO (box march, ubn_render_box) and DirectMPIGO (NDC march, ubn_render_ndc),
csrc/render_bounded.cu, against model.forward under no_grad, an fp64 restatement and the reference's own GPU path.

* alphainv_last bit-identical to forward's; n_shaded equal to forward's kept samples up to the ray's stop; n_marched the samples
  of the 32-sample chunks up to the stop, clamped to the ray's own n_steps;
* rgb_marched within 1e-5 of forward and of fp64 (forward's survivors up to the stop, their fp32 weights, the k0 read with
  F.grid_sample in float64, the rgbnet and the sums in float64); depth within a bound from the number of summed terms (box depths
  are sums of w * step_id and reach S_max);
* box ray geometry, the S_max overflow, mask caches, batching, whole frames within 64 B per ray, the reference, and the routing of
  render.render_rays / render_viewpoints with fused_frame at its default and on.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.util import assert_equal

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
RK_BOX = dict(near=0.2, far=1e9, bg=1., rand_bkgd=False, stepsize=0.5, render_depth=True)
RK_NDC = dict(near=0., far=1., bg=1, rand_bkgd=False, stepsize=0.5, render_depth=True)
LO, HI = [-1.0, -1.3, -0.6], [1.1, 1.2, 0.8]          # a non-cubic box
# (k0 channels, viewbase_pe, width); None: no rgbnet, sigmoid(k0)
BOX_SHAPES = {'c12': (12, 4, 128), 'c9': (9, 4, 64), 'sig': None}
NDC_SHAPES = {'c9': (9, 0, 64), 'sig': None}
U = 2.0 ** -24


# ---- fixtures ---------------------------------------------------------------------------------------------------------------
def _shell_rays(n, g, radius=3.0):
    c = torch.tensor([(a + b) / 2 for a, b in zip(LO, HI)])
    o = torch.randn(n, 3, generator=g)
    o = c + o / o.norm(dim=-1, keepdim=True) * radius
    tgt = c + (torch.rand(n, 3, generator=g) - 0.5) * torch.tensor([b - a for a, b in zip(LO, HI)])
    d = tgt - o
    return o.to(DEV), d.to(DEV), (d / d.norm(dim=-1, keepdim=True)).to(DEV)


def _box(shape, thres, scene, nv=40 ** 3, n=2048, seed=3, mask_p=1.0, **kw):
    """DirectVoxGO on an object-in-box scene.  'dense': density N(0, 1) (alpha_init 1e-2), rays rarely stop; 'opaque': a solid
    ball of high density in the middle of the box, most rays that reach it stop there."""
    from unboundednerfpytorch_b200 import models
    g = torch.Generator().manual_seed(seed)
    sh = BOX_SHAPES[shape]
    args = dict(rgbnet_dim=0) if sh is None else dict(rgbnet_dim=sh[0], viewbase_pe=sh[1], rgbnet_width=sh[2], rgbnet_direct=True)
    args.update(kw)
    m = models.DirectVoxGO(xyz_min=LO, xyz_max=HI, num_voxels=nv, num_voxels_base=nv, alpha_init=1e-2, fast_color_thres=thres,
                           rgbnet_depth=3, **args)
    with torch.no_grad():
        X, Y, Z = [int(v) for v in m.world_size]
        ax = [torch.linspace(-1, 1, k) for k in (X, Y, Z)]
        r2 = sum(a ** 2 for a in torch.meshgrid(*ax, indexing='ij'))
        d = torch.randn(X, Y, Z, generator=g)
        if scene == 'opaque':
            d = d + torch.where(r2 < 0.5, 40.0, 0.0)
        m.density.grid.copy_(d[None, None])
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
        m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=g) < mask_p)
    ro, rd, vd = _shell_rays(n, g)
    return m.to(DEV), ro, rd, vd


def _ndc(shape, thres, scene, depth=32, nv=48 ** 3, n=2048, seed=5, mask_p=1.0):
    """DirectMPIGO on seeded grids.  'dense': density N(-1, 3); 'opaque': four planes of high density half way through."""
    from unboundednerfpytorch_b200 import models
    g = torch.Generator().manual_seed(seed)
    sh = NDC_SHAPES[shape]
    m = models.DirectMPIGO(xyz_min=[-1.4, -1.1, -1.], xyz_max=[1.4, 1.1, 1.], num_voxels=nv, mpi_depth=depth,
                           rgbnet_dim=0 if sh is None else sh[0], rgbnet_width=64, fast_color_thres=thres)
    with torch.no_grad():
        d = torch.randn(m.density.grid.shape, generator=g) * 3.0 - 1.0
        if scene == 'opaque':
            Z = d.shape[-1]
            d[..., Z // 2:Z // 2 + 4] += 40.0
        m.density.grid.copy_(d)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
        m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=g) < mask_p)
    ro = torch.cat([(torch.rand(n, 2, generator=g) - 0.5) * 3.0, -torch.ones(n, 1)], -1)
    rd = torch.cat([torch.randn(n, 2, generator=g) * 0.3, 2.0 + torch.randn(n, 1, generator=g) * 0.02], -1)
    vd = rd / rd.norm(dim=-1, keepdim=True)
    return m.to(DEV), ro.to(DEV), rd.to(DEV), vd.to(DEV)


def _render(m, ro, rd, vd, rk):
    N = ro.shape[0]
    ns = torch.full((N,), -1, dtype=torch.int32, device=DEV)
    nm = torch.full((N,), -1, dtype=torch.int32, device=DEV)
    with torch.no_grad():
        assert m.render_fused_ok(ro, rk)
        out = m.render_fused(ro, rd, vd, n_shaded=ns, n_marched=nm, **rk)
    return out, ns, nm


def _records(m, ro, rd, rk):
    """Forward's march records (the very march forward runs): weights, alphainv_last, raw_alpha, ray_id, step_id (sorted by
    (ray, step)), each ray's own number of steps, and the sample points of the records."""
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import march, ops
    with torch.no_grad():
        if hasattr(m, 'mpi_depth'):
            cfg, S = m._ndc_cfg(rk)
            descs = [G.grid_desc(g.grid, *g._bounds(), 0) for g in (m.density, m.k0, m.act_shift)]
            w, last, alpha, _, rid, sid = march.NdcMarch.apply(m.density.grid, m.k0.grid, m.act_shift.grid, ro, rd,
                                                               m.mask_cache.mask, cfg, *descs)
            n_steps = torch.full((ro.shape[0],), S, dtype=torch.int64, device=DEV)
            pts = ops.sample_ndc_pts_on_rays(ro.contiguous(), rd.contiguous(), m.xyz_min, m.xyz_max, S)[0][rid, sid]
        else:
            cfg = m._box_cfg(rk)
            ddesc = G.grid_desc(m.density.grid, *m.density._bounds(), 0)
            kdesc = G.grid_desc(m.k0.grid, *m.k0._bounds(), 0)
            w, last, alpha, _, rid, sid = march.BoxMarch.apply(m.density.grid, m.k0.grid, ro, rd, m.mask_cache.mask, cfg, ddesc,
                                                               kdesc)
            stepdist = m._stepdist(rk['stepsize'])
            t_min, t_max = ops.infer_t_minmax(ro.contiguous(), rd.contiguous(), m.xyz_min, m.xyz_max, rk['near'], 1e9)
            n_steps = torch.clamp(ops.infer_n_samples(rd.contiguous(), t_min, t_max, stepdist).long(), max=cfg.s_max)
            p, _, prid = ops.sample_pts_on_rays(ro.contiguous(), rd.contiguous(), m.xyz_min, m.xyz_max, rk['near'], 1e9, stepdist)[:3]
            cnt = torch.bincount(prid, minlength=ro.shape[0])
            start = torch.cumsum(cnt, 0) - cnt
            pts = p[start[rid] + sid]
    return dict(w=w, last=last, alpha=alpha, rid=rid, sid=sid, n_steps=n_steps, pts=pts)


def _stop(rec, N, thres):
    """Per ray, the step at which the transmittance scan stops (the ray's n_steps when it never does), from the listed samples:
    T = float(double(T) * (1 - alpha)), stop at T < 1e-3.  At threshold 0 every queried sample is listed and forward returns all
    of them; above it forward returns only the kept ones and never one after the stop (None: not derivable)."""
    if thres > 0:
        return None
    rid, sid = rec['rid'].cpu().numpy(), rec['sid'].cpu().numpy()
    alpha = rec['alpha'].double().cpu().numpy()
    stop = rec['n_steps'].cpu().numpy().copy()
    T = np.ones(N, dtype=np.float32)
    done = np.zeros(N, dtype=bool)
    for i in range(len(rid)):                     # records are in (ray, step) order
        r = rid[i]
        if done[r]:
            continue
        T[r] = np.float32(np.float64(T[r]) * (1.0 - alpha[i]))
        if np.float64(T[r]) < 1e-3:
            done[r] = True
            stop[r] = sid[i]
    return torch.as_tensor(stop, device=DEV)


def _fp64(m, rec, upto, vd, bg):
    """rgb_marched, depth and the depth error bound from the survivors up to the stop: fp32 weights, the k0 read with F.grid_sample
    in float64, the rgbnet and the sums in float64."""
    from unboundednerfpytorch_b200.models import _view_embed
    N = vd.shape[0]
    rid, sid, w = rec['rid'][upto], rec['sid'][upto], rec['w'][upto].double()
    p = rec['pts'][upto].double()
    mn, mx = m.xyz_min.double(), m.xyz_max.double()
    ind = ((p - mn) / (mx - mn)).flip((-1,)) * 2 - 1
    grid = m.k0.grid.detach().double().contiguous()
    feat = F.grid_sample(grid, ind.reshape(1, 1, 1, -1, 3), mode='bilinear', align_corners=True).reshape(grid.shape[1], -1).T
    if m.rgbnet is None:
        rgb = torch.sigmoid(feat)
    else:
        l1, l2, l3 = m.rgbnet[0], m.rgbnet[2][0], m.rgbnet[3]
        emb = _view_embed(vd.double(), m.viewfreq.double())[rid]
        h = torch.relu(torch.cat([feat, emb], -1) @ l1.weight.double().T + l1.bias.double())
        h = torch.relu(h @ l2.weight.double().T + l2.bias.double())
        rgb = torch.sigmoid(h @ l3.weight.double().T + l3.bias.double())
    col = torch.zeros(N, 3, dtype=torch.float64, device=DEV).index_add_(0, rid, w[:, None] * rgb)
    col = col + rec['last'].double()[:, None] * float(bg)
    term = sid.double() if not hasattr(m, 'mpi_depth') else (sid.double() + 0.5) / rec['n_steps'][0].double()
    depth = torch.zeros(N, dtype=torch.float64, device=DEV).index_add_(0, rid, w * term)
    # a sequential fp32 sum of n rounded products: |error| <= (n + 1) u sum |w term| (+ the rounding of the term itself)
    n = torch.bincount(rid, minlength=N).double()
    bound = (n + 2) * U * depth + 1e-12
    return col, depth, bound


def _check(m, ro, rd, vd, rk, thres, scene):
    N = ro.shape[0]
    out, ns, nm = _render(m, ro, rd, vd, rk)
    with torch.no_grad():
        fwd = m(ro, rd, vd, **rk)
    rec = _records(m, ro, rd, rk)
    assert_equal(rec['last'], fwd['alphainv_last'], 'records are forward\'s')
    assert_equal(out['alphainv_last'], fwd['alphainv_last'], 'alphainv_last')
    stop = _stop(rec, N, thres)
    upto = torch.ones_like(rec['rid'], dtype=torch.bool) if stop is None else rec['sid'] <= stop[rec['rid']]
    assert_equal(ns, torch.bincount(rec['rid'][upto], minlength=N).to(torch.int32), 'n_shaded')
    n_steps = rec['n_steps']
    if stop is not None:
        assert_equal(nm, torch.clamp((stop // 32 + 1) * 32, max=n_steps).to(torch.int32), 'n_marched')
    else:           # at least the chunk of the last kept sample, whole chunks or the ray's end
        last_kept = torch.full((N,), -1, dtype=torch.int64, device=DEV).scatter_reduce_(0, rec['rid'], rec['sid'], 'amax')
        assert bool((nm.long() >= torch.clamp((last_kept // 32 + 1) * 32, max=n_steps) * (last_kept >= 0)).all())
        assert bool(((nm.long() % 32 == 0) | (nm.long() == n_steps)).all()) and bool((nm.long() <= n_steps).all())
    if scene == 'opaque':
        assert (out['alphainv_last'] < 1e-3).float().mean() > 0.1          # many rays stop early
    assert int(ns.sum()) > 0
    err = (out['rgb_marched'] - fwd['rgb_marched']).abs().max().item()
    assert err <= 1e-5, err
    col, depth, bound = _fp64(m, rec, upto, vd, rk['bg'])
    e64 = (out['rgb_marched'].double() - col).abs().max().item()
    assert e64 <= 1e-5, e64
    d_out = out['depth'].double()
    assert bool(((d_out - depth).abs() <= bound).all()), ((d_out - depth).abs() / bound).max().item()
    assert bool(((d_out - fwd['depth'].double()).abs() <= 2 * bound).all()), ((d_out - fwd['depth']).abs() / bound).max().item()
    return out, fwd


BOX_CASES = [(s, t, sc) for s in BOX_SHAPES for t in (0.0, 1e-4) for sc in ('dense', 'opaque')]
NDC_CASES = [(s, t, sc) for s in NDC_SHAPES for t in (0.0, 1e-3) for sc in ('dense', 'opaque')]


@pytest.mark.parametrize('shape,thres,scene', BOX_CASES, ids=[f'{s}-t{t:g}-{sc}' for s, t, sc in BOX_CASES])
def test_box_render_matches_forward_and_fp64(shape, thres, scene):
    m, ro, rd, vd = _box(shape, thres, scene, seed=len(shape) + int(thres > 0))
    _check(m, ro, rd, vd, RK_BOX, thres, scene)


@pytest.mark.parametrize('shape,thres,scene', NDC_CASES, ids=[f'{s}-t{t:g}-{sc}' for s, t, sc in NDC_CASES])
def test_ndc_render_matches_forward_and_fp64(shape, thres, scene):
    m, ro, rd, vd = _ndc(shape, thres, scene, seed=len(shape) + int(thres > 0))
    _check(m, ro, rd, vd, RK_NDC, thres, scene)


def test_box_ray_geometry_and_rays_without_steps():
    """Rays that miss the box, start inside it, have zero direction components, run along a face or an edge, or the diagonals."""
    m, _, _, _ = _box('c12', 1e-4, 'dense')
    lo, hi = torch.tensor(LO), torch.tensor(HI)
    c = (lo + hi) / 2
    o, d = [], []
    o += [torch.tensor([5., 5., 5.]), torch.tensor([-4., 0., 0.])]; d += [torch.tensor([1., 0.2, 0.1]), torch.tensor([0., 1., 0.])]
    o += [c, c + 0.1]; d += [torch.tensor([0.3, -0.2, 0.9]), torch.tensor([-1., 0.5, 0.])]
    o += [torch.tensor([-3., 0.1, 0.2])]; d += [torch.tensor([1., 0., 0.])]
    o += [torch.tensor([-3., float(HI[1]), 0.1])]; d += [torch.tensor([1., 0., 0.])]
    o += [torch.tensor([-3., float(HI[1]), float(LO[2])])]; d += [torch.tensor([1., 0., 0.])]
    o += [lo - (hi - lo) * 0.5]; d += [hi - lo]
    o += [hi]; d += [lo - hi]
    ro, rd = torch.stack(o).to(DEV), torch.stack(d).to(DEV)
    vd = rd / rd.norm(dim=-1, keepdim=True)
    out, fwd = _check(m, ro, rd, vd, RK_BOX, 1e-4, 'dense')
    assert_equal(out['alphainv_last'][:2], torch.ones(2, device=DEV), 'alphainv_last of a miss')
    assert_equal(out['rgb_marched'][:2], torch.ones(2, 3, device=DEV), 'rgb = bg of a miss')
    assert_equal(out['depth'][:2], torch.zeros(2, device=DEV), 'depth of a miss')


def test_box_overflow_raises_as_forward(monkeypatch):
    from unboundednerfpytorch_b200 import march
    m, ro, rd, vd = _box('c12', 1e-4, 'dense', n=256)
    monkeypatch.setattr(march, 'box_s_max', lambda *a: 16)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match='s_max'):
            m(ro, rd, vd, **RK_BOX)
        assert m.render_fused_ok(ro, RK_BOX)
        with pytest.raises(RuntimeError, match='s_max'):
            m.render_fused(ro, rd, vd, **RK_BOX)


@pytest.mark.parametrize('model', ['box', 'ndc'])
def test_mask_cache_with_holes_and_all_zero(model):
    thres = 1e-4 if model == 'box' else 1e-3
    if model == 'box':
        m, ro, rd, vd = _box('c12', thres, 'opaque', mask_p=0.7)
        rk = RK_BOX
    else:
        m, ro, rd, vd = _ndc('c9', thres, 'opaque', mask_p=0.7)
        rk = RK_NDC
    _check(m, ro, rd, vd, rk, thres, 'opaque')
    with torch.no_grad():
        m.mask_cache.mask.zero_()
    out, ns, _ = _render(m, ro, rd, vd, rk)
    N = ro.shape[0]
    assert int(ns.abs().sum()) == 0
    assert_equal(out['alphainv_last'], torch.ones(N, device=DEV), 'alphainv_last without survivors')
    assert_equal(out['rgb_marched'], torch.full((N, 3), float(rk['bg']), device=DEV), 'rgb = bg without survivors')
    assert_equal(out['depth'], torch.zeros(N, device=DEV), 'depth without survivors')


@pytest.mark.parametrize('model,shape,scene', [('box', 'c12', 'dense'), ('box', 'c9', 'opaque'), ('box', 'sig', 'dense'),
                                               ('ndc', 'c9', 'dense'), ('ndc', 'sig', 'opaque')])
def test_batching_permutation_and_rerun_give_the_same_bits(model, shape, scene):
    if model == 'box':
        m, ro, rd, vd = _box(shape, 0.0, scene, n=20000)
        rk = RK_BOX
    else:
        m, ro, rd, vd = _ndc(shape, 0.0, scene, n=20000)
        rk = RK_NDC
    N = ro.shape[0]
    whole, ns, nm = _render(m, ro, rd, vd, rk)
    again, ns2, nm2 = _render(m, ro, rd, vd, rk)
    chunks = [m.render_fused(a, b, c, **rk) for a, b, c in zip(ro.split(8192), rd.split(8192), vd.split(8192))]
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(1)).to(DEV)
    permuted = m.render_fused(ro[perm], rd[perm], vd[perm], **rk)
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(N, device=DEV)
    assert_equal(ns, ns2, 'n_shaded rerun')
    assert_equal(nm, nm2, 'n_marched rerun')
    for k in ('rgb_marched', 'depth', 'alphainv_last'):
        assert_equal(whole[k], again[k], k + ' rerun')
        assert_equal(whole[k], torch.cat([c[k] for c in chunks]), k + ' chunks')
        assert_equal(whole[k], permuted[k][inv], k + ' permuted')


def _frame(model):
    from unboundednerfpytorch_b200 import rays as R
    if model == 'box':
        m, _, _, _ = _box('c12', 1e-4, 'opaque', nv=160 ** 3, n=1)
        H, W = 800, 800
        K = np.array([[1111., 0., 400.], [0., 1111., 400.], [0., 0., 1.]])
        c2w = torch.tensor([[1., 0., 0., 0.05], [0., 1., 0., -0.05], [0., 0., 1., 3.0]])
        ndc, rk = False, RK_BOX
    else:
        m, _, _, _ = _ndc('c9', 1e-3, 'dense', depth=128, nv=256 ** 3, n=1)
        H, W = 756, 1008
        K = np.array([[815., 0., 504.], [0., 815., 378.], [0., 0., 1.]])
        c2w = torch.tensor([[1., 0., 0., 0.], [0., 1., 0., 0.], [0., 0., 1., 0.]])
        ndc, rk = True, RK_NDC
    ro, rd, vd = R._rays_of_a_view(H, W, K, c2w, ndc, False, False, False, 'center', device=DEV)
    return m, ro.reshape(-1, 3), rd.reshape(-1, 3), vd.reshape(-1, 3), rk


@pytest.mark.parametrize('model', ['box', 'ndc'])
def test_whole_frame_in_one_call_within_64_bytes_per_ray(model):
    m, ro, rd, vd, rk = _frame(model)
    N = ro.shape[0]
    with torch.no_grad():
        assert m.render_fused_ok(ro, rk)
        m.render_fused(ro[:16], rd[:16], vd[:16], **rk)          # host geometry cached, mask resolved
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = m.render_fused(ro, rd, vd, **rk)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base - sum(v.numel() * v.element_size() for v in out.values())
    assert extra <= 64 * N, (extra, N)
    assert (out['alphainv_last'] < 0.999).float().mean() > 0.05          # the frame sees the scene
    sl = slice(N // 2, N // 2 + 4096)
    with torch.no_grad():
        fwd = m(ro[sl], rd[sl], vd[sl], **rk)
    assert_equal(out['alphainv_last'][sl], fwd['alphainv_last'], 'alphainv_last')
    assert (out['rgb_marched'][sl] - fwd['rgb_marched']).abs().max() <= 1e-5


def test_box_vs_reference_gpu():
    """A reduced shape against the reference's own dvgo.py over its own CUDA extension (oracle/_ref)."""
    from tests.test_gpu_dvgo_reference import _quiet, _ref_gpu_dvgo
    ref_gpu_py, ns, ref_dvgo = _ref_gpu_dvgo()
    m, ro, rd, vd = _box('c12', 1e-4, 'opaque', nv=48 ** 3, n=2048, seed=7)
    rk = dict(near=0.2, far=1e9, bg=1., stepsize=0.5, render_depth=True)
    state = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}
    kw = {k: v for k, v in m.get_kwargs().items() if k != 'voxel_size_ratio'}
    # built on the host like ours, then moved (voxel_size, and with it the step length, as the CPU rounds it)
    ref = _quiet(ref_dvgo.DirectVoxGO, **kw)
    ref.load_state_dict(state, strict=True)
    ref = ref.to(DEV)
    assert float(ref.voxel_size) == float(m.voxel_size)
    ref_gpu_py.default_cuda(True)
    try:
        with torch.no_grad():
            a = ref(ro, rd, vd, **rk)
    finally:
        ref_gpu_py.default_cuda(False)
    out, _, _ = _render(m, ro, rd, vd, rk)
    assert a['ray_id'].numel() > 10000
    assert_equal(out['alphainv_last'], a['alphainv_last'], 'alphainv_last vs the reference')
    assert (out['rgb_marched'] - a['rgb_marched']).abs().max() <= 1e-5


def test_ndc_vs_reference_gpu():
    """A reduced shape against the reference's own dmpigo.py over its own CUDA extension (oracle/_ref)."""
    from tests.test_gpu_dvgo_reference import _quiet, _ref_gpu_dvgo
    ref_gpu_py, ns, _ = _ref_gpu_dvgo()
    m, ro, rd, vd = _ndc('c9', 1e-3, 'opaque', depth=64, nv=96 ** 3, n=2048, seed=9)
    state = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}
    kw = {k: v for k, v in m.get_kwargs().items() if k != 'voxel_size_ratio'}
    rk = dict(RK_NDC)
    ref_gpu_py.default_cuda(True)
    try:
        ref = _quiet(ns.dmpigo.DirectMPIGO, **kw)
        ref.load_state_dict(state, strict=True)
        with torch.no_grad():
            a = ref.to(DEV)(ro, rd, vd, global_step=None, **rk)
    finally:
        ref_gpu_py.default_cuda(False)
    out, _, _ = _render(m, ro, rd, vd, rk)
    assert a['ray_id'].numel() > 10000
    assert_equal(out['alphainv_last'], a['alphainv_last'], 'alphainv_last vs the reference')
    assert (out['rgb_marched'] - a['rgb_marched']).abs().max() <= 1e-5


# ---- routing ----------------------------------------------------------------------------------------------------------------
def _run(m, ro, rd, vd, rk, **kw):
    from unboundednerfpytorch_b200 import _cabi, render as RD
    timer, _cabi.TIMER = _cabi.TIMER, _cabi.KernelTimer()
    try:
        out = RD.render_rays(m, ro, rd, vd, rk, **kw)
        return out, set(_cabi.TIMER.records)
    finally:
        _cabi.TIMER = timer


def _chunk_loop(m, ro, rd, vd, rk):
    from unboundednerfpytorch_b200 import render as RD
    outs = {k: [] for k in RD.KEYS}
    with torch.no_grad():
        for a, b, c in zip(ro.split(8192), rd.split(8192), vd.split(8192)):
            ret = m(a, b, c, **dict(rk, render_depth=True, coherent_rays=False))
            for k in RD.KEYS:
                outs[k].append(ret[k].reshape(a.shape[0], -1))
    return {k: torch.cat(v) for k, v in outs.items()}


def _models():
    for shape in BOX_SHAPES:
        yield ('box', shape) + _box(shape, 1e-4, 'opaque', n=10000) + (RK_BOX, 'render_box')
    for shape in NDC_SHAPES:
        yield ('ndc', shape) + _ndc(shape, 1e-3, 'dense', n=10000) + (RK_NDC, 'render_ndc')


def test_routing_default_keeps_the_chunk_loop():
    from unboundednerfpytorch_b200 import render as RD
    for kind, shape, m, ro, rd, vd, rk, name in _models():
        out, keys = _run(m, ro, rd, vd, rk)
        assert name not in keys and f'march_{kind}_density_fwd' in keys, (kind, shape, keys)
        want = _chunk_loop(m, ro, rd, vd, rk)
        for k in RD.KEYS:
            assert_equal(out[k], want[k], f'{kind}/{shape} {k}')


def test_routing_fused_frame_takes_the_fused_render():
    from unboundednerfpytorch_b200 import render as RD
    for kind, shape, m, ro, rd, vd, rk, name in _models():
        out, keys = _run(m, ro, rd, vd, rk, fused_frame=True)
        assert keys == {name}, (kind, shape, keys)
        want = m.render_fused(ro, rd, vd, **rk)
        for k in RD.KEYS:
            assert_equal(out[k], want[k].reshape(ro.shape[0], -1), f'{kind}/{shape} {k}')


def test_routing_fused_frame_outside_the_coverage():
    from unboundednerfpytorch_b200 import models, render as RD
    g = torch.Generator().manual_seed(0)
    ro, rd, vd = _shell_rays(5000, g)
    torch.manual_seed(0)
    outside = [
        models.DirectVoxGO(xyz_min=LO, xyz_max=HI, num_voxels=32 ** 3, num_voxels_base=32 ** 3, alpha_init=1e-2,
                           fast_color_thres=1e-4, density_type='TensoRFGrid', density_config=dict(n_comp=8, n_comp_xy=8),
                           k0_type='TensoRFGrid', k0_config=dict(n_comp=24), rgbnet_dim=12, rgbnet_direct=True),
        _box('c12', 1e-4, 'dense', n=1, rgbnet_direct=False)[0],
        _box('c12', 1e-4, 'dense', n=1, rgbnet_width=64)[0],                  # (12, 4, 64): not a covered width
        _box('c9', 1e-4, 'dense', n=1, rgbnet_width=128)[0],                  # (9, 4, 128)
    ]
    for m in outside:
        m = m.to(DEV)
        with torch.no_grad():
            assert not m.render_fused_ok(ro, RK_BOX)
        out, keys = _run(m, ro, rd, vd, RK_BOX, fused_frame=True)
        assert 'render_box' not in keys, keys
        want = _chunk_loop(m, ro, rd, vd, RK_BOX)
        for k in RD.KEYS:
            assert_equal(out[k], want[k], k)
    m, ro, rd, vd = _box('c12', 1e-4, 'dense', n=5000)
    rk_t = dict(RK_BOX, bg=torch.tensor(1.0, device=DEV))
    with torch.no_grad():
        assert m.render_fused_ok(ro, RK_BOX) and not m.render_fused_ok(ro, rk_t)
    out, keys = _run(m, ro, rd, vd, rk_t, fused_frame=True)
    assert 'render_box' not in keys and 'march_box_density_fwd' in keys, keys
    with torch.enable_grad():
        assert not m.render_fused_ok(ro, RK_BOX)
    mn, ro, rd, vd = _ndc('c9', 1e-3, 'dense', n=5000)
    with torch.no_grad():
        assert mn.render_fused_ok(ro, RK_NDC) and not mn.render_fused_ok(ro, dict(RK_NDC, bg=torch.ones(3, device=DEV)))
    with torch.enable_grad():
        assert not mn.render_fused_ok(ro, RK_NDC)


def test_routing_of_contracted_models_is_the_same_under_both_values():
    from tests.test_gpu_render_fused import RK, _model
    from tests.util import seeded_rays
    from unboundednerfpytorch_b200 import render as RD
    ro, rd, vd = seeded_rays(10000, 21, DEV)
    for kind, shape, F_ in (('dcvgo', 'c12', 0), ('fg', 'sig', 0), ('fg', 'c12', 4)):
        m = _model(kind, shape, 0.0, 'dense', F_=F_)
        a, ka = _run(m, ro, rd, vd, RK)
        b, kb = _run(m, ro, rd, vd, RK, fused_frame=True)
        assert ka == kb, (ka, kb)
        assert ('render_contracted' in ka) == (F_ == 0)
        for k in RD.KEYS:
            assert_equal(a[k], b[k], k)


@pytest.mark.parametrize('model', ['box', 'ndc'])
def test_render_viewpoints_fused_frame(model, capsys):
    from unboundednerfpytorch_b200 import render
    if model == 'box':
        m, _, _, _ = _box('c12', 1e-4, 'opaque')
        H, W = 48, 64
        K = np.array([[60., 0., 32.], [0., 60., 24.], [0., 0., 1.]])
        c2w = np.array([[1, 0, 0, 0.05], [0, 1, 0, -0.05], [0, 0, 1, 3.0]], dtype=np.float32)
        ndc, rk = False, dict(RK_BOX)
    else:
        m, _, _, _ = _ndc('c9', 1e-3, 'dense')
        H, W = 60, 80
        K = np.array([[70., 0., 40.], [0., 70., 30.], [0., 0., 1.]])
        c2w = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
        ndc, rk = True, dict(RK_NDC)
    a = render.render_viewpoints(None, m, [c2w], [[H, W]], [K], ndc, rk, chunk=1024)
    b = render.render_viewpoints(None, m, [c2w], [[H, W]], [K], ndc, rk, chunk=1024, fused_frame=True, gt_imgs=a[0],
                                 eval_ssim=True)
    assert np.abs(a[0] - b[0]).max() <= 1e-5
    assert np.array_equal(a[2], b[2])                                        # bgmaps: alphainv_last, bit for bit
    assert (a[2] < 0.999).mean() > 0.1
    # depth: sums of w * term in another order; a term is at most S_max (box) or 1 (NDC)
    d_scale = 512.0 if model == 'box' else 1.0
    assert np.abs(a[1] - b[1]).max() <= 64 * U * d_scale
    out = capsys.readouterr().out
    ssim = float(out.split('Ssim')[1].split()[0])
    assert ssim > 0.999
