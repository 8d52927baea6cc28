"""GPU: the fused whole-frame render of the contracted models (models._ContractedBase.render_fused -> ubn_render_contracted,
csrc/render.cu) against model.forward under no_grad and against an fp64 restatement.

* alphainv_last bit-identical to forward's;
* n_shaded equal, per ray, to forward's returned samples up to the ray's stop (forward lists zero-weight samples after the stop
  when fast_color_thres is 0; the fused march leaves the ray there);
* rgb_marched and depth within 1e-5 of forward, and within 1e-5 of fp64: forward's survivors up to the stop, their (fp32) weights,
  the k0 read with F.grid_sample in float64, the rgbnet and the sums in float64;
* one call, 8192-ray chunks, a permutation and a second run give the same bits;
* edge cases, a full 1600x1067 frame in one call within 64 B per ray of extra memory, and the routing of render.render_rays
  (FourierGridModel with Fourier slabs keeps the chunk loop).
"""
import numpy as np
import pytest
import torch

from tests.util import assert_equal, seeded_rays

DEV = 'cuda:0'
RK = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, render_depth=True)
SHAPES = {'c12': dict(C=12, rgbnet=True, pe=4), 'c3': dict(C=3, rgbnet=True, pe=8), 'sig': dict(C=3, rgbnet=False, pe=4)}


def _model(kind, shape, thres, scene, F_=0, world=24, seed=0, norm='inf'):
    """FourierGridModel (kind 'fg', P = 2 F_ + 1 slabs; the fused render covers F_ = 0) or DirectContractedVoxGO ('dcvgo') with
    random grids.  scene 'dense': density N(0, 1), rays rarely stop; 'opaque': a solid sphere of high density in the middle of the scene, most rays stop early."""
    from unboundednerfpytorch_b200 import models
    sh = SHAPES[shape]
    dim = sh['C'] if sh['rgbnet'] else 0
    torch.manual_seed(seed)
    if kind == 'fg':
        m = models.FourierGridModel(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=world ** 3,
                                    num_voxels_base_density=world ** 3, num_voxels_rgb=world ** 3, num_voxels_base_rgb=world ** 3,
                                    num_voxels_viewdir=-1, alpha_init=1e-4, fast_color_thres=thres, rgbnet_dim=dim,
                                    fourier_freq_num=F_, contracted_norm=norm, viewbase_pe=sh['pe'])
    else:
        m = models.DirectContractedVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=world ** 3, num_voxels_base=world ** 3,
                                         alpha_init=1e-4, fast_color_thres=thres, rgbnet_dim=dim, contracted_norm=norm,
                                         viewbase_pe=sh['pe'])
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        d = torch.randn(m.density.grid.shape, generator=g)
        if scene == 'opaque':
            X, Y, Z = m.density.grid.shape[2:]
            ax = [torch.linspace(-1, 1, n) for n in (X, Y, Z)]
            r = torch.stack(torch.meshgrid(*ax, indexing='ij'), -1).norm(dim=-1)
            d = d + torch.where(r < 0.5, 40.0, 0.0)
        m.density.grid.copy_(d)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
    return m.to(DEV)


def _render(m, ro, rd, vd, rk=RK):
    ns = torch.full((ro.shape[0],), -1, dtype=torch.int32, device=DEV)
    with torch.no_grad():
        assert m.render_fused_ok(ro, rk)
        out = m.render_fused(ro, rd, vd, n_shaded=ns, **rk)
    return out, ns


def _stop_steps(m, fwd, N, S):
    """Per ray, the step at which forward's transmittance scan stops (S when it never does), from forward's listed samples: the
    kernel's recurrence T = float(double(T) * (1 - alpha)), stop at T < 1e-3.  With fast_color_thres > 0 forward keeps only a
    subset of the listed samples, but it never returns one after the stop, so the count below needs the stop only at threshold 0."""
    A = np.zeros((N, S))
    listed = np.zeros((N, S), dtype=bool)
    rid, sid = fwd['ray_id'].cpu().numpy(), fwd['step_id'].cpu().numpy()
    A[rid, sid] = fwd['raw_alpha'].double().cpu().numpy()
    listed[rid, sid] = True
    T = np.ones(N, dtype=np.float32)
    stop = np.full(N, S)
    for s in range(S):
        live = (stop == S) & listed[:, s]
        T = np.where(live, (T.astype(np.float64) * (1.0 - A[:, s])).astype(np.float32), T)
        stop[live & (T.astype(np.float64) < 1e-3)] = s        # the kernel compares the float T with the double 1e-3
    return stop


def _expected_n_shaded(m, fwd, N, S):
    stop = torch.as_tensor(_stop_steps(m, fwd, N, S), device=DEV)
    rid, sid = fwd['ray_id'], fwd['step_id']
    upto = sid <= stop[rid]
    return torch.bincount(rid[upto], minlength=N).to(torch.int32), upto


def _fp64(m, ro, rd, vd, fwd, upto, rk):
    """rgb_marched, depth from forward's survivors up to the stop: weights (fp32, as the kernel uses them), k0 features read in
    float64, the rgbnet and the sums in float64."""
    from oracle import cpu_ref
    from unboundednerfpytorch_b200.models import _view_embed
    N = ro.shape[0]
    rid, sid = fwd['ray_id'][upto], fwd['step_id'][upto]
    w = fwd['weights'][upto].double()
    t = fwd['t'][upto].double()
    pts, _, _ = m._sample_dense(ro, rd, rk['stepsize'])
    F_ = m.k0.num_freqs if m.k0.num_freqs and m.k0.num_freqs > 0 else 0
    feat = cpu_ref.fourier_grid_forward(m.k0.grid.detach().double().contiguous(), pts[rid, sid].double(), m.xyz_min.double(),
                                        m.xyz_max.double(), F_)
    if m.rgbnet is None:
        rgb = torch.sigmoid(feat)
    else:
        l1, l2, l3 = m.rgbnet[0], m.rgbnet[2][0], m.rgbnet[3]
        emb = _view_embed(vd.double(), m.viewfreq.double())[rid]
        x = torch.cat([feat, emb], -1)
        h = torch.relu(x @ l1.weight.double().T + l1.bias.double())
        h = torch.relu(h @ l2.weight.double().T + l2.bias.double())
        rgb = torch.sigmoid(h @ l3.weight.double().T + l3.bias.double())
    col = torch.zeros(N, 3, dtype=torch.float64, device=DEV).index_add_(0, rid, w[:, None] * rgb)
    if m.RENDER_USES_BG:
        col = col + fwd['alphainv_last'].double()[:, None] * float(rk['bg'])
    depth = torch.zeros(N, dtype=torch.float64, device=DEV).index_add_(0, rid, w * (1 - 1 / (1 + t)))
    return col, depth


CASES = [(k, s, t, sc) for k in ('fg', 'dcvgo') for s in SHAPES for t in (0.0, 1e-4) for sc in ('dense', 'opaque')]


@pytest.mark.gpu
@pytest.mark.parametrize('kind,shape,thres,scene', CASES, ids=[f'{k}-{s}-t{t:g}-{sc}' for k, s, t, sc in CASES])
def test_fused_render_matches_forward_and_fp64(kind, shape, thres, scene):
    m = _model(kind, shape, thres, scene, seed=len(kind) + len(shape))
    N = 600
    ro, rd, vd = seeded_rays(N, 11, DEV)
    out, ns = _render(m, ro, rd, vd)
    nm = torch.full((N,), -1, dtype=torch.int32, device=DEV)
    with torch.no_grad():
        m.render_fused(ro, rd, vd, n_marched=nm, **RK)
        fwd = m(ro, rd, vd, **RK)
    S = fwd['n_max']
    assert_equal(out['alphainv_last'], fwd['alphainv_last'], 'alphainv_last')
    want_ns, upto = _expected_n_shaded(m, fwd, N, S)
    assert_equal(ns, want_ns, 'n_shaded')
    # marched: every 32-sample chunk up to the one the ray stops in (the whole ray when it never stops)
    stop = torch.as_tensor(_stop_steps(m, fwd, N, S), device=DEV)
    assert_equal(nm, torch.clamp((stop // 32 + 1) * 32, max=S).to(torch.int32), 'n_marched')
    if scene == 'opaque':
        assert (out['alphainv_last'] < 1e-3).float().mean() > 0.3          # most rays stop early
        assert ((ns % 16) != 0).any()                                         # stops inside partly filled tiles
    else:
        assert int(ns.sum()) > 0
    err_rgb = (out['rgb_marched'] - fwd['rgb_marched']).abs().max().item()
    err_d = (out['depth'] - fwd['depth']).abs().max().item()
    assert err_rgb <= 1e-5 and err_d <= 1e-5, (err_rgb, err_d)
    col, depth = _fp64(m, ro, rd, vd, fwd, upto, RK)
    e64_rgb = (out['rgb_marched'].double() - col).abs().max().item()
    e64_d = (out['depth'].double() - depth).abs().max().item()
    assert e64_rgb <= 1e-5 and e64_d <= 1e-5, (e64_rgb, e64_d)


@pytest.mark.gpu
@pytest.mark.parametrize('kind,shape,scene', [('dcvgo', 'c12', 'dense'), ('fg', 'c3', 'opaque'), ('fg', 'sig', 'dense')])
def test_batching_permutation_and_rerun_give_the_same_bits(kind, shape, scene):
    m = _model(kind, shape, 0.0, scene, seed=3)
    N = 20000
    ro, rd, vd = seeded_rays(N, 5, DEV)
    whole, ns = _render(m, ro, rd, vd)
    again, ns2 = _render(m, ro, rd, vd)
    chunks = [m.render_fused(a, b, c, **RK) for a, b, c in zip(ro.split(8192), rd.split(8192), vd.split(8192))]
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(1)).to(DEV)
    permuted = m.render_fused(ro[perm], rd[perm], vd[perm], **RK)
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(N, device=DEV)
    assert_equal(ns, ns2, 'n_shaded rerun')
    for k in ('rgb_marched', 'depth', 'alphainv_last'):
        assert_equal(whole[k], again[k], k + ' rerun')
        assert_equal(whole[k], torch.cat([c[k] for c in chunks]), k + ' chunks')
        assert_equal(whole[k], permuted[k][inv], k + ' permuted')


@pytest.mark.gpu
def test_zero_and_one_ray():
    m = _model('dcvgo', 'c12', 0.0, 'dense')
    ro, rd, vd = seeded_rays(1, 2, DEV)
    out = m.render_fused(ro[:0], rd[:0], vd[:0], **RK)
    assert all(out[k].shape[0] == 0 for k in out)
    out, ns = _render(m, ro, rd, vd)
    with torch.no_grad():
        fwd = m(ro, rd, vd, **RK)
    assert_equal(out['alphainv_last'], fwd['alphainv_last'], 'alphainv_last')
    assert (out['rgb_marched'] - fwd['rgb_marched']).abs().max() <= 1e-5


@pytest.mark.gpu
def test_rays_without_survivors_and_a_mask_cache_with_holes():
    m = _model('dcvgo', 'c12', 1e-4, 'opaque')
    N = 3000
    ro, rd, vd = seeded_rays(N, 9, DEV)
    g = torch.Generator(device=DEV).manual_seed(4)
    with torch.no_grad():
        m.mask_cache.mask &= torch.rand(m.mask_cache.mask.shape, generator=g, device=DEV) > 0.3
    out, ns = _render(m, ro, rd, vd)
    with torch.no_grad():
        fwd = m(ro, rd, vd, **RK)
    assert_equal(out['alphainv_last'], fwd['alphainv_last'], 'alphainv_last')
    want_ns, _ = _expected_n_shaded(m, fwd, N, fwd['n_max'])
    assert_equal(ns, want_ns, 'n_shaded')
    assert (out['rgb_marched'] - fwd['rgb_marched']).abs().max() <= 1e-5
    with torch.no_grad():
        m.mask_cache.mask.zero_()
    out, ns = _render(m, ro, rd, vd)
    assert int(ns.abs().sum()) == 0
    assert_equal(out['alphainv_last'], torch.ones(N, device=DEV), 'alphainv_last without survivors')
    assert_equal(out['rgb_marched'], torch.ones(N, 3, device=DEV), 'rgb = bg without survivors')
    assert_equal(out['depth'], torch.zeros(N, device=DEV), 'depth without survivors')


@pytest.mark.gpu
@pytest.mark.parametrize('shape', ['c12', 'c3'])
def test_fouriergrid_all_samples_surviving(shape):
    """FourierGridModel at fourier_freq_num 0 with every one of 512+ samples kept (no ray stops): 32 full tiles per ray."""
    rk = dict(RK, stepsize=0.07)
    m = _model('fg', shape, 0.0, 'dense', seed=2)
    with torch.no_grad():
        m.density.grid.fill_(-30.0)                                         # alpha ~ 0: no ray stops, every sample survives
    N = 200
    ro, rd, vd = seeded_rays(N, 13, DEV)
    out, ns = _render(m, ro, rd, vd, rk)
    with torch.no_grad():
        fwd = m(ro, rd, vd, **rk)
    S = fwd['n_max']
    assert S >= 512
    assert int(ns.min()) == S
    assert_equal(out['alphainv_last'], fwd['alphainv_last'], 'alphainv_last')
    assert (out['rgb_marched'] - fwd['rgb_marched']).abs().max() <= 1e-5
    assert (out['depth'] - fwd['depth']).abs().max() <= 1e-5
    _, upto = _expected_n_shaded(m, fwd, N, S)
    col, depth = _fp64(m, ro, rd, vd, fwd, upto, rk)
    assert (out['rgb_marched'].double() - col).abs().max() <= 1e-5
    assert (out['depth'].double() - depth).abs().max() <= 1e-5


@pytest.mark.gpu
def test_full_frame_in_one_call_within_64_bytes_per_ray():
    from unboundednerfpytorch_b200 import rays as R
    m = _model('dcvgo', 'c12', 0.0, 'dense', world=64, norm='l2')
    H, W = 1067, 1600
    K = np.array([[float(W), 0, W / 2], [0, float(W), H / 2], [0, 0, 1]], dtype=np.float64)
    c2w = torch.tensor([[1., 0., 0., 0.15], [0., 1., 0., -0.10], [0., 0., 1., 0.35]])
    ro, rd, vd = R._rays_of_a_view(H, W, K, c2w, False, False, False, False, 'center', device=DEV)
    ro, rd, vd = ro.reshape(-1, 3), rd.reshape(-1, 3), vd.reshape(-1, 3)
    N = ro.shape[0]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = m.render_fused(ro, rd, vd, **RK)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base - sum(v.numel() * v.element_size() for v in out.values())
    assert extra <= 64 * N, (extra, N)
    sl = slice(N // 2, N // 2 + 4096)
    with torch.no_grad():
        fwd = m(ro[sl], rd[sl], vd[sl], **RK)
    assert_equal(out['alphainv_last'][sl], fwd['alphainv_last'], 'alphainv_last')
    assert (out['rgb_marched'][sl] - fwd['rgb_marched']).abs().max() <= 1e-5


@pytest.mark.gpu
def test_render_rays_routing():
    from unboundednerfpytorch_b200 import _cabi, render as RD
    ro, rd, vd = seeded_rays(10000, 21, DEV)

    def run(m, rk=RK):
        timer, _cabi.TIMER = _cabi.TIMER, _cabi.KernelTimer()
        try:
            out = RD.render_rays(m, ro, rd, vd, rk)
            return out, set(_cabi.TIMER.records)
        finally:
            _cabi.TIMER = timer

    def chunk_loop(m, rk):
        outs = {k: [] for k in RD.KEYS}
        with torch.no_grad():
            for a, b, c in zip(ro.split(8192), rd.split(8192), vd.split(8192)):
                ret = m(a, b, c, **dict(rk, render_depth=True, coherent_rays=False))
                for k in RD.KEYS:
                    outs[k].append(ret[k].reshape(a.shape[0], -1))
        return {k: torch.cat(v) for k, v in outs.items()}

    for kind, shape, F_ in (('dcvgo', 'c12', 0), ('dcvgo', 'sig', 0), ('fg', 'c3', 0), ('fg', 'c12', 0), ('fg', 'sig', 0)):
        m = _model(kind, shape, 0.0, 'dense', F_=F_)
        out, keys = run(m)
        assert keys == {'render_contracted'}, keys
        want = m.render_fused(ro, rd, vd, **RK)
        for k in RD.KEYS:
            assert_equal(out[k], want[k].reshape(ro.shape[0], -1), k)
    # outside the coverage: FourierGridModel with Fourier slabs (9 and 11), a 15-channel k0, an rgbnet at a viewbase_pe the kernels
    # do not take, FourierGridModel with rand_bkgd -> the chunk loop, unchanged
    for F_, shape in ((4, 'c12'), (5, 'c3'), (4, 'sig')):
        m = _model('fg', shape, 0.0, 'dense', F_=F_)
        out, keys = run(m)
        assert 'render_contracted' not in keys and 'march_density_fwd' in keys, keys
        want = chunk_loop(m, RK)
        for k in RD.KEYS:
            assert_equal(out[k], want[k], k)
    from unboundednerfpytorch_b200 import models
    torch.manual_seed(0)                               # rgbnet_dim 3 at viewbase_pe 4: not a covered (C, pe) pair
    mpe = models.DirectContractedVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=24 ** 3, num_voxels_base=24 ** 3,
                                       alpha_init=1e-4, fast_color_thres=0.0, rgbnet_dim=3, viewbase_pe=4).to(DEV)
    out, keys = run(mpe)
    assert 'render_contracted' not in keys and 'march_density_fwd' in keys, keys
    want = chunk_loop(mpe, RK)
    for k in RD.KEYS:
        assert_equal(out[k], want[k], k)
    m15 = models.FourierGridModel(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=24 ** 3, num_voxels_base_density=24 ** 3,
                                  num_voxels_rgb=24 ** 3, num_voxels_base_rgb=24 ** 3, num_voxels_viewdir=-1, alpha_init=1e-4,
                                  fast_color_thres=0.0, rgbnet_dim=15, fourier_freq_num=2).to(DEV)
    out, keys = run(m15)
    assert 'render_contracted' not in keys and 'march_density_fwd' in keys, keys
    want = chunk_loop(m15, RK)
    for k in RD.KEYS:
        assert_equal(out[k], want[k], k)
    m = _model('fg', 'c12', 0.0, 'dense', F_=0)
    rk = dict(RK, rand_bkgd=True)
    with torch.no_grad():
        assert m.render_fused_ok(ro, RK) and not m.render_fused_ok(ro, rk)
    torch.manual_seed(5)
    out, keys = run(m, rk)
    assert 'render_contracted' not in keys and 'march_density_fwd' in keys, keys
    torch.manual_seed(5)
    want = chunk_loop(m, rk)
    for k in RD.KEYS:
        assert_equal(out[k], want[k], k)
    with torch.enable_grad():
        assert not m.render_fused_ok(ro, RK)
