"""GPU: the fused whole-frame render of FourierGridModel with Fourier slabs (render_kwargs['fused_slabs'] ->
models._ContractedBase.render_fused -> ubn_render_fourier, csrc/render_fourier.cu) against model.forward under no_grad and
against an fp64 restatement, at 7, 9 and 11 slabs.

* alphainv_last bit-identical to forward's; n_shaded equal to forward's samples up to the stop; n_marched the 32-sample chunks
  up to the stop;
* rgb_marched and depth within 1e-5 of forward and of fp64 (forward's survivors up to the stop, the k0 read, the rgbnet and
  the sums in float64);
* one call, 8192-ray chunks, a permutation and a rerun give the same bits; zero and one ray; rays without survivors, rays whose
  every sample survives, rays of one kept sample each (a 16-row tile spans 16 rays, every slot of the warp in use); a 1600x1067 frame in one
  call within 64 B per ray of extra memory;
* routing: with the key, covered models take exactly render_fourier; everything outside the coverage keeps the chunk loop bit for
  bit; render_viewpoints takes the key through render_kwargs.
"""
import numpy as np
import pytest
import torch

from tests.test_gpu_render_fused import DEV, RK, _expected_n_shaded, _fp64, _model, _stop_steps
from tests.util import assert_equal, seeded_rays

pytestmark = pytest.mark.gpu
RKS = dict(RK, fused_slabs=True)
SLABS = {7: 3, 9: 4, 11: 5}                                # P -> fourier_freq_num


def _render(m, ro, rd, vd, rk=RKS):
    ns = torch.full((ro.shape[0],), -1, dtype=torch.int32, device=DEV)
    nm = torch.full((ro.shape[0],), -1, dtype=torch.int32, device=DEV)
    with torch.no_grad():
        assert m.render_fused_ok(ro, rk)
        out = m.render_fused(ro, rd, vd, n_shaded=ns, n_marched=nm, **rk)
    return out, ns, nm


def _check_against_forward(m, ro, rd, vd, rk=RKS):
    N = ro.shape[0]
    out, ns, nm = _render(m, ro, rd, vd, rk)
    with torch.no_grad():
        fwd = m(ro, rd, vd, **rk)
    S = fwd['n_max']
    assert_equal(out['alphainv_last'], fwd['alphainv_last'], 'alphainv_last')
    want_ns, upto = _expected_n_shaded(m, fwd, N, S)
    assert_equal(ns, want_ns, 'n_shaded')
    if m.fast_color_thres <= 0:
        stop = torch.as_tensor(_stop_steps(m, fwd, N, S), device=DEV)
        assert_equal(nm, torch.clamp((stop // 32 + 1) * 32, max=S).to(torch.int32), 'n_marched')
    else:
        # forward returns only the samples whose weight passes the threshold, so its listed samples (and with them the stop) are
        # not all known here: the march reached at least the chunk of every returned sample
        last = torch.full((N,), -1, dtype=torch.int64, device=DEV).scatter_reduce_(0, fwd['ray_id'], fwd['step_id'], 'amax')
        reached = torch.where(last >= 0, torch.clamp((last // 32 + 1) * 32, max=S), 0)
        assert bool((nm.long() >= reached).all() and (nm <= S).all()), 'n_marched'
    err_rgb = (out['rgb_marched'] - fwd['rgb_marched']).abs().max().item()
    err_d = (out['depth'] - fwd['depth']).abs().max().item()
    assert err_rgb <= 1e-5 and err_d <= 1e-5, (err_rgb, err_d)
    col, depth = _fp64(m, ro, rd, vd, fwd, upto, rk)
    e64_rgb = (out['rgb_marched'].double() - col).abs().max().item()
    e64_d = (out['depth'].double() - depth).abs().max().item()
    assert e64_rgb <= 1e-5 and e64_d <= 1e-5, (e64_rgb, e64_d)
    return out, ns


CASES = [(P, t, sc) for P in SLABS for t in (0.0, 1e-4) for sc in ('dense', 'opaque')]


@pytest.mark.parametrize('P,thres,scene', CASES, ids=[f'p{P}-t{t:g}-{sc}' for P, t, sc in CASES])
def test_fourier_render_matches_forward_and_fp64(P, thres, scene):
    m = _model('fg', 'c12', thres, scene, F_=SLABS[P], seed=P)
    assert m.k0.grid.shape[0] == P and m.density.grid.shape[0] == P
    ro, rd, vd = seeded_rays(600, 11, DEV)
    out, ns = _check_against_forward(m, ro, rd, vd)
    if scene == 'opaque':
        assert (out['alphainv_last'] < 1e-3).float().mean() > 0.1          # many rays stop early
        assert ((ns % 16) != 0).any()
    else:
        assert int(ns.sum()) > 0


@pytest.mark.parametrize('P', [7, 11])
def test_batching_permutation_and_rerun_give_the_same_bits(P):
    m = _model('fg', 'c12', 0.0, 'opaque', F_=SLABS[P], seed=3)
    N = 20000
    ro, rd, vd = seeded_rays(N, 5, DEV)
    whole, ns, _ = _render(m, ro, rd, vd)
    again, ns2, _ = _render(m, ro, rd, vd)
    with torch.no_grad():
        chunks = [m.render_fused(a, b, c, **RKS) for a, b, c in zip(ro.split(8192), rd.split(8192), vd.split(8192))]
        perm = torch.randperm(N, generator=torch.Generator().manual_seed(1)).to(DEV)
        permuted = m.render_fused(ro[perm], rd[perm], vd[perm], **RKS)
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(N, device=DEV)
    assert_equal(ns, ns2, 'n_shaded rerun')
    for k in ('rgb_marched', 'depth', 'alphainv_last'):
        assert_equal(whole[k], again[k], k + ' rerun')
        assert_equal(whole[k], torch.cat([c[k] for c in chunks]), k + ' chunks')
        assert_equal(whole[k], permuted[k][inv], k + ' permuted')


def test_zero_and_one_ray():
    m = _model('fg', 'c12', 0.0, 'dense', F_=3)
    ro, rd, vd = seeded_rays(1, 2, DEV)
    with torch.no_grad():
        out = m.render_fused(ro[:0], rd[:0], vd[:0], **RKS)
    assert all(out[k].shape[0] == 0 for k in out)
    _check_against_forward(m, ro, rd, vd)


def test_rays_without_survivors():
    m = _model('fg', 'c12', 1e-4, 'dense', F_=4)
    with torch.no_grad():
        m.density.grid.fill_(-30.0)                                          # alpha ~ 1e-13 < fast_color_thres everywhere
    N = 3000
    ro, rd, vd = seeded_rays(N, 9, DEV)
    out, ns, _ = _render(m, ro, rd, vd)
    with torch.no_grad():
        fwd = m(ro, rd, vd, **RKS)
    assert int(ns.abs().sum()) == 0
    assert_equal(out['alphainv_last'], fwd['alphainv_last'], 'alphainv_last')
    assert_equal(out['alphainv_last'], torch.ones(N, device=DEV), 'alphainv_last without survivors')
    assert_equal(out['rgb_marched'], torch.zeros(N, 3, device=DEV), 'rgb without survivors')
    assert_equal(out['depth'], torch.zeros(N, device=DEV), 'depth without survivors')


@pytest.mark.parametrize('P', [7, 9, 11])
def test_all_samples_surviving(P):
    """Every one of 512+ samples kept (no ray stops): 32 full tiles per ray, a ray's sums carried across its tiles."""
    rk = dict(RKS, stepsize=0.07)
    m = _model('fg', 'c12', 0.0, 'dense', F_=SLABS[P], seed=2)
    with torch.no_grad():
        m.density.grid.fill_(-30.0)
    ro, rd, vd = seeded_rays(200, 13, DEV)
    out, ns = _check_against_forward(m, ro, rd, vd, rk)
    assert int(ns.min()) >= 512


def test_one_kept_sample_per_ray_fills_every_slot():
    """An opaque sphere behind empty space with a threshold: a ray that hits it keeps exactly its first sample inside (alpha ~ 1
    stops it), a ray that misses keeps none.  A 16-row tile then spans 16 rays, one per slot of the warp."""
    m = _model('fg', 'c12', 1e-4, 'dense', F_=3, seed=4)
    with torch.no_grad():
        X, Y, Z = m.density.grid.shape[2:]
        ax = [torch.linspace(-1, 1, n) for n in (X, Y, Z)]
        r = torch.stack(torch.meshgrid(*ax, indexing='ij'), -1).norm(dim=-1)
        m.density.grid.copy_(torch.where(r < 0.5, 300.0, -30.0).expand_as(m.density.grid).to(DEV))
    ro, rd, vd = seeded_rays(8000, 17, DEV, spread=0.2)
    out, ns = _check_against_forward(m, ro, rd, vd)
    assert int(ns.max()) <= 2 and (ns == 1).float().mean() > 0.3, torch.bincount(ns.long()).tolist()


def test_full_frame_in_one_call_within_64_bytes_per_ray():
    from unboundednerfpytorch_b200 import rays as R
    m = _model('fg', 'c12', 0.0, 'dense', F_=4, world=64, norm='l2')
    H, W = 1067, 1600
    K = np.array([[float(W), 0, W / 2], [0, float(W), H / 2], [0, 0, 1]], dtype=np.float64)
    c2w = torch.tensor([[1., 0., 0., 0.15], [0., 1., 0., -0.10], [0., 0., 1., 0.35]])
    ro, rd, vd = R._rays_of_a_view(H, W, K, c2w, False, False, False, False, 'center', device=DEV)
    ro, rd, vd = ro.reshape(-1, 3), rd.reshape(-1, 3), vd.reshape(-1, 3)
    N = ro.shape[0]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        out = m.render_fused(ro, rd, vd, **RKS)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base - sum(v.numel() * v.element_size() for v in out.values())
    assert extra <= 64 * N, (extra, N)
    sl = slice(N // 2, N // 2 + 4096)
    with torch.no_grad():
        fwd = m(ro[sl], rd[sl], vd[sl], **RKS)
    assert_equal(out['alphainv_last'][sl], fwd['alphainv_last'], 'alphainv_last')
    assert (out['rgb_marched'][sl] - fwd['rgb_marched']).abs().max() <= 1e-5


def _run(m, ro, rd, vd, rk):
    from unboundednerfpytorch_b200 import _cabi, render as RD
    timer, _cabi.TIMER = _cabi.TIMER, _cabi.KernelTimer()
    try:
        out = RD.render_rays(m, ro, rd, vd, rk)
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


def _fg(rgbnet_dim, viewbase_pe, F_):
    from unboundednerfpytorch_b200 import models
    torch.manual_seed(0)
    return models.FourierGridModel(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=24 ** 3, num_voxels_base_density=24 ** 3,
                                   num_voxels_rgb=24 ** 3, num_voxels_base_rgb=24 ** 3, num_voxels_viewdir=-1, alpha_init=1e-4,
                                   fast_color_thres=0.0, rgbnet_dim=rgbnet_dim, fourier_freq_num=F_,
                                   viewbase_pe=viewbase_pe).to(DEV)


def test_render_rays_routing_with_fused_slabs():
    from unboundednerfpytorch_b200 import render as RD
    ro, rd, vd = seeded_rays(10000, 21, DEV)
    for P, F_ in SLABS.items():
        m = _model('fg', 'c12', 0.0, 'dense', F_=F_)
        out, keys = _run(m, ro, rd, vd, RKS)
        assert keys == {'render_fourier'}, keys
        with torch.no_grad():
            want = m.render_fused(ro, rd, vd, **RKS)
        for k in RD.KEYS:
            assert_equal(out[k], want[k].reshape(ro.shape[0], -1), k)
        out, keys = _run(m, ro, rd, vd, RK)                                  # without the key: the chunk loop, as before
        assert 'render_fourier' not in keys and 'march_density_fwd' in keys, keys
    # outside the coverage, with the key: the chunk loop, bit for bit
    uncovered = {'pe 8': _fg(12, 8, 3), 'C = 3': _fg(3, 4, 3), 'C = 15': _fg(15, 4, 3), 'P = 5': _fg(12, 4, 2)}
    for what, m in uncovered.items():
        out, keys = _run(m, ro, rd, vd, RKS)
        assert 'render_fourier' not in keys and 'render_contracted' not in keys and 'march_density_fwd' in keys, (what, keys)
        want = _chunk_loop(m, ro, rd, vd, RKS)
        for k in RD.KEYS:
            assert_equal(out[k], want[k], f'{what}: {k}')
    m = _model('fg', 'c12', 0.0, 'dense', F_=3)
    rk = dict(RKS, rand_bkgd=True)
    with torch.no_grad():
        assert m.render_fused_ok(ro, RKS) and not m.render_fused_ok(ro, rk)
    torch.manual_seed(5)
    out, keys = _run(m, ro, rd, vd, rk)
    assert 'render_fourier' not in keys and 'march_density_fwd' in keys, keys
    torch.manual_seed(5)
    want = _chunk_loop(m, ro, rd, vd, rk)
    for k in RD.KEYS:
        assert_equal(out[k], want[k], 'rand_bkgd: ' + k)
    with torch.enable_grad():
        assert not m.render_fused_ok(ro, RKS)


def test_gradients_enabled_keep_the_training_forward():
    """With gradients on, the key changes nothing: render_fused_ok declines, and model(...) with the key -- the call of
    render_rays' chunk loop and of a training step whose render_kwargs carry it -- is forward without it: the same outputs bit for
    bit and the same gradients.  (render_rays itself runs under no_grad, so the caller's gradient mode never reaches its routing.)"""
    m = _model('fg', 'c12', 1e-4, 'opaque', F_=3, seed=8)
    ro, rd, vd = seeded_rays(3000, 23, DEV)
    outs, grads = [], []
    for rk in (RKS, RK):
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            assert not m.render_fused_ok(ro, rk)
            ret = m(ro, rd, vd, **rk)
            assert ret['rgb_marched'].requires_grad
            (ret['rgb_marched'].square().sum() + ret['depth'].sum()).backward()
        outs.append({k: ret[k].detach() for k in ('rgb_marched', 'depth', 'alphainv_last')})
        grads.append({n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None})
    for k in outs[0]:
        assert_equal(outs[0][k], outs[1][k], k)
    assert grads[0].keys() == grads[1].keys() and len(grads[0]) > 0
    for n in grads[0]:                  # the grid gradients are scattered with float atomics: equal up to summation order
        g0, g1 = grads[0][n], grads[1][n]
        assert (g0 - g1).abs().max() <= 1e-5 * g1.abs().max() + 1e-12, n


def test_render_viewpoints_with_fused_slabs(capsys):
    from unboundednerfpytorch_b200 import render
    m = _model('fg', 'c12', 1e-4, 'opaque', F_=4, seed=6)
    H, W = 48, 64
    K = np.array([[60., 0., 32.], [0., 60., 24.], [0., 0., 1.]])
    c2w = np.array([[1, 0, 0, 0.05], [0, 1, 0, -0.05], [0, 0, 1, 0.3]], dtype=np.float32)
    a = render.render_viewpoints(None, m, [c2w], [[H, W]], [K], False, dict(RK), chunk=1024)
    b = render.render_viewpoints(None, m, [c2w], [[H, W]], [K], False, dict(RKS), chunk=1024, gt_imgs=a[0], eval_ssim=True)
    assert np.array_equal(a[2], b[2])                                        # bgmaps: alphainv_last, bit for bit
    assert (a[2] < 0.999).mean() > 0.1
    assert np.abs(a[0] - b[0]).max() <= 1e-5
    out = capsys.readouterr().out
    assert float(out.split('Ssim')[1].split()[0]) > 0.999
