"""The width-64 tensor-core rgbnet (DirectMPIGO of llff_default: rgbnet_dim 9, rgbnet_width 64, viewbase_pe 0, so
12 -> 64 -> 64 -> 3 with the 3 view-direction columns folded into the per-ray bias) against fp64, at the ray layouts where the
backward's bookkeeping changes, and through DirectMPIGO.

The kernels are the width-128 ones with the hidden width as a template parameter (csrc/shade_tc.cu): every sizing of a layer,
the panel save layout ([tile][W/4 column quads][128 rows][4]), the ReLU mask words (W/32 chunks per 128-row tile) and every
bias / gradient index change with it.  The judge is the one of tests/test_gpu_rgbnet_layouts.py -- elementwise
|got - want| <= TAU * B with B the same expression on absolute values -- over a width- and K-generic fp64 reference.

Launch 1 of the width-64 backward runs 8 warps per CTA and one CTA per SM (3xTF32 needs 230 registers per thread), so its grid
and warp ranges are those of the 8-warp width-128 backward: the bounds8_* layouts put a ray boundary at every one of its
warp-range boundaries."""
import math

import pytest
import torch

from tests.test_gpu_rgbnet_layouts import AROUND8, LAYOUTS, SMALL, TAU, TAU_TC1, TINY, UNIT, judge, partition

DEV = 'cuda:0'
K, W = 9, 64
BWD_WARPS = 8              # launch 1 of the width-64 backward: 8 warps per CTA, at most 132 CTAs (one per SM)


# ---- fp64 reference, any K and width ----------------------------------------------------------------------------------
def ref64(feat, vb, ray_id, W1k, W2, b2, W3, b3, g_rgb, chunk=1 << 18):
    """rgb and every gradient of rgb = sigmoid(W3 relu(W2 relu(W1k x + vb[ray]) + b2) + b3) in fp64, and for each the bound B:
    the same expression on the absolute values of every operand, ReLU masks kept (the algebra of ref64 in
    tests/test_gpu_rgbnet_layouts.py, sized from the inputs)."""
    d = lambda x: x.double()
    W1k, W2, b2, W3, b3 = map(d, (W1k, W2, b2, W3, b3))
    aW1, aW2, ab2, aW3, ab3 = (x.abs() for x in (W1k, W2, b2, W3, b3))
    (M, k), (N, w), dev = feat.shape, vb.shape, feat.device
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=dev)
    want = dict(rgb=z(M, 3), g_feat=z(M, k), g_vb=z(N, w), dW1k=z(w, k), dW2=z(w, w), db2=z(w), dW3=z(3, w), db3=z(3))
    bound = {key: torch.zeros_like(v) for key, v in want.items()}
    dz1_rows = z(M, w)
    for lo in range(0, M, chunk):
        sl = slice(lo, min(M, lo + chunk))
        x, r, g = d(feat[sl]), ray_id[sl], d(g_rgb[sl])
        v = d(vb[r])
        z1 = x @ W1k.t() + v
        m1 = (z1 > 0).double()
        h1 = z1 * m1
        z2 = h1 @ W2.t() + b2
        m2 = (z2 > 0).double()
        h2 = z2 * m2
        y = torch.sigmoid(h2 @ W3.t() + b3)
        dz3 = g * y * (1 - y)
        dZ2 = (dz3 @ W3) * m2
        dZ1 = (dZ2 @ W2) * m1
        Bh1 = (x.abs() @ aW1.t() + v.abs()) * m1
        Bh2 = (Bh1 @ aW2.t() + ab2) * m2
        By = y * (1 - y) * (Bh2 @ aW3.t() + ab3) + y
        Bdz3 = g.abs() * (y * (1 - y) + (1 - 2 * y).abs() * By)
        BdZ2 = (Bdz3 @ aW3) * m2
        BdZ1 = (BdZ2 @ aW2) * m1
        want['rgb'][sl], bound['rgb'][sl] = y, By
        want['g_feat'][sl], bound['g_feat'][sl] = dZ1 @ W1k, BdZ1 @ aW1
        want['g_vb'].index_add_(0, r, dZ1)
        bound['g_vb'].index_add_(0, r, BdZ1)
        dz1_rows[sl] = dZ1
        for key, a, b, ba, bb in (('dW1k', dZ1, x, BdZ1, x.abs()), ('dW2', dZ2, h1, BdZ2, Bh1), ('dW3', dz3, h2, Bdz3, Bh2)):
            want[key] += a.t() @ b
            bound[key] += ba.t() @ bb
        want['db2'] += dZ2.sum(0)
        bound['db2'] += BdZ2.sum(0)
        want['db3'] += dz3.sum(0)
        bound['db3'] += Bdz3.sum(0)
    return want, bound, dz1_rows


def reference(inp):
    return ref64(*(inp[k] for k in ('feat', 'vb', 'ray_id', 'W1k', 'W2', 'b2', 'W3', 'b3', 'g_rgb')))


def min_preact(inp, idx):
    x = inp['feat'][idx].double()
    z1 = x @ inp['W1k'].double().t() + inp['vb'][inp['ray_id'][idx]].double()
    z2 = torch.relu(z1) @ inp['W2'].double().t() + inp['b2'].double()
    return torch.minimum(z1.abs().amin(1), z2.abs().amin(1))


def make_inputs(ray_id, N, seed, thresh=1e-5, max_rounds=8):
    """Seeded nn.Linear-scaled weights (fan-in 12 = 9 features + 3 view columns for layer 1), per-ray view bias and features;
    ReLU-ambiguous samples (an fp64 pre-activation within `thresh` of zero) get their feature row redrawn, never dropped."""
    g = torch.Generator().manual_seed(seed)
    M = ray_id.numel()
    u = lambda *s, a: ((torch.rand(*s, generator=g) * 2 - 1) * a)
    p = dict(W1k=u(W, K, a=1 / math.sqrt(K + 3)), W2=u(W, W, a=1 / math.sqrt(W)), b2=u(W, a=1 / math.sqrt(W)),
             W3=u(3, W, a=1 / math.sqrt(W)), b3=torch.randn(3, generator=g) * 0.1)
    inp = dict(feat=torch.randn(M, K, generator=g), vb=torch.randn(N, W, generator=g) * 0.5, ray_id=ray_id,
               g_rgb=torch.randn(M, 3, generator=g), **p)
    inp = {k: v.to(DEV) for k, v in inp.items()}
    idx = torch.arange(M, device=DEV)
    for _ in range(max_rounds):
        amb = idx[min_preact(inp, idx) <= thresh]
        if amb.numel() == 0:
            return inp
        inp['feat'][amb] = torch.randn(amb.numel(), K, generator=g).to(DEV)
        idx = amb
    raise AssertionError(f'{idx.numel()} samples still ReLU-ambiguous after {max_rounds} redraws')


def run(inp, mode='tc3'):
    """Forward + backward through _ShadeFn.apply with vb as a leaf, and the forward again under no_grad; the launch counter
    and timer show that the kernels ran."""
    from unboundednerfpytorch_b200 import _cabi, shade as shade_mod
    timer = _cabi.KernelTimer()
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(shade_mod, 'MODE', mode)
        mp.setattr(_cabi, 'TIMER', timer)
        leaves = {k: inp[k].clone().requires_grad_(True) for k in ('feat', 'vb', 'W1k', 'W2', 'b2', 'W3', 'b3')}
        args = [leaves['feat'], leaves['vb'], inp['ray_id']] + [leaves[k] for k in ('W1k', 'W2', 'b2', 'W3', 'b3')]
        rgb = shade_mod._ShadeFn.apply(*args, True)
        rgb.backward(inp['g_rgb'])
        with torch.no_grad():
            rgb_ng = shade_mod._ShadeFn.apply(*args, False)
    assert set(timer.summary()) == {'rgbnet_fwd', 'rgbnet_bwd'}
    got = dict(rgb=rgb.detach(), g_feat=leaves['feat'].grad, g_vb=leaves['vb'].grad)
    got.update({'d' + k: leaves[k].grad for k in ('W1k', 'W2', 'b2', 'W3', 'b3')})
    return got, rgb_ng


# ---- 3xTF32 against fp64 ------------------------------------------------------------------------------------------------
BIG = 1_200_000
CASES = ([(lay, M) for lay in ('aligned16', 'offset16', 'len4_o1', 'alternating', 'one_ray_first', 'sparse_odd', 'bounds8_0',
                               'randint') for M in SMALL]
         + [(lay, M) for lay in ('offset16', 'len4_o2', 'alternating', 'sparse_odd', 'bounds8_m1', 'bounds8_0', 'bounds8_p1',
                                 'geometric250', 'randint') for M in AROUND8]
         + [(lay, BIG) for lay in ('len4_o1', 'alternating', 'sparse_odd', 'bounds8_m1', 'bounds8_p1', 'geometric250', 'randint')])


@pytest.mark.gpu
@pytest.mark.parametrize('layout,M', CASES, ids=[f'{lay}-{M}' for lay, M in CASES])
def test_w64_layout_vs_fp64(layout, M):
    """tc3: rgb, g_feat, g_vb and the six parameter gradients within TAU * B of fp64; rays without samples get exactly zero;
    the no_grad forward is bit-identical to the grad-enabled one."""
    ray_id, N = LAYOUTS[layout](M)
    assert ray_id.numel() == M and bool((ray_id[1:] >= ray_id[:-1]).all()) and int(ray_id.max()) < N
    inp = make_inputs(ray_id, N, seed=M + 64)
    want, bound, _ = reference(inp)
    got, rgb_ng = run(inp)
    assert got['g_feat'].shape == (M, K) and got['g_vb'].shape == (N, W) and got['dW2'].shape == (W, W)
    assert torch.equal(rgb_ng, got['rgb']), 'no_grad forward differs from the grad-enabled one'
    empty = torch.bincount(inp['ray_id'], minlength=N) == 0
    assert not bool(got['g_vb'][empty].any()), 'rays without samples got a nonzero g_vb'
    judge(got, want, bound, f'{layout} M={M} width 64')


def test_w64_bounds_layouts_follow_the_launch():
    """CPU: the bounds8 layouts put a ray start at every warp-range boundary of the width-64 launch 1 (8 warps, one CTA per SM)."""
    for M in AROUND8 + (BIG,):
        ranges = partition(M, BWD_WARPS)
        assert len(ranges) - 1 == min(132, -(-(-(-M // UNIT)) // BWD_WARPS)) * BWD_WARPS
        for nm, shift in (('m1', -1), ('0', 0), ('p1', 1)):
            ids = LAYOUTS[f'bounds8_{nm}'](M)[0]
            b = torch.tensor([UNIT * u + shift for u in ranges[1:-1]])
            assert bool((ids[b] != ids[b - 1]).all())


# ---- single-pass TF32 -----------------------------------------------------------------------------------------------------
TC1_CASES = [('aligned16', 129), ('len4_o1', 4099), ('alternating', 4099), ('sparse_odd', AROUND8[1]), ('bounds8_p1', AROUND8[0]),
             ('bounds8_m1', AROUND8[2])]


def _tc1_inputs(ray_id, N, seed):
    """Pre-activations far from zero (as _tc1_inputs of tests/test_gpu_rgbnet_layouts.py), so that single-pass TF32 keeps every
    ReLU mask of fp64, and a one-signed upstream gradient so that a ray's sum does not cancel."""
    inp = make_inputs(ray_id, N, seed)
    g = torch.Generator().manual_seed(seed + 1)
    sign = lambda *s: (torch.randint(0, 2, s, generator=g) * 2 - 1).float().to(DEV)
    inp['feat'] *= 0.3
    inp['vb'] = sign(N, W) * (1.5 + torch.rand(N, W, generator=g).to(DEV))
    inp['b2'] = sign(W) * 25.0
    inp['W3'] *= 0.05
    inp['g_rgb'] = (torch.rand(ray_id.numel(), 3, generator=g) + 0.25).to(DEV)
    assert float(min_preact(inp, torch.arange(ray_id.numel(), device=DEV)).min()) > 0.2
    return inp


def _rss_bound(inp):
    """per ray: sqrt(sum over its samples of ||B(dZ1)||^2)"""
    x, r = inp['feat'].double(), inp['ray_id']
    W1k, W2, b2, W3, b3 = (inp[k].double() for k in ('W1k', 'W2', 'b2', 'W3', 'b3'))
    z1 = x @ W1k.t() + inp['vb'][r].double()
    z2 = torch.relu(z1) @ W2.t() + b2
    y = torch.sigmoid(torch.relu(z2) @ W3.t() + b3)
    BdZ1 = (((inp['g_rgb'].double() * y * (1 - y)).abs() @ W3.abs()) * (z2 > 0) @ W2.abs()) * (z1 > 0)
    rss = torch.zeros(inp['vb'].shape[0], dtype=torch.float64, device=x.device)
    rss.index_add_(0, r, BdZ1.pow(2).sum(1))
    return rss.sqrt()


@pytest.mark.gpu
@pytest.mark.parametrize('layout,M', TC1_CASES, ids=[f'{lay}-{M}' for lay, M in TC1_CASES])
def test_w64_tc1_rays(layout, M):
    """UBN_RGBNET_MODE=tc1 at width 64: rays without samples exactly zero, and every ray's g_vb within TAU_TC1 of the per-ray
    bound sqrt(sum ||B(dZ1)||^2), the check that rejects one sample moved to the neighbouring ray."""
    ray_id, N = LAYOUTS[layout](M)
    inp = _tc1_inputs(ray_id, N, M)
    want, _, _ = reference(inp)
    got, rgb_ng = run(inp, mode='tc1')
    assert torch.equal(rgb_ng, got['rgb'])
    g_vb, w = got['g_vb'], want['g_vb']
    empty = torch.bincount(inp['ray_id'], minlength=N) == 0
    assert not bool(g_vb[empty].any()), 'rays without samples got a nonzero g_vb'
    r = float(((g_vb.double() - w).norm(dim=1) / (_rss_bound(inp) + TINY))[~empty].max())
    assert r <= TAU_TC1, f'per-ray norm error {r:.2e} of the bound'
    rel = float(((got['rgb'].double() - want['rgb']).abs() / want['rgb']).max())
    assert rel <= 4e-3, f'rgb relative error {rel:.2e}'


# ---- the C ABI refuses what it has no kernel for -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('n_feat,n_hidden', [(12, 64), (3, 64), (9, 128), (9, 32), (12, 256)])
def test_unsupported_pairs_raise(n_feat, n_hidden):
    from unboundednerfpytorch_b200 import _cabi
    from unboundednerfpytorch_b200._cabi import c_i64, c_int, check, ptr, stream_of
    lib = _cabi.load()
    M, N = 64, 4
    f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=DEV)
    feat, vb, ray_id = f(M, n_feat), f(N, n_hidden), torch.zeros(M, dtype=torch.int64, device=DEV)
    W1k, W2, b2, W3, b3, rgb = f(n_hidden, n_feat), f(n_hidden, n_hidden), f(n_hidden), f(3, n_hidden), f(3), f(M, 3)
    h1, h2 = f(128, n_hidden), f(128, n_hidden)
    m = torch.zeros(4 * n_hidden, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match='CUDA error'):
        check(lib.ubn_rgbnet_fwd_tc_kw(c_int(n_feat), c_int(n_hidden), ptr(feat), ptr(vb), ptr(ray_id), ptr(W1k), ptr(W2), ptr(b2),
                                       ptr(W3), ptr(b3), c_i64(M), ptr(rgb), ptr(h1), ptr(h2), ptr(m), c_int(4), stream_of(feat)))
    with pytest.raises(RuntimeError, match='CUDA error'):
        check(lib.ubn_rgbnet_bwd_tc_fused_kw(c_int(n_feat), c_int(n_hidden), ptr(feat), ptr(ray_id), ptr(W1k), ptr(W2), ptr(W3),
                                             ptr(rgb), ptr(h1), ptr(h2), ptr(rgb), c_i64(M), ptr(feat), ptr(vb), ptr(W1k), ptr(W2),
                                             ptr(b2), ptr(W3), ptr(b3), ptr(m), ptr(m), c_int(4), stream_of(feat)))
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_w64_without_panel_saves_or_masks_raises():
    """Width 64 writes its saves in the panel layout and runs the backward with both ReLU masks only."""
    from unboundednerfpytorch_b200 import _cabi
    from unboundednerfpytorch_b200._cabi import c_i64, c_int, check, ptr, stream_of
    lib = _cabi.load()
    M, N = 64, 4
    f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=DEV)
    feat, vb, ray_id = f(M, K), f(N, W), torch.zeros(M, dtype=torch.int64, device=DEV)
    W1k, W2, b2, W3, b3, rgb = f(W, K), f(W, W), f(W), f(3, W), f(3), f(M, 3)
    h1, h2 = f(128, W), f(128, W)
    m = torch.zeros(4 * W, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match='CUDA error'):       # saves without bit 2
        check(lib.ubn_rgbnet_fwd_tc_kw(c_int(K), c_int(W), ptr(feat), ptr(vb), ptr(ray_id), ptr(W1k), ptr(W2), ptr(b2), ptr(W3),
                                       ptr(b3), c_i64(M), ptr(rgb), ptr(h1), ptr(h2), ptr(m), c_int(0), stream_of(feat)))
    for flags, m2, m1 in ((0, m, m), (4, None, m), (4, m, None)):
        with pytest.raises(RuntimeError, match='CUDA error'):
            check(lib.ubn_rgbnet_bwd_tc_fused_kw(c_int(K), c_int(W), ptr(feat), ptr(ray_id), ptr(W1k), ptr(W2), ptr(W3), ptr(rgb),
                                                 ptr(h1), ptr(h2), ptr(rgb), c_i64(M), ptr(feat), ptr(vb), ptr(W1k), ptr(W2), ptr(b2),
                                                 ptr(W3), ptr(b3), ptr(m2), ptr(m1), c_int(flags), stream_of(feat)))
    # the forward without saves needs no panel bit
    check(lib.ubn_rgbnet_fwd_tc_kw(c_int(K), c_int(W), ptr(feat), ptr(vb), ptr(ray_id), ptr(W1k), ptr(W2), ptr(b2), ptr(W3),
                                   ptr(b3), c_i64(M), ptr(rgb), None, None, None, c_int(0), stream_of(feat)))
    torch.cuda.synchronize()
    assert torch.equal(rgb, torch.full_like(rgb, 0.5))


# ---- DirectMPIGO --------------------------------------------------------------------------------------------------------
def _timed(fn):
    from unboundednerfpytorch_b200 import _cabi
    timer = _cabi.KernelTimer()
    prev, _cabi.TIMER = _cabi.TIMER, timer
    try:
        out = fn()
    finally:
        _cabi.TIMER = prev
    return out, timer.summary()


@pytest.mark.gpu
def test_dmpigo_llff_default_runs_the_kernel():
    """DirectMPIGO at the llff_default shape (rgbnet_dim 9, width 64, mpi_depth 128, 255-step rays) shades with the tensor-core
    rgbnet in forward and forward_ops, forward and backward; raw_rgb is within 1e-5 of scale of the torch (cuBLAS) rgbnet on the
    same survivors, and the rgbnet's gradients within the 5e-4 the reference comparison of tests/test_gpu_mpi.py allows."""
    from tests.test_gpu_callers_unchanged import _stat
    from tests.test_gpu_mpi import RK, _ndc_scene
    from unboundednerfpytorch_b200 import shade as shade_mod
    m, ro, rd, vd = _ndc_scene(9, depth=128, nv=256 ** 3, seed=9, dmean=-1.0)
    assert shade_mod.supported(m.rgbnet, 9)

    def step(fwd):
        m.zero_grad(set_to_none=True)
        out = fwd(ro, rd, vd, global_step=None, **RK)
        (out['rgb_marched'].pow(2).sum() + (out['raw_rgb'] * out['weights'].detach()[:, None]).sum()).backward()
        return out, {k: p.grad.clone() for k, p in m.named_parameters() if k.startswith('rgbnet')}

    results = {}
    for name, fwd in (('forward', m.forward), ('forward_ops', m.forward_ops)):
        (out, grads), timed = _timed(lambda: step(fwd))
        assert timed.get('rgbnet_fwd', (0, 0))[1] == 1 and timed.get('rgbnet_bwd', (0, 0))[1] == 1, (name, timed)
        results[name] = (out, grads)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(shade_mod, 'supported', lambda *a, **k: False)
        (out_t, grads_t), timed = _timed(lambda: step(m.forward))
        assert 'rgbnet_fwd' not in timed
    out, grads = results['forward']
    assert out['ray_id'].numel() > 100000
    assert torch.equal(out['ray_id'], out_t['ray_id'])
    assert _stat(out['raw_rgb'], out_t['raw_rgb']) <= 1e-5
    assert _stat(out['rgb_marched'], out_t['rgb_marched']) <= 1e-5
    assert _stat(results['forward_ops'][0]['raw_rgb'], out_t['raw_rgb']) <= 1e-5
    for k in grads_t:
        assert _stat(grads[k], grads_t[k]) <= 5e-4, k


@pytest.mark.gpu
@pytest.mark.parametrize('dim,width', [(9, 128), (3, 64), (12, 64)])
def test_dmpigo_other_shapes_stay_on_torch(dim, width):
    from tests.test_gpu_mpi import RK
    from unboundednerfpytorch_b200 import models, shade as shade_mod
    m = models.DirectMPIGO(xyz_min=[-1.4, -1.1, -1.], xyz_max=[1.4, 1.1, 1.], num_voxels=32 ** 3, mpi_depth=16,
                           rgbnet_dim=dim, rgbnet_width=width, fast_color_thres=0.0).to(DEV)
    assert not shade_mod.supported(m.rgbnet, dim)
    g = torch.Generator().manual_seed(0)
    ro = torch.cat([(torch.rand(256, 2, generator=g) - 0.5) * 2, -torch.ones(256, 1)], -1).to(DEV)
    rd = torch.cat([torch.randn(256, 2, generator=g) * 0.3, 2.0 * torch.ones(256, 1)], -1).to(DEV)
    vd = rd / rd.norm(dim=-1, keepdim=True)
    out, timed = _timed(lambda: m(ro, rd, vd, global_step=None, **RK))
    assert out['ray_id'].numel() > 0 and 'rgbnet_fwd' not in timed and 'rgbnet_bwd' not in timed


@pytest.mark.gpu
def test_dmpigo_w64_training_lowers_the_loss():
    """40 steps of forward + backward + TV + MaskedAdam on a teacher / student pair, every one through the width-64 kernels."""
    import torch.nn.functional as F
    from tests.test_gpu_mpi import RK, _ndc_scene
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    teacher, ro, rd, vd = _ndc_scene(9, depth=32, nv=48 ** 3, seed=1, dmean=0.0)
    student, _, _, _ = _ndc_scene(9, depth=32, nv=48 ** 3, seed=2, dmean=-2.0, dstd=0.1, thres=1e-4)
    with torch.no_grad():
        student.mask_cache.mask.fill_(True)
        target = teacher(ro, rd, vd, **RK)['rgb_marched']
    cfg = dict(lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])
    opt = create_optimizer_or_freeze_model(student, cfg, global_step=0)
    losses = []

    def train():
        for it in range(1, 41):
            ret = student(ro, rd, vd, global_step=it, **RK)
            opt.zero_grad(set_to_none=True)
            loss = F.mse_loss(ret['rgb_marched'], target)
            loss.backward()
            student.density_total_variation_add_grad(1e-6 / len(ro), it < 20)
            student.k0_total_variation_add_grad(1e-7 / len(ro), it < 20)
            opt.step()
            losses.append(loss.item())
    _, timed = _timed(train)
    assert timed['rgbnet_fwd'][1] == 40 and timed['rgbnet_bwd'][1] == 40
    assert losses[-1] < 0.9 * losses[0], losses[::5]
    assert all(torch.isfinite(p).all() for p in student.parameters())
