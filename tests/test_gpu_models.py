"""GPU parity tests of the model-level hot path (fused march through the C ABI + rgbnet + composite):
vs the golden fixtures recorded from the reference's Python, vs the CPU oracle on fresh seeded inputs, fused vs
op-by-op composition, and size-independent properties at the BASELINE size (8192 rays x 512 samples)."""
import pytest
import torch

from tests.util import assert_close, assert_equal, load_golden, seeded_rays

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
FLOAT_KEYS = ('rgb_marched', 'alphainv_last', 'weights', 'raw_rgb', 'raw_alpha', 'raw_density', 'depth', 't', 's')


def _loss(ret, lw, dev):
    loss = (ret['rgb_marched'] * lw['rgb'].to(dev)).sum() + (ret['alphainv_last'] * lw['last'].to(dev)).sum()
    return loss + 0.01 * (ret['raw_rgb'].pow(2).sum(-1) * ret['weights'].detach()).sum() + 0.1 * ret['weights'].pow(2).sum()


def _build(cls, rec):
    m = cls(**rec['kwargs'])
    m.load_state_dict(rec['state'])
    return m.to(DEV)


def _check_against_golden(m, rec, fwd, name, grad_rtol=5e-5):
    rk, ref = rec['render_kwargs'], rec['ret']
    m.zero_grad()
    ret = fwd(rec['rays_o'].to(DEV), rec['rays_d'].to(DEV), rec['viewdirs'].to(DEV), global_step=None, **rk)
    assert_equal(ret['ray_id'], ref['ray_id'], name + ' ray_id')           # which samples survive: bit exact
    if 'step_id' in ref:
        assert_equal(ret['step_id'], ref['step_id'], name + ' step_id')
    for k in FLOAT_KEYS:
        if k in ref:
            assert_close(ret[k], ref[k], rtol=2e-5, atol=2e-6, what=f'{name} {k}')
    if 'wsum_mid' in ref:
        assert_close(ret['wsum_mid'], ref['wsum_mid'], rtol=2e-5, atol=2e-6, what=name + ' wsum_mid')
    _loss(ret, rec['loss_w'], DEV).backward()
    for pname, p in m.named_parameters():
        if pname in ref['grads']:
            g = ref['grads'][pname]
            scale = g.abs().max().item() + 1e-12
            assert_close(p.grad, g, rtol=grad_rtol, atol=1e-5 * scale + 1e-9, what=f'{name} grad {pname}')


@pytest.mark.parametrize('name', ['fouriergrid_thres', 'fouriergrid_opaque'])
@pytest.mark.parametrize('path', ['fused', 'ops'])
def test_fouriergrid_model_golden(name, path):
    from unboundednerfpytorch_b200 import models
    rec = load_golden('l2_models.pt')[name]
    m = _build(models.FourierGridModel, rec)
    _check_against_golden(m, rec, m.forward if path == 'fused' else m.forward_ops, f'{name}/{path}')


@pytest.mark.parametrize('name', ['dcvgo_inf', 'dcvgo_l2_opaque'])
@pytest.mark.parametrize('path', ['fused', 'ops'])
def test_dcvgo_model_golden(name, path):
    from unboundednerfpytorch_b200 import models
    rec = load_golden('l2_models.pt')[name]
    m = _build(models.DirectContractedVoxGO, rec)
    _check_against_golden(m, rec, m.forward if path == 'fused' else m.forward_ops, f'{name}/{path}')


def test_dvgo_model_golden():
    """BASELINE config 1 family (bounded DVGO): sampling + forward + grads vs the reference python."""
    from unboundednerfpytorch_b200 import models, ops
    rec = load_golden('l2_models.pt')['dvgo']
    m = _build(models.DirectVoxGO, rec)
    out = ops.sample_pts_on_rays(rec['rays_o'].to(DEV).contiguous(), rec['rays_d'].to(DEV).contiguous(), m.xyz_min, m.xyz_max,
                                 0.2, 1e9, rec['stepdist'])
    for a, b, nm in zip(out, rec['sample'], ('pts', 'mask_outbbox', 'ray_id', 'step_id', 'N_steps', 't_min', 't_max')):
        (assert_close if a.dtype == torch.float32 else assert_equal)(a, b, what=nm)
    _check_against_golden(m, rec, m.forward, 'dvgo')


def test_dvgo_config1_fixture_64cubed_1024_rays():
    """SURVEY.md 8c / BASELINE config 1: DVGO 64^3 DenseGrid, 1024 rays, stepsize 0.5 -- the fixture was produced by the reference's
    own dvgo.py on CPU (torch F.grid_sample path; oracle/make_golden.py::golden_cfg1), the grids are regenerated from the seed."""
    from tests.util import cfg1_scene
    from unboundednerfpytorch_b200 import models
    rec = load_golden('l2_cfg1.pt')
    kw, dens, k0, net, ro, rd, vd = cfg1_scene(rec['seed'])
    m = models.DirectVoxGO(**kw)
    with torch.no_grad():
        m.density.grid.copy_(dens)
        m.k0.grid.copy_(k0)
    m.load_state_dict(net, strict=False)
    m = m.to(DEV)
    with torch.no_grad():
        ret = m(ro.to(DEV), rd.to(DEV), vd.to(DEV), **rec['render_kwargs'])
    assert ret['ray_id'].numel() == rec['n_survivors']
    assert_equal(torch.bincount(ret['ray_id'], minlength=1024).to(torch.int32), rec['per_ray_count'], 'survivors per ray')
    for k in ('rgb_marched', 'depth', 'alphainv_last'):
        assert_close(ret[k], rec[k], rtol=1e-5, atol=1e-5 * float(rec[k].abs().max()), what=f'cfg1 {k}')
    wsum = torch.zeros(1024, device=DEV).index_add_(0, ret['ray_id'], ret['weights'])
    assert_close(wsum, rec['weights_sum'], rtol=1e-5, atol=1e-6, what='cfg1 weights sum')


def _fresh_model(flavor, world, F_, thres, seed, dens_mean=0.0, dens_std=1.0, norm='inf'):
    from unboundednerfpytorch_b200 import models
    torch.manual_seed(seed)
    if flavor == 'fouriergrid':
        kw = dict(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=world ** 3, num_voxels_base_density=world ** 3,
                  num_voxels_rgb=world ** 3, num_voxels_base_rgb=world ** 3, num_voxels_viewdir=-1, alpha_init=1e-4,
                  fast_color_thres=thres, rgbnet_dim=12, fourier_freq_num=F_, contracted_norm=norm)
        m = models.FourierGridModel(**kw)
    else:
        kw = dict(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=world ** 3, num_voxels_base=world ** 3, alpha_init=1e-4,
                  fast_color_thres=thres, rgbnet_dim=12, contracted_norm=norm)
        m = models.DirectContractedVoxGO(**kw)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=g) * dens_std + dens_mean)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
        if flavor == 'dcvgo':
            m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=g) > 0.1)
    return m, kw


@pytest.mark.parametrize('flavor,world,F_,thres,mean,norm', [
    ('fouriergrid', 40, 4, 0.0, 0.0, 'inf'),       # dense mode: every nominal sample is live (roofline configuration)
    ('fouriergrid', 40, 3, 1e-4, 6.0, 'l2'),       # realistic: rays terminate, two threshold masks
    ('dcvgo', 48, 0, 0.0, 0.0, 'inf'),
    ('dcvgo', 48, 0, 1e-4, 6.0, 'l2'),
])
def test_model_vs_cpu_oracle_seeded(oracle, flavor, world, F_, thres, mean, norm):
    """Fresh seeded scene (not a fixture): fused CUDA path vs the CPU oracle restatement, forward and backward."""
    m, kw = _fresh_model(flavor, world, F_, thres, 777, dens_mean=mean, dens_std=3.0 if mean else 1.0, norm=norm)
    state = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}
    N = 96
    ro, rd, vd = seeded_rays(N, 778)
    p = oracle.params_from_state(flavor, kw, state, requires_grad=True)
    ref = oracle.model_forward(flavor, p, ro, rd, vd, 0.5, bg=1)
    m = m.to(DEV)
    ret = m(ro.to(DEV), rd.to(DEV), vd.to(DEV), global_step=None, is_train=False, near=0., far=1e9, bg=1, rand_bkgd=False,
            stepsize=0.5, render_depth=True)
    assert_equal(ret['ray_id'], ref['ray_id'], 'ray_id')
    assert_equal(ret['step_id'], ref['step_id'], 'step_id')
    for k in FLOAT_KEYS:
        # raw_density: interpolated N(0,1) grid values that cancel towards 0 in the slab mean; its error is set by fp32
        # rounding of the sin/cos-warped sample coordinate (x (X-1)/2 x grid slope), i.e. absolute, not relative
        # ... and of the ray direction itself: torch-CPU and torch-CUDA evaluate d/||d|| differently in the last bit, the
        # kernel follows torch-CUDA (what the reference runs), the oracle runs torch-CPU; one ulp of d is amplified by
        # t (<= 192) x 2^(F-1) x (X-1)/2 on the way to a voxel index.  Tight raw_density parity is asserted against the
        # op-by-op CUDA composition in test_full_size_properties_8192x512.
        atol = (2e-3 if F_ >= 3 else 5e-5) if k == 'raw_density' else 2e-6
        assert_close(ret[k], ref[k].reshape(ret[k].shape), rtol=2e-5, atol=atol, what=k)
    g = torch.Generator().manual_seed(5)
    lw = dict(rgb=torch.randn(N, 3, generator=g), last=torch.randn(N, generator=g))
    _loss(ret, lw, DEV).backward()
    _loss(ref, lw, 'cpu').backward()
    for mine, theirs, nm in ((m.density.grid.grad, p['density_grid'].grad, 'density'), (m.k0.grid.grad, p['k0_grid'].grad, 'k0'),
                             (m.rgbnet[0].weight.grad, p['rgbnet']['W1'].grad, 'W1')):
        # scatter weights inherit the fp32 rounding of the (sin/cos-warped, x(X-1)/2) sample coordinate: up to ~1e-5..1e-4
        # absolute on a trilinear weight for the 2^3-frequency slabs, times the per-sample gradient (~ scale)
        scale = theirs.abs().max().item() + 1e-12
        assert_close(mine, theirs, rtol=5e-5, atol=(1e-3 if F_ >= 3 else 1e-5) * scale + 1e-9, what='grad ' + nm)


@pytest.mark.parametrize('flavor', ['fouriergrid', 'dcvgo'])
def test_full_size_properties_8192x512(flavor):
    """BASELINE size: 8192 rays x 512 nominal samples (world 153 => S = 512).  The CPU oracle would take minutes here,
    so parity is carried by size-independent properties: fused == op-by-op composition of the individually verified ops,
    the telescoping identity sum(w) + T_last == 1, sortedness / histogram of ray_id, and determinism of the forward."""
    F_ = 1 if flavor == 'fouriergrid' else 0
    m, _ = _fresh_model(flavor, 153, F_, 0.0, 777)
    m = m.to(DEV)
    N = 8192
    ro, rd, vd = seeded_rays(N, 777, DEV)
    rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, render_depth=True)
    with torch.no_grad():
        a = m(ro, rd, vd, global_step=None, **rk)
        b = m.forward_ops(ro, rd, vd, global_step=None, **rk)
        a2 = m(ro, rd, vd, global_step=None, **rk)
    assert a['n_max'] == 512
    # which samples survive: identical up to threshold bands (a 1-ulp difference between torch's elementwise point
    # arithmetic -- its 3-vector norm kernel in particular -- and the in-kernel one can flip a cumdist / mask-cache-rounding
    # decision): <= 1e-4 of the samples
    ka, kb = a['ray_id'] * 512 + a['step_id'], b['ray_id'] * 512 + b['step_id']
    in_b, in_a = torch.isin(ka, kb), torch.isin(kb, ka)
    flips = int((~in_b).sum() + (~in_a).sum())
    assert flips <= 1e-4 * ka.numel(), f'{flips} membership flips out of {ka.numel()}'
    for k in ('weights', 'raw_alpha', 'raw_density'):
        assert_close(a[k][in_b], b[k].reshape(-1)[in_a], rtol=2e-5, atol=2e-6, what=k + ' fused vs ops')
    for k in ('rgb_marched', 'alphainv_last', 'depth'):
        bad = ((a[k] - b[k]).abs() > 2e-6 + 2e-5 * b[k].abs()).reshape(N, -1).any(-1)
        assert int(bad.sum()) <= max(flips, 0) * 2, f'{k}: {int(bad.sum())} rays differ with {flips} flips'
    for k in ('rgb_marched', 'alphainv_last', 'weights', 'depth', 'raw_alpha'):
        assert_equal(a[k], a2[k], k + ' deterministic')
    if flavor == 'fouriergrid':
        assert a['weights'].numel() == N * 512
    assert (a['ray_id'][1:] >= a['ray_id'][:-1]).all()
    wsum = torch.zeros(N, device=DEV, dtype=torch.float64).index_add_(0, a['ray_id'], a['weights'].double())
    assert ((wsum + a['alphainv_last'].double()) - 1).abs().max() < 5e-5


def test_training_step_reduces_loss():
    """fwd + bwd + TV + MaskedAdam on a teacher/student pair: the drop-in pieces compose into a working optimiser step."""
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    teacher, _ = _fresh_model('dcvgo', 32, 0, 1e-4, 1, dens_mean=4.0, dens_std=3.0)
    student, _ = _fresh_model('dcvgo', 32, 0, 0.0, 2, dens_mean=0.0, dens_std=0.1)
    teacher, student = teacher.to(DEV), student.to(DEV)
    with torch.no_grad():
        student.act_shift.copy_(teacher.act_shift)
    cfg = dict(lrate_density=1e-1, lrate_k0=1e-1, lrate_rgbnet=1e-3, lrate_decay=20, skip_zero_grad_fields=['density', 'k0'])
    opt = create_optimizer_or_freeze_model(student, cfg, global_step=0)
    rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5)
    ro, rd, vd = seeded_rays(2048, 3, DEV)
    with torch.no_grad():
        target = teacher(ro, rd, vd, **rk)['rgb_marched']
    losses = []
    for it in range(1, 31):
        ret = student(ro, rd, vd, global_step=it, is_train=True, **rk)
        opt.zero_grad(set_to_none=True)
        loss = torch.nn.functional.mse_loss(ret['rgb_marched'], target)
        loss.backward()
        student.density_total_variation_add_grad(1e-6 / len(ro), it < 10)
        student.k0_total_variation_add_grad(1e-7 / len(ro), it < 10)
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.999 * losses[0] and all(b <= a * 1.0001 for a, b in zip(losses, losses[1:])), losses
    assert all(torch.isfinite(p).all() for p in student.parameters())


@pytest.mark.parametrize('mode', ['simt', 'tc3', 'tc3w4', 'tc1', 'tc3+tcbwd', 'tc3+fused', 'tc3+fusedh2', 'tc3+fused4', 'tc1+fused'])
def test_fused_rgbnet_vs_torch(mode, monkeypatch):
    """csrc/shade.cu (fp32 FFMA) and csrc/shade_tc.cu (tensor cores: 3xTF32 fp32-grade, single-pass TF32 preview) vs the torch
    nn.Sequential they replace: forward and every gradient."""
    from unboundednerfpytorch_b200 import models, shade as shade_mod
    monkeypatch.setattr(shade_mod, 'BWD_MODE', {'tcbwd': 'tc3', 'fused': 'fused', 'fusedh2': 'fused', 'fused4': 'fused4'}.get(mode.split('+')[-1], 'simt'))
    monkeypatch.setattr(shade_mod, 'USE_MASKS', not mode.endswith('fusedh2'))      # 'fusedh2': both backward launches re-read the saves (A/B of the ReLU masks)
    mode = mode.split('+')[0]
    monkeypatch.setattr(shade_mod, 'MODE', mode)
    fwd_tol = dict(rtol=1e-5, atol=1e-6) if mode != 'tc1' else dict(rtol=5e-3, atol=5e-3)
    torch.manual_seed(3)
    net = models._make_rgbnet(39, 128, 3).to(DEV)
    with torch.no_grad():
        net[3].bias.normal_(0, 0.1)
    for M, n_rays in ((1, 1), (77, 5), (300, 300), (20000, 37), (150001, 613)):
        g = torch.Generator().manual_seed(M)
        k0 = torch.randn(M, 12, generator=g).to(DEV).requires_grad_(True)
        emb = torch.randn(n_rays, 27, generator=g).to(DEV)
        ray_id = torch.sort(torch.randint(0, n_rays, (M,), generator=g))[0].to(DEV)
        gr = torch.randn(M, 3, generator=g).to(DEV)
        # ReLU' is discontinuous: a pre-activation within fp32 rounding of zero legitimately gets a different mask from two fp32
        # implementations and changes that sample's gradient wholesale.  Keep the comparison about arithmetic: drop the (few)
        # samples whose fp64 pre-activations come within 1e-5 of zero (1e-2 for the single-pass TF32 mode).
        with torch.no_grad():
            x64 = torch.cat([k0, emb[ray_id]], -1).double()
            z1 = x64 @ net[0].weight.double().t() + net[0].bias.double()
            z2 = torch.relu(z1) @ net[2][0].weight.double().t() + net[2][0].bias.double()
            ok = (torch.minimum(z1.abs().amin(1), z2.abs().amin(1)) > (5e-2 if mode == 'tc1' else 1e-5))
        if M > 1 and bool(ok.any()):
            k0 = k0.detach()[ok].clone().requires_grad_(True)
            ray_id, gr = ray_id[ok].contiguous(), gr[ok].contiguous()
        ref = torch.sigmoid(net(torch.cat([k0, emb[ray_id]], -1)))
        net.zero_grad(); k0.grad = None
        (ref * gr).sum().backward()
        want = [k0.grad.clone()] + [p.grad.clone() for p in net.parameters()]
        net.zero_grad(); k0.grad = None
        out = shade_mod.shade(net, k0, emb, ray_id)
        assert_close(out, ref, what=f'rgb M={M} {mode}', **fwd_tol)
        if mode == 'tc1' and shade_mod.BWD_MODE not in ('fused', 'fused4'):
            continue
        (out * gr).sum().backward()
        got = [k0.grad] + [p.grad for p in net.parameters()]
        for a, b, nm in zip(got, want, ['k0', 'W1', 'b1', 'W2', 'b2', 'W3', 'b3']):
            scale = b.abs().max().item() + 1e-12
            if mode == 'tc1':            # single TF32 pass on truncated operands: ~1e-3 relative per product, judged in norm
                rel = float((a - b).norm() / (b.norm() + 1e-30))
                assert rel <= 8e-2, f'grad {nm} M={M} tf32x1: relative Frobenius error {rel:.2e}'
            else:
                # parameter gradients are fp32 sums over M samples whose partial sums reach `scale`: two summation orders differ
                # by a few ulp(scale) * sqrt(#adds) -- judged at the north-star 1e-5 of the largest element; k0 is per sample
                assert_close(a, b, rtol=2e-5, atol=(2e-6 if nm == 'k0' else 1e-5) * scale + 1e-9, what=f'grad {nm} M={M}')


@pytest.mark.parametrize('flavor,F_,thres', [('fouriergrid', 4, 0.0), ('fouriergrid', 2, 1e-4), ('dcvgo', 0, 1e-4)])
def test_density_scatter_variants_agree(flavor, F_, thres):
    """ubn_set_density_scatter 0 / 1: per-sample scatter vs the two-phase run-merging scatter of the fused march backward -- the same
    addends, merged before or inside the L2 reductions: density-grid gradients agree to fp32 summation order, everything else
    is untouched."""
    from unboundednerfpytorch_b200 import ops
    m, _ = _fresh_model(flavor, 40, F_, thres, 13, dens_mean=5.0 if thres else 0.0, dens_std=3.0 if thres else 1.0)
    m = m.to(DEV)
    ro, rd, vd = seeded_rays(700, 17, DEV)
    rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, render_depth=True)
    grads = []
    try:
        for variant in (0, 1):
            ops.set_density_scatter(variant)
            assert ops.get_density_scatter() == variant
            m.zero_grad(set_to_none=True)
            ret = m(ro, rd, vd, global_step=None, **rk)
            (ret['rgb_marched'].sum() + 1e-2 * ret['depth'].sum() + 0.1 * ret['raw_rgb'].pow(2).sum()).backward()
            grads.append({k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None})
    finally:
        ops.set_density_scatter(1)
    a, b = grads
    assert a.keys() == b.keys()
    scale = float(a['density.grid'].abs().max())
    assert scale > 0
    assert float((a['density.grid'] - b['density.grid']).abs().max()) <= 1e-5 * scale
    assert float((a['density.grid'].double().sum() - b['density.grid'].double().sum()).abs()) <= 1e-5 * float(a['density.grid'].double().abs().sum())
    for k in a:
        if k != 'density.grid':
            s_ = float(a[k].abs().max()) + 1e-30
            assert float((a[k] - b[k]).abs().max()) <= 1e-5 * s_, k


def test_rgbnet_dw2_long_sample_sum_vs_fp64():
    """dW2 = sum over ALL samples of dZ2^T H1 is a split-K tensor-core GEMM.  A tensor-core fp32 accumulator need not round to
    nearest, so one accumulator chain per CTA over hundreds of 32-sample chunks could carry a bias that grows linearly with the
    chain.  k_shade_dw2_tc therefore restarts the MMA accumulator every 32-sample chunk and keeps an fp32 round-to-nearest
    running sum in registers.  This test makes the chains long (1.2 M samples, ~280 chunks per CTA) and judges dW2 -- and
    the other sample sums -- against an fp64 evaluation at 1e-5 of the tensor scale."""
    from unboundednerfpytorch_b200 import models, shade as shade_mod
    assert shade_mod.MODE == 'tc3' and shade_mod.BWD_MODE == 'fused'
    torch.manual_seed(5)
    net = models._make_rgbnet(39, 128, 3).to(DEV)
    M, n_rays = 1_200_007, 2048
    g = torch.Generator().manual_seed(M)
    k0 = torch.randn(M, 12, generator=g).to(DEV)
    emb = torch.randn(n_rays, 27, generator=g).to(DEV)
    ray_id = torch.sort(torch.randint(0, n_rays, (M,), generator=g))[0].to(DEV)
    gr = (torch.rand(M, 3, generator=g) + 0.25).to(DEV)            # one-signed upstream gradient: partial sums grow steadily
    with torch.no_grad():                                          # drop ReLU-ambiguous samples (see test_fused_rgbnet_vs_torch)
        x64 = torch.cat([k0, emb[ray_id]], -1).double()
        z1 = x64 @ net[0].weight.double().t() + net[0].bias.double()
        z2 = torch.relu(z1) @ net[2][0].weight.double().t() + net[2][0].bias.double()
        ok = torch.minimum(z1.abs().amin(1), z2.abs().amin(1)) > 1e-5
        del x64, z1, z2
    k0, ray_id, gr = k0[ok].clone(), ray_id[ok].contiguous(), gr[ok].contiguous()
    net64 = models._make_rgbnet(39, 128, 3).to(DEV).double()
    net64.load_state_dict({k: v.double() for k, v in net.state_dict().items()})
    want = {}
    for lo in range(0, k0.shape[0], 200_000):                       # fp64 yardstick, chunked to bound memory
        sl = slice(lo, lo + 200_000)
        out64 = torch.sigmoid(net64(torch.cat([k0[sl], emb[ray_id[sl]]], -1).double()))
        (out64 * gr[sl].double()).sum().backward()
    want = [p.grad.clone() for p in net64.parameters()]
    k0 = k0.requires_grad_(True)
    out = shade_mod.shade(net, k0, emb, ray_id)
    (out * gr).sum().backward()
    for a, b, nm in zip([p.grad for p in net.parameters()], want, ['W1', 'b1', 'W2', 'b2', 'W3', 'b3']):
        scale = float(b.abs().max())
        err = float((a.double() - b).abs().max()) / scale
        print(f'[dw2-long] grad {nm}: max error {err:.2e} of scale')
        assert err <= 1e-5, f'grad {nm}: {err:.2e} of scale vs fp64'


def test_progressive_growing_and_occupancy_utilities(oracle):
    """SURVEY 8a row a13: scale_volume_grid / update_occupancy_cache / voxel_count_views / maskout_near_cam_vox / hit_coarse_geo as
    grid-native kernels (csrc/grid_utils.cu), each against the reference's own torch composition (FourierGrid_model.py:375-456)
    evaluated with torch ops on the same GPU: masks and counts element for element, resampled grids to fp32 rounding."""
    import torch.nn.functional as F
    from unboundednerfpytorch_b200 import grid as G
    m, kw = _fresh_model('fouriergrid', 24, 2, 1e-4, 5, dens_mean=1.0, dens_std=3.0)
    m = m.to(DEV)
    g = torch.Generator().manual_seed(11)

    # ---- voxel_count_views vs the reference composition on torch-CPU autograd (oracle.dense_grid_forward = F.grid_sample) ----
    H = W = 12
    ro = (torch.rand(2 * H, W, 3, generator=g) - 0.5)
    rd = torch.randn(2 * H, W, 3, generator=g)
    cnt = m.voxel_count_views(ro.flatten(0, 1).to(DEV), rd.flatten(0, 1).to(DEV), [H * W, H * W], near=0.0, far=1e9, stepsize=0.5,
                              irregular_shape=True)
    ws = [int(v) for v in m.world_size_density]
    ref = torch.zeros(1, 1, *ws)
    n_samples = int(torch.tensor([w + 1.0 for w in ws]).norm() / 0.5) + 1
    rng = torch.arange(n_samples)[None].float()
    for o_, d_ in zip(ro.flatten(0, 1).split(H * W), rd.flatten(0, 1).split(H * W)):
        ones = torch.zeros(1, 1, *ws, requires_grad=True)
        vec = torch.where(d_ == 0, torch.full_like(d_, 1e-6), d_)
        a, b = (m.xyz_max.cpu() - o_) / vec, (m.xyz_min.cpu() - o_) / vec
        t_min = torch.minimum(a, b).amax(-1).clamp(min=0.0, max=1e9)
        interpx = t_min[..., None] + 0.5 * m.voxel_size_density.cpu() * rng / d_.norm(dim=-1, keepdim=True)
        pts = o_[..., None, :] + d_[..., None, :] * interpx[..., None]
        oracle.dense_grid_forward(ones, pts, m.xyz_min.cpu(), m.xyz_max.cpu()).sum().backward()
        ref += (ones.grad > 1)
    assert cnt.shape == ref.shape and float(cnt.max()) == 2.0
    mism = (cnt.cpu() != ref).float().mean().item()
    assert mism < 2e-4, mism            # voxels whose accumulated weight sits within float noise of the threshold 1

    # ---- scale_volume_grid: layout contract + F.interpolate (ATen upsample_trilinear3d) on the same device ----
    before_k0 = m.k0.grid.detach().clone()
    before_d = m.density.grid.detach().clone()
    m.scale_volume_grid(30 ** 3, 30 ** 3)
    size = tuple(int(v) for v in m.world_size_rgb)
    want_k0 = F.interpolate(before_k0.contiguous(), size=size, mode='trilinear', align_corners=True)
    want_d = F.interpolate(before_d.contiguous(), size=size, mode='trilinear', align_corners=True)
    assert m.k0.grid.stride()[1] == 1 and m.k0.grid.shape == want_k0.shape
    assert_close(m.k0.grid, want_k0, rtol=1e-6, atol=1e-6, what='scale_volume_grid k0')
    assert_close(m.density.grid, want_d, rtol=1e-6, atol=1e-6, what='scale_volume_grid density')

    # ---- update_occupancy_cache: the reference's meshgrid -> density -> activate -> max_pool3d -> AND, in torch ops ----
    with torch.no_grad():
        m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, generator=g) > 0.2)
    occ0 = m.mask_cache.mask.clone()
    ms = occ0.shape
    axes = [torch.linspace(float(m.xyz_min[a]), float(m.xyz_max[a]), ms[a], device=DEV) for a in range(3)]
    xyz = torch.stack(torch.meshgrid(*axes, indexing='ij'), -1)
    with torch.no_grad():
        alpha = F.max_pool3d(m.activate_density(m.density(xyz)[None, None]), kernel_size=3, padding=1, stride=1)[0, 0]
    want_mask = occ0 & (alpha > m.fast_color_thres)
    m.update_occupancy_cache()
    assert (m.mask_cache.mask & ~occ0).sum() == 0
    flips = int((m.mask_cache.mask != want_mask).sum())
    assert flips <= 1e-4 * want_mask.numel(), f'{flips} cells differ from the torch composition'
    assert 0.05 < float(m.mask_cache.mask.float().mean()) < 0.95, 'degenerate occupancy test scene'

    # ---- maskout_near_cam_vox vs the reference loop (FourierGrid_model.py:375-388) in torch ops ----
    cams = (torch.rand(23, 3, generator=g) - 0.5).to(DEV)
    near_clip = 0.35
    want_grid = m.density.grid.detach().clone().contiguous()
    ind_norm = ((cams - m.xyz_min) / (m.xyz_max - m.xyz_min)).flip((-1,)) * 2 - 1
    F_ = m.density.nerf_pos_num_freq
    freqs = 2 ** torch.linspace(0, F_ - 1, F_, device=DEV)
    emb = [ind_norm] + [f(fr * ind_norm) for fr in freqs for f in (torch.sin, torch.cos)]
    wsd = [int(v) for v in m.world_size_density]
    lat = torch.stack(torch.meshgrid(*[torch.linspace(-1, 1, wsd[a], device=DEV) for a in range(3)], indexing='ij'), -1)
    for i, cam in enumerate(emb):
        nearest = torch.stack([(lat.unsqueeze(-2) - co).pow(2).sum(-1).sqrt().amin(-1) for co in cam.split(10)]).amin(0)
        want_grid[i][0][nearest <= near_clip] = -100
    m.maskout_near_cam_vox(cams, near_clip)
    n_hit = int((want_grid == -100).sum())
    assert n_hit > 0
    diff = int((m.density.grid.detach() != want_grid).sum())
    assert diff <= 1e-4 * want_grid.numel(), f'{diff} voxels differ from the reference loop ({n_hit} masked)'

    # the model still renders, and hit_coarse_geo has the reference's shape / dtype contract
    ro1, rd1, vd1 = seeded_rays(64, 3, DEV)
    out = m(ro1, rd1, vd1, near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5)
    assert torch.isfinite(out['rgb_marched']).all()
    hit = m.hit_coarse_geo(ro1, rd1, near=0., far=1e9, stepsize=0.5)
    assert hit.shape == (64,) and hit.dtype == torch.bool


def test_reduce_tv_step_single_process_matches_tv_then_step():
    """dist.reduce_tv_step at world 1 == total_variation_add_grad on both grids + MaskedAdam.step() (run_train.py:281-289)."""
    from unboundednerfpytorch_b200 import dist as D, models
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    outs = []
    for use_tail in (False, True):
        torch.manual_seed(3)
        m = models.FourierGridModel(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=20 ** 3,
                                    num_voxels_base_density=20 ** 3, num_voxels_rgb=20 ** 3, num_voxels_base_rgb=20 ** 3,
                                    num_voxels_viewdir=-1, alpha_init=1e-4, fast_color_thres=0, rgbnet_dim=12,
                                    fourier_freq_num=2).to(DEV)
        opt = create_optimizer_or_freeze_model(m, dict(lrate_density=0.1, lrate_k0=0.1, lrate_rgbnet=1e-3, lrate_decay=20,
                                                       skip_zero_grad_fields=['density', 'k0']), 0)
        g = torch.Generator().manual_seed(9)
        for p in m.parameters():
            if not p.requires_grad:
                continue
            grad = (torch.randn(p.shape, generator=g) * (torch.rand(p.shape, generator=g) > 0.5)).to(DEV)
            p.grad = torch.empty_like(p, memory_format=torch.preserve_format).copy_(grad)     # same layout as the parameter
        if use_tail:
            D.reduce_tv_step(opt, m.tv_terms(1e-3, 1e-4, True))
        else:
            m.density_total_variation_add_grad(1e-3, True)
            m.k0_total_variation_add_grad(1e-4, True)
            opt.step()
        outs.append({k: v.detach().clone() for k, v in m.state_dict().items()})
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k


@pytest.mark.parametrize('flavor,F_', [('fouriergrid', 3), ('dcvgo', 0)])
def test_psnr_delta_vs_oracle(flavor, F_):
    """BASELINE.json metric, second half: "PSNR delta vs ref" (SURVEY.md 8d protocol, no datasets offline; see
    oracle/psnr_check.py).  Gate: |PSNR(cuda, GT) - PSNR(oracle, GT)| <= 0.01 dB, student images agree to > 90 dB."""
    from oracle.psnr_check import psnr_delta
    r = psnr_delta(flavor, F_, DEV)
    print(f"[psnr] {flavor}: PSNR(oracle, GT) = {r['psnr_oracle']:.4f} dB, PSNR(cuda, GT) = {r['psnr_cuda']:.4f} dB, "
          f"delta = {r['delta_db']:+.2e} dB, PSNR(cuda vs oracle) = {r['psnr_cuda_vs_oracle']:.1f} dB")
    assert r['gt_std'] > 0.02, 'degenerate teacher image'
    assert 5.0 < r['psnr_oracle'] < 60.0, 'student should differ visibly from the teacher'
    assert abs(r['delta_db']) <= 0.01
    assert r['psnr_cuda_vs_oracle'] > 90.0


def test_psnr_gate_of_the_single_pass_tf32_mode(monkeypatch):
    """The opt-in reduced-precision rgbnet mode (UBN_RGBNET_MODE=tc1: one TF32 pass per product instead of the 3-pass split) is not
    held to the 1e-5 parity bar; its gate is BASELINE.json's image metric: rendered PSNR within 0.01 dB of the reference."""
    from oracle.psnr_check import psnr_delta
    from unboundednerfpytorch_b200 import shade as shade_mod
    monkeypatch.setattr(shade_mod, 'MODE', 'tc1')
    for flavor, F_ in (('fouriergrid', 3), ('dcvgo', 0)):
        r = psnr_delta(flavor, F_, DEV)
        print(f"[psnr tf32x1] {flavor}: delta = {r['delta_db']:+.2e} dB, PSNR(cuda vs oracle) = {r['psnr_cuda_vs_oracle']:.1f} dB")
        assert abs(r['delta_db']) <= 0.01
        assert r['psnr_cuda_vs_oracle'] > 45.0


@pytest.mark.parametrize('flavor,F_,thres', [('fouriergrid', 4, 0.0), ('fouriergrid', 2, 1e-4), ('dcvgo', 0, 1e-4)])
def test_feature_kernel_families_agree(flavor, F_, thres):
    """Pass B in its four forms (ubn_set_feature_kernel 0 / 1 / 2 / 3: warp-cooperative, lane-per-sample forward, lane-per-sample
    forward + backward, lane-per-sample forward + slab-major scatter): identical survivors and records, features / rgb equal to fp32 rounding, k0 gradients equal to the
    atomics' summation order; and the lane-per-sample forward is BIT-identical to the stand-alone grid op (ATen corner order +
    torch-CUDA slab-mean order), i.e. to what F.grid_sample(...).mean(0) returns in the reference."""
    from unboundednerfpytorch_b200 import ops
    m, _ = _fresh_model(flavor, 40, F_, thres, 11, dens_mean=5.0 if thres else 0.0, dens_std=3.0 if thres else 1.0)
    m = m.to(DEV)
    ro, rd, vd = seeded_rays(700, 12, DEV)
    rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, render_depth=True)
    outs, grads = [], []
    default = ops.get_feature_kernel()
    try:
        for variant in (0, 1, 2, 3, 4, 5, 6):
            ops.set_feature_kernel(variant)
            assert ops.get_feature_kernel() == variant
            m.zero_grad(set_to_none=True)
            ret = m(ro, rd, vd, global_step=None, **rk)
            (ret['rgb_marched'].sum() + 0.1 * ret['raw_rgb'].pow(2).sum()).backward()
            outs.append(ret)
            grads.append(m.k0.grid.grad.detach().clone())
    finally:
        ops.set_feature_kernel(default)
    for ret in outs[1:]:
        assert torch.equal(ret['ray_id'], outs[0]['ray_id']) and torch.equal(ret['step_id'], outs[0]['step_id'])
        for k in ('weights', 'raw_density', 't'):
            assert torch.equal(ret[k], outs[0][k]), k
        assert_close(ret['raw_rgb'], outs[0]['raw_rgb'], rtol=1e-5, atol=1e-6, what='raw_rgb across kernel families')
        assert_close(ret['rgb_marched'], outs[0]['rgb_marched'], rtol=1e-5, atol=1e-6, what='rgb_marched across kernel families')
    for gk in grads[1:]:
        # the families round the features differently, so a handful of rgbnet pre-activations within rounding distance of zero get
        # another ReLU mask (see tests/parity_at_size.py): element-wise agreement up to a tiny fraction of the tensor
        scale = float(grads[0].abs().max())
        beyond = ((gk - grads[0]).abs() > 1e-5 * scale + 1e-4 * grads[0].abs()).float().mean().item()
        assert beyond <= 1e-3, f'k0 grad across kernel families: {beyond:.2e} of the elements beyond tolerance'
    # bit parity of the lane-per-sample forward with what the REFERENCE computes: F.grid_sample over the slabs + .mean(0) in torch
    # (oracle.cpu_ref.fourier_grid_forward on CUDA tensors = FourierGrid_grid.py:60-78 / grid.py:50-61 verbatim)
    from oracle import cpu_ref
    for variant in (3, 6):          # both lane-per-sample gathers (32 samples x 1 lane, 8 samples x 3 quad lanes per instruction)
        with torch.no_grad():
            ops.set_feature_kernel(variant)
            try:
                (w, last, alpha, dens, k0, ray_id, step_id, t, inner), _ = m._march(ro, rd, 0.5)
            finally:
                ops.set_feature_kernel(default)
            pts, _, _ = m._sample_dense(ro, rd, 0.5)
            want = cpu_ref.fourier_grid_forward(m.k0.grid.detach().contiguous(), pts[ray_id, step_id], m.xyz_min, m.xyz_max,
                                                F_ if flavor == 'fouriergrid' else 0)
        assert torch.equal(k0, want), f'variant {variant}: {int((k0 != want).sum())} of {k0.numel()} feature values differ from grid_sample + mean'
