"""metrics.rgb_ssim (csrc/metrics.cu) against the reference's utils.rgb_ssim, element by element, and its use by
render.render_viewpoints and by the reference's unmodified run_render.render_viewpoints.

Tolerances: every map element within 1e-10 of the reference's, the mean within 1e-12.  The reference filters the fp32-rounded
images and products in fp64, so the kernel differs from it only in the order of the fp64 sums.  A reordered sum of f <= 32 taps
of values <= max_val**2 moves a moment by a few ulps of max_val**2, ~1e-15 for max_val = 1; the variance cancels that against
mu**2 without amplifying the absolute error, and the map divides it by sigma00 + sigma11 + c2 >= c2 = 9e-4, so a map element
moves by ~1e-12 and the mean of many by less.  On the CPU two fp64 orders agreed within 1.2e-12 per element and 2e-15 on the
mean, 100x inside the bounds; fp32 moments miss them by orders of magnitude (up to 9.5e-5 on the map, 2.5e-7 on the mean).
For max_val = 255 both the moments and c1, c2 scale by 255**2, so the same bounds hold."""
import os
import re
import sys
import types

import numpy as np
import pytest
import torch

from oracle import ssim_ref
from tests.util import ROOT, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
PY = os.path.join(ROOT, 'oracle', '_ref', 'py')
MAP_TOL, MEAN_TOL = 1e-10, 1e-12


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


@pytest.fixture(scope='module')
def ref():
    """The reference's own utils / run_render / dvgo, staged by __graft_entry__.build() into git-ignored oracle/_ref/py/."""
    if not os.path.exists(os.path.join(PY, 'FourierGrid', 'run_render.py')):
        if os.environ.get('UBN_ALLOW_NO_REF') == '1':
            pytest.skip('oracle/_ref/py not staged (UBN_ALLOW_NO_REF=1)')
        pytest.fail('oracle/_ref/py/FourierGrid/run_render.py is missing: run __graft_entry__.build() where the reference exists')
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
    # run_render.py's imports that its render_viewpoints does not reach: video writing, colour maps, style transfer
    _stub('imageio', imwrite=unused, mimwrite=unused)
    _stub('matplotlib').__path__ = []
    _stub('matplotlib.pyplot', get_cmap=unused)
    _stub('FourierGrid.arf', ARF=unused)
    sys.path.insert(0, PY)
    try:
        from FourierGrid import dcvgo, dmpigo, dvgo, run_render, utils
    finally:
        sys.path.remove(PY)
    return types.SimpleNamespace(utils=utils, run_render=run_render, dvgo=dvgo, dcvgo=dcvgo, dmpigo=dmpigo)


def _compare(got_map, got_mean, want_map, want_mean, what):
    got_map = got_map.cpu().numpy() if isinstance(got_map, torch.Tensor) else got_map
    assert got_map.dtype == np.float64 and got_map.shape == want_map.shape, what
    nan = np.isnan(want_map)
    assert np.array_equal(np.isnan(got_map), nan), f'{what}: NaN positions differ'
    if (~nan).any():
        err = np.abs(got_map[~nan] - want_map[~nan]).max()
        assert err <= MAP_TOL, f'{what}: map max abs err {err:.3e}'
    if np.isnan(want_mean):
        assert np.isnan(got_mean), what
    else:
        assert abs(float(got_mean) - float(want_mean)) <= MEAN_TOL, f'{what}: mean {float(got_mean)!r} vs {float(want_mean)!r}'


# ---------------------------------------------------------------------------------------------------------------------------
# against the reference's maps and means
# ---------------------------------------------------------------------------------------------------------------------------
def test_small_goldens_numpy_and_tensor_input():
    """Every frame kind, a single output row and column, filter_size 1 / 10 / 32, non-default sigma / k1 / k2, max_val 255, a NaN
    pixel; numpy input (returns np.float64 / a float64 ndarray) and CUDA tensors (CUDA float64 tensors) give the same bits."""
    from unboundednerfpytorch_b200 import metrics
    for name, g in load_golden('l2_ssim/small.pt').items():
        kw = dict(g['kwargs'])
        mean = metrics.rgb_ssim(g['img0'], g['img1'], g['max_val'], **kw)
        m = metrics.rgb_ssim(g['img0'], g['img1'], g['max_val'], return_map=True, **kw)
        assert type(mean) is np.float64 and isinstance(m, np.ndarray), name
        _compare(m, mean, g['map'], g['mean'], name)
        a, b = torch.from_numpy(g['img0']).to(DEV), torch.from_numpy(g['img1']).to(DEV)
        tmean = metrics.rgb_ssim(a, b, g['max_val'], **kw)
        tmap = metrics.rgb_ssim(a, b, g['max_val'], return_map=True, **kw)
        assert tmean.is_cuda and tmean.dtype == torch.float64 and tmean.dim() == 0, name
        assert tmap.is_cuda and tmap.dtype == torch.float64, name
        assert np.array_equal(tmap.cpu().numpy(), m, equal_nan=True), name
        assert np.array_equal(tmean.cpu().numpy(), mean, equal_nan=True), name


def test_large_goldens():
    from unboundednerfpytorch_b200 import metrics
    for name, g in load_golden('l2_ssim/large.pt').items():
        a, b = ssim_ref.ssim_frames(g['kind'], g['H'], g['W'], g['seed'])
        mean = metrics.rgb_ssim(a, b, g['max_val'], **g['kwargs'])
        assert abs(mean - g['mean']) <= MEAN_TOL, (name, mean, g['mean'])


@pytest.mark.parametrize('kind', ['noise', 'ramp', 'flat', 'near'])
@pytest.mark.parametrize('W,H', [(1008, 756), (1237, 822), (1600, 1067)])
def test_against_staged_reference_at_render_sizes(ref, kind, W, H):
    from unboundednerfpytorch_b200 import metrics
    a, b = ssim_ref.ssim_frames(kind, H, W, seed=W + H)
    want = ref.utils.rgb_ssim(a, b, max_val=1, return_map=True)
    ta, tb = torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)
    _compare(metrics.rgb_ssim(ta, tb, 1, return_map=True), metrics.rgb_ssim(ta, tb, 1).item(), want, np.mean(want),
             f'{kind} {W}x{H}')


# ---------------------------------------------------------------------------------------------------------------------------
# shapes, degenerate inputs, determinism
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('f', [11, 1, 10, 32])
def test_every_tile_remainder_against_fp64(f):
    """Map sizes Ho = 32 q + r and Wo = 32 q' + r' with r and r' each taking every value 0 .. 31 (tiles are 32 x 32), against the
    fp64 restatement of oracle/ssim_ref.py.  r = 1 gives an image exactly filter_size tall, r = 0 one exactly filter_size wide."""
    from unboundednerfpytorch_b200 import metrics
    for r in range(32):
        ho = 32 * ((r // 2) % 2) + (r or 32)
        wo = 32 * ((r // 3) % 2) + ((7 * r + 1) % 32 or 32)
        H, W = ho + f - 1, wo + f - 1
        a, b = ssim_ref.ssim_frames('noise' if r % 2 else 'ramp', H, W, seed=100 + r)
        want_map, want_mean = ssim_ref.rgb_ssim_fp64(a, b, 1, filter_size=f)
        ta, tb = torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)
        _compare(metrics.rgb_ssim(ta, tb, 1, filter_size=f, return_map=True), metrics.rgb_ssim(ta, tb, 1, filter_size=f).item(),
                 want_map, want_mean, f'f={f} {H}x{W}')


@pytest.mark.parametrize('kind,H,W,f', [('noise', 756, 1008, 11), ('ramp', 64, 80, 11), ('flat', 50, 41, 1), ('near', 45, 70, 32),
                                        ('ramp', 10, 10, 10)])
def test_identical_frames_score_exactly_one(kind, H, W, f):
    from unboundednerfpytorch_b200 import metrics
    a, _ = ssim_ref.ssim_frames(kind, H, W, seed=5)
    t = torch.from_numpy(a).to(DEV)
    m = metrics.rgb_ssim(t, t.clone(), 1, filter_size=f, return_map=True)
    assert bool((m == 1.0).all()), f'{int((m != 1.0).sum())} map elements differ from 1'
    assert metrics.rgb_ssim(t, t.clone(), 1, filter_size=f).item() == 1.0
    assert metrics.rgb_ssim(a, a.copy(), 1, filter_size=f) == 1.0


def test_nan_pixel_poisons_exactly_its_windows():
    from unboundednerfpytorch_b200 import metrics
    H, W, f = 100, 90, 11
    a, b = ssim_ref.ssim_frames('noise', H, W, seed=9)
    nans = [(0, 0, 0), (50, 47, 1), (99, 89, 2), (33, 5, 1)]
    for y, x, c in nans:
        (a if y % 2 else b)[y, x, c] = np.nan
    expect = np.zeros((H - f + 1, W - f + 1, 3), bool)
    for y, x, c in nans:
        expect[max(0, y - f + 1):y + 1, max(0, x - f + 1):x + 1, c] = True
    m = metrics.rgb_ssim(a, b, 1, return_map=True)
    assert np.array_equal(np.isnan(m), expect)
    assert np.isnan(metrics.rgb_ssim(a, b, 1))
    want_map, _ = ssim_ref.rgb_ssim_fp64(a, b, 1)
    assert np.abs(m[~expect] - want_map[~expect]).max() <= MAP_TOL


def test_two_calls_give_the_same_bits():
    from unboundednerfpytorch_b200 import metrics
    a, b = ssim_ref.ssim_frames('near', 1067, 1600, seed=3)
    ta, tb = torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)
    m1, m2 = (metrics.rgb_ssim(ta, tb, 1, return_map=True) for _ in range(2))
    s1, s2 = (metrics.rgb_ssim(ta, tb, 1) for _ in range(2))
    assert torch.equal(m1, m2)
    assert s1.view(torch.int64).item() == s2.view(torch.int64).item()


def test_runs_on_the_callers_stream():
    from unboundednerfpytorch_b200 import metrics
    a, b = ssim_ref.ssim_frames('ramp', 300, 400, seed=4)
    ta, tb = torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)
    want = metrics.rgb_ssim(ta, tb, 1).item()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)              # a busy stream: the result is only right if the kernel queues behind it
        tb2 = tb * 1.0
        got = metrics.rgb_ssim(ta, tb2, 1)
    torch.cuda.current_stream().wait_stream(s)
    assert got.item() == want


# ---------------------------------------------------------------------------------------------------------------------------
# render_viewpoints
# ---------------------------------------------------------------------------------------------------------------------------
def _model(seed=3):
    from unboundednerfpytorch_b200 import models
    torch.manual_seed(seed)
    m = models.DirectContractedVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=32 ** 3, num_voxels_base=32 ** 3, alpha_init=1e-2,
                                     fast_color_thres=1e-4, rgbnet_dim=12, contracted_norm='l2')
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        m.density.grid.copy_(torch.randn(m.density.grid.shape, generator=g) * 3 + 2)
        m.k0.grid.copy_(torch.randn(m.k0.grid.shape, generator=g))
    return m.to(DEV)


def _views(H=45, W=61):
    K = np.array([[60., 0., W / 2], [0., 60., H / 2], [0., 0., 1.]])
    poses = [np.array([[1., 0., 0., 0.1], [0., 1., 0., -0.2], [0., 0., 1., 0.3]], dtype=np.float32),
             np.array([[0., 0., 1., -0.3], [0., 1., 0., 0.0], [-1., 0., 0., 0.2]], dtype=np.float32)]
    gt = [np.random.RandomState(i).rand(H, W, 3).astype(np.float32) for i in range(2)]
    return poses, [(H, W)] * 2, [K] * 2, gt


def _printed(out, key):
    lines = [ln for ln in out.splitlines() if ln.startswith(key + ' ')]
    assert len(lines) == 1, out
    return lines[0], float(re.fullmatch(rf'{key} (\S+) \(avg\)', lines[0]).group(1))


def test_render_viewpoints_eval_ssim(ref, capsys):
    from unboundednerfpytorch_b200 import render as RD
    m = _model()
    poses, HW, Ks, gt = _views()
    rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, render_depth=True)
    capsys.readouterr()
    plain = RD.render_viewpoints(None, m, poses, HW, Ks, False, rk, gt_imgs=gt, chunk=512)
    psnr_plain, _ = _printed(capsys.readouterr().out, 'Psnr')
    scored = RD.render_viewpoints(None, m, poses, HW, Ks, False, rk, gt_imgs=gt, eval_ssim=True, chunk=512)
    out = capsys.readouterr().out
    psnr_line, _ = _printed(out, 'Psnr')
    _, ssim = _printed(out, 'Ssim')
    assert out.index('Psnr') < out.index('Ssim')
    assert psnr_line == psnr_plain
    for x, y in zip(plain, scored):
        assert x.dtype == y.dtype and np.array_equal(x, y)
    want = np.mean([ref.utils.rgb_ssim(rgb, g, max_val=1) for rgb, g in zip(scored[0], gt)])
    assert abs(ssim - want) <= MEAN_TOL, (ssim, want)
    # nothing to score: no ground truth, or a scaled render
    with pytest.raises(NotImplementedError):
        RD.render_viewpoints(None, m, poses, HW, Ks, False, rk, gt_imgs=gt, render_factor=2, eval_ssim=True)
    with pytest.raises(NotImplementedError):
        RD.render_viewpoints(None, m, poses, HW, Ks, False, rk, eval_ssim=True)
    with pytest.raises(NotImplementedError):
        RD.render_viewpoints(None, m, poses, HW, Ks, False, rk, gt_imgs=gt, eval_lpips_alex=True)


class Cfg(dict):
    """The attribute-and-key access of the reference's mmengine Config."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None


def test_reference_run_render_scores_on_the_gpu_under_install_metrics(ref, capsys):
    """The reference's own run_render.render_viewpoints, unmodified, on this package's model: with install_metrics its
    utils.rgb_ssim is metrics.rgb_ssim, and the printed Ssim agrees with the same call on scipy."""
    import warnings
    from unboundednerfpytorch_b200 import legacy, metrics
    m = _model(5)
    poses, HW, Ks, gt = _views(37, 50)
    cfg = Cfg(model='DVGO', data=Cfg(dataset_type='llff', flip_x=False, flip_y=False))
    rk = dict(near=0., far=1e9, bg=1, stepsize=0.5, inverse_y=False, flip_x=False, flip_y=False, render_depth=True)

    def run():
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            torch.set_default_tensor_type('torch.cuda.FloatTensor')     # run_FourierGrid.py:87, which the driver's rays rely on
        try:
            out = ref.run_render.render_viewpoints(cfg, m, torch.tensor(np.stack(poses), device=DEV), np.array(HW), np.stack(Ks),
                                                   False, rk, gt_imgs=gt, eval_ssim=True)
        finally:
            with warnings.catch_warnings():
                warnings.simplefilter('ignore')
                torch.set_default_tensor_type('torch.FloatTensor')
        return out, capsys.readouterr().out

    capsys.readouterr()
    with legacy.install_models(ref.run_render, ref.dvgo, ref.dcvgo, ref.dmpigo, ref.utils), \
            legacy.install_metrics(ref.run_render, ref.utils):
        assert ref.utils.rgb_ssim is metrics.rgb_ssim
        gpu, out_gpu = run()
    assert ref.utils.rgb_ssim is not metrics.rgb_ssim                     # restored
    cpu, out_cpu = run()
    _, s_gpu = _printed(out_gpu, 'Ssim')
    _, s_cpu = _printed(out_cpu, 'Ssim')
    assert abs(s_gpu - s_cpu) <= MEAN_TOL, (s_gpu, s_cpu)
    assert _printed(out_gpu, 'Psnr') == _printed(out_cpu, 'Psnr')
    for x, y in zip(gpu, cpu):
        assert np.array_equal(x, y)
