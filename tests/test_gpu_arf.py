"""arf.ARF and its kernels (csrc/color.cu) against fp64, against the reference's goldens, against the reference's own ARF on the
GPU, and inside the reference's unmodified run_render block render.

Bounds (u32 = 2^-24, u64 = 2^-53, gamma_n(u) = n u / (1 - n u)):

* Moments.  ubn_color_moments adds fp64 terms d_i = x_i - k_i (exact: x and k are fp32 of similar magnitude) and d_i d_j (one
  rounding each).  Every partial sum passes through at most D = 4 ceil(n / (4 * 256 * 1056)) + 40 additions: the grid-stride
  loop (4 pixels per group), a head and a tail pixel, 5 shuffle levels, 8 warps, the closing block's stride over at most 1056
  partials (<= 5) and again 5 + 8.  So |dS_ij| <= gamma_(D+1)(u64) sum|d_i d_j| and |dS_i| <= gamma_D(u64) sum|d_i|.  The mean
  k + S / n adds two roundings and the covariance S_ij / n - m_i m_j three and the errors of m_i, m_j (|m_i| <= E|d_i|), so
  |d mu_i| <= gamma_(D+3) (|k_i| + E|d_i|) and |d c_ij| <= 3 gamma_(D+4) (E|d_i d_j| + E|d_i| E|d_j|).  The two-pass numpy
  reference errs by far less.
* Affine.  Three dependent fmas per channel, one rounding each: |y - (T x + b)| <= gamma_3(u32) (|b| + |T| |x|) against the
  exact value of the same fp32 T, b; the fp64 evaluation adds < 4 u64 of the same scale, and the clamp is 1-Lipschitz.
* End to end.  T and b are the fp64 transform rounded once to fp32 and then applied as above: <= gamma_4(u32) (|b| + |T| |x|)
  + 1e-9 of the same scale for the fp64 moments and SVD (oracle.arf_ref.transform_rounding_bound); the reference's own fp32
  error is oracle.arf_ref.reference_fp32_bound."""
import importlib.util
import math
import os
import sys
import types
import warnings
from fractions import Fraction

import cv2
import numpy as np
import pytest
import torch

from oracle import arf_ref
from tests.util import ROOT, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
PY = os.path.join(ROOT, 'oracle', '_ref', 'py')
U64 = 2.0 ** -53
CTAS, THREADS = 1056, 256
SETS = ('random', 'random_landscape', 'near_grey', 'constant', 'one_pixel', 'outside')
REF_TOL = 1e-5


class Cfg(dict):
    """The attribute-and-key access of the reference's mmengine Config."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def write_png_bytes(path, rgb):
    ok, buf = cv2.imencode('.png', np.ascontiguousarray(rgb[..., ::-1]))
    assert ok
    buf.tofile(path)


class ImageioStub:
    """imageio as the reference's arf.py / run_render.py use it, on cv2 (PNG bytes only), with the videos captured."""

    def __init__(self):
        self.videos = []

    @staticmethod
    def imread(path):
        return np.ascontiguousarray(cv2.imread(path, cv2.IMREAD_UNCHANGED)[..., ::-1])

    @staticmethod
    def imwrite(path, a):
        cv2.imwrite(path, np.ascontiguousarray(np.asarray(a)[..., ::-1]))

    def mimwrite(self, path, frames, **kw):
        self.videos.append((path, np.asarray(frames), kw))


def _staged():
    if not os.path.exists(os.path.join(PY, 'FourierGrid', 'arf.py')):
        if os.environ.get('UBN_ALLOW_NO_REF') == '1':
            pytest.skip('oracle/_ref/py not staged (UBN_ALLOW_NO_REF=1)')
        pytest.fail('oracle/_ref/py/FourierGrid/arf.py is missing: run __graft_entry__.build() where the reference exists')


@pytest.fixture(scope='module')
def ref_arf():
    """The reference's own ARF class, loaded from the staged arf.py under a private module name (another test module may have
    stubbed FourierGrid.arf), its imageio bound to the cv2 stand-in."""
    _staged()
    spec = importlib.util.spec_from_file_location('_staged_reference_arf', os.path.join(PY, 'FourierGrid', 'arf.py'))
    mod = importlib.util.module_from_spec(spec)
    saved = sys.modules.get('imageio')
    sys.modules['imageio'] = ImageioStub()
    try:
        spec.loader.exec_module(mod)
    finally:
        if saved is None:
            del sys.modules['imageio']
        else:
            sys.modules['imageio'] = saved
    return mod


@pytest.fixture(scope='module')
def ref_render():
    """The reference's run_render / utils / dvgo, staged by __graft_entry__.build() into git-ignored oracle/_ref/py/."""
    _staged()
    from unboundednerfpytorch_b200 import functional as F_, legacy
    legacy.install()

    def unused(*a, **k):
        raise NotImplementedError('not on the path these tests drive')
    _stub('torch_scatter', segment_coo=F_.segment_coo, scatter_add=unused)
    _stub('torch_efficient_distloss', flatten_eff_distloss=F_.flatten_eff_distloss)
    if 'imageio' not in sys.modules:
        _stub('imageio', imwrite=unused, mimwrite=unused)
    if 'matplotlib' not in sys.modules:
        _stub('matplotlib').__path__ = []
        _stub('matplotlib.pyplot', get_cmap=unused)
    sys.path.insert(0, PY)
    try:
        from FourierGrid import run_render, utils
    finally:
        sys.path.remove(PY)
    return types.SimpleNamespace(run_render=run_render, utils=utils)


def _stylizer(kind, HW, tmp_path, style_id=34):
    from unboundednerfpytorch_b200.arf import ARF
    root = tmp_path / f'styles_{kind}'
    root.mkdir(exist_ok=True)
    write_png_bytes(str(root / f'{style_id}.jpg'), load_golden(f'l2_arf/style_{kind}.pt')['source'])
    return ARF(Cfg(arf=Cfg(style_root=str(root), style_id=style_id)), {'HW': np.array([HW])}, DEV)


# ---------------------------------------------------------------------------------------------------------------------------
# ubn_color_moments
# ---------------------------------------------------------------------------------------------------------------------------
def _depth(n):
    return 4 * math.ceil(n / (4 * THREADS * CTAS)) + 40


def _gamma64(n):
    return n * U64 / (1 - n * U64)


def _check_moments(x, mu, cov, what):
    x64 = x.reshape(-1, 3).astype(np.float64)
    n = len(x64)
    mu_ref, cov_ref = arf_ref.moments_fp64(x64)
    k = x64[0]
    d = np.abs(x64 - k)
    Ed = d.mean(0)
    D = _depth(n)
    tol_mu = 2 * _gamma64(D + 3) * (np.abs(k) + Ed)
    tol_cov = 3 * _gamma64(D + 4) * (d.T @ d / n + np.outer(Ed, Ed))
    assert (np.abs(mu - mu_ref) <= tol_mu).all(), f'{what}: mean {mu} vs {mu_ref}, tol {tol_mu}'
    err = np.abs(cov - cov_ref)
    assert (err <= tol_cov).all(), f'{what}: covariance err {err.max():.3e}, worst ratio {(err / tol_cov).max():.3f}'


MOMENT_SIZES = [1, 2, 3, 4, 5, 6, 7, 8, 9, 1021, 1022, 1023, 1024, 4 * THREADS * CTAS + 3, 3_000_001]


@pytest.mark.parametrize('n', MOMENT_SIZES)
def test_moments_against_fp64_at_every_offset(n):
    from unboundednerfpytorch_b200 import arf
    rs = np.random.RandomState(n % 1000)
    host = (0.4 + 0.2 * rs.randn(n + 2, 3)).astype(np.float32)
    host[0] = (3.0, -1.0, 0.5)                         # the shift pixel far from the mean
    flat = torch.from_numpy(host.reshape(-1)).to(DEV)
    for off in range(4):
        buf = torch.empty(3 * n + 8, dtype=torch.float32, device=DEV)
        view = buf[off:off + 3 * n].view(n, 3)
        view.copy_(flat[:3 * n].view(n, 3))
        assert view.storage_offset() == off
        mu, cov = arf.color_moments(view)
        assert mu.dtype == cov.dtype == np.float64
        assert np.array_equal(cov, cov.T)
        _check_moments(host[:n], mu, cov, f'n={n} offset={off}')
        mu2, cov2 = arf.color_moments(view)
        assert mu.tobytes() == mu2.tobytes() and cov.tobytes() == cov2.tobytes(), f'n={n} offset={off}: calls differ'


def test_moments_of_a_set_above_2_31_floats():
    """716 M pixels (8.6 GB, 2.148e9 floats > 2^31): channel c of pixel p is ((3 p + c) mod 256) / 256, so the set repeats every
    256 pixels and its moments are those of one period, computed exactly with fractions.  Every d and d_i d_j is a multiple of
    2^-16 below 1 and every partial sum below 2^30, so the fp64 sums are exact: the result is the exact moment up to the last
    division and product (a few ulp).  Then the transform y = x / 2 + 1 / 4 (exact in fp32) runs in place over the whole set."""
    from unboundednerfpytorch_b200 import arf
    n = 716_000_000
    assert 3 * n > 2 ** 31 and n % 256 == 0
    period = [[Fraction((3 * p + c) % 256, 256) for c in range(3)] for p in range(256)]
    mu_exact = [sum(px[c] for px in period) / 256 for c in range(3)]
    cov_exact = [[sum((px[i] - mu_exact[i]) * (px[j] - mu_exact[j]) for px in period) / 256 for j in range(3)] for i in range(3)]
    row = (torch.arange(768, device=DEV) % 256).float() / 256
    big = row.repeat(n // 256)
    try:
        mu, cov = arf.color_moments(big.view(n, 3))
        for i in range(3):
            assert abs(mu[i] - float(mu_exact[i])) <= 4 * U64 * abs(float(mu_exact[i])), (i, mu[i], float(mu_exact[i]))
            for j in range(3):
                assert abs(cov[i, j] - float(cov_exact[i][j])) <= 8 * U64 * 0.5, (i, j, cov[i, j], float(cov_exact[i][j]))
        mu2, cov2 = arf.color_moments(big.view(n, 3))
        assert mu.tobytes() == mu2.tobytes() and cov.tobytes() == cov2.tobytes()
        arf.color_affine(big.view(n, 3), 0.5 * np.eye(3), [0.25] * 3, out=big.view(n, 3))
        want = row * 0.5 + 0.25
        chunk = 768 * (1 << 18)
        for s in range(0, big.numel(), chunk):
            part = big[s:s + chunk].view(-1, 768)
            assert bool((part == want).all()), f'affine wrong in floats {s} .. {s + chunk}'
    finally:
        del big
        torch.cuda.empty_cache()


def test_non_finite_moments_name_the_set(tmp_path):
    st = _stylizer('portrait', (48, 64), tmp_path)
    x = arf_ref.content_set('random', (2, 10, 12, 3), 1)
    x[1, 3, 4, 2] = np.nan
    with pytest.raises(ValueError, match='content set'):
        st.match_colors_for_image_set(x, str(tmp_path))
    x[1, 3, 4, 2] = np.inf
    with pytest.raises(ValueError, match='content set'):
        st.match_colors_for_image_set(torch.from_numpy(x).to(DEV), str(tmp_path))


# ---------------------------------------------------------------------------------------------------------------------------
# ubn_color_affine
# ---------------------------------------------------------------------------------------------------------------------------
def _affine_case(n, seed):
    rs = np.random.RandomState(seed)
    x = rs.uniform(-0.5, 1.5, (n, 3)).astype(np.float32)
    T = (rs.randn(3, 3) * np.array([[1.0], [30.0], [0.3]])).astype(np.float32)
    b = (rs.randn(3) * 5).astype(np.float32)
    return x, T, b


def _check_affine(x, T, b, y, what):
    x64, T64, b64 = x.astype(np.float64), T.astype(np.float64), b.astype(np.float64)
    with np.errstate(invalid='ignore', over='ignore'):
        pre = (x64[:, None, :] * T64[None]).sum(-1) + b64                # no BLAS: IEEE inf / NaN arithmetic term by term
        want = np.clip(pre, 0., 1.)
        scale = np.abs(b64) + (np.abs(x64)[:, None, :] * np.abs(T64)[None]).sum(-1)
    nan = np.isnan(pre)
    assert np.array_equal(np.isnan(y), nan), f'{what}: NaN positions differ'
    inf = np.isinf(pre)
    assert np.array_equal(y[inf], want[inf]), f'{what}: clamp of an infinite value'
    fin = ~nan & ~inf
    tol = (arf_ref.gamma(3) + 4 * U64) * scale[fin]
    err = np.abs(y[fin] - want[fin])
    assert (err <= tol).all(), f'{what}: max err {err.max():.3e}, worst ratio {(err / np.maximum(tol, 1e-300)).max():.3f}'
    assert ((y[~nan] >= 0) & (y[~nan] <= 1)).all()


AFFINE_SIZES = [1, 2, 3, 4, 5, 6, 7, 8, 9, 1001, 1024, 4 * THREADS * CTAS + 5, 2_000_003]


@pytest.mark.parametrize('n', AFFINE_SIZES)
def test_affine_against_fp64_at_every_alignment_and_in_place(n):
    from unboundednerfpytorch_b200 import arf
    x, T, b = _affine_case(n, n % 997)
    if n >= 8:                                         # non-finite inputs: NaN and both infinities
        x[n // 2, 1] = np.nan
        x[n // 3, 0] = np.inf
        x[n - 1, 2] = -np.inf
    src = torch.from_numpy(x).to(DEV)
    results = []
    for off_in in range(4):
        bin_ = torch.empty(3 * n + 8, device=DEV)
        xin = bin_[off_in:off_in + 3 * n].view(n, 3)
        xin.copy_(src)
        for off_out in range(4):
            bout = torch.full((3 * n + 8,), -7.0, device=DEV)
            yout = bout[off_out:off_out + 3 * n].view(n, 3)
            arf.color_affine(xin, T, b, out=yout)
            assert bool((bout[:off_out] == -7).all()) and bool((bout[off_out + 3 * n:] == -7).all()), 'wrote outside out'
            results.append(yout.clone())
        assert xin.view(torch.int32).equal(src.view(torch.int32)), 'out-of-place call changed its input'
        arf.color_affine(xin, T, b, out=xin)                           # in place
        results.append(xin.clone())
    y0 = results[0].view(torch.int32)
    for i, r in enumerate(results[1:]):
        assert r.view(torch.int32).equal(y0), f'n={n}: result {i + 1} differs in bits from the aligned out-of-place one'
    _check_affine(x, T, b, results[0].cpu().numpy(), f'n={n}')


def test_affine_clamp_matches_torch_clamp():
    """With T = I and b = 0 each channel is fma(0, x2, fma(0, x1, fma(1, x0, 0))) = x0 for finite pixels: the result equals
    torch.clamp_(x, 0, 1) value for value, and a NaN pixel stays NaN where torch.clamp_ keeps it."""
    from unboundednerfpytorch_b200 import arf
    vals = np.array([-3e38, -1.5, -1e-30, 0.0, 1e-30, 0.25, 0.5, 1 - 2 ** -24, 1.0, 1 + 2 ** -23, 2.0, 3e38], np.float32)
    x = np.stack([np.roll(vals, i)[:3] for i in range(len(vals))] * 7).astype(np.float32)
    x[5] = np.nan
    x[17] = np.nan
    t = torch.from_numpy(x).to(DEV)
    y = arf.color_affine(t, np.eye(3), np.zeros(3))
    want = t.clone().clamp_(0.0, 1.0)
    assert torch.equal(torch.isnan(y), torch.isnan(want))
    ok = ~torch.isnan(want)
    assert torch.equal(y[ok], want[ok])


# ---------------------------------------------------------------------------------------------------------------------------
# ARF.match_colors_for_image_set
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', SETS)
def test_goldens_against_fp64_and_the_reference(name, tmp_path):
    g = load_golden(f'l2_arf/set_{name}.pt')
    style = load_golden(f'l2_arf/style_{g["style"]}.pt')
    st = _stylizer(g['style'], style['HW'], tmp_path)
    assert np.array_equal(st.np_style_img, style['np_style_img'])
    out, tf = st.match_colors_for_image_set(g['image_set'].copy(), str(tmp_path))
    got, got_tf = out.cpu().numpy(), tf.cpu().numpy()
    want, want_tf, T, b = arf_ref.match_colors_fp64(g['image_set'], style['np_style_img'])
    ours = arf_ref.transform_rounding_bound(g['image_set'], T, b)
    err = np.abs(got - want)
    assert (err <= ours).all(), f'{name}: vs fp64 {err.max():.3e}, worst ratio {(err / ours).max():.3f}'
    tf_tol = arf_ref.U32 * np.abs(want_tf) + 1e-9 * np.abs(want_tf).max()
    assert (np.abs(got_tf - want_tf) <= tf_tol).all(), f'{name}: color_tf vs fp64 {np.abs(got_tf - want_tf).max():.3e}'
    ref_px, ref_tf = arf_ref.reference_fp32_bound(g['image_set'], style['np_style_img'])
    err_ref = np.abs(got - g['out'])
    assert (err_ref <= ref_px + ours).all(), f'{name}: vs the reference {err_ref.max():.3e}'
    assert (np.abs(got_tf - g['color_tf']) <= ref_tf + tf_tol).all(), f'{name}: color_tf vs the reference'
    print(f'{name}: ours vs fp64 {err.max():.2e}, reference vs fp64 {np.abs(g["out"] - want).max():.2e}')


def test_types_shapes_devices_png_and_untouched_input(tmp_path):
    st = _stylizer('landscape', (48, 64), tmp_path)
    x = arf_ref.content_set('random', (3, 17, 29, 3), 5)
    out_np, tf_np = st.match_colors_for_image_set(x.copy(), str(tmp_path))
    for t, shape in ((out_np, x.shape), (tf_np, (4, 4))):
        assert isinstance(t, torch.Tensor) and t.dtype == torch.float32 and t.device == torch.device(DEV)
        assert tuple(t.shape) == shape
    assert torch.equal(tf_np[3], torch.tensor([0., 0., 0., 1.], device=DEV))
    png = cv2.imread(str(tmp_path / 'style_image.png'), cv2.IMREAD_UNCHANGED)[..., ::-1]
    assert np.array_equal(png, np.clip(st.np_style_img * 255.0, 0.0, 255.0).astype(np.uint8))
    xt = torch.from_numpy(x).to(DEV)
    before = xt.clone()
    out_t, tf_t = st.match_colors_for_image_set(xt, str(tmp_path))
    assert torch.equal(xt, before), 'the input tensor was modified'
    assert out_t.data_ptr() != xt.data_ptr()
    assert torch.equal(out_t, out_np) and torch.equal(tf_t, tf_np)
    flat, _ = st.match_colors_for_image_set(x.reshape(-1, 3).copy(), str(tmp_path))        # any shape ending in 3
    assert torch.equal(flat.view(x.shape), out_np)
    odd = xt.permute(0, 2, 1, 3)                                                           # a non-contiguous view
    out_odd, _ = st.match_colors_for_image_set(odd, str(tmp_path))
    assert tuple(out_odd.shape) == tuple(odd.shape)                 # its moments are summed in another order
    assert torch.allclose(out_odd, out_np.permute(0, 2, 1, 3), rtol=0, atol=1e-5)


@pytest.mark.parametrize('kind,shape', [('random', (4, 270, 480, 3)), ('random', (8, 432, 576, 3)),
                                        ('outside', (3, 300, 400, 3))])
def test_against_the_staged_reference_on_the_gpu(ref_arf, kind, shape, tmp_path):
    """The reference's ARF (fp32 cuBLAS covariance and transform) on the same GPU, at 1e-5 on pixels and color_tf, for
    well-conditioned sets up to ~2 M pixels (the reference's covariance error grows with the pixel count)."""
    x = arf_ref.content_set(kind, shape, sum(shape))
    mu, cov = arf_ref.moments_fp64(x)
    assert np.linalg.eigvalsh(cov).min() >= 1e-3
    root = tmp_path / 'styles'
    root.mkdir()
    write_png_bytes(str(root / '34.jpg'), load_golden('l2_arf/style_portrait.pt')['source'])
    cfg = Cfg(arf=Cfg(style_root=str(root), style_id=34))
    data_dict = {'HW': np.array([shape[1:3]])}
    from unboundednerfpytorch_b200.arf import ARF
    ours = ARF(cfg, data_dict, DEV)
    ref_imageio = ref_arf.imageio
    ref_arf.imageio = ImageioStub()
    try:
        ref = ref_arf.ARF(cfg, data_dict, DEV)
        assert np.array_equal(ours.np_style_img, ref.np_style_img)
        r_out, r_tf = ref.match_colors_for_image_set(x.copy(), str(tmp_path))
    finally:
        ref_arf.imageio = ref_imageio
    o_out, o_tf = ours.match_colors_for_image_set(x.copy(), str(tmp_path))
    want, want_tf, _, _ = arf_ref.match_colors_fp64(x, ours.np_style_img)
    o_out, r_out, o_tf, r_tf = (t.cpu().numpy() for t in (o_out, r_out, o_tf, r_tf))
    msg = (f'{kind} {shape}: ours-ref {np.abs(o_out - r_out).max():.2e} (tf {np.abs(o_tf - r_tf).max():.2e}); vs fp64: ours '
           f'{np.abs(o_out - want).max():.2e} (tf {np.abs(o_tf - want_tf).max():.2e}), '
           f'reference {np.abs(r_out - want).max():.2e} '
           f'(tf {np.abs(r_tf - want_tf).max():.2e})')
    print(msg)
    assert np.abs(o_out - r_out).max() <= REF_TOL and np.abs(o_tf - r_tf).max() <= REF_TOL, msg


def test_peak_device_memory_of_a_numpy_call(ref_arf, tmp_path):
    shape = (16, 270, 480, 3)
    x = arf_ref.content_set('random', shape, 11)
    st = _stylizer('portrait', shape[1:3], tmp_path)
    st.match_colors_for_image_set(x[:1].copy(), str(tmp_path))           # warm up
    torch.cuda.synchronize()

    def peak(fn):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        res = fn()
        torch.cuda.synchronize()
        p = torch.cuda.max_memory_allocated() - base
        del res
        return p
    ours = peak(lambda: st.match_colors_for_image_set(x, str(tmp_path)))
    root = tmp_path / 'styles_portrait'
    cfg = Cfg(arf=Cfg(style_root=str(root), style_id=34))
    ref_imageio = ref_arf.imageio
    ref_arf.imageio = ImageioStub()
    try:
        ref = ref_arf.ARF(cfg, {'HW': np.array([shape[1:3]])}, DEV)
        theirs = peak(lambda: ref.match_colors_for_image_set(x, str(tmp_path)))
    finally:
        ref_arf.imageio = ref_imageio
    print(f'peak device memory of a {x.nbytes / 2 ** 20:.1f} MiB set: ours {ours / 2 ** 20:.2f} MiB, '
          f'reference {theirs / 2 ** 20:.2f} MiB')
    assert ours <= x.nbytes + 2 ** 20, (ours, x.nbytes)


def test_runs_on_the_callers_stream(tmp_path):
    st = _stylizer('portrait', (48, 64), tmp_path)
    x = torch.from_numpy(arf_ref.content_set('random', (2, 300, 400, 3), 4)).to(DEV)
    want, want_tf = st.match_colors_for_image_set(x, str(tmp_path))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)              # a busy stream: the result is only right if the kernels queue behind it
        x2 = x * 1.0
        got, got_tf = st.match_colors_for_image_set(x2, str(tmp_path))
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(got, want) and torch.equal(got_tf, want_tf)


# ---------------------------------------------------------------------------------------------------------------------------
# the reference's own block render (run_render.py:146-177)
# ---------------------------------------------------------------------------------------------------------------------------
def _look_at(cam):
    back = cam / np.linalg.norm(cam)
    right = np.cross([0., 0., 1.], back)
    right /= np.linalg.norm(right)
    up = np.cross(back, right)
    return np.stack([right, up, back, cam], 1).astype(np.float32)


def _write_block_checkpoints(dirname, n_blocks):
    from unboundednerfpytorch_b200 import ckpt, models
    for i in range(n_blocks):
        torch.manual_seed(40 + i)
        m = models.FourierGridModel(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=32 ** 3, num_voxels_rgb=32 ** 3,
                                    num_voxels_base_density=32 ** 3, num_voxels_base_rgb=32 ** 3, num_voxels_viewdir=-1,
                                    alpha_init=1e-2, fast_color_thres=1e-4, rgbnet_dim=12, fourier_freq_num=2).to(DEV)
        with torch.no_grad():
            m.density.grid.normal_(0., 6.)
            m.k0.grid.normal_(0., 2.)
            last = [mod for mod in m.rgbnet.modules() if isinstance(mod, torch.nn.Linear)][-1]
            last.weight.mul_(30.)             # saturated, independent channels: a colourful, well-conditioned rendered set
            last.bias.normal_(0., 1.)
        ckpt.save_checkpoint(0, m, None, os.path.join(dirname, f'fine_last_{i}.tar'))


def test_reference_block_render_stylizes_through_install_arf(ref_render, monkeypatch, tmp_path):
    """run_render.run_render, unmodified, with block_num = 2 and render_train: two FourierGridModel block checkpoints, each
    block's rendered set recoloured by ARF, one stylized video.  Under install_models + install_arf the stylizer is arf.ARF;
    every match_colors_for_image_set result agrees with the same run on the reference's ARF at 1e-5."""
    from unboundednerfpytorch_b200 import arf, legacy
    rr = ref_render.run_render
    n_blocks, per_block, H, W, style_id = 2, 2, 24, 32, 5
    expdir = tmp_path / 'exp'
    expdir.mkdir()
    _write_block_checkpoints(str(expdir), n_blocks)
    styles = tmp_path / 'styles'
    styles.mkdir()
    write_png_bytes(str(styles / f'{style_id}.jpg'), load_golden('l2_arf/style_landscape.pt')['source'])
    n_views = n_blocks * per_block
    poses = np.stack([_look_at(np.array([2.5 * np.cos(a), 2.5 * np.sin(a), 0.3]))
                      for a in np.linspace(0, 2 * np.pi, n_views, endpoint=False)])
    K = np.array([[30., 0., W / 2], [0., 30., H / 2], [0., 0., 1.]], dtype=np.float32)
    cfg = Cfg(basedir=str(tmp_path), expname='exp', model='FourierGrid', arf=Cfg(style_root=str(styles), style_id=style_id),
              data=Cfg(ndc=False, white_bkgd=True, inverse_y=False, flip_x=False, flip_y=False, dataset_type='mega'),
              fine_model_and_render=Cfg(stepsize=0.5))

    def args():
        return types.SimpleNamespace(block_num=n_blocks, num_per_block=per_block, render_train=True, render_test=False,
                                     render_video=False, dump_images=False, eval_ssim=False, eval_lpips_alex=False,
                                     eval_lpips_vgg=False, ft_path='')

    images = torch.rand(n_views, H, W, 3, generator=torch.Generator().manual_seed(0))

    def data_dict():                    # run_render narrows i_train in place: a fresh dict per run
        return {'near': 0.1, 'far': 1e9, 'i_train': np.arange(n_views), 'i_test': np.arange(0),
                'poses': torch.tensor(poses, device=DEV), 'HW': np.array([[H, W]] * n_views), 'Ks': np.stack([K] * n_views),
                'images': images}

    def run(stylizer_cls):
        stub = ImageioStub()
        record = []
        real = stylizer_cls.match_colors_for_image_set

        def recording(self, image_set, train_save_dir):
            out, tf = real(self, image_set, train_save_dir)
            record.append((np.array(image_set, copy=True), out.cpu().numpy(), tf.cpu().numpy(), self.np_style_img))
            return out, tf
        monkeypatch.setattr(stylizer_cls, 'match_colors_for_image_set', recording)
        monkeypatch.setattr(rr, 'imageio', stub)
        monkeypatch.setattr(rr, 'ARF', stylizer_cls)
        monkeypatch.setenv('TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD', '1')     # utils.load_model: model_kwargs hold numpy arrays
        dd = data_dict()
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            torch.set_default_tensor_type('torch.cuda.FloatTensor')  # run_FourierGrid.py:87, which the driver's rays rely on
        try:
            with legacy.install_models(rr, ref_render.utils):
                if stylizer_cls is arf.ARF:
                    with legacy.install_arf(rr):
                        assert rr.ARF is arf.ARF
                        rr.run_render(args(), cfg, dd, DEV)
                else:
                    rr.run_render(args(), cfg, dd, DEV)
        finally:
            with warnings.catch_warnings():
                warnings.simplefilter('ignore')
                torch.set_default_tensor_type('torch.FloatTensor')
            monkeypatch.undo()
        return record, stub.videos

    spec = importlib.util.spec_from_file_location('_staged_reference_arf_render', os.path.join(PY, 'FourierGrid', 'arf.py'))
    ref_mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_mod)
    ref_mod.imageio = ImageioStub()
    ours, videos = run(arf.ARF)
    theirs, ref_videos = run(ref_mod.ARF)
    assert len(ours) == len(theirs) == n_blocks
    for i, ((xi, oi, ti, si), (xr, orr, tr, sr)) in enumerate(zip(ours, theirs)):
        assert xi.shape == (per_block, H, W, 3) and np.array_equal(xi, xr), f'block {i}: the rendered sets differ'
        assert np.array_equal(si, sr), f'block {i}: style images differ'
        want, want_tf, _, _ = arf_ref.match_colors_fp64(xi, si)
        eig = np.linalg.eigvalsh(arf_ref.moments_fp64(xi)[1])
        msg = (f'block {i} (content eigenvalues {eig}): ours-ref {np.abs(oi - orr).max():.2e} (tf {np.abs(ti - tr).max():.2e}); '
               f'vs fp64: ours {np.abs(oi - want).max():.2e}, reference {np.abs(orr - want).max():.2e}')
        print(msg)
        assert eig.min() >= 1e-3, msg                 # the regime where the reference's fp32 transform holds 1e-5
        assert np.abs(oi - orr).max() <= REF_TOL and np.abs(ti - tr).max() <= REF_TOL, msg
    for vids in (videos, ref_videos):
        assert len(vids) == 1
    (path, frames, kw), (rpath, rframes, _) = videos[0], ref_videos[0]
    assert os.path.basename(path) == f'video.rgb.style.{style_id}.mp4' and path == rpath
    assert os.path.dirname(path) == os.path.join(str(tmp_path), 'exp', 'render_train_fine_last')
    assert frames.shape == (n_views, H, W, 3) and frames.dtype == np.uint8 and rframes.shape == frames.shape
    stacked = np.concatenate([o for _, o, _, _ in ours]).astype(np.float64)
    assert np.array_equal(frames, (255 * np.clip(stacked, 0, 1)).astype(np.uint8))
    assert np.abs(frames.astype(int) - rframes.astype(int)).max() <= 1
    assert kw == dict(fps=15, quality=8)
