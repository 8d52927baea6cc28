"""CPU: the host side of the ARF stylizer (arf.ARF) -- the fp64 restatement of oracle/arf_ref.py against the reference's goldens
(tests/golden/l2_arf/, oracle/make_golden_arf.py), the style image's load and resize bit for bit, the input checks, and
legacy.install_arf.

The goldens are the reference's fp32 CPU arithmetic; oracle.arf_ref.reference_fp32_bound derives, from that arithmetic at each
fixture's pixel count, how far its result may lie from the fp64 transfer (first order in u = 2^-24, worst-case summation).  The
well-conditioned sets are held to bounds of 1e-4 .. 2e-3 (observed: ~1e-7).  For the near-grey set (smallest content eigenvalue
~1e-6) the bound exceeds 1: the reference's covariance error there reaches the eigenvalue itself, and its output is pinned only
by the clamp (observed: 2.4e-4 on pixels and 5.6e-2 on color_tf)."""
import ast
import os
import subprocess
import sys
import types

import cv2
import numpy as np
import pytest
import torch

from oracle import arf_ref
from tests.util import ROOT, load_golden

SETS = ('random', 'random_landscape', 'near_grey', 'constant', 'one_pixel', 'outside')


class Cfg(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None


def _style(kind):
    return load_golden(f'l2_arf/style_{kind}.pt')


def write_png_bytes(path, rgb):
    ok, buf = cv2.imencode('.png', np.ascontiguousarray(rgb[..., ::-1]))
    assert ok
    buf.tofile(path)


def _host_stylizer(path, HW):
    """An ARF whose style image stays on the host: the constructor itself requires a CUDA device."""
    from unboundednerfpytorch_b200.arf import ARF
    st = ARF.__new__(ARF)
    st.w, st.h, st.device = HW[1], HW[0], torch.device('cpu')
    st.style_img = st.load_style_img(path)
    return st


@pytest.mark.parametrize('name', SETS)
def test_fp64_restatement_within_the_references_fp32_bound(name):
    g = load_golden(f'l2_arf/set_{name}.pt')
    style = _style(g['style'])['np_style_img']
    out, tf, _, _ = arf_ref.match_colors_fp64(g['image_set'], style)
    px_bound, tf_bound = arf_ref.reference_fp32_bound(g['image_set'], style)
    assert g['out'].shape == g['image_set'].shape and g['out'].dtype == np.float32
    assert g['color_tf'].shape == (4, 4)
    err = np.abs(g['out'] - out)
    assert (err <= px_bound).all(), f'{name}: max err {err.max():.3e}, worst ratio {(err / px_bound).max():.3f}'
    tf_err = np.abs(g['color_tf'] - tf)
    assert (tf_err <= tf_bound).all(), f'{name}: color_tf err {tf_err.max():.3e}'
    assert np.array_equal(g['color_tf'][3], [0, 0, 0, 1])
    if name in ('random', 'random_landscape', 'outside'):
        assert px_bound.max() < 5e-3 and tf_bound.max() < 5e-3, (px_bound.max(), tf_bound.max())


@pytest.mark.parametrize('kind', ['portrait', 'landscape'])
def test_load_style_img_is_the_references_bit_for_bit(kind, tmp_path):
    s = _style(kind)
    path = str(tmp_path / '34.jpg')
    write_png_bytes(path, s['source'])
    st = _host_stylizer(path, s['HW'])
    assert st.np_style_img.dtype == np.float32
    assert st.np_style_img.shape == s['np_style_img'].shape
    assert np.array_equal(st.np_style_img, s['np_style_img'])
    assert (st.np_style_img.shape[0] > st.np_style_img.shape[1]) == (kind == 'portrait')
    assert torch.equal(st.style_img, torch.from_numpy(s['np_style_img']))


def test_style_image_checks(tmp_path):
    from unboundednerfpytorch_b200.arf import ARF
    with pytest.raises(FileNotFoundError):
        ARF.read_style_image(str(tmp_path / 'missing.jpg'))
    bad = {'grey.png': np.zeros((8, 9), np.uint8), 'rgba.png': np.zeros((8, 9, 4), np.uint8),
           'deep.png': np.zeros((8, 9, 3), np.uint16)}
    for name, img in bad.items():
        cv2.imwrite(str(tmp_path / name), img)
        with pytest.raises(ValueError):
            ARF.read_style_image(str(tmp_path / name))
    (tmp_path / 'junk.jpg').write_bytes(b'not an image')
    with pytest.raises(ValueError):
        ARF.read_style_image(str(tmp_path / 'junk.jpg'))


def test_constructor_checks(tmp_path):
    from unboundednerfpytorch_b200.arf import ARF
    write_png_bytes(str(tmp_path / '5.jpg'), arf_ref.style_source('portrait', 1))
    data_dict = {'HW': np.array([[48, 64]])}
    with pytest.raises(AssertionError):
        ARF(Cfg(), data_dict, 'cuda')
    with pytest.raises(ValueError):                           # no CPU path
        ARF(Cfg(arf=Cfg(style_root=str(tmp_path), style_id=5)), data_dict, 'cpu')


@pytest.mark.parametrize('image_set', [np.zeros((2, 3, 3), np.float64), np.zeros((2, 3, 3), np.float16),
                                       np.zeros((2, 3, 3), np.uint8), torch.zeros(2, 3, 3), torch.zeros(2, 3, 3).double(),
                                       [[0.0, 0.0, 0.0]]])
def test_set_types_other_than_float32_raise_type_error(image_set, tmp_path):
    s = _style('portrait')
    path = str(tmp_path / '34.jpg')
    write_png_bytes(path, s['source'])
    st = _host_stylizer(path, s['HW'])
    with pytest.raises(TypeError):
        st.match_colors_for_image_set(image_set, str(tmp_path))


@pytest.mark.parametrize('image_set', [np.zeros((0, 3), np.float32), np.zeros((4, 0, 3), np.float32),
                                       np.zeros((4, 4, 4), np.float32), np.zeros((), np.float32)])
def test_empty_or_non_rgb_sets_raise_value_error(image_set, tmp_path):
    s = _style('portrait')
    path = str(tmp_path / '34.jpg')
    write_png_bytes(path, s['source'])
    st = _host_stylizer(path, s['HW'])
    with pytest.raises(ValueError):
        st.match_colors_for_image_set(image_set, str(tmp_path))


def test_transform_is_independent_of_the_svd_basis():
    """color_transform of the product module against the oracle's, and with the covariances' SVD bases rotated within a
    repeated eigenvalue (the isotropic case) or with flipped signs: T and b do not move."""
    from unboundednerfpytorch_b200 import arf
    rs = np.random.RandomState(3)
    for _ in range(5):
        A, B = rs.randn(3, 3), rs.randn(3, 3)
        cov_c, cov_s = A @ A.T / 10, B @ B.T / 10
        mu_c, mu_s = rs.rand(3), rs.rand(3)
        T, b = arf.color_transform(mu_c, cov_c, mu_s, cov_s)
        T_ref, b_ref = arf_ref.transform_fp64(mu_c, cov_c, mu_s, cov_s)
        assert np.allclose(T, T_ref, rtol=1e-12, atol=1e-12) and np.allclose(b, b_ref, rtol=1e-12, atol=1e-12)
    T, _ = arf.color_transform(np.zeros(3), 0.04 * np.eye(3), np.zeros(3), 0.09 * np.eye(3))
    assert np.allclose(T, 1.5 * np.eye(3), rtol=1e-14)
    T, _ = arf.color_transform(np.zeros(3), np.zeros((3, 3)), np.zeros(3), 0.09 * np.eye(3))     # every sigma at the clamp
    assert np.allclose(T, 0.3e4 * np.eye(3), rtol=1e-14)


def test_install_arf_patches_and_restores():
    from unboundednerfpytorch_b200 import arf, legacy

    class Original:
        pass
    run_render = types.ModuleType('run_render')
    run_render.ARF = Original
    other = types.ModuleType('other')
    with legacy.install_arf(run_render, other) as patch:
        assert run_render.ARF is arf.ARF
        assert not hasattr(other, 'ARF')
        assert len(patch.saved) == 1
    assert run_render.ARF is Original
    patch = legacy.install_arf(run_render)
    assert run_render.ARF is arf.ARF
    patch.restore()
    assert run_render.ARF is Original
    assert 'ARF' not in legacy.model_names()


def test_product_module_never_imports_oracle():
    src = open(os.path.join(ROOT, 'unboundednerfpytorch_b200', 'arf.py')).read()
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.Import):
            assert not any(a.name.split('.')[0] == 'oracle' for a in node.names)
        elif isinstance(node, ast.ImportFrom):
            assert node.level > 0 or (node.module or '').split('.')[0] != 'oracle'
    code = 'import sys; import unboundednerfpytorch_b200.arf; print(any(m.split(".")[0] == "oracle" for m in sys.modules))'
    out = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, check=True).stdout
    assert out.strip() == 'False'
