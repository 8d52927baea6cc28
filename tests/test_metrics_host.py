"""CPU: the host side of metrics.rgb_ssim -- its filter taps against the reference's, its input checks, the fp64 restatement
of oracle/ssim_ref.py against the reference's maps and means (tests/golden/l2_ssim/), and legacy.install_metrics."""
import types

import numpy as np
import pytest

from tests.util import load_golden


def test_taps_are_the_references_bit_for_bit():
    from unboundednerfpytorch_b200 import metrics
    taps = load_golden('l2_ssim/taps.pt')
    assert sorted({n for n, _ in taps}) == list(range(1, 33))                # odd and even sizes
    for (n, sigma), want in taps.items():
        got = metrics.gaussian_taps(n, sigma)
        assert got.dtype == np.float64 and got.shape == (n,)
        assert np.array_equal(got, want), (n, sigma)
        assert np.array_equal(got, got[::-1]), (n, sigma)                   # symmetric: convolution = correlation


def _img(H=16, W=16, C=3, dtype=np.float32):
    return np.zeros((H, W, C), dtype)


@pytest.mark.parametrize('a,b', [(np.zeros((16, 16), np.float32),) * 2,                  # 2-D
                                 (_img(C=4), _img(C=4)),                                    # 4 channels
                                 (_img(), _img(W=17))])                                     # shapes differ
def test_shape_checks_raise_assertion_error(a, b):
    from unboundednerfpytorch_b200 import metrics
    with pytest.raises(AssertionError):
        metrics.rgb_ssim(a, b, 1.0)


@pytest.mark.parametrize('dtype', [np.float64, np.float16, np.uint8])
def test_dtypes_other_than_float32_raise_type_error(dtype):
    from unboundednerfpytorch_b200 import metrics
    with pytest.raises(TypeError):
        metrics.rgb_ssim(_img(), _img(dtype=dtype), 1.0)
    with pytest.raises(TypeError):
        metrics.rgb_ssim(_img(dtype=dtype), _img(), 1.0)


def test_cpu_tensors_raise_type_error():
    import torch
    from unboundednerfpytorch_b200 import metrics
    with pytest.raises(TypeError):
        metrics.rgb_ssim(torch.zeros(16, 16, 3), torch.zeros(16, 16, 3), 1.0)


@pytest.mark.parametrize('H,W,kw', [(10, 16, {}), (16, 10, {}), (12, 40, dict(filter_size=13)), (40, 40, dict(filter_size=33)),
                                    (16, 16, dict(filter_size=0))])
def test_sizes_raise_value_error(H, W, kw):
    from unboundednerfpytorch_b200 import metrics
    with pytest.raises(ValueError):
        metrics.rgb_ssim(_img(H, W), _img(H, W), 1.0, **kw)


def test_fp64_restatement_matches_the_reference():
    """oracle.ssim_ref.rgb_ssim_fp64 (its own taps, its own summation order) against the reference's scipy maps: the same bounds
    the GPU test holds the kernel to."""
    from oracle import ssim_ref
    for name, g in load_golden('l2_ssim/small.pt').items():
        m, mean = ssim_ref.rgb_ssim_fp64(g['img0'], g['img1'], g['max_val'], **g['kwargs'])
        assert m.shape == g['map'].shape, name
        nan = np.isnan(g['map'])
        assert np.array_equal(np.isnan(m), nan), name
        assert np.abs(m[~nan] - g['map'][~nan]).max() <= 1e-10, name
        if name == 'nan':
            assert np.isnan(mean) and np.isnan(g['mean'])
        else:
            assert abs(mean - g['mean']) <= 1e-12, name
    for name, g in load_golden('l2_ssim/large.pt').items():
        a, b = ssim_ref.ssim_frames(g['kind'], g['H'], g['W'], g['seed'])
        _, mean = ssim_ref.rgb_ssim_fp64(a, b, g['max_val'], **g['kwargs'])
        assert abs(mean - g['mean']) <= 1e-12, name


def test_install_metrics_patches_and_restores():
    from unboundednerfpytorch_b200 import legacy, metrics

    def original(*a, **k):
        return 'scipy'
    utils = types.ModuleType('utils')
    utils.rgb_ssim = original
    other = types.ModuleType('other')                     # a module without rgb_ssim is left alone
    with legacy.install_metrics(utils, other) as patch:
        assert utils.rgb_ssim is metrics.rgb_ssim
        assert not hasattr(other, 'rgb_ssim')
        assert len(patch.saved) == 1
    assert utils.rgb_ssim is original
    patch = legacy.install_metrics(utils)
    assert utils.rgb_ssim is metrics.rgb_ssim
    patch.restore()
    assert utils.rgb_ssim is original
    assert 'rgb_ssim' not in legacy.model_names()          # install_models does not touch the metric


def test_ssim_kernels_have_no_spills(tmp_path):
    """csrc/metrics.cu compiles for sm_90a with no stack frame and no spills (ptxas -v)."""
    import os
    import re
    import subprocess
    from tests.util import ROOT
    from unboundednerfpytorch_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip('needs nvcc')
    flags = [f for f in build.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC', '-fvisibility=hidden', '--cudart', 'static')]
    res = subprocess.run([nvcc, '-cubin', os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc', 'metrics.cu'),
                          '-o', str(tmp_path / 'm.cubin'), '-Xptxas', '-v'] + flags, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    props = re.findall(r'Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                       r'spill loads', log)
    assert sorted(n for n, *_ in props if 'ssim' in n) == sorted(n for n, *_ in props) and len(props) == 2, log
    for name, *sizes in props:
        assert sizes == ['0', '0', '0'], (name, sizes)
