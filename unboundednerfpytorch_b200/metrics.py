"""Image-quality metrics of the evaluation step (FourierGrid/utils.py:77-125).

``rgb_ssim`` is the reference's ``utils.rgb_ssim`` -- same signature, same arguments, same result types -- computed by
``ubn_rgb_ssim`` (csrc/metrics.cu) on the GPU instead of scipy's convolve2d on the CPU.  The kernel keeps the reference's
precision: the products img**2 and img0*img1 are fp32, the filtered moments and everything after them fp64.  LPIPS is not here:
it needs pretrained network weights."""
import ctypes

import numpy as np
import torch

from . import _cabi
from .ops import _Guard


def gaussian_taps(filter_size, filter_sigma):
    """The normalised 1-D Gaussian filter of utils.py:90-95 (float64), evaluated with the same numpy operations in the same
    order, so the taps are the reference's bit for bit.  Symmetric: odd sizes centre a tap on 0, even sizes straddle it."""
    half = filter_size // 2
    offset = (2 * half - filter_size + 1) / 2
    z2 = ((np.arange(filter_size) - half + offset) / filter_sigma) ** 2
    taps = np.exp(-0.5 * z2)
    taps /= np.sum(taps)
    return taps


def _check_dtype(img, on_host):
    if on_host:
        ok = isinstance(img, np.ndarray) and img.dtype == np.float32
    else:
        ok = isinstance(img, torch.Tensor) and img.dtype == torch.float32 and img.is_cuda
    if not ok:
        raise TypeError('rgb_ssim takes two float32 numpy arrays or two float32 CUDA tensors, got '
                        f'{type(img).__name__} of dtype {getattr(img, "dtype", None)} (no conversion: the reference squares '
                        'float64 input in float64)')


def rgb_ssim(img0, img1, max_val, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03, return_map=False):
    """SSIM of two [H, W, 3] images, as utils.rgb_ssim.  numpy input is uploaded to the current CUDA device and the result comes
    back as np.float64 (or a float64 [H - f + 1, W - f + 1, 3] map with ``return_map``); CUDA tensor input gives a CUDA float64
    tensor, 0-dim or the map, on the caller's stream.

    Raises AssertionError for anything but two 3-D, 3-channel images of one shape (the reference's asserts), TypeError for
    anything but float32, ValueError when H or W is smaller than filter_size (scipy's 'valid' mode) or filter_size is outside
    1 .. 32."""
    assert len(img0.shape) == 3
    assert img0.shape[-1] == 3
    assert tuple(img0.shape) == tuple(img1.shape)
    on_host = isinstance(img0, np.ndarray)
    _check_dtype(img0, on_host)
    _check_dtype(img1, on_host)
    if not 1 <= filter_size <= _cabi.SSIM_MAX_TAPS or int(filter_size) != filter_size:
        raise ValueError(f'filter_size must be an integer in 1 .. {_cabi.SSIM_MAX_TAPS}, got {filter_size}')
    filter_size = int(filter_size)
    H, W = int(img0.shape[0]), int(img0.shape[1])
    if H < filter_size or W < filter_size:
        raise ValueError(f'a {H}x{W} image is smaller than the {filter_size}-tap filter (no valid output)')
    taps = gaussian_taps(filter_size, filter_sigma)
    c1 = (k1 * max_val) ** 2
    c2 = (k2 * max_val) ** 2
    if on_host:
        dev = torch.device('cuda', torch.cuda.current_device())
        a = torch.from_numpy(np.ascontiguousarray(img0)).to(dev)
        b = torch.from_numpy(np.ascontiguousarray(img1)).to(dev)
    else:
        if img0.device != img1.device:
            raise ValueError(f'img0 is on {img0.device}, img1 on {img1.device}')
        a, b = img0.contiguous(), img1.contiguous()
    ssim_map = torch.empty((H - filter_size + 1, W - filter_size + 1, 3), dtype=torch.float64, device=a.device) if return_map \
        else None
    scratch = torch.empty(_cabi.SSIM_MAX_CTAS, dtype=torch.float64, device=a.device)
    mean = torch.empty((), dtype=torch.float64, device=a.device)
    host_taps = (ctypes.c_double * filter_size)(*taps.tolist())
    with _Guard(a) as lib:
        _cabi.check(lib.ubn_rgb_ssim(_cabi.ptr(a), _cabi.ptr(b), _cabi.c_i64(H), _cabi.c_i64(W), _cabi.c_int(filter_size), host_taps,
                                     ctypes.c_double(c1), ctypes.c_double(c2), _cabi.ptr(ssim_map), _cabi.ptr(scratch),
                                     _cabi.ptr(mean), _cabi.stream_of(a)))
    out = ssim_map if return_map else mean
    if on_host:
        return out.cpu().numpy() if return_map else np.float64(out.item())
    return out
