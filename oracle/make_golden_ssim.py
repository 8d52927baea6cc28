"""oracle/make_golden_ssim.py -- TEST INFRASTRUCTURE ONLY.  Generates tests/golden/l2_ssim/.

Runs the reference's UNMODIFIED utils.rgb_ssim (FourierGrid/utils.py:79-125, scipy convolve2d on the CPU) over the oracle
stand-ins of oracle/stubs.py on seeded frame pairs (oracle.ssim_ref.ssim_frames) and records:

* ``taps.pt``: the 1-D filter the reference passes to convolve2d, for filter_size 1 .. 32 at three sigmas, read off the call
  itself (a recording wrapper around scipy.signal.convolve2d);
* ``small.pt``: small frames with both images, the map and the mean -- every frame kind, a single output row and a single output
  column, filter_size 1 / 10 / 32, non-default filter_sigma / k1 / k2, max_val 255 on 0..255 images, and one NaN pixel;
* ``large.pt``: frames at render sizes, stored as kind, seed and shape (the test regenerates the pixels) with the mean only.

    python -m oracle.make_golden_ssim      # from the repo root, where the reference checkout exists
"""
import os
import sys

import numpy as np
import scipy.signal

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden import SEED, _save  # noqa: E402  (installs the stand-ins and the reference path)
from oracle.ssim_ref import ssim_frames  # noqa: E402
from FourierGrid import utils as ref_utils  # noqa: E402

SIGMAS = (1.5, 0.8, 3.0)


def golden_taps():
    seen = []
    real = scipy.signal.convolve2d

    def record(z, f, mode):
        seen.append(np.array(f, dtype=np.float64).ravel())
        return real(z, f, mode=mode)
    rec = {}
    scipy.signal.convolve2d = record
    try:
        for sigma in SIGMAS:
            for n in range(1, 33):
                seen.clear()
                z = np.zeros((n, n, 3), np.float32)
                ref_utils.rgb_ssim(z, z, max_val=1, filter_size=n, filter_sigma=sigma)
                rec[(n, sigma)] = seen[0]
    finally:
        scipy.signal.convolve2d = real
    _save(os.path.join('l2_ssim', 'taps.pt'), rec)


SMALL = {
    # name: (kind, H, W, seed offset, rgb_ssim keywords)
    'noise': ('noise', 24, 31, 0, {}),
    'ramp': ('ramp', 29, 40, 1, {}),
    'flat': ('flat', 20, 26, 2, {}),
    'near': ('near', 27, 33, 3, {}),
    'one_row': ('noise', 11, 37, 4, {}),
    'one_col': ('ramp', 35, 11, 5, {}),
    'f1': ('noise', 9, 13, 6, dict(filter_size=1)),
    'f10': ('ramp', 21, 25, 7, dict(filter_size=10)),
    'f32': ('near', 40, 45, 8, dict(filter_size=32)),
    'params': ('noise', 26, 30, 9, dict(filter_sigma=0.8, k1=0.05, k2=0.1)),
    'max255': ('noise', 22, 28, 10, dict(max_val=255)),
    'nan': ('near', 20, 24, 11, {}),
}

LARGE = {
    'noise_1008x756': ('noise', 756, 1008, 20, {}),
    'ramp_1237x822': ('ramp', 822, 1237, 21, {}),
}


def _case(kind, H, W, seed, kw):
    a, b = ssim_frames(kind, H, W, seed)
    kw = dict(kw)
    max_val = kw.pop('max_val', 1)
    if max_val == 255:
        a, b = np.round(a * 255).astype(np.float32), np.round(b * 255).astype(np.float32)
    return a, b, max_val, kw


def golden_small():
    rec = {}
    for name, (kind, H, W, off, kw) in SMALL.items():
        a, b, max_val, kw = _case(kind, H, W, SEED + off, kw)
        if name == 'nan':
            a[7, 13, 1] = np.nan
        m = ref_utils.rgb_ssim(a, b, max_val, return_map=True, **kw)
        rec[name] = dict(img0=a, img1=b, max_val=max_val, kwargs=kw, map=m, mean=np.mean(m))
    _save(os.path.join('l2_ssim', 'small.pt'), rec)


def golden_large():
    rec = {}
    for name, (kind, H, W, off, kw) in LARGE.items():
        a, b, max_val, kw = _case(kind, H, W, SEED + off, kw)
        rec[name] = dict(kind=kind, H=H, W=W, seed=SEED + off, max_val=max_val, kwargs=kw,
                         mean=ref_utils.rgb_ssim(a, b, max_val, **kw))
    _save(os.path.join('l2_ssim', 'large.pt'), rec)


if __name__ == '__main__':
    golden_taps()
    golden_small()
    golden_large()
