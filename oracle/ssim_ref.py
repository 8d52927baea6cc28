"""oracle/ssim_ref.py -- TEST INFRASTRUCTURE ONLY (CPU oracle of the SSIM score; never imported by the product path).

The evaluation score of utils.rgb_ssim (FourierGrid/utils.py:79-125) restated from the formula in fp64 numpy, and the seeded
frame pairs the SSIM goldens (oracle/make_golden_ssim.py), tests and scripts/bench_ssim.py are generated from."""
import numpy as np


def ssim_frames(kind, H, W, seed):
    """A seeded float32 [H, W, 3] frame pair for the SSIM tests: 'noise' (uniform), 'ramp' (smooth ramps and a slow wave: the
    variances are differences of nearly equal moments), 'flat' (constant colours with 1e-3 perturbations), 'near' (a textured
    frame and the same frame plus 1e-4 noise).  Regenerated from np.random.RandomState(seed), so large frames need no fixture."""
    rs = np.random.RandomState(seed)
    yy, xx = np.meshgrid(np.linspace(0., 1., H), np.linspace(0., 1., W), indexing='ij')
    if kind == 'noise':
        a, b = rs.rand(H, W, 3), rs.rand(H, W, 3)
    elif kind == 'ramp':
        s = rs.rand(2, 3, 3)
        a = np.stack([0.1 + 0.4 * s[0, c, 0] * xx + 0.4 * s[0, c, 1] * yy + 0.05 * np.sin(6 * xx + 3 * s[0, c, 2]) for c in range(3)], -1)
        b = np.stack([0.1 + 0.4 * s[1, c, 0] * xx + 0.4 * s[1, c, 1] * yy + 0.05 * np.cos(5 * yy + 3 * s[1, c, 2]) for c in range(3)], -1)
    elif kind == 'flat':
        base = rs.rand(3)
        a = base + 1e-3 * rs.randn(H, W, 3)
        b = base + 1e-3 * rs.randn(H, W, 3)
    elif kind == 'near':
        a = 0.5 + 0.3 * np.sin(9 * xx + 4 * yy)[..., None] + 0.1 * rs.rand(H, W, 3)
        b = a + 1e-4 * rs.randn(H, W, 3)
    else:
        raise ValueError(kind)
    return a.astype(np.float32), b.astype(np.float32)


def rgb_ssim_fp64(img0, img1, max_val, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03):
    """SSIM with a separable Gaussian window ('valid' positions only), in fp64: returns (map [H-f+1, W-f+1, 3], mean).  The squared
    and cross images are rounded to fp32 before filtering, as the reference's float32 numpy products are; the window is the
    normalised Gaussian centred at (f - 1) / 2, symmetric, so filtering is a correlation along H, then along W."""
    from numpy.lib.stride_tricks import sliding_window_view
    x, y = np.asarray(img0, np.float32), np.asarray(img1, np.float32)
    g = np.exp(-0.5 * ((np.arange(filter_size) - (filter_size - 1) / 2) / filter_sigma) ** 2)
    g = g / g.sum()

    def blur(z):
        z = sliding_window_view(np.asarray(z, np.float64), filter_size, axis=0) @ g
        return sliding_window_view(z, filter_size, axis=1) @ g

    mx, my = blur(x), blur(y)
    vx = np.maximum(blur(x * x) - mx * mx, 0.)
    vy = np.maximum(blur(y * y) - my * my, 0.)
    cxy = blur(x * y) - mx * my
    cxy = np.sign(cxy) * np.minimum(np.sqrt(vx * vy), np.abs(cxy))
    C1, C2 = (k1 * max_val) ** 2, (k2 * max_val) ** 2
    m = (2 * mx * my + C1) * (2 * cxy + C2) / ((mx * mx + my * my + C1) * (vx + vy + C2))
    return m, m.mean()
