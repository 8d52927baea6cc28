"""oracle/arf_ref.py -- TEST INFRASTRUCTURE ONLY (CPU oracle of the ARF colour transfer; never imported by the product path).

ARF.match_colors_for_image_set (FourierGrid/arf.py:60-89) restated in fp64 numpy with two-pass moments, the error bounds the
tests hold the reference and this package to, and the seeded style images and content sets the ARF goldens
(oracle/make_golden_arf.py), tests and scripts/bench_arf.py are generated from."""
import numpy as np

U32 = 2.0 ** -24                      # unit roundoff of fp32
SIG_MIN, SIG_MAX = 1e-8, 1e8          # arf.py:77-78


def gamma(n, u=U32):
    """gamma_n = n u / (1 - n u): the relative error bound of n successive roundings (Higham, Accuracy and Stability, 3.1)."""
    return n * u / (1 - n * u)


# ---------------------------------------------------------------------------------------------------------------------------
# seeded inputs
# ---------------------------------------------------------------------------------------------------------------------------
def style_source(kind, seed):
    """A seeded 8-bit RGB style image: 'portrait' (120 x 75) or 'landscape' (90 x 131) -- two colour ramps, a wave and noise."""
    H, W = {'portrait': (120, 75), 'landscape': (90, 131)}[kind]
    rs = np.random.RandomState(seed)
    yy, xx = np.meshgrid(np.linspace(0., 1., H), np.linspace(0., 1., W), indexing='ij')
    s = rs.rand(3, 3)
    img = np.stack([0.15 + 0.5 * s[c, 0] * xx + 0.3 * s[c, 1] * yy + 0.1 * np.sin(7 * xx * (c + 1) + 5 * s[c, 2])
                    for c in range(3)], -1)
    img = img + 0.08 * rs.rand(H, W, 3)
    return np.clip(np.round(img * 255), 0, 255).astype(np.uint8)


def content_set(kind, shape, seed):
    """A seeded float32 content set of ``shape`` (..., 3):
    'random'    -- uniform pixels with a little shared grey (well conditioned: every covariance eigenvalue >= 0.025);
    'near_grey' -- a uniform grey level plus 1e-3 normal noise per channel (smallest covariance eigenvalue ~1e-6);
    'constant'  -- one colour with few mantissa bits (its sums are exact in fp32, so every eigenvalue is 0 and hits the clamp);
    'outside'   -- uniform in [-0.5, 1.5] (values outside [0, 1], which the transform's clamp meets)."""
    rs = np.random.RandomState(seed)
    n = int(np.prod(shape[:-1]))
    if kind == 'random':
        u = rs.rand(n, 3)
        x = 0.7 * u + 0.3 * u.mean(1, keepdims=True)
    elif kind == 'near_grey':
        x = rs.uniform(0.2, 0.8, (n, 1)) + 1e-3 * rs.randn(n, 3)
    elif kind == 'constant':
        x = np.broadcast_to(np.array([0.375, 0.5, 0.8125]), (n, 3))
    elif kind == 'outside':
        x = rs.uniform(-0.5, 1.5, (n, 3))
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(x.reshape(shape)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------------
# the transfer in fp64
# ---------------------------------------------------------------------------------------------------------------------------
def moments_fp64(pixels):
    """Two-pass fp64 mean and population covariance of the RGB pixels of an array [..., 3]."""
    x = np.asarray(pixels, np.float64).reshape(-1, 3)
    mu = x.mean(0)
    d = x - mu
    return mu, d.T @ d / len(x)


def transform_fp64(mu_c, cov_c, mu_s, cov_s):
    """arf.py:71-81 in fp64: T = cov_s^(1/2) cov_c^(-1/2) through the SVD with the singular values clamped, b = mu_s - T mu_c."""
    u_c, sig_c, _ = np.linalg.svd(cov_c)
    u_s, sig_s, _ = np.linalg.svd(cov_s)
    scl_s = np.diag(np.sqrt(np.clip(sig_s, SIG_MIN, SIG_MAX)))
    scl_c = np.diag(1 / np.sqrt(np.clip(sig_c, SIG_MIN, SIG_MAX)))
    T = u_s @ scl_s @ u_s.T @ u_c @ scl_c @ u_c.T
    return T, mu_s - T @ mu_c


def match_colors_fp64(image_set, style_img):
    """(recoloured set in fp64 [..., 3], color_tf [4, 4], T, b): arf.py:60-89 with every step in fp64."""
    T, b = transform_fp64(*moments_fp64(image_set), *moments_fp64(style_img))
    x = np.asarray(image_set, np.float64)
    out = np.clip(x @ T.T + b, 0., 1.)
    tf = np.eye(4)
    tf[:3, :3], tf[:3, 3] = T, b
    return out, tf, T, b


# ---------------------------------------------------------------------------------------------------------------------------
# error bounds
# ---------------------------------------------------------------------------------------------------------------------------
def apply_bound(image_set, T, b, u=U32):
    """|fp32 evaluation - exact| per element of clamp(T x + b) for the fp32 T, b given, evaluated as three dependent fmas (one
    rounding each, ubn_color_affine's order) or as a 3-term dot product plus an add (the reference's matmul): gamma_3 and
    gamma_4 of (|b| + |T| |x|).  The clamp is 1-Lipschitz, so the bound holds after it.  Uses gamma_4, which covers both."""
    x = np.abs(np.asarray(image_set, np.float64))
    return gamma(4, u) * (np.abs(b) + x @ np.abs(T).T)


def transform_rounding_bound(image_set, T, b):
    """|this package's fp32 result - the fp64 transfer| per element.  T and b are the fp64 transform rounded once to fp32
    (|dT| <= u |T|, |db| <= u |b|) and applied with three fmas (gamma_3): together <= (u + gamma_3) (|b| + |T| |x|) <
    gamma_4 (|b| + |T| |x|).  The fp64 moments and SVD add a relative error of order cond * 1e-16 (<= 1e-9 for every eigenvalue
    >= 1e-8, the clamp), covered by the 1e-9 term."""
    x = np.abs(np.asarray(image_set, np.float64))
    return (gamma(4) + 1e-9) * (np.abs(b) + x @ np.abs(T).T)


def reference_fp32_bound(image_set, style_img):
    """First-order bound of |reference (fp32, arf.py:60-89) - match_colors_fp64| -> (per element of the set, per element of
    color_tf), derived from the reference's fp32 arithmetic at this pixel count n:

    * mean(0) of n values: |d mu| <= gamma_n mean|x| (any summation order);
    * cov = (X - mu)^T (X - mu) / n: the centring adds u |d| + |d mu|, the n-term dot products gamma_n, the division u, so
      |dC_ij| <= (gamma_n + 2u) E|d_i||d_j| + |d mu_i| E|d_j| + |d mu_j| E|d_i|; the fp32 SVD is backward stable, which adds
      about 10 u ||C||;
    * f(C) = C^(-1/2) and g(C) = C^(1/2) (singular values clamped to [1e-8, 1e8]): by the Daleckii-Krein formula the Frechet
      derivative is bounded by the largest divided difference of f, |f'(lambda_min)| = lambda_min^(-3/2) / 2 and
      |g'(lambda_min)| = lambda_min^(-1/2) / 2, with lambda_min lowered by ||dC|| and raised to the clamp;
    * T = g(C_s) f(C_c) as a chain of six fp32 3 x 3 products: + 30 u ||g|| ||f||; b = mu_s - mu_c T^T: |db| <= |d mu_s| +
      ||dT|| ||mu_c|| + ||T|| |d mu_c| + 4 u (|mu_s| + ||T|| ||mu_c||);
    * the set, y = T (x - mu_c) + mu_s, as the reference evaluates it (x T^T + b in fp32): ||dT|| |x - mu_c| + ||T|| |d mu_c| +
      |d mu_s| + 4 u (|mu_s| + ||T|| ||mu_c||) (the rounding of b) + gamma_4 (|b| + |T| |x|); the clamp is 1-Lipschitz.  The
      first term is written about mu_c because the transform moves the mean exactly onto mu_s: a constant set comes out as mu_s
      whatever T is.

    Everything is first order in u; a factor 2 covers the second-order terms.  Where the set is nearly grey, ||dC|| reaches
    lambda_min and the bound exceeds 1: the reference's fp32 result there is not determined by its inputs to any digit, and only
    the clamp to [0, 1] constrains it."""
    def side(z):
        z = np.asarray(z, np.float64).reshape(-1, 3)
        n = len(z)
        mu, C = moments_fp64(z)
        d = np.abs(z - mu)
        Ed = d.mean(0)
        dmu = gamma(n) * np.abs(z).mean(0)
        dC = (gamma(n) + 2 * U32) * (d.T @ d / n) + np.outer(dmu, Ed) + np.outer(Ed, dmu)
        dC = np.linalg.norm(dC) + 10 * U32 * np.linalg.norm(C, 2)
        lam = max(np.linalg.eigvalsh(C).min() - dC, SIG_MIN)
        return mu, C, dmu, dC, lam

    mu_c, C_c, dmu_c, dC_c, lam_c = side(image_set)
    mu_s, C_s, dmu_s, dC_s, lam_s = side(style_img)
    T, b = transform_fp64(mu_c, C_c, mu_s, C_s)
    nf = 1 / np.sqrt(max(np.linalg.eigvalsh(C_c).min(), SIG_MIN))           # ||C_c^(-1/2)||
    ng = np.sqrt(max(np.linalg.eigvalsh(C_s).max(), SIG_MIN))               # ||C_s^(1/2)||
    dF = dC_c / (2 * lam_c ** 1.5)
    dG = dC_s / (2 * np.sqrt(lam_s))
    dT = ng * dF + dG * (nf + dF) + 30 * U32 * ng * nf
    nT = np.linalg.norm(T, 2)
    db = (np.linalg.norm(dmu_s) + dT * np.linalg.norm(mu_c) + nT * np.linalg.norm(dmu_c)
          + 4 * U32 * (np.linalg.norm(mu_s) + nT * np.linalg.norm(mu_c)))
    x = np.asarray(image_set, np.float64)
    px = 2 * (dT * np.linalg.norm(x - mu_c, axis=-1, keepdims=True) + nT * np.linalg.norm(dmu_c) + np.linalg.norm(dmu_s)
              + 4 * U32 * (np.linalg.norm(mu_s) + nT * np.linalg.norm(mu_c)) + apply_bound(x, T, b))
    tf = np.zeros((4, 4))
    tf[:3, :3], tf[:3, 3] = 2 * dT, 2 * db
    return px, tf
