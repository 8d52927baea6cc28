"""Host-side checks of DirectVoxGO and the box march's record bound (no GPU): constructor keywords, get_kwargs, state-dict names
and shapes, and march.box_s_max against an fp32 restatement of the reference's n_steps (render_utils_kernel.cu:12-79) on
adversarial rays."""
import numpy as np
import pytest
import torch

LO, HI = [-1.0, -1.3, -0.6], [1.1, 1.2, 0.8]


@pytest.mark.parametrize('rgbnet_dim', [0, 12])
def test_constructor_kwargs_and_state_dict(rgbnet_dim):
    from unboundednerfpytorch_b200 import models
    m = models.DirectVoxGO(xyz_min=LO, xyz_max=HI, num_voxels=40 ** 3, num_voxels_base=40 ** 3, alpha_init=1e-2,
                           fast_color_thres=1e-4, rgbnet_dim=rgbnet_dim, rgbnet_direct=True, rgbnet_width=128, viewbase_pe=4)
    kw = m.get_kwargs()
    assert set(kw) == {'xyz_min', 'xyz_max', 'num_voxels', 'num_voxels_base', 'alpha_init', 'voxel_size_ratio', 'mask_cache_path',
                       'mask_cache_thres', 'mask_cache_world_size', 'fast_color_thres', 'density_type', 'k0_type',
                       'density_config', 'k0_config', 'rgbnet_dim', 'rgbnet_direct', 'rgbnet_full_implicit', 'rgbnet_depth',
                       'rgbnet_width', 'viewbase_pe'}
    ws = [int(v) for v in m.world_size]
    sd = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    C = 3 if rgbnet_dim == 0 else rgbnet_dim
    want = {'xyz_min': (3,), 'xyz_max': (3,), 'act_shift': (1,), 'density.grid': (1, 1, *ws), 'density.xyz_min': (3,),
            'density.xyz_max': (3,), 'k0.grid': (1, C, *ws), 'k0.xyz_min': (3,), 'k0.xyz_max': (3,), 'mask_cache.mask': tuple(ws),
            'mask_cache.xyz2ijk_scale': (3,), 'mask_cache.xyz2ijk_shift': (3,)}
    if rgbnet_dim:
        dim0 = 3 + 3 * 4 * 2 + rgbnet_dim
        want.update({'viewfreq': (4,), 'rgbnet.0.weight': (128, dim0), 'rgbnet.0.bias': (128,), 'rgbnet.2.0.weight': (128, 128),
                     'rgbnet.2.0.bias': (128,), 'rgbnet.3.weight': (3, 128), 'rgbnet.3.bias': (3,)})
    assert sd == want
    # a fresh model from its own kwargs has the same state-dict layout (ckpt.load_model)
    m2 = models.DirectVoxGO(**kw)
    assert {k: tuple(v.shape) for k, v in m2.state_dict().items()} == want


def test_mask_cache_path_defers_to_a_state_dict(tmp_path):
    """A host-built model with mask_cache_path resolves the coarse mask only on a CUDA device; a state dict that carries the mask
    supersedes the file (so a fine checkpoint loads without the coarse file it names)."""
    from unboundednerfpytorch_b200 import models
    m = models.DirectVoxGO(xyz_min=LO, xyz_max=HI, num_voxels=20 ** 3, num_voxels_base=20 ** 3, alpha_init=1e-2,
                           mask_cache_path=str(tmp_path / 'missing_coarse.tar'))
    assert m._pending_mask is not None
    sd = m.state_dict()
    sd['mask_cache.mask'] = torch.rand(sd['mask_cache.mask'].shape) < 0.5
    m.load_state_dict(sd)
    assert m._pending_mask is None
    assert torch.equal(m.mask_cache.mask, sd['mask_cache.mask'])


def _n_steps_fp32(o, d, lo, hi, near, stepdist):
    """render_utils_kernel.cu:12-79 restated in numpy fp32 (the division / min / max / ceil of infer_t_minmax, infer_n_samples)."""
    f = np.float32
    o, d, lo, hi = (np.asarray(v, dtype=f) for v in (o, d, lo, hi))
    v = np.where(d == 0, f(1e-6), d)
    a = (hi - o) / v
    b = (lo - o) / v
    t_min = max(min(max(np.minimum(a, b)), f(1e9)), f(near))
    t_max = max(min(min(np.maximum(a, b)), f(1e9)), f(near))
    rnorm = np.sqrt(f(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), dtype=f)
    return int(max(np.ceil(f(f(f(t_max - t_min) * rnorm) / f(stepdist))), 1.0))


def test_s_max_bounds_adversarial_rays():
    from unboundednerfpytorch_b200 import march
    rng = np.random.default_rng(0)
    lo, hi = np.array(LO), np.array(HI)
    c = (lo + hi) / 2
    for stepdist in (0.5 * 2.1 / 160, 0.5 * 2.1 / 100, 0.013, 0.1):
        s_max = march.box_s_max(LO, HI, stepdist)
        rays = [(lo - (hi - lo), hi - lo), (hi + 1e-3, lo - hi), (lo, hi - lo), (hi, lo - hi)]           # longest diagonals
        rays += [(np.array([-5., 0.1, 0.2]), np.array([1., 0., 0.])), (np.array([0.1, -5., 0.2]), np.array([0., 3., 0.])),
                 (np.array([0.1, 0.2, -5.]), np.array([0., 0., 1e-3]))]                                       # axis-parallel
        rays += [(c, rng.normal(size=3)) for _ in range(50)]                                                  # origin inside
        rays += [(np.array([-9., 0.3, 0.1]), np.array([1., 0., 0.]))] * 2                                    # zero components
        rays += [(np.array([-3., float(HI[1]), float(LO[2])]), np.array([1., 0., 0.]))]                       # along an edge
        for _ in range(500):                                                                                  # random chords
            o = c + rng.normal(size=3) * 6
            rays.append((o, c + (rng.random(3) - 0.5) * (hi - lo) - o))
        n = [_n_steps_fp32(o, d, LO, HI, near, stepdist) for o, d in rays for near in (0.0, 0.2)]
        assert max(n) <= s_max, (stepdist, max(n), s_max)
        assert max(n) >= s_max - 8          # the bound is tight: the diagonals reach it
        # near beyond t_max: one sample at o + d * near
        assert _n_steps_fp32(lo - 1, np.array([1., 1., 1.]), LO, HI, 100.0, stepdist) == 1


@pytest.mark.parametrize('tag', ['coarse', 'fine'])
def test_constructor_against_reference_fixture(tag):
    """get_kwargs and state-dict names / shapes against what the reference's dvgo.py recorded (tests/golden/l2_dvgo/)."""
    from tests.util import load_golden
    from unboundednerfpytorch_b200 import models
    rec = load_golden(f'l2_dvgo/{tag}.pt')
    m = models.DirectVoxGO(**rec['kwargs'])
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == rec['state_shapes']
    ours, ref = m.get_kwargs(), rec['get_kwargs']
    assert set(ours) == set(ref)
    for k, v in ref.items():
        if isinstance(v, (np.ndarray, torch.Tensor)):
            assert np.array_equal(np.asarray(ours[k]), np.asarray(v)), k
        else:
            assert ours[k] == v, k
