"""render.py: the reference's render driver surface (run_render.py:15-114) and the two multi-GPU render modes at world = 1."""
import numpy as np
import pytest
import torch

from tests.util import assert_close

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


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


def test_render_viewpoints_matches_the_chunk_loop_of_the_reference_driver():
    from unboundednerfpytorch_b200 import rays as R, render as RD
    m = _model()
    H, W = 37, 53                                   # 1961 rays: not a multiple of the chunk size used below
    K = np.array([[60., 0., W / 2], [0., 60., H / 2], [0., 0., 1.]])
    poses = [np.array([[1., 0., 0., 0.1], [0., 1., 0., -0.2], [0., 0., 1., 0.3]], dtype=np.float32),
             np.array([[0., 0., 1., -0.3], [0., 1., 0., 0.0], [-1., 0., 0., 0.2]], dtype=np.float32)]
    rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, inverse_y=False, render_depth=True)
    gt = [np.random.RandomState(i).rand(H, W, 3).astype(np.float32) for i in range(2)]
    rgbs, depths, bgmaps = RD.render_viewpoints(None, m, poses, [(H, W)] * 2, [K] * 2, False, rk, gt_imgs=gt, verbose=False, chunk=512)
    assert rgbs.shape == (2, H, W, 3) and depths.shape == (2, H, W, 1) and bgmaps.shape == (2, H, W, 1)
    for i, c2w in enumerate(poses):
        ro, rd, vd = R.get_rays_of_a_view(H, W, K, torch.tensor(c2w), False, False, False, False)
        with torch.no_grad():
            chunks = [m(a, b, c, **rk) for a, b, c in zip(ro.view(-1, 3).split(8192), rd.view(-1, 3).split(8192), vd.view(-1, 3).split(8192))]
        want = torch.cat([c['rgb_marched'] for c in chunks]).reshape(H, W, 3)
        assert_close(torch.from_numpy(rgbs[i]), want, rtol=1e-5, atol=1e-6, what=f'frame {i}')       # chunking does not change a ray
    # flips / rotations / factor like the reference's post-processing
    # same chunk size as above: the per-ray bias table is one cuBLAS GEMM per chunk, whose kernel (and last bit) depends on the row count
    r2, _, _ = RD.render_viewpoints(None, m, poses[:1], [(H, W)], [K], False, rk, verbose=False, render_video_flipy=True, render_video_rot90=1,
                                    chunk=512)
    assert np.array_equal(r2[0], np.rot90(np.flip(rgbs[0], axis=0), k=1, axes=(0, 1)))
    r3, _, _ = RD.render_viewpoints(None, m, poses[:1], [(H, W)], [K], False, rk, verbose=False, render_factor=2)
    assert r3.shape == (1, H // 2, W // 2, 3)
    with pytest.raises(NotImplementedError):
        RD.render_viewpoints(None, m, poses[:1], [(H, W)], [K], False, rk, eval_ssim=True)


def test_block_idw_composite_world1_and_visibility_gate():
    from tests.util import seeded_rays
    from unboundednerfpytorch_b200 import render as RD
    m = _model(5)
    ro, rd, vd = seeded_rays(3000, 4, DEV)
    rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5)
    want = RD.render_rays(m, ro, rd, vd, rk)['rgb_marched']
    rgb, info = RD.render_blocks_idw(m, ro, rd, vd, rk, centroid=[0.5, 0., 0.], cam_origin=[0., 0., 0.])
    assert bool(info['visible']) and abs(float(info['weight']) - 0.5 ** -4) < 1e-3
    assert_close(rgb, want, rtol=1e-6, atol=1e-6, what='one visible block: the composite is that block')      # w * rgb / w
    with torch.no_grad():
        m.density.grid.fill_(-50.0)                  # an empty block: nothing accumulates -> gated out, weight 0
    rgb2, info2 = RD.render_blocks_idw(m, ro, rd, vd, rk, centroid=[0.5, 0., 0.], cam_origin=[0., 0., 0.])
    assert not bool(info2['visible']) and float(info2['den']) == 0.0

