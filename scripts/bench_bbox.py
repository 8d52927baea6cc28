"""Time the scene-bounds passes of bbox.py against the reference's torch compositions on the same GPU and print one JSON line.

    python scripts/bench_bbox.py [--steps 10] [--warmup 2]

Shapes: compute_bbox_by_cam_frustrm's bounded branch at a 100-view 800 x 800 Blender-like camera set (64 M rays) and its
unbounded-inward branch at 200 views of 1297 x 840 (the 360-degree scenes); compute_bbox_by_coarse_geo's reduction on a 160^3
DenseGrid density.  Each leg runs this library's call (one reduction launch) and the reference's composition over this library's
per-view rays (bbox_compute.py: rays.get_rays_of_a_view, then the near / far points, amin / amax and torch.minimum / maximum; or
the meshgrid / linspace lattice, density, activate_density, mask, amin / amax), checks that both give the same bits, and reports
CUDA-event times per call.  The card's name and power limit are read in the same run."""
import argparse
import contextlib
import io
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_dvgo import _gpu, _time  # noqa: E402


def _cfg(**kw):
    ns = types.SimpleNamespace
    d = dict(dataset_type='blender', ndc=False, inverse_y=False, flip_x=False, flip_y=False, unbounded_inward=False,
             unbounded_inner_r=1.0)
    d.update(kw)
    return ns(model='DVGO', data=ns(**d))


def _cameras(n, H, W, radius, seed):
    g = torch.Generator().manual_seed(seed)
    poses = []
    for _ in range(n):
        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
        d = torch.randn(3, generator=g, dtype=torch.float64)
        poses.append(torch.cat([q, (d / d.norm() * radius)[:, None]], 1).numpy())
    f = 1.1 * W
    K = np.array([[f, 0, 0.5 * W], [0, f, 0.5 * H], [0, 0, 1]])
    return np.array([[H, W]] * n), np.array([K] * n), np.array(poses, dtype=np.float32)


def _torch_frustum(cfg, HW, Ks, poses, near, far, near_clip):
    from unboundednerfpytorch_b200 import rays
    xyz_min = torch.tensor([np.inf] * 3, device='cuda')
    xyz_max = -xyz_min
    for (H, W), K, c2w in zip(HW, Ks, poses):
        ro, rd, vd = rays.get_rays_of_a_view(H=H, W=W, K=K, c2w=c2w, ndc=False, inverse_y=False, flip_x=False, flip_y=False)
        if cfg.data.unbounded_inward:
            pts = ro + rd * near_clip
            xyz_min, xyz_max = torch.minimum(xyz_min, pts.amin((0, 1))), torch.maximum(xyz_max, pts.amax((0, 1)))
        else:
            pts = torch.stack([ro + vd * near, ro + vd * far])
            xyz_min, xyz_max = torch.minimum(xyz_min, pts.amin((0, 1, 2))), torch.maximum(xyz_max, pts.amax((0, 1, 2)))
    if cfg.data.unbounded_inward:
        center = (xyz_min + xyz_max) * 0.5
        radius = (center - xyz_min).max() * cfg.data.unbounded_inner_r
        xyz_min, xyz_max = center - radius, center + radius
    return xyz_min, xyz_max


def _torch_coarse_geo(model, thres):
    interp = torch.stack(torch.meshgrid(*[torch.linspace(0, 1, int(n), device='cuda') for n in model.world_size], indexing='ij'), -1)
    dense_xyz = model.xyz_min * (1 - interp) + model.xyz_max * interp
    alpha = model.activate_density(model.density(dense_xyz))
    active = dense_xyz[alpha > thres]
    return active.amin(0), active.amax(0)


def _leg(ours, ref, args):
    a, b = ours(), ref()
    same = all(torch.equal(x, y) for x, y in zip(a, b))
    t_ours = _time(lambda i: ours(), args.steps, args.warmup)
    t_ref = _time(lambda i: ref(), args.steps, args.warmup)
    return dict(ms=round(t_ours, 4), torch_ms=round(t_ref, 4), speedup=round(t_ref / t_ours, 2), bit_identical=same,
                xyz_min=a[0].tolist(), xyz_max=a[1].tolist())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()
    from unboundednerfpytorch_b200 import bbox, models
    name, power = _gpu()
    out = dict(gpu=name, power_limit=power)
    run_args = types.SimpleNamespace(block_num=2)

    HW, Ks, poses = _cameras(100, 800, 800, 4.0, 1)
    cfg = _cfg()
    out['frustum_bounded_100x800x800'] = _leg(
        lambda: bbox.compute_bbox_by_cam_frustrm(run_args, cfg, HW, Ks, poses, np.arange(100), 2.0, 6.0),
        lambda: _torch_frustum(cfg, HW, Ks, poses, 2.0, 6.0, None), args)

    HW, Ks, poses = _cameras(200, 840, 1297, 3.0, 2)
    cfg = _cfg(dataset_type='llff', unbounded_inward=True, unbounded_inner_r=1.0)
    out['frustum_unbounded_200x1297x840'] = _leg(
        lambda: bbox.compute_bbox_by_cam_frustrm(run_args, cfg, HW, Ks, poses, np.arange(200), 0.0, 1e9, near_clip=0.1),
        lambda: _torch_frustum(cfg, HW, Ks, poses, 0.0, 1e9, 0.1), args)

    g = torch.Generator().manual_seed(3)
    with contextlib.redirect_stdout(io.StringIO()):
        m = models.DirectVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=160 ** 3, num_voxels_base=160 ** 3, alpha_init=1e-6,
                               rgbnet_dim=0)
    X, Y, Z = [int(v) for v in m.world_size]
    with torch.no_grad():
        r2 = sum(a ** 2 for a in torch.meshgrid(*[torch.linspace(-1, 1, k) for k in (X, Y, Z)], indexing='ij'))
        m.density.grid.copy_((20.0 * (0.4 - r2) + 2.0 * torch.randn(X, Y, Z, generator=g))[None, None])
    m = m.cuda()
    thres = 1e-3                     # configs/default.py fine_model_and_render.bbox_thres
    out['coarse_geo_160'] = _leg(lambda: bbox.coarse_geo_bounds(m, thres), lambda: _torch_coarse_geo(m, thres), args)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
