"""Time DirectContractedVoxGO.update_occupancy_cache_lt_nviews on its kernel against the reference's composition on the same GPU
and print one JSON line.

    python scripts/bench_lt_nviews.py [--steps 3] [--warmup 1] [--views 20]

Shape: a 160^3 density world (bg_len 0.2, inf contraction), 20 training views of 640 x 480 (0.3 MP) around the scene, the truck
stepsize 0.5 (S = 534 samples per ray).  The reference leg is the unmodified dcvgo.py staged under oracle/_ref/py (dcvgo.py:195-213:
per view a grid.DenseGrid ones grid, sample_ray of every 8192-ray chunk as a [8192, S, 3] tensor, grid_sample's autograd backward),
with CUDA as the default tensor type as run_FourierGrid.py sets it; the legacy modules stand in for the extension imports it never
calls on this path.  Both legs start from an all-true mask; the JSON reports CUDA-event milliseconds per call, the speedup and the
number of voxels whose mask differs (atomic summation order can flip voxels whose weight sum is within rounding of 1).  The card's
name and power limit are read in the same run."""
import argparse
import contextlib
import io
import json
import os
import sys
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_dvgo import _gpu, _time  # noqa: E402


def _reference_dcvgo():
    py = os.path.join(ROOT, 'oracle', '_ref', 'py')
    if not os.path.exists(os.path.join(py, 'FourierGrid', 'dcvgo.py')):
        return None
    from unboundednerfpytorch_b200 import functional as F_, legacy
    legacy.install()
    sys.modules['torch_scatter'] = types.SimpleNamespace(segment_coo=F_.segment_coo, scatter_add=None)
    sys.modules['torch_efficient_distloss'] = types.SimpleNamespace(flatten_eff_distloss=F_.flatten_eff_distloss)
    sys.path.insert(0, py)
    from FourierGrid import dcvgo
    return dcvgo


@contextlib.contextmanager
def _cuda_default():
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        torch.set_default_tensor_type('torch.cuda.FloatTensor')
    try:
        yield
    finally:
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            torch.set_default_tensor_type('torch.FloatTensor')


def _views(n, H, W, radius=3.0):
    """rays_o_tr / rays_d_tr [n*H*W, 3] of n cameras on a ring looking at the origin, imsz."""
    from unboundednerfpytorch_b200 import rays
    K = np.array([[0.8 * W, 0, W / 2], [0, 0.8 * W, H / 2], [0, 0, 1]], dtype=np.float32)
    os_, ds = [], []
    for i in range(n):
        a = 2 * np.pi * i / n
        cam = np.array([radius * np.cos(a), radius * np.sin(a), 0.3 * np.sin(3 * a)])
        back = cam / np.linalg.norm(cam)
        right = np.cross([0., 0., 1.], back)
        right /= np.linalg.norm(right)
        c2w = np.stack([right, np.cross(back, right), back, cam], 1).astype(np.float32)
        o, d, _ = rays.get_rays_of_a_view(H, W, K, torch.tensor(c2w, device='cuda'), False, False, False, False)
        os_.append(o.reshape(-1, 3))
        ds.append(d.reshape(-1, 3))
    return torch.cat(os_), torch.cat(ds), [H * W] * n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--views', type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark measures the GPU'
    from unboundednerfpytorch_b200 import models
    name, power = _gpu()
    kw = dict(num_voxels=160 ** 3, num_voxels_base=160 ** 3, alpha_init=1e-2, fast_color_thres=1e-4, rgbnet_dim=12, bg_len=0.2,
              contracted_norm='inf')
    lo, hi = [-1.] * 3, [1.] * 3
    ours = models.DirectContractedVoxGO(lo, hi, **kw).cuda()
    rays_o, rays_d, imsz = _views(args.views, 480, 640)
    rk = dict(near=0., far=1e9, bg=1, stepsize=0.5)
    S = int(2 / 2.4 * int(ours.world_size[0]) / 0.5 + 1) * 2
    out = dict(metric='update_occupancy_cache_lt_nviews, DirectContractedVoxGO', gpu=name, power_limit=power,
               shape=dict(world=[int(v) for v in ours.world_size], views=args.views, rays_per_view=imsz[0], samples_per_ray=S))

    def run_ours(i):
        ours.mask_cache.mask.fill_(True)
        ours.update_occupancy_cache_lt_nviews(rays_o, rays_d, imsz, rk, 3)
    out['ms'] = round(_time(run_ours, args.steps, args.warmup), 3)
    out['samples_per_s'] = round(args.views * imsz[0] * S / (out['ms'] * 1e-3), 1)

    dcvgo = _reference_dcvgo()
    if dcvgo is None:
        out['reference'] = 'unavailable: oracle/_ref/py is not staged'
    else:
        with _cuda_default():
            ref = dcvgo.DirectContractedVoxGO(torch.tensor(lo), torch.tensor(hi), **kw).cuda()

        def run_ref(i):
            ref.mask_cache.mask.fill_(True)
            with _cuda_default(), contextlib.redirect_stdout(io.StringIO()):
                ref.update_occupancy_cache_lt_nviews(rays_o, rays_d, imsz, rk, 3)
        ref_steps = max(1, min(args.steps, 2))
        out['reference_ms'] = round(_time(run_ref, ref_steps, min(args.warmup, 1)), 3)
        out['speedup'] = round(out['reference_ms'] / out['ms'], 2)
        out['mask_flips'] = int((ours.mask_cache.mask != ref.mask_cache.mask).sum())
        out['mask_kept'] = round(float(ours.mask_cache.mask.float().mean()), 4)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
