"""oracle/make_golden_bbox.py -- TEST INFRASTRUCTURE ONLY.  Generates tests/golden/l2_bbox/.

Runs the reference's UNMODIFIED FourierGrid/bbox_compute.py on CPU over the oracle stand-ins of oracle/stubs.py, plus a stand-in
for FourierGrid.load_everything (whose loaders need datasets and packages this checkout does not have): its load_existing_model is
reduced to utils.load_model(dvgo.DirectVoxGO, path), the path bbox_compute.py:140 has commented out.  Records:

* ``frustum.pt``: compute_bbox_by_cam_frustrm on small synthetic camera sets (odd H and W, per-view H, W and K) in all four branches
  -- bounded with and without NDC, unbounded-inward, nerfpp (by dataset type and by cfg.model 'FourierGrid') and Waymo -- with
  inverse_y / flip_x / flip_y set in turn; and FourierGrid_compute_bbox_by_cam_frustrm_mega, which the dispatch does not reach;
* ``coarse_geo.pt``: compute_bbox_by_coarse_geo on tests/golden/l2_dvgo/coarse_last.tar at a threshold that keeps part of the
  lattice and at one that keeps none (the whole-lattice fallback), on tests/golden/l2_tensorf/model_last.tar (a TensoRF density),
  and the world_size / voxel_size of the fine DirectVoxGO the reference builds on the first result, as run_train.py:379-385 does.

    python -m oracle.make_golden_bbox      # from the repo root, where the reference checkout exists
"""
import contextlib
import io
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_golden import OUT, SEED, _save  # noqa: E402  (installs the stand-ins and the reference path)
from oracle.make_golden_dvgo import KW_FINE, _allow_numpy  # noqa: E402
from FourierGrid import dvgo as ref_dvgo  # noqa: E402
from FourierGrid import utils as ref_utils  # noqa: E402

_le = types.ModuleType('FourierGrid.load_everything')
_le.__doc__ = 'oracle stand-in (oracle/make_golden_bbox.py)'
_le.load_existing_model = lambda args, cfg, cfg_train, path, device=None: (ref_utils.load_model(ref_dvgo.DirectVoxGO, path), None, 0)
sys.modules['FourierGrid.load_everything'] = _le
from FourierGrid import bbox_compute as ref_bbox  # noqa: E402

DIR = os.path.join(OUT, 'l2_bbox')


def _ns(**kw):
    return types.SimpleNamespace(**kw)


def _cfg(dataset_type='blender', model='DVGO', ndc=False, inverse_y=False, flip_x=False, flip_y=False, unbounded_inward=False,
         unbounded_inner_r=1.0, boundary_ratio=0.0):
    return _ns(model=model, data=_ns(dataset_type=dataset_type, ndc=ndc, inverse_y=inverse_y, flip_x=flip_x, flip_y=flip_y,
                                     unbounded_inward=unbounded_inward, unbounded_inner_r=unbounded_inner_r,
                                     boundary_ratio=boundary_ratio))


def _look_at(eye, target, up=(0., 0., 1.)):
    """c2w [3,4] (OpenGL convention: the camera looks along -z)."""
    eye, target, up = (np.asarray(v, dtype=np.float64) for v in (eye, target, up))
    f = target - eye
    f /= np.linalg.norm(f)
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    u = np.cross(r, f)
    return np.stack([r, u, -f, eye], 1)


def _cameras(gen, n, hw_choices, forward_facing=False):
    """n views on a shell around the origin (or, forward-facing, near the z = 0 plane looking down -z), per-view H, W and K."""
    HW, Ks, poses = [], [], []
    for i in range(n):
        H, W = hw_choices[i % len(hw_choices)]
        f = 0.9 * W + 7.0 * float(torch.rand(1, generator=gen))
        K = np.array([[f, 0, 0.5 * W + float(torch.rand(1, generator=gen)) - 0.5], [0, f * 1.01, 0.5 * H], [0, 0, 1]])
        if forward_facing:
            eye = (torch.rand(3, generator=gen).numpy() - 0.5) * np.array([0.4, 0.3, 0.1])
            c2w = _look_at(eye, eye + np.array([0.02, -0.01, -1.0]), up=(0., 1., 0.))
        else:
            d = torch.randn(3, generator=gen).numpy()
            eye = d / np.linalg.norm(d) * (3.0 + float(torch.rand(1, generator=gen)))
            c2w = _look_at(eye, (torch.rand(3, generator=gen).numpy() - 0.5) * 0.3)
        HW.append((H, W))
        Ks.append(K)
        poses.append(c2w)
    return np.array(HW), np.array(Ks), torch.tensor(np.array(poses), dtype=torch.float32)


CASES = {
    # tag: (cfg keywords, near, far, near_clip, camera-set keywords)
    'bounded': (dict(), 0.3, 4.2, None, dict(n=5, hw_choices=[(7, 9), (11, 5), (6, 13)])),
    'bounded_invy_flipx': (dict(inverse_y=True, flip_x=True), 0.5, 6.0, None, dict(n=4, hw_choices=[(9, 7), (5, 11)])),
    'bounded_ndc': (dict(dataset_type='llff', ndc=True, flip_y=True), 0.0, 1.0, None,
                    dict(n=4, hw_choices=[(9, 13), (7, 11)], forward_facing=True)),
    'unbounded': (dict(dataset_type='llff', unbounded_inward=True, unbounded_inner_r=0.8, flip_y=True), 0.0, 1e9, 0.15,
                  dict(n=5, hw_choices=[(11, 9), (7, 13)])),
    'nerfpp': (dict(dataset_type='nerfpp', inverse_y=True, unbounded_inner_r=1.0), 0.0, 1e9, 0.3,
               dict(n=4, hw_choices=[(13, 7)])),
    'fouriergrid': (dict(dataset_type='tankstemple', model='FourierGrid', flip_x=True, flip_y=True, unbounded_inner_r=1.2), 0.0,
                    1e9, 0.05, dict(n=3, hw_choices=[(5, 9), (9, 5)])),
    'waymo': (dict(dataset_type='waymo', unbounded_inner_r=0.9), 0.1, 1e9, 0.1, dict(n=6, hw_choices=[(7, 9)])),
}


def golden_frustum():
    gen = torch.Generator().manual_seed(SEED + 60)
    rec = {}
    args = _ns(block_num=1)
    for tag, (ckw, near, far, near_clip, camkw) in CASES.items():
        HW, Ks, poses = _cameras(gen, **camkw)
        i_train = np.arange(len(HW))[::-1][: max(1, len(HW) - 1)].copy()   # a proper, reordered subset of the views
        cfg = _cfg(**ckw)
        kw = {} if near_clip is None else dict(near_clip=near_clip)
        with contextlib.redirect_stdout(io.StringIO()):
            lo, hi = ref_bbox.compute_bbox_by_cam_frustrm(args, cfg, HW, Ks, poses, i_train, near, far, **kw)
        rec[tag] = dict(cfg=ckw, HW=HW, Ks=Ks, poses=poses, i_train=i_train, near=near, far=far, near_clip=near_clip,
                        xyz_min=lo.clone(), xyz_max=hi.clone())
    HW, Ks, poses = _cameras(gen, n=5, hw_choices=[(7, 9)])
    cfg = _cfg(dataset_type='mega', model='FourierGrid', unbounded_inner_r=1.1, boundary_ratio=0.25)
    i_train = np.array([0, 2, 3, 4])
    with contextlib.redirect_stdout(io.StringIO()):
        lo, hi = ref_bbox.FourierGrid_compute_bbox_by_cam_frustrm_mega(cfg, HW, Ks, poses, i_train, None)
    rec['mega'] = dict(cfg=dict(dataset_type='mega', model='FourierGrid', unbounded_inner_r=1.1, boundary_ratio=0.25), HW=HW, Ks=Ks,
                       poses=poses, i_train=i_train, near=None, far=None, near_clip=None, xyz_min=lo.clone(), xyz_max=hi.clone())
    _save(os.path.join('l2_bbox', 'frustum.pt'), rec)


THRES_SOME, THRES_NONE = 0.05, 1.0     # 59 of 3740 coarse lattice points exceed 0.05; alpha <= 1 everywhere, so 1.0 keeps none


def golden_coarse_geo():
    _allow_numpy()
    rec = {}
    torch.manual_seed(SEED + 61)
    for tag, rel, thres in (('dvgo_some', 'l2_dvgo/coarse_last.tar', THRES_SOME), ('dvgo_none', 'l2_dvgo/coarse_last.tar', THRES_NONE),
                            ('tensorf', 'l2_tensorf/model_last.tar', 0.1)):
        with contextlib.redirect_stdout(io.StringIO()):
            lo, hi = ref_bbox.compute_bbox_by_coarse_geo(ref_dvgo.DirectVoxGO, os.path.join(OUT, rel), thres, 'cpu', None,
                                                         _ns(fine_train=None))
        rec[tag] = dict(path=rel, thres=thres, xyz_min=lo.clone(), xyz_max=hi.clone())
    # the fine stage on the first bounds (run_train.py:379-385 -> create_new_model, dvgo branch)
    lo, hi = rec['dvgo_some']['xyz_min'], rec['dvgo_some']['xyz_max']
    fine_kw = {k: v for k, v in KW_FINE.items() if k not in ('xyz_min', 'xyz_max')}
    cwd = os.getcwd()
    os.chdir(os.path.join(OUT, 'l2_dvgo'))
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            fine = ref_dvgo.DirectVoxGO(xyz_min=lo, xyz_max=hi, mask_cache_path='coarse_last.tar', mask_cache_thres=1e-3, **fine_kw)
    finally:
        os.chdir(cwd)
    rec['fine'] = dict(kwargs=fine_kw, world_size=fine.world_size.clone(), voxel_size=float(fine.voxel_size),
                       voxel_size_ratio=float(fine.voxel_size_ratio), xyz_min=fine.xyz_min.clone(), xyz_max=fine.xyz_max.clone())
    _save(os.path.join('l2_bbox', 'coarse_geo.pt'), rec)


if __name__ == '__main__':
    torch.set_num_threads(4)
    golden_frustum()
    golden_coarse_geo()
