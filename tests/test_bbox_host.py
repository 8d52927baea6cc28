"""CPU: bbox.compute_bbox_by_cam_frustrm's dispatch (bbox_compute.py:117-128) and its host branches, Waymo and Mega-NeRF, which
read camera centres only, against the reference's results in tests/golden/l2_bbox/frustum.pt."""
import types

import pytest
import torch

from tests.util import load_golden


def _cfg(dataset_type='blender', model='DVGO', ndc=False, inverse_y=False, flip_x=False, flip_y=False, unbounded_inward=False,
         unbounded_inner_r=1.0, boundary_ratio=0.0):
    ns = types.SimpleNamespace
    return ns(model=model, data=ns(dataset_type=dataset_type, ndc=ndc, inverse_y=inverse_y, flip_x=flip_x, flip_y=flip_y,
                                   unbounded_inward=unbounded_inward, unbounded_inner_r=unbounded_inner_r,
                                   boundary_ratio=boundary_ratio))


def test_dispatch():
    from unboundednerfpytorch_b200.bbox import frustum_branch
    assert frustum_branch(_cfg('waymo', model='FourierGrid', unbounded_inward=True)) == 'waymo'
    assert frustum_branch(_cfg('nerfpp', unbounded_inward=True)) == 'nerfpp'
    assert frustum_branch(_cfg('mega', model='FourierGrid')) == 'nerfpp'
    assert frustum_branch(_cfg('blender', model='FourierGrid')) == 'nerfpp'
    assert frustum_branch(_cfg('llff', unbounded_inward=True)) == 'unbounded'
    assert frustum_branch(_cfg('llff', ndc=True)) == 'bounded'
    assert frustum_branch(_cfg('blender')) == 'bounded'


def _equal(a, b):
    a = a.detach().cpu()
    assert a.dtype == torch.float32 and a.shape == (3,)
    assert torch.equal(a, b), (a, b)


def test_waymo_golden(capsys):
    from unboundednerfpytorch_b200 import bbox
    g = load_golden('l2_bbox/frustum.pt')['waymo']
    for block_num in (1, 4):
        lo, hi = bbox.compute_bbox_by_cam_frustrm(types.SimpleNamespace(block_num=block_num), _cfg(**g['cfg']), g['HW'], g['Ks'],
                                                  g['poses'], g['i_train'], g['near'], g['far'], near_clip=g['near_clip'])
        _equal(lo, g['xyz_min'])
        _equal(hi, g['xyz_max'])
        out = capsys.readouterr().out
        assert ('compute_bbox_by_cam_frustrm: finish' in out) == (block_num <= 1)


def test_mega_golden():
    from unboundednerfpytorch_b200 import bbox
    g = load_golden('l2_bbox/frustum.pt')['mega']
    lo, hi = bbox.FourierGrid_compute_bbox_by_cam_frustrm_mega(_cfg(**g['cfg']), g['HW'], g['Ks'], g['poses'], g['i_train'], None)
    _equal(lo, g['xyz_min'])
    _equal(hi, g['xyz_max'])
    # poses as a NumPy array and i_train as a list select the same views
    lo2, _ = bbox.FourierGrid_compute_bbox_by_cam_frustrm_mega(_cfg(**g['cfg']), g['HW'], g['Ks'], g['poses'].numpy(),
                                                               list(g['i_train']), None)
    _equal(lo2, g['xyz_min'])


def test_inward_branches_need_near_clip():
    from unboundednerfpytorch_b200 import bbox
    g = load_golden('l2_bbox/frustum.pt')['unbounded']
    with pytest.raises(TypeError):
        bbox.compute_bbox_by_cam_frustrm(types.SimpleNamespace(block_num=2), _cfg(**g['cfg']), g['HW'], g['Ks'], g['poses'],
                                         g['i_train'], g['near'], g['far'])
