"""Host-side checks of TensoRFGrid and the TensoRF DirectVoxGO (no GPU): a seeded construction gives the reference's parameter
names, shapes and values (tests/golden/l2_tensorf/, written by oracle/make_golden_tensorf.py), the factors are stored
channels-last, get_kwargs, the create_grid dispatch and its error for unknown types."""
import os

import pytest
import torch

from tests.util import ROOT, assert_equal

GOLD = os.path.join(ROOT, 'tests', 'golden', 'l2_tensorf')
GRID_TAGS = ['r3xy2_c1', 'r3xy2_c3', 'r3xy2_c12', 'r8_c1', 'r24_c12']


def _load(name):
    return torch.load(os.path.join(GOLD, name), map_location='cpu', weights_only=False)


@pytest.mark.parametrize('tag', GRID_TAGS)
def test_seeded_construction_matches_reference(tag):
    from unboundednerfpytorch_b200 import grid as G
    g = _load(f'grid_{tag}.pt')
    torch.manual_seed(g['seed'])
    ours = G.create_grid('TensoRFGrid', channels=g['channels'], world_size=torch.tensor(g['world_size']), xyz_min=g['xyz_min'],
                         xyz_max=g['xyz_max'], config=g['config'])
    assert isinstance(ours, G.TensoRFGrid)
    sd = ours.state_dict()
    assert list(sd) == list(g['state'])
    for k, v in g['state'].items():
        assert_equal(sd[k], v, k)
    R, A, B = None, None, None
    for name in G.TENSORF_FACTORS:
        t = getattr(ours, name)
        _, R, A, B = t.shape
        assert t.stride() == (A * B * R, 1, B * R, R), f'{name} is not stored channels-last'
    assert ('f_vec' in sd) == (g['channels'] > 1)
    assert f"n_comp={g['config']['n_comp']}" in repr(ours)


def test_model_kwargs_and_state_dict():
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import models
    m = _load('model.pt')
    ours = models.DirectVoxGO(**m['kwargs'])
    assert isinstance(ours.density, G.TensoRFGrid) and isinstance(ours.k0, G.TensoRFGrid)
    assert {k: tuple(v.shape) for k, v in ours.state_dict().items()} == m['state_shapes']
    kw = ours.get_kwargs()
    assert set(kw) == set(m['get_kwargs'])
    for k in ('density_type', 'k0_type', 'density_config', 'k0_config', 'num_voxels', 'rgbnet_dim'):
        assert kw[k] == m['kwargs'][k]
    # a fresh model from its own kwargs has the same state-dict layout (ckpt.load_model), and loads the state the reference wrote
    again = models.DirectVoxGO(**kw)
    again.load_state_dict(m['state'])
    for k, v in m['state'].items():
        assert_equal(again.state_dict()[k], v, k)


def test_reference_checkpoint_loads():
    """model_last.tar, written by the reference's classes after a scale_volume_grid, loads through ckpt.load_model."""
    from unboundednerfpytorch_b200 import ckpt, models
    path = os.path.join(GOLD, 'model_last.tar')
    ours = ckpt.load_model(models.DirectVoxGO, path)
    ref = torch.load(path, map_location='cpu', weights_only=False)['model_state_dict']
    for k, v in ref.items():
        assert_equal(ours.state_dict()[k], v, k)


def test_unknown_grid_type_raises():
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import models
    with pytest.raises(NotImplementedError):
        G.create_grid('CPGrid', channels=1, world_size=[4, 4, 4], xyz_min=[0.] * 3, xyz_max=[1.] * 3, config={})
    with pytest.raises(NotImplementedError):
        models.DirectVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=8 ** 3, num_voxels_base=8 ** 3, alpha_init=1e-2,
                           k0_type='CPGrid')


def test_other_models_keep_rejecting_tensorf():
    from unboundednerfpytorch_b200 import models
    with pytest.raises(NotImplementedError):
        models.DirectContractedVoxGO(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels=8 ** 3, num_voxels_base=8 ** 3,
                                     alpha_init=1e-2, density_type='TensoRFGrid', density_config=dict(n_comp=2))
