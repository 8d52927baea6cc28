"""CPU: DirectMPIGO's host-side surface against what the reference's own dmpigo.py computed (fixtures of
oracle/make_golden_mpi.py): grid resolution, act_shift initialisation, get_kwargs, state-dict names / shapes, strict loading of
reference state dicts, the NDC sample count, s and the TV weights."""
import numpy as np
import pytest
import torch

from tests.util import load_golden


def _ctor_cases():
    return load_golden('l2_mpi/constructor.pt')


def _model(kwargs):
    from unboundednerfpytorch_b200 import models
    kw = dict(kwargs, xyz_min=np.array(kwargs['xyz_min'], dtype=np.float32), xyz_max=np.array(kwargs['xyz_max'], dtype=np.float32))
    return models.DirectMPIGO(**kw)


@pytest.mark.parametrize('i', range(4))
def test_constructor_matches_reference(i):
    c = _ctor_cases()[i]
    m = _model(c['kwargs'])
    assert torch.equal(m.world_size, c['world_size'])
    assert m.voxel_size_ratio == c['voxel_size_ratio']
    assert torch.equal(m.act_shift.grid.detach(), c['act_shift']), 'act_shift initial values differ'
    assert not m.act_shift.grid.requires_grad
    kw = {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in m.get_kwargs().items()}
    assert kw == c['get_kwargs']
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == c['state_shapes']
    # the weights each method passes to its grid, recorded on the grid's own call like the fixture records the reference's
    for name in ('density', 'k0'):
        calls = []
        getattr(m, name).total_variation_add_grad = lambda wx, wy, wz, dense, calls=calls: calls.append((float(wx), float(wy),
                                                                                                           float(wz), dense))
        getattr(m, f'{name}_total_variation_add_grad')(c['tv_weight'], True)
        assert calls == [(*c['tv'][name], True)], name
    assert {g: w[:3] for g, w in m.tv_terms(c['tv_weight'], c['tv_weight']).items()} == {
        m.density.grid: c['tv']['density'], m.k0.grid: c['tv']['k0']}


@pytest.mark.parametrize('tag', ['mpi_rgb9', 'mpi_rgb0'])
def test_reference_state_dict_loads_strictly(tag):
    rec = load_golden(f'l2_mpi/{tag}.pt')
    m = _model(rec['kwargs'])
    m.load_state_dict(rec['state'], strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, rec['state'][k]), k
    if rec['kwargs'].get('rgbnet_dim', 0) > 0:
        assert m.viewfreq.numel() == 0            # viewbase_pe defaults to 0: the view embedding is viewdirs itself


@pytest.mark.parametrize('tag', ['mpi_rgb9', 'mpi_rgb0'])
def test_ndc_sample_count_and_s(tag):
    rec = load_golden(f'l2_mpi/{tag}.pt')
    m = _model(rec['kwargs'])
    S = m._n_samples(rec['render_kwargs']['stepsize'])
    assert S == rec['ret']['n_max'] == int((rec['kwargs']['mpi_depth'] - 1) / 0.5) + 1
    # s = (step_id + 0.5) / N_samples: recover step_id from the recorded s and recompute it with the same torch ops
    step_id = torch.round(rec['ret']['s'] * S - 0.5).long()
    assert torch.equal((step_id + 0.5) / S, rec['ret']['s'])


def test_llff_default_shapes():
    """llff_default: mpi_depth 128, stepsize 0.5 -> 255 samples per ray; LLFF's rgbnet is 12 -> 64 -> 64 -> 3."""
    from unboundednerfpytorch_b200 import models
    m = models.DirectMPIGO(xyz_min=[-1.4, -1.1, -1.], xyz_max=[1.4, 1.1, 1.], num_voxels=48 ** 3, mpi_depth=128, rgbnet_dim=9,
                           rgbnet_width=64, fast_color_thres=1e-3)
    assert m._n_samples(0.5) == 255
    assert m.voxel_size_ratio == 2.0
    assert [tuple(p.shape) for p in m.rgbnet.parameters()] == [(64, 12), (64,), (64, 64), (64,), (3, 64), (3,)]
    assert m.k0.grid.stride(1) == 1                # channels-last k0, as the fused NDC march reads it
