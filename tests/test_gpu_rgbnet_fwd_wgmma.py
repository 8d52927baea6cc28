"""GPU: the warpgroup-MMA rgbnet forward (k_shade_fwd_wgmma, ubn_set_fwd_engine(1), the default at width 128 and 12 features)
against fp64, at the sizes where its 64-sample tiles, its two alternating consumer warpgroups and its persistent grid change
hands: one sample, a tile just below, at and above 64 and 128 rows (the panel block), 4097, and about a million samples.  The
ray layouts put one sample on each ray, one ray across every tile, and ray boundaries on and one sample off the tile edges.

* rgb and the saved H1 / H2 (read back out of the panel layout) within TAU * B of fp64 at 3xTF32 (B: the same expression on
  absolute values, as in test_gpu_rgbnet_layouts.py), within the single-pass tolerance of test_gpu_models.py at tc1;
* every H1 mask bit equal to (saved H1 > 0), and nothing written past n_pts (sentinel-filled buffers);
* the no-save and row-major forms give the panel form's rgb bit for bit;
* the backward (launch 1 + the wgmma dW2) fed by these saves: every gradient within TAU * B of fp64 at 3xTF32; at tc1 no
  further from fp64 than with the mma.sync forward's saves (ubn_set_fwd_engine(0)), with a 50 % margin;
* the mma.sync forward (k_shade_fwd_tc, ubn_set_fwd_engine(0)) held to the same 3xTF32 checks, since the default no longer
  runs it."""
import math

import pytest
import torch

from tests.test_gpu_rgbnet_layouts import TAU, TAU_TC1, TINY, _from_lengths, _tc1_inputs, judge, make_inputs, ratios, \
    reference, run_engine

DEV = 'cuda:0'
TILE = 64
SIZES = (1, 63, 64, 65, 127, 128, 129, 4097, 1_000_003)
SENT = -7.25                           # never a saved activation (those are >= 0)
SENT_MASK = -0x5A5A5A5B                # 0xA5A5A5A5 as int32


def _layout(name, M):
    if name == 'one_per_ray':
        return torch.arange(M), M
    if name == 'one_ray':
        return torch.zeros(M, dtype=torch.int64), 1
    if name == 'tile_edges':           # rays of 64 and 128 samples, every boundary on a tile edge
        return _from_lengths([TILE * (1 + i % 2) for i in range(M // TILE + 1)], M)
    if name == 'off_edges':            # the same rays shifted by one sample, and a 37-sample ray in every third
        return _from_lengths([1] + [37 if i % 3 == 2 else TILE * (1 + i % 2) for i in range(M // TILE + 1)], M)
    raise KeyError(name)


LAYOUTS = ('one_per_ray', 'one_ray', 'tile_edges', 'off_edges')


def _forward(inp, mode, save=True, panel=True, engine=1):
    """one ubn_rgbnet_fwd_tc call into sentinel-filled outputs: rgb [M + 64, 3], H1 / H2 [rows + 128, 128], masks"""
    from unboundednerfpytorch_b200 import ops
    from unboundednerfpytorch_b200._cabi import c_i64, c_int, check, ptr, stream_of
    M = inp['feat'].shape[0]
    rows = -(-M // 128) * 128 + 128
    rgb = torch.full((M + TILE, 3), SENT, device=DEV)
    h1 = torch.full((rows, 128), SENT, device=DEV) if save else None
    h2 = torch.full((rows, 128), SENT, device=DEV) if save else None
    m1 = torch.full((rows * 4,), SENT_MASK, dtype=torch.int32, device=DEV) if save and panel else None
    ops.set_fwd_engine(engine)
    try:
        with ops._Guard(inp['feat']) as lib:
            check(lib.ubn_rgbnet_fwd_tc(*(ptr(inp[k]) for k in ('feat', 'vb', 'ray_id', 'W1k', 'W2', 'b2', 'W3', 'b3')), c_i64(M),
                                        ptr(rgb), ptr(h1), ptr(h2), ptr(m1),
                                        c_int((1 if mode == 'tc1' else 0) | (4 if panel and save else 0)), stream_of(inp['feat'])))
        torch.cuda.synchronize()
    finally:
        ops.set_fwd_engine(1)
    return rgb, h1, h2, m1


def _unpanel(p):
    """[rows / 128][32 quads][128 rows][4] -> [rows][128]"""
    return p.reshape(-1, 32, 128, 4).permute(0, 2, 1, 3).reshape(-1, 128)


def _hidden64(inp):
    """H1, H2 in fp64 and their bounds (as ref64: the same expressions on absolute values, ReLU masks kept)"""
    d = lambda x: x.double()
    x, v = d(inp['feat']), d(inp['vb'][inp['ray_id']])
    W1k, W2, b2 = d(inp['W1k']), d(inp['W2']), d(inp['b2'])
    z1 = x @ W1k.t() + v
    m1 = (z1 > 0).double()
    h1, Bh1 = z1 * m1, (x.abs() @ W1k.abs().t() + v.abs()) * m1
    z2 = h1 @ W2.t() + b2
    m2 = (z2 > 0).double()
    return h1, Bh1, z2 * m2, (Bh1 @ W2.abs().t() + b2.abs()) * m2


def _inputs(layout, M, mode):
    ray_id, N = _layout(layout, M)
    assert ray_id.numel() == M and int(ray_id.max()) < N
    return (_tc1_inputs if mode == 'tc1' else make_inputs)(ray_id, N, M + len(layout), DEV)


def _close(got, want, bound, mode, what):
    if mode == 'tc3':
        r = float(((got.double() - want).abs() / (bound + TINY / TAU)).max())
        assert r <= TAU, f'{what}: |got - want| / B = {r:.2e} > {TAU:.0e}'
    else:
        torch.testing.assert_close(got.double(), want, rtol=5e-3, atol=5e-3, msg=lambda m: f'{what}: {m}')


@pytest.mark.gpu
@pytest.mark.parametrize('M', SIZES)
@pytest.mark.parametrize('layout', LAYOUTS)
@pytest.mark.parametrize('mode', ('tc3', 'tc1'))
def test_fwd_wgmma_saves_vs_fp64(mode, layout, M):
    inp = _inputs(layout, M, mode)
    want, bound, _ = reference(inp)
    rgb, h1p, h2p, m1 = _forward(inp, mode)
    _close(rgb[:M], want['rgb'], bound['rgb'], mode, 'rgb')
    assert bool((rgb[M:] == SENT).all()), 'rgb written past n_pts'
    h1, h2 = _unpanel(h1p), _unpanel(h2p)
    w1, b1, w2, b2 = _hidden64(inp)
    _close(h1[:M], w1, b1, mode, 'H1')
    _close(h2[:M], w2, b2, mode, 'H2')
    assert bool((h1[M:] == SENT).all()) and bool((h2[M:] == SENT).all()), 'H1 / H2 rows written past n_pts'
    # mask words [rows / 128][4 chunks][128 rows], bit e of chunk c = unit 32 c + e
    words = m1.reshape(-1, 4, 128).permute(0, 2, 1).reshape(-1, 4).long() & 0xFFFFFFFF
    bits = (words[:, :, None] >> torch.arange(32, device=DEV)) & 1
    assert torch.equal(bits.reshape(-1, 128)[:M].bool(), h1[:M] > 0), 'mask bits differ from saved H1 > 0'
    assert bool((m1.reshape(-1, 4, 128).permute(0, 2, 1).reshape(-1, 4)[M:] == SENT_MASK).all()), 'mask words written past n_pts'
    # the other two forms of the kernel: same arithmetic, same bits
    rgb_ns = _forward(inp, mode, save=False)[0]
    rgb_rm, h1r, h2r, _ = _forward(inp, mode, panel=False)
    assert torch.equal(rgb_ns, rgb) and torch.equal(rgb_rm, rgb), 'no-save / row-major forward differs from the panel form'
    assert torch.equal(h1r[:M], h1[:M]) and torch.equal(h2r[:M], h2[:M]), 'row-major saves differ from the panel saves'
    assert bool((h1r[M:] == SENT).all()) and bool((h2r[M:] == SENT).all()), 'row-major rows written past n_pts'


@pytest.mark.gpu
@pytest.mark.parametrize('M', SIZES)
@pytest.mark.parametrize('layout', LAYOUTS)
@pytest.mark.parametrize('mode', ('tc3', 'tc1'))
def test_fwd_wgmma_gradients_vs_fp64(mode, layout, M):
    from unboundednerfpytorch_b200 import ops
    inp = _inputs(layout, M, mode)
    want, bound, _ = reference(inp)
    got, rgb_ng = run_engine(inp, mode, 'fused', True)
    assert torch.equal(rgb_ng, got['rgb']), 'no_grad forward differs from the grad-enabled one'
    ops.set_fwd_engine(0)
    try:
        ref_got, ref_ng = run_engine(inp, mode, 'fused', True)
    finally:
        ops.set_fwd_engine(1)
    if mode == 'tc3':
        judge(got, want, bound, f'{layout} M={M} wgmma forward')
        assert torch.equal(ref_ng, ref_got['rgb']), 'mma.sync: no_grad forward differs from the grad-enabled one'
        judge(ref_got, want, bound, f'{layout} M={M} mma.sync forward')
        return
    # single pass: relative to the bound, as the dW2 engines are judged; no worse than the mma.sync forward's saves
    r_wg = ratios(got, want, {k: v * TAU_TC1 / TAU for k, v in bound.items()})
    r_mma = ratios(ref_got, want, {k: v * TAU_TC1 / TAU for k, v in bound.items()})
    bad = {k: f'{r_wg[k]:.2e} vs {r_mma[k]:.2e}' for k in r_wg if not r_wg[k] <= max(TAU, 1.5 * r_mma[k])}
    assert not bad, f'tc1 gradients from the wgmma forward further from fp64 than from mma.sync: {bad}'
    assert math.isfinite(sum(r_wg.values()))
