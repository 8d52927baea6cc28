"""GPU: grad_W2 of the width-128 rgbnet backward from the warpgroup-MMA kernel (k_shade_dw2_wgmma, the default dW2 engine)
element by element against fp64, and against the mma.sync kernel (k_shade_dw2_tc, ubn_set_dw2_engine(0)).

The sizes cover a single sample, chunks of 32 samples just below, at and above a boundary, one chunk per CTA of a full grid
(132 x 32) and one sample more (the first CTA takes a second, one-row chunk), and the sizes of the benchmark.  3xTF32 is held to
the bound of test_gpu_rgbnet_layouts.py, |got - want| <= TAU * B with B the same sums over absolute values; single-pass TF32 to
TAU_TC1 * B on inputs whose pre-activations stay far from zero (so the single-pass forward keeps every fp64 ReLU mask)."""
import math

import pytest
import torch

from tests.test_gpu_rgbnet_layouts import TAU, TAU_TC1, TINY, min_preact, ref64

DEV = 'cuda:0'
SIZES = (1, 31, 32, 33, 129, 132 * 32, 132 * 32 + 1, 1 << 20, 4_194_304)
RAY_LEN = 512


def _inputs(M, K, seed, single_pass):
    g = torch.Generator().manual_seed(seed)
    N = -(-M // RAY_LEN)
    u = lambda *s, a: ((torch.rand(*s, generator=g) * 2 - 1) * a)
    inp = dict(W1k=u(128, K, a=1 / math.sqrt(K + 27)), W2=u(128, 128, a=1 / math.sqrt(128)), b2=u(128, a=1 / math.sqrt(128)),
               W3=u(3, 128, a=1 / math.sqrt(128)), b3=torch.randn(3, generator=g) * 0.1, vb=torch.randn(N, 128, generator=g) * 0.5,
               feat=torch.randn(M, K, generator=g), g_rgb=torch.randn(M, 3, generator=g),
               ray_id=torch.arange(M) // RAY_LEN)
    if single_pass:                    # as _tc1_inputs of test_gpu_rgbnet_layouts.py: |z| >~ 0.5 everywhere
        sign = lambda *s: (torch.randint(0, 2, s, generator=g) * 2 - 1).float()
        inp['feat'] *= 0.3
        inp['vb'] = sign(N, 128) * (1.5 + torch.rand(N, 128, generator=g))
        inp['b2'] = sign(128) * 25.0
        inp['W3'] *= 0.05
        inp['g_rgb'] = torch.rand(M, 3, generator=g) + 0.25
    inp = {k: v.to(DEV) for k, v in inp.items()}
    idx = torch.arange(M, device=DEV)
    for _ in range(8):                 # redraw ReLU-ambiguous samples (two correct fp32 evaluations may disagree on the mask)
        amb = idx[min_preact(inp['feat'][idx], inp['vb'], inp['ray_id'][idx], inp['W1k'], inp['W2'], inp['b2']) <= 1e-5]
        if amb.numel() == 0:
            return inp
        inp['feat'][amb] = (torch.randn(amb.numel(), K, generator=g) * (0.3 if single_pass else 1.0)).to(DEV)
        idx = amb
    raise AssertionError('samples still ReLU-ambiguous after 8 redraws')


def _dw2_ref64(inp, chunk=1 << 18):
    """dW2 = sum over samples of dZ2^T H1 in fp64 and its bound B, for any feature count (the dW2 part of ref64)"""
    d = lambda x: x.double()
    W1k, W2, b2, W3, b3 = map(d, (inp[k] for k in ('W1k', 'W2', 'b2', 'W3', 'b3')))
    want = torch.zeros(128, 128, dtype=torch.float64, device=DEV)
    bound = torch.zeros_like(want)
    M = inp['feat'].shape[0]
    for lo in range(0, M, chunk):
        sl = slice(lo, min(M, lo + chunk))
        x, v, g = d(inp['feat'][sl]), d(inp['vb'][inp['ray_id'][sl]]), d(inp['g_rgb'][sl])
        z1 = x @ W1k.t() + v
        m1 = (z1 > 0).double()
        h1 = z1 * m1
        z2 = h1 @ W2.t() + b2
        m2 = (z2 > 0).double()
        y = torch.sigmoid((z2 * m2) @ W3.t() + b3)
        dZ2 = ((g * y * (1 - y)) @ W3) * m2
        Bh1 = (x.abs() @ W1k.abs().t() + v.abs()) * m1
        Bh2 = (Bh1 @ W2.abs().t() + b2.abs()) * m2
        By = y * (1 - y) * (Bh2 @ W3.abs().t() + b3.abs()) + y
        BdZ2 = ((g.abs() * (y * (1 - y) + (1 - 2 * y).abs() * By)) @ W3.abs()) * m2
        want += dZ2.t() @ h1
        bound += BdZ2.t() @ Bh1
    return want, bound


def _run_dw2(inp, mode, engine):
    from unboundednerfpytorch_b200 import ops, shade as shade_mod
    ops.set_dw2_engine(engine)
    try:
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(shade_mod, 'MODE', mode)
            mp.setattr(shade_mod, 'BWD_MODE', 'fused')
            mp.setattr(shade_mod, 'USE_MASKS', True)
            W2 = inp['W2'].clone().requires_grad_(True)
            args = [inp['feat'], inp['vb'], inp['ray_id'], inp['W1k'], W2, inp['b2'], inp['W3'], inp['b3']]
            shade_mod._ShadeFn.apply(*args, True).backward(inp['g_rgb'])
    finally:
        ops.set_dw2_engine(1)
    return W2.grad


def _ratio(got, want, bound, tau):
    return float(((got.double() - want).abs() / (bound + TINY / tau)).max())


@pytest.mark.gpu
@pytest.mark.parametrize('K', (12, 15))
@pytest.mark.parametrize('M', SIZES)
@pytest.mark.parametrize('mode', ('tc3', 'tc1'))
def test_dw2_wgmma_vs_fp64(mode, M, K):
    inp = _inputs(M, K, seed=M + K, single_pass=mode == 'tc1')
    if K == 12:
        want, bound, _ = ref64(*(inp[k] for k in ('feat', 'vb', 'ray_id', 'W1k', 'W2', 'b2', 'W3', 'b3', 'g_rgb')))
        want, bound = want['dW2'], bound['dW2']
    else:
        want, bound = _dw2_ref64(inp)
    tau = TAU if mode == 'tc3' else TAU_TC1
    wg, mma = _run_dw2(inp, mode, 1), _run_dw2(inp, mode, 0)
    r_wg, r_mma = _ratio(wg, want, bound, tau), _ratio(mma, want, bound, tau)
    assert r_wg <= tau, f'wgmma dW2: |got - want| / B = {r_wg:.2e} > {tau:.0e} (mma.sync engine: {r_mma:.2e})'
    assert r_mma <= tau, f'mma.sync dW2: |got - want| / B = {r_mma:.2e} > {tau:.0e}'
    # the two engines issue the same products: they differ by the tensor cores' accumulation order only
    r_pair = _ratio(wg, mma.double(), bound, tau)
    assert r_pair <= tau, f'wgmma vs mma.sync dW2: {r_pair:.2e} of B'
