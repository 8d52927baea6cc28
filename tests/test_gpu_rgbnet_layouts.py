"""The rgbnet kernels (csrc/shade_tc.cu, csrc/shade.cu) against a plain fp64 evaluation, at the ray layouts and sizes where the
backward's bookkeeping changes.

k_shade_bwd_tc walks contiguous ranges of 16-sample units per warp, carries the open ray's view-bias sum across units, turns up
to 4 ray segments per unit into indicator rows of an MMA operand (more than 4 fall back to per-sample adds) and reads bit-packed
ReLU masks.  A sample landing on the wrong ray, a ray emitted twice or never, or a swapped mask bit moves grad_view_bias by one
sample's share -- invisible in W1 / b1 after the sum over rays, so grad_view_bias is read here directly from _ShadeFn.apply.

Every output is judged element by element as |got - want| <= TAU * B, where B is the same expression evaluated in fp64 on the
absolute values of its operands (ReLU masks kept): a short ray is judged on its own magnitude, not hidden by a large neighbour.
test_checker_rejects_misplaced_samples (CPU) shows that TAU is tight enough to reject one sample moved to the neighbouring ray or
one sample's dZ1 dropped."""
import math

import pytest
import torch

DEV = 'cuda:0'
TAU = 1e-5                # elementwise |got - want| <= TAU * B (worst seen on an H100 80GB HBM3: 1.1e-6, g_vb)
TINY = 1e-30
TAU_TC1 = 4e-3            # single-pass TF32: per-ray ||got - want|| <= TAU_TC1 * sqrt(sum over the ray's samples of ||B(dZ1)||^2)
                          # (worst seen on an H100: 1.0e-3; one moved sample: >= 1.9e-2)
UNIT = 16
NUM_SMS = 132             # kNumSMs of the library (H100 SXM)
OUTS = ('rgb', 'g_feat', 'g_vb', 'dW1k', 'dW2', 'db2', 'dW3', 'db3')
WORST = {}                # check name -> worst |got - want| / B seen in this session


# ---- fp64 reference ----------------------------------------------------------------------------------------------------
def ref64(feat, vb, ray_id, W1k, W2, b2, W3, b3, g_rgb, chunk=1 << 18):
    """rgb and every gradient of rgb = sigmoid(W3 relu(W2 relu(W1k x + vb[ray]) + b2) + b3) in fp64 (the definitions above
    k_shade_bwd_tc), with g_vb = index_add of dZ1 over ray_id; and for each output the bound B: the same expression on the
    absolute values of every operand, the ReLU masks kept.  B also carries the forward's error into the backward (rgb into
    dz3, H1 / H2 into dW2 / dW3).  Chunked over samples to bound memory."""
    d = lambda x: x.double()
    W1k, W2, b2, W3, b3 = map(d, (W1k, W2, b2, W3, b3))
    aW1, aW2, ab2, aW3, ab3 = (x.abs() for x in (W1k, W2, b2, W3, b3))
    M, N, dev = feat.shape[0], vb.shape[0], feat.device
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=dev)
    want = dict(rgb=z(M, 3), g_feat=z(M, 12), g_vb=z(N, 128), dW1k=z(128, 12), dW2=z(128, 128), db2=z(128), dW3=z(3, 128), db3=z(3))
    bound = {k: torch.zeros_like(v) for k, v in want.items()}
    dz1_rows = z(M, 128)              # kept for the fakes of the self-check
    for lo in range(0, M, chunk):
        sl = slice(lo, min(M, lo + chunk))
        x, r, g = d(feat[sl]), ray_id[sl], d(g_rgb[sl])
        v = d(vb[r])
        z1 = x @ W1k.t() + v
        m1 = (z1 > 0).double()
        h1 = z1 * m1
        z2 = h1 @ W2.t() + b2
        m2 = (z2 > 0).double()
        h2 = z2 * m2
        y = torch.sigmoid(h2 @ W3.t() + b3)
        dz3 = g * y * (1 - y)
        dZ2 = (dz3 @ W3) * m2
        dZ1 = (dZ2 @ W2) * m1
        Bz1 = x.abs() @ aW1.t() + v.abs()
        Bh1 = Bz1 * m1
        Bh2 = (Bh1 @ aW2.t() + ab2) * m2
        By = y * (1 - y) * (Bh2 @ aW3.t() + ab3) + y
        Bdz3 = g.abs() * (y * (1 - y) + (1 - 2 * y).abs() * By)
        BdZ2 = (Bdz3 @ aW3) * m2
        BdZ1 = (BdZ2 @ aW2) * m1
        want['rgb'][sl], bound['rgb'][sl] = y, By
        want['g_feat'][sl], bound['g_feat'][sl] = dZ1 @ W1k, BdZ1 @ aW1
        want['g_vb'].index_add_(0, r, dZ1)
        bound['g_vb'].index_add_(0, r, BdZ1)
        dz1_rows[sl] = dZ1
        for k, a, b, ba, bb in (('dW1k', dZ1, x, BdZ1, x.abs()), ('dW2', dZ2, h1, BdZ2, Bh1), ('dW3', dz3, h2, Bdz3, Bh2)):
            want[k] += a.t() @ b
            bound[k] += ba.t() @ bb
        want['db2'] += dZ2.sum(0)
        bound['db2'] += BdZ2.sum(0)
        want['db3'] += dz3.sum(0)
        bound['db3'] += Bdz3.sum(0)
    return want, bound, dz1_rows


def ratios(got, want, bound):
    """name -> worst |got - want| / (B + TINY / TAU): <= TAU is a pass."""
    vals = [((got[k].double() - want[k]).abs() / (bound[k] + TINY / TAU)).max() for k in OUTS if k in got and got[k].numel()]
    return dict(zip([k for k in OUTS if k in got and got[k].numel()], torch.stack(vals).tolist()))


def judge(got, want, bound, what):
    r = ratios(got, want, bound)
    for k, v in r.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
    bad = {k: f'{v:.2e}' for k, v in r.items() if not v <= TAU}
    assert not bad, f'{what}: |got - want| / B above TAU = {TAU:.0e}: {bad}'


def min_preact(feat, vb, ray_id, W1k, W2, b2):
    x = feat.double()
    z1 = x @ W1k.double().t() + vb[ray_id].double()
    z2 = torch.relu(z1) @ W2.double().t() + b2.double()
    return torch.minimum(z1.abs().amin(1), z2.abs().amin(1))


def make_inputs(ray_id, N, seed, dev, edit=None, thresh=1e-5):
    """Seeded weights, per-ray view bias and per-sample features, changed by `edit(inputs)` if given.  ReLU-ambiguous samples
    (an fp64 pre-activation within `thresh` of zero: two correct fp32 evaluations may disagree on the mask) then get their
    feature row redrawn -- never dropped, which would change the ray layout."""
    g = torch.Generator().manual_seed(seed)
    M = ray_id.numel()
    u = lambda *s, a: ((torch.rand(*s, generator=g) * 2 - 1) * a)
    p = dict(W1k=u(128, 12, a=1 / math.sqrt(39)), W2=u(128, 128, a=1 / math.sqrt(128)), b2=u(128, a=1 / math.sqrt(128)),
             W3=u(3, 128, a=1 / math.sqrt(128)), b3=torch.randn(3, generator=g) * 0.1)
    vb = torch.randn(N, 128, generator=g) * 0.5
    feat = torch.randn(M, 12, generator=g)
    g_rgb = torch.randn(M, 3, generator=g)
    p = {k: v.to(dev) for k, v in p.items()}
    inp = dict(feat=feat.to(dev), vb=vb.to(dev), ray_id=ray_id.to(dev), g_rgb=g_rgb.to(dev), **p)
    if edit is not None:
        edit(inp)
    return redraw(inp, g, thresh)


def redraw(inp, g, thresh=1e-5, max_rounds=8):
    idx = torch.arange(inp['ray_id'].numel(), device=inp['feat'].device)
    for _ in range(max_rounds):
        amb = idx[min_preact(inp['feat'][idx], inp['vb'], inp['ray_id'][idx], inp['W1k'], inp['W2'], inp['b2']) <= thresh]
        if amb.numel() == 0:
            return inp
        inp['feat'][amb] = torch.randn(amb.numel(), 12, generator=g).to(inp['feat'].device)
        idx = amb
    raise AssertionError(f'{idx.numel()} samples still ReLU-ambiguous after {max_rounds} redraws')


def reference(inp):
    return ref64(*(inp[k] for k in ('feat', 'vb', 'ray_id', 'W1k', 'W2', 'b2', 'W3', 'b3', 'g_rgb')))


# ---- ray layouts -------------------------------------------------------------------------------------------------------
def partition(M, warps):
    """Python mirror of unit_grid + the warp ranges of k_shade_bwd_tc: first unit of every warp's range, and the end."""
    n_units = -(-M // UNIT)
    n_w = min(NUM_SMS, -(-n_units // warps)) * warps
    return [n_units * w // n_w for w in range(n_w + 1)]


def _from_lengths(lengths, M):
    ids = torch.repeat_interleave(torch.arange(len(lengths)), torch.tensor(lengths))[:M]
    return ids, int(ids[-1]) + 1


def _from_starts(starts, M):
    ind = torch.zeros(M, dtype=torch.int64)
    ind[torch.tensor(sorted({s for s in starts if 0 <= s < M} | {0}))] = 1
    ids = ind.cumsum(0) - 1
    return ids, int(ids[-1]) + 1


def _geometric(M, mean, seed):
    g = torch.Generator().manual_seed(seed)
    lens = (1 + (-torch.log1p(-torch.rand(M // 4 + 16, generator=g)) * (mean - 1)).floor()).long()
    cut = int((lens.cumsum(0) < M).sum()) + 1
    return lens[:cut].tolist()


def _alternating(M):
    """Runs of 1-3-sample rays (more than 4 segments per unit: the per-sample path) up to offset 12 of a unit, then a ray of
    40+ samples that starts inside that non-fitting unit and continues into fitting units."""
    lens, pos, k = [], 0, 0
    while pos < M:
        target = (pos // UNIT + 2 + k % 2) * UNIT + 12
        while pos < target:
            lens.append(min(1 + len(lens) % 3, target - pos))
            pos += lens[-1]
        lens.append(40 + 23 * (k % 3))
        pos += lens[-1]
        k += 1
    return _from_lengths(lens, M)


def _bounds(M, warps, shift):
    """A ray boundary at every warp-range (and so every CTA) boundary of the kernel's partition, moved by `shift` samples."""
    return _from_starts([UNIT * u + shift for u in partition(M, warps)[1:-1]], M)


def _sparse(M):
    ids = 2 * _from_lengths(_geometric(M, 20, M), M)[0] + 3      # odd ids only, the first is 3
    return ids, 4 * int(ids[-1]) + 64


def _randint(M):
    n = max(1, M // 245) + 1
    return torch.sort(torch.randint(0, n, (M,), generator=torch.Generator().manual_seed(M)))[0], n


LAYOUTS = {
    'aligned16': lambda M: _from_lengths([UNIT] * (-(-M // UNIT)), M),
    'offset16': lambda M: _from_lengths([8] + [UNIT] * (-(-M // UNIT)), M),
    'len4_o0': lambda M: _from_lengths([4] * (-(-M // 4)), M),
    'len4_o1': lambda M: _from_lengths([3] + [4] * (-(-M // 4)), M),
    'len4_o2': lambda M: _from_lengths([2] + [4] * (-(-M // 4)), M),
    'len4_o3': lambda M: _from_lengths([1] + [4] * (-(-M // 4)), M),
    'alternating': _alternating,
    'one_ray_first': lambda M: (torch.zeros(M, dtype=torch.int64), 3),
    'one_ray_last': lambda M: (torch.full((M,), 4, dtype=torch.int64), 5),
    'sparse_odd': _sparse,
    **{f'bounds{w}_{nm}': (lambda M, w=w, s=s: _bounds(M, w, s)) for w in (8, 4) for nm, s in (('m1', -1), ('0', 0), ('p1', 1))},
    'geometric250': lambda M: _from_lengths(_geometric(M, 250, M), M),
    'randint': _randint,
}

SMALL = (1, 15, 16, 17, 31, 32, 33, 127, 128, 129)
AROUND8 = (UNIT * 1056 - 1, UNIT * 1056, UNIT * 1056 + 1)       # n_units around n_warps = 132 CTAs x 8 warps
AROUND4 = (UNIT * 528 - 1, UNIT * 528, UNIT * 528 + 1)          # the same for 4 warps
BIG = 2_000_003
CASES = ([(lay, M) for lay in ('aligned16', 'offset16', 'len4_o0', 'len4_o1', 'len4_o2', 'len4_o3', 'alternating', 'one_ray_first',
                              'one_ray_last', 'sparse_odd', 'bounds8_0', 'randint') for M in SMALL]
         + [(lay, M) for lay in ('aligned16', 'offset16', 'len4_o0', 'len4_o1', 'alternating', 'one_ray_first', 'sparse_odd',
                                 'bounds8_m1', 'bounds8_0', 'bounds8_p1', 'geometric250', 'randint') for M in AROUND8]
         + [(lay, M) for lay in ('aligned16', 'offset16', 'len4_o2', 'bounds4_m1', 'bounds4_0', 'bounds4_p1') for M in AROUND4]
         + [(lay, BIG) for lay in ('offset16', 'len4_o1', 'alternating', 'one_ray_last', 'sparse_odd', 'bounds8_m1', 'bounds8_p1',
                                   'bounds4_m1', 'geometric250', 'randint')])

# (forward MODE, BWD_MODE, USE_MASKS)
ENGINES = (('tc3', 'fused', True), ('tc3', 'fused', False), ('tc3', 'fused4', True), ('tc3', 'tc3', True), ('tc3', 'simt', True),
           ('tc3w4', 'fused', True), ('simt', 'fused', True), ('simt', 'simt', True))


def run_engine(inp, mode, bwd, masks):
    """Forward + backward through _ShadeFn.apply with vb as a leaf, and the forward again under no_grad (the kSave = false
    instantiations)."""
    from unboundednerfpytorch_b200 import shade as shade_mod
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(shade_mod, 'MODE', mode)
        mp.setattr(shade_mod, 'BWD_MODE', bwd)
        mp.setattr(shade_mod, 'USE_MASKS', masks)
        leaves = {k: inp[k].clone().requires_grad_(True) for k in ('feat', 'vb', 'W1k', 'W2', 'b2', 'W3', 'b3')}
        args = [leaves['feat'], leaves['vb'], inp['ray_id']] + [leaves[k] for k in ('W1k', 'W2', 'b2', 'W3', 'b3')]
        rgb = shade_mod._ShadeFn.apply(*args, True)
        rgb.backward(inp['g_rgb'])
        with torch.no_grad():
            rgb_ng = shade_mod._ShadeFn.apply(*args, False)
    got = dict(rgb=rgb.detach(), g_feat=leaves['feat'].grad, g_vb=leaves['vb'].grad)
    got.update({'d' + k: leaves[k].grad for k in ('W1k', 'W2', 'b2', 'W3', 'b3')})
    return got, rgb_ng


def engines_for(layout):
    w = 4 if layout.startswith('bounds4') else 8 if layout.startswith('bounds8') else None
    if w is None:
        return ENGINES
    # the boundaries mirror one partition: 4-warp layouts are for the 4-warp backward, 8-warp layouts for the 8-warp ones
    return [e for e in ENGINES if (e[1] == 'fused4') == (w == 4)]


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    if WORST:
        print('\n[rgbnet-layouts] worst |got - want| / B: ' + ', '.join(f'{k} {v:.2e}' for k, v in sorted(WORST.items())))


@pytest.mark.gpu
@pytest.mark.parametrize('layout,M', CASES, ids=[f'{lay}-{M}' for lay, M in CASES])
def test_rgbnet_layout_vs_fp64(layout, M):
    """Every engine: rgb, g_feat, g_vb and the six parameter gradients within TAU * B of fp64; rays without samples get exactly
    zero; the no_grad forward is bit-identical to the grad-enabled one."""
    ray_id, N = LAYOUTS[layout](M)
    assert ray_id.numel() == M and bool((ray_id[1:] >= ray_id[:-1]).all()) and int(ray_id.max()) < N
    inp = make_inputs(ray_id, N, seed=M, dev=DEV)
    want, bound, _ = reference(inp)
    empty = torch.bincount(inp['ray_id'], minlength=N) == 0
    fails = []
    for mode, bwd, masks in engines_for(layout):
        what = f'{layout} M={M} {mode}+{bwd}{"" if masks else " (no masks)"}'
        got, rgb_ng = run_engine(inp, mode, bwd, masks)
        try:
            assert torch.equal(rgb_ng, got['rgb']), f'{what}: no_grad forward differs from the grad-enabled one'
            assert not bool(got['g_vb'][empty].any()), f'{what}: rays without samples got a nonzero g_vb'
            judge(got, want, bound, what)
        except AssertionError as e:
            fails.append(str(e))
    assert not fails, '\n'.join(fails)


# single-pass TF32 truncates every operand toward zero, so its error along a ray is coherent (~1e-3 of the ray's magnitude):
# one moved sample is only visible above it on rays of up to ~100 samples.  The short-ray layouts get the per-ray norm
# check; the long-ray ones the exact zeros and the relative error only.
TC1_CASES = [('aligned16', 129), ('len4_o1', 4099), ('alternating', 4099), ('sparse_odd', AROUND8[1]), ('bounds8_p1', AROUND8[0]),
             ('bounds8_m1', AROUND8[2]), ('geometric250', AROUND8[2]), ('randint', AROUND8[0])]
TC1_LONG_RAYS = ('geometric250', 'randint')


def _tc1_inputs(ray_id, N, seed, dev):
    """Inputs whose pre-activations stay far from zero (|z| >~ 0.5), so that single-pass TF32 (~1e-3 relative) keeps every
    ReLU mask of the fp64 reference: vb and b2 carry a large signed offset per column.  The masks are then constant along a
    ray, so a ray's g_vb is a fixed linear map of its sum of dz3; a one-signed upstream gradient keeps that sum from
    cancelling, which would make the per-ray relative error meaningless."""
    inp = make_inputs(ray_id, N, seed, dev)
    g = torch.Generator().manual_seed(seed + 1)
    sign = lambda *s: (torch.randint(0, 2, s, generator=g) * 2 - 1).float().to(dev)
    inp['feat'] *= 0.3
    inp['vb'] = sign(N, 128) * (1.5 + torch.rand(N, 128, generator=g).to(dev))
    inp['b2'] = sign(128) * 25.0
    inp['W3'] *= 0.05                                    # H2 ~ 25: keep the sigmoid out of saturation, where 1 - rgb rounds away
    inp['g_rgb'] = (torch.rand(ray_id.numel(), 3, generator=g) + 0.25).to(dev)
    assert float(min_preact(inp['feat'], inp['vb'], inp['ray_id'], inp['W1k'], inp['W2'], inp['b2']).min()) > 0.2
    return inp


def tc1_ray_ratio(g_vb, want, rss):
    """per ray: ||got - want|| / sqrt(sum over its samples of ||B(dZ1)||^2)"""
    return (g_vb.double() - want).norm(dim=1) / (rss + TINY)


@pytest.mark.gpu
@pytest.mark.parametrize('layout,M', TC1_CASES, ids=[f'{lay}-{M}' for lay, M in TC1_CASES])
def test_rgbnet_tc1_rays(layout, M):
    """Single-pass TF32 (tc1 + fused): rays without samples exactly zero, every ray's g_vb within the relative Frobenius error
    the model-level test allows, and every sample on its own ray: a per-ray norm check that one moved sample fails."""
    ray_id, N = LAYOUTS[layout](M)
    inp = _tc1_inputs(ray_id, N, M, DEV)
    want, bound, dz1 = reference(inp)
    got, _ = run_engine(inp, 'tc1', 'fused', True)
    g_vb, w = got['g_vb'], want['g_vb']
    empty = torch.bincount(inp['ray_id'], minlength=N) == 0
    assert not bool(g_vb[empty].any()), 'rays without samples got a nonzero g_vb'
    live = ~empty
    rel = ((g_vb.double() - w).norm(dim=1) / w.norm(dim=1))[live]
    assert float(rel.max()) <= 8e-2, f'worst per-ray relative Frobenius error {float(rel.max()):.2e}'
    Bz = _rss_bound(inp)
    r = float(tc1_ray_ratio(g_vb, w, Bz)[live].max())
    key = 'tc1 g_vb per ray' + (' (long rays)' if layout in TC1_LONG_RAYS else '')
    WORST[key] = max(WORST.get(key, 0.0), r)
    if layout in TC1_LONG_RAYS:
        return
    assert r <= TAU_TC1, f'per-ray norm error {r:.2e} of the bound'
    for p in (M // 2, M // 3, M // 5):                   # the same check rejects one sample moved to the neighbouring ray
        i = _boundary_sample(inp['ray_id'].cpu(), p)
        rf = float(tc1_ray_ratio(_moved(inp['ray_id'], dz1, w, i).float(), w, Bz).max())
        WORST['tc1 moved-sample fake (min)'] = min(WORST.get('tc1 moved-sample fake (min)', math.inf), rf)
        assert rf > 2 * TAU_TC1, f'sample {i} moved to the ray before it is only {rf:.2e} of the bound'


def _rss_bound(inp):
    """per ray: sqrt(sum over its samples of ||B(dZ1)||^2), B(dZ1) as in ref64 without the forward's error"""
    x, r = inp['feat'].double(), inp['ray_id']
    W1k, W2, b2, W3, b3 = (inp[k].double() for k in ('W1k', 'W2', 'b2', 'W3', 'b3'))
    rss = torch.zeros(inp['vb'].shape[0], dtype=torch.float64, device=x.device)
    for lo in range(0, x.shape[0], 1 << 18):
        sl = slice(lo, lo + (1 << 18))
        z1 = x[sl] @ W1k.t() + inp['vb'][r[sl]].double()
        z2 = torch.relu(z1) @ W2.t() + b2
        y = torch.sigmoid(torch.relu(z2) @ W3.t() + b3)
        BdZ1 = (((inp['g_rgb'][sl].double() * y * (1 - y)).abs() @ W3.abs()) * (z2 > 0) @ W2.abs()) * (z1 > 0)
        rss.index_add_(0, r[sl], BdZ1.pow(2).sum(1))
    return rss.sqrt()


# ---- dead units: exact zeros pin the bit layout of the ReLU masks ------------------------------------------------------
DEAD_B2 = (0, 11, 20, 31, 43, 86, 125)      # b2[c] = -1e3: columns 8 j + 2 t + e over every j & 3, t and e
DEAD_VB_ALL = (3, 14, 57, 96)               # vb[:, c'] = -1e3 on every ray
DEAD_VB_SOME = (33, 70, 119)                # ... on the even rays only


@pytest.mark.gpu
@pytest.mark.parametrize('layout,M', [('geometric250', AROUND8[2]), ('aligned16', 129), ('len4_o1', 4099)])
def test_rgbnet_dead_units_exact_zero(layout, M):
    """Hidden units that are off for every sample (b2[c] = -1e3, or vb[:, c'] = -1e3 on every ray) and units off on some rays
    only: every gradient that flows only through them is exactly 0.0 in every engine, which a ReLU mask bit read from the
    wrong position (t and e swapped, another j & 3) would break.  A unit with an all-zero upstream gradient adds exactly 0.0
    to g_feat."""
    ray_id, N = LAYOUTS[layout](M)
    even = torch.arange(N, device=DEV) % 2 == 0
    some = torch.zeros(N, 128, dtype=torch.bool, device=DEV)
    some[even.nonzero()[:, 0][:, None], torch.tensor(DEAD_VB_SOME, device=DEV)[None]] = True
    zu = 1 if M > 2 * UNIT else 0                       # one unit with an all-zero upstream gradient

    def edit(inp):
        inp['b2'][list(DEAD_B2)] = -1e3
        inp['vb'][:, list(DEAD_VB_ALL)] = -1e3
        inp['vb'][some] = -1e3
        inp['g_rgb'][UNIT * zu:UNIT * zu + UNIT] = 0

    inp = make_inputs(ray_id, N, seed=M + 7, dev=DEV, edit=edit)
    want, bound, _ = reference(inp)
    dead_vb = some.clone()
    dead_vb[:, list(DEAD_VB_ALL)] = True
    fails = []
    for mode, bwd, masks in ENGINES:
        what = f'{layout} M={M} {mode}+{bwd}{"" if masks else " (no masks)"}'
        got, _ = run_engine(inp, mode, bwd, masks)
        zeros = {'db2[c]': got['db2'][list(DEAD_B2)], 'dW2[c, :]': got['dW2'][list(DEAD_B2)],
                 'dW3[:, c]': got['dW3'][:, list(DEAD_B2)], "dW2[:, c']": got['dW2'][:, list(DEAD_VB_ALL)],
                 "dW1k[c', :]": got['dW1k'][list(DEAD_VB_ALL)], "g_vb[ray, c']": got['g_vb'][dead_vb],
                 'g_feat of the zero-gradient unit': got['g_feat'][UNIT * zu:UNIT * zu + UNIT]}
        try:
            for k, v in zeros.items():
                assert not bool(v.any()), f'{what}: {k} not exactly zero ({int((v != 0).sum())} elements, max {float(v.abs().max()):.2e})'
            judge(got, want, bound, what)
        except AssertionError as e:
            fails.append(str(e))
    assert not fails, '\n'.join(fails)


# ---- CPU: the layouts have the structure they are named for, and the check is tight enough to see misplaced samples ----
def unit_segments(ray_id):
    """number of ray segments in every full 16-sample unit (what k_shade_bwd_tc calls nseg)"""
    n = ray_id.numel() // UNIT
    u = ray_id[:n * UNIT].view(n, UNIT)
    return 1 + (u[:, 1:] != u[:, :-1]).sum(1)


def test_layouts_have_their_structure():
    M = AROUND8[2]
    seg = {lay: unit_segments(LAYOUTS[lay](M)[0]) for lay in ('aligned16', 'offset16', 'len4_o0', 'len4_o1', 'len4_o2', 'len4_o3')}
    assert bool((seg['aligned16'] == 1).all()) and bool((seg['offset16'] == 2).all()) and bool((seg['len4_o0'] == 4).all())
    for o in (1, 2, 3):
        assert bool((seg[f'len4_o{o}'] == 5).all())
    ids = LAYOUTS['aligned16'](M)[0]
    assert bool((ids[UNIT::UNIT] != ids[UNIT - 1:-1:UNIT]).all())           # every unit starts a ray
    # alternating: a unit with more than 4 segments whose last ray runs on through the whole next unit
    ids = LAYOUTS['alternating'](M)[0]
    s = unit_segments(ids)
    n = s.numel()
    last = ids[UNIT - 1:n * UNIT:UNIT]
    nxt = ids[2 * UNIT - 1:n * UNIT:UNIT]
    assert int(((s[:-1] > 4) & (last[:-1] == nxt)).sum()) > 100
    for w in (8, 4):
        for nm, shift in (('m1', -1), ('0', 0), ('p1', 1)):
            ids = LAYOUTS[f'bounds{w}_{nm}'](M)[0]
            b = torch.tensor([UNIT * u + shift for u in partition(M, w)[1:-1]])
            assert bool((ids[b] != ids[b - 1]).all())                         # a ray starts at every range boundary + shift
    ids, N = LAYOUTS['sparse_odd'](M)
    assert int(ids[0]) > 0 and bool((ids % 2 == 1).all()) and N > 2 * int(ids.max())
    for lay, n_rays in (('one_ray_first', 3), ('one_ray_last', 5)):
        ids, N = LAYOUTS[lay](M)
        assert N == n_rays and int(ids.min()) == int(ids.max()) == (0 if lay.endswith('first') else N - 1)
    ids = LAYOUTS['geometric250'](BIG)[0]
    assert 200 < BIG / (int(ids[-1]) + 1) < 300



def _boundary_sample(ray_id, p):
    """A sample next to the ray boundary nearest to sample p: the first sample of its ray (it has a ray before it)."""
    starts = ((ray_id[1:] != ray_id[:-1]).nonzero()[:, 0] + 1)
    assert starts.numel(), 'layout has a single ray'
    return int(starts[(starts - p).abs().argmin()])


def _moved(ray_id, dz1, g_vb, i):
    """g_vb with sample i's dZ1 on the ray before it instead of its own."""
    fake = g_vb.clone()
    fake[ray_id[i]] -= dz1[i]
    fake[ray_id[i - 1]] += dz1[i]
    return fake


SELF_CASES = [(lay, 4099) for lay in ('aligned16', 'offset16', 'len4_o0', 'len4_o1', 'len4_o2', 'len4_o3', 'alternating',
                                      'sparse_odd', 'randint')] + \
             [('bounds8_m1', AROUND8[2]), ('bounds8_p1', AROUND8[0]), ('bounds4_0', AROUND4[2]), ('geometric250', AROUND8[2])]


@pytest.mark.parametrize('layout,M', SELF_CASES, ids=[f'{lay}-{M}' for lay, M in SELF_CASES])
def test_checker_rejects_misplaced_samples(layout, M):
    """fp64 reference rounded to fp32 passes at TAU; the same with one sample moved to the neighbouring ray (at a unit boundary
    and at a warp-range boundary) or one sample's dZ1 dropped fails."""
    ray_id, N = LAYOUTS[layout](M)
    inp = make_inputs(ray_id, N, seed=M, dev='cpu')
    want, bound, dz1 = reference(inp)
    honest = {k: v.float() for k, v in want.items()}
    worst = max(ratios(honest, want, bound).values())
    assert worst <= TAU / 20, f'fp32 rounding alone is {worst:.2e} of B'
    warps = 4 if layout.startswith('bounds4') else 8
    at = {'unit': UNIT * (-(-M // UNIT) // 2 + 1), 'warp range': UNIT * partition(M, warps)[len(partition(M, warps)) // 2]}
    for where, p in at.items():
        i = _boundary_sample(ray_id, p)
        assert abs(i - p) < 64 or layout.startswith(('randint', 'geometric')), (where, i, p)
        assert bool(dz1[i].any())
        r = ratios({'g_vb': _moved(ray_id, dz1, want['g_vb'], i).float()}, want, bound)['g_vb']
        assert r > 10 * TAU, f'{layout}: sample {i} moved at a {where} boundary is only {r:.2e} of B'
        dropped = want['g_vb'].clone()
        dropped[ray_id[i]] -= dz1[i]
        r = ratios({'g_vb': dropped.float()}, want, bound)['g_vb']
        assert r > 10 * TAU, f'{layout}: sample {i} dZ1 dropped at a {where} boundary is only {r:.2e} of B'
