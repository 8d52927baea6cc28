"""The march's grid-gradient scatters (csrc/march.cu, march_feature.cu, march_ndc.cu) against a plain fp64 adjoint, element by
element, with no MLP in between.

Every scatter is driven through its autograd Function (march.March, NdcMarch, BoxMarch) with a seeded upstream gradient on one
output per grid: the k0 features (k0 grid), and raw_density (contracted) or raw_alpha (NDC / box) for the density grid.  Through
raw_density the scatter receives exactly the upstream value per survivor; through raw_alpha it receives the reference's raw2alpha
derivative interval * min(e, 1e10) * (1 + e)^(-interval - 1) of the survivor's fp32 raw density, evaluated here in fp64.

The fp64 reference uses the kernel's own cells: sample points from the op path (bit-identical to the kernels'), the reference's
normalisation and Fourier embedding, unnormalisation, floor and clamp all in fp32 on the GPU as ATen does them; only the 8 corner
weights and the index_add of w * g / P are fp64.  (An fp64 coordinate chain would move a corner weight by ~ulp * (X - 1) / 2, far
above 1e-5 of a small weight.)  The fp64 gather from the same cells reproduces the kernels' forward features and densities within
TAU_FWD of their bound, which shows that both sides agree on the cells.

Every grid element is judged as |got - want| <= TAU * B, B = sum of |w| * |g| / P over its addends (fp64), and an element without
addends must come out exactly 0.0 (a stray or doubled write).  The cases sit where the scatters' bookkeeping changes: every slab
count of the reference's configs (P = 1 .. 9 on the specialised kernels, P = 11 = fourier_freq_num 5 on the generic ones), every
k0 kernel selection and both density scatters, non-cubic odd-sized grids, the x-range split boundaries of the slab-major scatter,
equal-cell merges across its groups of 4 and 32-sample chunks, ragged survivor chunks, the run scatter's run lengths and its
shared-memory limit, box faces / edges / corners, and every record alignment of the 36- and 12-byte NDC / box records.  Each
structural claim is asserted from the kernel's own ray_id / step_id and the reference cells.  test_checker_rejects_faults (CPU)
shows that TAU rejects one moved, dropped or doubled sample, a sin / cos slab swap and a dropped x-range boundary plane."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

DEV = 'cuda:0'
TAU = 1e-5                # scatter: |got - want| <= TAU * B element by element (worst seen on an H100 80GB HBM3: 1.1e-6, and
                          # 3.2e-6 of B + |prefill| when adding into pre-filled buffers)
TAU_FWD = 1e-6            # forward self-check: kernel features / density within TAU_FWD of the fp64 gather's bound (worst seen 3.7e-7)
WORST = {}                # check -> worst |got - want| / B in this session
RUN_SMEM_LIMIT = 40 * 1024    # the run scatter of k_march_density_bwd is used while 4 warps x (S + 33) floats fit in it
BG = 0.2                  # bg_len of the contracted models


# ---- fp64 reference ----------------------------------------------------------------------------------------------------
def slab_coords(pts, mn, mx, n_freqs):
    """[P, M, 3] normalised coordinates of every slab in world-axis order (x -> grid dim X), fp32 on the device of pts: the
    reference's ind_norm (grid.py:55, without the .flip, a permutation) and nerf_pos_embed (FourierGrid_grid.py:21-36)."""
    from oracle.cpu_ref import nerf_pos_embed
    mn = torch.as_tensor(mn, dtype=torch.float32, device=pts.device)
    mx = torch.as_tensor(mx, dtype=torch.float32, device=pts.device)
    n = ((pts - mn) / (mx - mn)) * 2 - 1
    if n_freqs <= 0:
        return n[None]
    P = 1 + 2 * n_freqs
    return nerf_pos_embed(n, n_freqs).reshape(-1, P, 3).permute(1, 0, 2)


def cells(coords, shape):
    """ATen's unnormalisation ((c + 1) / 2) * (size - 1), the clamped base voxel and the fractions, all fp32."""
    size = torch.tensor(shape, dtype=torch.float32, device=coords.device)
    c = ((coords + 1) / 2) * (size - 1)
    x0 = torch.minimum(torch.clamp(torch.floor(c), min=0), size - 2)
    return x0.long(), c - x0


def _corners(x0, f, shape):
    """(voxel index inside the slab [.., M], fp64 weight [.., M]) of the 8 corners of every cell."""
    X, Y, Z = shape
    f = f.double()
    for corner in range(8):
        bx, by, bz = corner >> 2, (corner >> 1) & 1, corner & 1
        w = ((f[..., 2] if bz else 1 - f[..., 2]) * (f[..., 1] if by else 1 - f[..., 1])) * (f[..., 0] if bx else 1 - f[..., 0])
        yield ((x0[..., 0] + bx) * Y + x0[..., 1] + by) * Z + x0[..., 2] + bz, w


def ref_scatter(x0, f, g, shape):
    """want[P, X, Y, Z, C] = sum over samples, slabs and corners of w * g / P in fp64, and its bound B (|w| * |g| / P)."""
    P, C = x0.shape[0], g.shape[1]
    X, Y, Z = shape
    gP = g.double() / P
    agP = gP.abs()
    want = torch.zeros(P, X * Y * Z, C, dtype=torch.float64, device=g.device)
    bound = torch.zeros_like(want)
    for s in range(P):
        for idx, w in _corners(x0[s], f[s], shape):
            want[s].index_add_(0, idx, w[:, None] * gP)
            bound[s].index_add_(0, idx, w.abs()[:, None] * agP)
    return want.view(P, X, Y, Z, C), bound.view(P, X, Y, Z, C)


def ref_gather(x0, f, grid):
    """Forward of the same cells in fp64: mean over slabs of the trilinear reads of grid[P, X, Y, Z, C], and its bound."""
    P, X, Y, Z, C = grid.shape
    flat = grid.double().reshape(P, -1, C)
    val = torch.zeros(x0.shape[1], C, dtype=torch.float64, device=grid.device)
    bound = torch.zeros_like(val)
    for s in range(P):
        for idx, w in _corners(x0[s], f[s], (X, Y, Z)):
            v = flat[s][idx]
            val += w[:, None] * v
            bound += w.abs()[:, None] * v.abs()
    return val / P, bound / P


def ratio(got, want, bound, base=None):
    """(worst |got - base - want| / (B + |base|) over elements with addends, elements without addends that differ from base)"""
    got = got.double()
    base = torch.zeros_like(got) if base is None else base.double()
    lim = bound + base.abs()
    empty = bound == 0
    stray = int((got[empty] != base[empty]).sum())
    live = ~empty
    r = float(((got - base - want).abs()[live] / lim[live]).max()) if bool(live.any()) else 0.0
    return r, stray


def judge(got, want, bound, what, key, base=None, tau=TAU):
    r, stray = ratio(got, want, bound, base)
    WORST[key] = max(WORST.get(key, 0.0), r)
    print(f'[march-scatter] {what}: worst |got - want| / B = {r:.2e}')
    assert stray == 0, f'{what}: {stray} elements without addends are not exactly {"the prefill" if base is not None else "0.0"}'
    assert r <= tau, f'{what}: |got - want| / B = {r:.2e} above {tau:.0e}'


def as_pxyzc(t):
    """[P, C, X, Y, Z] grid (contiguous or channels-last) or its gradient -> [P, X, Y, Z, C] view."""
    return t.permute(0, 2, 3, 4, 1)


def channels_last(t):
    """[P, X, Y, Z, C] values -> a [P, C, X, Y, Z] tensor with the channels-last strides of grid.zeros_grid."""
    return t.contiguous().permute(0, 4, 1, 2, 3)


def raw2alpha_grad(raw, shift, interval, g):
    """fp64 d raw_alpha / d raw_density * g of the reference's Raw2Alpha (render_utils_kernel.cu:431-443) at the fp32 raw
    density raw; the kernel adds shift in fp32 before its exp."""
    e = torch.exp((raw + np.float32(shift)).double())
    return interval * e.clamp(max=1e10) * (1 + e).pow(-interval - 1) * g.double()


# ---- kernel selections -----------------------------------------------------------------------------------------------
@pytest.fixture
def selections():
    """Restores the process-wide kernel selections after the test."""
    from unboundednerfpytorch_b200 import ops
    fk, ds = ops.get_feature_kernel(), ops.get_density_scatter()
    try:
        yield ops
    finally:
        ops.set_feature_kernel(fk)
        ops.set_density_scatter(ds)


def run_smem_ok(S):
    return 4 * 4 * (S + 33) <= RUN_SMEM_LIMIT


# ---- contracted march (FourierGridModel / DirectContractedVoxGO) -----------------------------------------------------
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def x_rays(n, g, x=-1.19, yz=0.95):
    """Rays along +x at fixed (y, z): their slab-0 cells walk through every x plane."""
    o = torch.cat([torch.full((n, 1), x), (torch.rand(n, 2, generator=g) * 2 - 1) * yz], 1)
    o[:, 0] += torch.rand(n, generator=g) * 0.4
    d = torch.zeros(n, 3)
    d[:, 0] = 1
    return o, d


def random_rays(n, g):
    return (torch.rand(n, 3, generator=g) * 2 - 1) * 0.9, torch.randn(n, 3, generator=g)


def far_rays(n, g):
    """Rays far outside the unit cube: every sample lies in the outer shell of the contracted space."""
    o = torch.cat([torch.full((n, 1), 60.0), (torch.rand(n, 2, generator=g) * 2 - 1) * 20], 1)
    d = torch.zeros(n, 3)
    d[:, 0] = 1
    return o, d


def ragged_planes(X):
    """Per-x-plane density of the ragged scene (X = 41, stepsize 0.5: ~2.8 samples per cell on the x rays), alive -6 / dead -40:
    planes 0-12 alive (a first chunk that is all survivors when the ray starts far enough left, and a chunk whose survivors
    straddle the x-range boundary at plane 10), one denser plane 27 in a dead stretch (for rays starting near cx = 4.2 its one
    survivor is sample 63: lane 31 of the second chunk), planes 31-33, and a dead outer shell (34-40: chunks without survivors,
    and no survivors at all on rays from far away)."""
    assert X == 41
    D = torch.full((X,), -40.0)
    D[0:13] = -6.0
    D[27] = -3.0
    D[31:34] = -6.0
    return D


class Contracted:
    """A FourierGrid / DCVGO-style scene built on raw grids (any shape, any slab count) and driven through march.March."""

    def __init__(self, P, shape, norm='inf', world_len=41, stepsize=0.1, n_x=192, n_rand=96, n_far=0, thres=0.0, seed=0):
        from unboundednerfpytorch_b200 import march
        from unboundednerfpytorch_b200 import grid as G
        self.P, self.shape, self.norm, self.thres = P, tuple(shape), norm, thres
        self.n_freqs = (P - 1) // 2
        X, Y, Z = shape
        g = _gen(1000 * P + seed)
        if thres > 0:       # ragged: the density is set by slab 0 alone, stripes of very negative density along x
            dens = torch.zeros(P, 1, X, Y, Z)
            dens[0, 0] = P * ragged_planes(X)[:, None, None] + 0.3 * torch.randn(X, Y, Z, generator=g)
        else:
            dens = torch.randn(P, 1, X, Y, Z, generator=g)
        self.dgrid = dens.to(DEV)
        self.kvals = torch.randn(P, X, Y, Z, 12, generator=g).to(DEV)
        parts = [x_rays(n_x, g), random_rays(n_rand, g)] + ([far_rays(n_far, g)] if n_far else [])
        self.ro = torch.cat([p[0] for p in parts]).to(DEV)
        self.rd = torch.cat([p[1] for p in parts]).to(DEV)
        self.mn = (torch.tensor([-1.] * 3) - BG).tolist()
        self.mx = (torch.tensor([1.] * 3) + BG).tolist()
        self.t_table = march.t_schedule(world_len, stepsize, BG, 1.5, DEV)
        self.S = self.t_table.numel()
        self.cfg = march.make_cfg([0.] * 3, [1.] * 3, BG, norm, self.S, 0.0, 0.5, thres)
        self.ddesc = G.grid_desc(self.dgrid, self.mn, self.mx, self.n_freqs)
        self.kdesc = G.grid_desc(channels_last(self.kvals), self.mn, self.mx, self.n_freqs)
        self.world_len, self.stepsize = world_len, stepsize

    def points(self, ray_id, step_id):
        from unboundednerfpytorch_b200 import models
        ns = types.SimpleNamespace(scene_center=torch.zeros(3, device=DEV), scene_radius=torch.ones(3, device=DEV), bg_len=BG,
                                   T_BOUNDARY=1.5, contracted_norm=self.norm, _world_len=lambda: self.world_len)
        pts, _, _ = models._ContractedBase._sample_dense(ns, self.ro, self.rd, self.stepsize)
        return pts[ray_id, step_id]

    def run(self, g_feat=None, g_dens=None, dbuf=None, kbuf=None):
        from unboundednerfpytorch_b200 import march
        dg = self.dgrid.clone().requires_grad_(True)
        kg = channels_last(self.kvals).clone().requires_grad_(True)
        if dbuf is not None:
            dg._ubn_grad_buffer = dbuf
        if kbuf is not None:
            kg._ubn_grad_buffer = kbuf
        out = march.March.apply(dg, kg, self.ro, self.rd, self.t_table, None, self.cfg, self.ddesc, self.kdesc,
                                self.thres <= 0, False)
        feat, dens, ray_id, step_id = out[4], out[3], out[5], out[6]
        if g_feat is not None:
            ((feat * g_feat).sum() + (dens * g_dens).sum()).backward()
        return dict(feat=feat.detach(), dens=dens.detach(), ray_id=ray_id, step_id=step_id, gk=kg.grad, gd=dg.grad)


def slab0_runs(ray_id, step_id, v0, S):
    """Equal-cell structure of consecutive survivors in slab 0, as the slab-major scatter (one x-range) groups them: rank of a
    survivor in its 32-sample chunk, pairs of neighbours in one cell that straddle a group of 4 / a chunk, and the longest run."""
    n = ray_id.numel()
    chunk = step_id // 32
    key = ray_id * (S // 32 + 1) + chunk
    idx = torch.arange(n, device=ray_id.device)
    start = torch.ones(n, dtype=torch.bool, device=ray_id.device)
    start[1:] = key[1:] != key[:-1]
    first = torch.cummax(torch.where(start, idx, torch.zeros_like(idx)), 0)[0]
    rank = idx - first
    same = (ray_id[1:] == ray_id[:-1]) & (v0[1:] == v0[:-1])
    same_chunk = same & ~start[1:]
    run_id = torch.cumsum(torch.cat([torch.ones(1, dtype=torch.long, device=ray_id.device), (~same_chunk).long()]), 0)
    return dict(group=int((same_chunk & (rank[:-1] % 4 == 3)).sum()), chunk=int((same & start[1:]).sum()),
                longest=int(torch.bincount(run_id).max()), rank=rank, key=key)


def part_bounds(X, n_split):
    return [((X - 1) * p) // n_split for p in range(1, n_split)]


C_SHAPE = (23, 37, 41)           # odd X * Y * Z: the slabs alternate in parity; X - 1 = 22 is not divisible by 4
C_SHAPE4 = (41, 23, 37)          # X - 1 = 40 is
CONTRACTED = {
    'P1': dict(P=1, shape=C_SHAPE),
    'P3': dict(P=3, shape=C_SHAPE4),
    'P5': dict(P=5, shape=C_SHAPE),
    'P7': dict(P=7, shape=C_SHAPE),
    'P7-l2': dict(P=7, shape=C_SHAPE4, norm='l2'),
    'P9': dict(P=9, shape=C_SHAPE4, n_far=32),
    'P9-l2': dict(P=9, shape=C_SHAPE, norm='l2'),
    'P11': dict(P=11, shape=C_SHAPE),
    'P9-X2': dict(P=9, shape=(2, 37, 41)),
    'P7-X3': dict(P=7, shape=(3, 23, 37)),
    'P5-X5': dict(P=5, shape=(5, 37, 41)),
    'P1-X3': dict(P=1, shape=(3, 23, 41)),
    'P9-ragged': dict(P=9, shape=C_SHAPE4, thres=1e-4, world_len=41, stepsize=0.5, n_x=768, n_rand=64, n_far=16),
    'P1-ragged': dict(P=1, shape=C_SHAPE4, thres=1e-4, world_len=41, stepsize=0.5, n_x=768, n_rand=64, n_far=16),
    'P7-longS': dict(P=7, shape=C_SHAPE, world_len=41, stepsize=0.025, n_x=48, n_rand=24),
    'P1-longS': dict(P=1, shape=C_SHAPE4, world_len=41, stepsize=0.025, n_x=48, n_rand=24),
}
# (feature kernel, density scatter): every k0 selection with the default run scatter, and the per-sample density scatter
SELECTIONS = [(fk, 1) for fk in range(7)] + [(5, 0)]


def _shape_str(shape):
    return 'x'.join(map(str, shape))


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(CONTRACTED))
def test_contracted_scatter_vs_fp64(case, selections):
    """k0 and density scatters of the contracted march under every kernel selection against the fp64 adjoint."""
    ops = selections
    spec = dict(CONTRACTED[case])
    sc = Contracted(**spec)
    P, shape, S = sc.P, sc.shape, sc.S
    X = shape[0]
    ops.set_feature_kernel(5)
    base = sc.run()
    ray_id, step_id = base['ray_id'], base['step_id']
    M = ray_id.numel()
    assert M > 1000, f'{case}: only {M} survivors'
    cs = slab_coords(sc.points(ray_id, step_id), sc.mn, sc.mx, sc.n_freqs)
    x0, f = cells(cs, shape)
    gen = torch.Generator(DEV).manual_seed(M)
    g_feat = torch.randn(M, 12, device=DEV, generator=gen)
    g_dens = torch.randn(M, device=DEV, generator=gen)
    want_k, bound_k = ref_scatter(x0, f, g_feat, shape)
    want_d, bound_d = ref_scatter(x0, f, g_dens[:, None], shape)
    fk_want, fk_bound = ref_gather(x0, f, sc.kvals)
    fd_want, fd_bound = ref_gather(x0, f, as_pxyzc(sc.dgrid))
    tag = f'contracted P={P} {_shape_str(shape)} {sc.norm} S={S}'
    side = 'run scatter' if run_smem_ok(S) else 'per-sample fallback'
    print(f'[coverage] {tag}: {M} survivors of {sc.ro.shape[0]} rays; density scatter mode 1 -> {side}')
    if case.endswith('longS'):
        assert not run_smem_ok(S), f'{case}: S = {S} should exceed the run scatter'
    else:
        assert run_smem_ok(S)
    _contracted_structure(case, sc, ray_id, step_id, cs, x0, f)

    fails = []
    for fk, ds in SELECTIONS:
        ops.set_feature_kernel(fk)
        ops.set_density_scatter(ds)
        got = sc.run(g_feat, g_dens)
        what = f'{tag} fk={fk} ds={ds}'
        try:
            assert torch.equal(got['ray_id'], ray_id) and torch.equal(got['step_id'], step_id), f'{what}: survivors differ'
            judge(got['feat'][:, :, None], fk_want[:, :, None], fk_bound[:, :, None], what + ' k0 forward self-check',
                  'forward self-check', tau=TAU_FWD)
            judge(got['dens'][:, None, None], fd_want[:, :, None], fd_bound[:, :, None], what + ' density forward self-check',
                  'forward self-check', tau=TAU_FWD)
            judge(as_pxyzc(got['gk']), want_k, bound_k, what + ' k0 scatter', f'k0 P={P}')
            judge(as_pxyzc(got['gd']), want_d, bound_d, what + ' density scatter', f'density P={P} ds={ds}')
        except AssertionError as e:
            fails.append(str(e))
    assert not fails, '\n'.join(fails)


def _contracted_structure(case, sc, ray_id, step_id, cs, x0, f):
    """The structural claims of each case, from the kernel's survivors and the reference cells."""
    P, (X, Y, Z), S = sc.P, sc.shape, sc.S
    tag = f'{case} ({_shape_str(sc.shape)})'
    bx0 = x0[0, :, 0]
    v0 = (x0[0, :, 0] * Y + x0[0, :, 1]) * Z + x0[0, :, 2]
    if sc.thres > 0:
        _ragged_structure(tag, sc, ray_id, step_id, bx0)
        return
    if X >= 5:      # every x-range boundary plane of the 2- and 4-way split, and the base planes on either side, get survivors
        for n_split in (2, 4):
            for b in part_bounds(X, n_split):
                planes = [p for p in (b - 1, b, b + 1) if p <= X - 2]      # X - 1 is never the base of a cell
                cnt = [int((bx0 == p).sum()) for p in planes]
                print(f'[coverage] {tag}: n_split {n_split} boundary plane {b}: survivors on base planes {planes} = {cnt}')
                assert min(cnt) > 0, f'{tag}: boundary {b} of the {n_split}-way split not covered: {cnt}'
    else:           # empty parts / single-plane parts
        for n_split in (2, 4):
            lo = [0] + part_bounds(X, n_split)
            hi = part_bounds(X, n_split) + [X]
            sizes = [h - l for l, h in zip(lo, hi)]
            print(f'[coverage] {tag}: {n_split}-way split planes per part {sizes}')
        assert 0 in [h - l for l, h in zip([0] + part_bounds(X, 4), part_bounds(X, 4) + [X])]
    # the outer shell: samples within 1 % of a face of the contracted domain, in the last cell along that axis
    last = ((x0[0] == torch.tensor([X - 2, Y - 2, Z - 2], device=DEV)) | (x0[0] == 0)) & (cs[0].abs() > 0.99)
    shell = int(last.any(1).sum())
    print(f'[coverage] {tag}: {shell} survivors in the outer shell')
    assert shell > 0
    runs = slab0_runs(ray_id, step_id, v0, S)
    print(f"[coverage] {tag}: slab-0 equal-cell neighbours straddling a group of 4: {runs['group']}, a 32-sample chunk: "
          f"{runs['chunk']}; longest run {runs['longest']}")
    if X >= 5:
        assert runs['group'] > 0 and runs['chunk'] > 0 and runs['longest'] > 5


def _ragged_structure(tag, sc, ray_id, step_id, bx0):
    X, S, N = sc.shape[0], sc.S, sc.ro.shape[0]
    n_chunks = -(-S // 32)
    key = ray_id * n_chunks + step_id // 32
    cnt = torch.bincount(key, minlength=N * n_chunks).view(N, n_chunks)
    live_rays = cnt.sum(1) > 0
    zero_chunks = int((cnt[live_rays] == 0).sum())
    one = cnt.view(-1)[key] == 1
    lane31 = int((one & (step_id % 32 == 31)).sum())
    full = int((cnt == 32).sum())
    part = torch.bucketize(bx0.contiguous(), torch.tensor(part_bounds(X, 4), device=DEV), right=True)
    pmin = torch.full((N * n_chunks,), 9, dtype=torch.long, device=DEV).scatter_reduce(0, key, part, 'amin')
    pmax = torch.full((N * n_chunks,), -1, dtype=torch.long, device=DEV).scatter_reduce(0, key, part, 'amax')
    split = int(((pmax > pmin) & (pmax >= 0)).sum())
    empty_rays = int((~live_rays).sum())
    print(f'[coverage] {tag}: ragged chunks: {zero_chunks} empty inside live rays, {int(one.sum())} with one survivor '
          f'({lane31} on lane 31), {full} full; {split} chunks split across 4-way x-ranges; {empty_rays} rays without survivors')
    assert zero_chunks > 0 and int(one.sum()) > 0 and lane31 > 0 and full > 0 and split > 0 and empty_rays > 0


@pytest.mark.gpu
def test_contracted_scatter_accumulates_into_persistent_buffers(selections):
    """Persistent gradient buffers (dist.PeerTail): both scatters add into pre-filled channels-last / contiguous buffers and end
    at prefill + fp64 within TAU * (B + |prefill|), with every element without addends untouched."""
    ops = selections
    sc = Contracted(P=9, shape=C_SHAPE)
    ops.set_feature_kernel(5)
    base = sc.run()
    ray_id, step_id = base['ray_id'], base['step_id']
    M = ray_id.numel()
    x0, f = cells(slab_coords(sc.points(ray_id, step_id), sc.mn, sc.mx, sc.n_freqs), sc.shape)
    gen = torch.Generator(DEV).manual_seed(7)
    g_feat = torch.randn(M, 12, device=DEV, generator=gen)
    g_dens = torch.randn(M, device=DEV, generator=gen)
    want_k, bound_k = ref_scatter(x0, f, g_feat, sc.shape)
    want_d, bound_d = ref_scatter(x0, f, g_dens[:, None], sc.shape)
    kpre = torch.randn(sc.kvals.shape, device=DEV, generator=gen)
    dpre = torch.randn(sc.dgrid.shape, device=DEV, generator=gen)
    for fk, ds in ((5, 1), (3, 0), (0, 1)):
        ops.set_feature_kernel(fk)
        ops.set_density_scatter(ds)
        kbuf, dbuf = channels_last(kpre).clone(), dpre.clone()
        got = sc.run(g_feat, g_dens, dbuf=dbuf, kbuf=kbuf)
        assert got['gk'] is kbuf and got['gd'] is dbuf
        what = f'contracted P=9 {_shape_str(sc.shape)} prefilled buffers fk={fk} ds={ds}'
        judge(as_pxyzc(kbuf), want_k, bound_k, what + ' k0', 'k0 prefilled', base=kpre)
        judge(as_pxyzc(dbuf), want_d, bound_d, what + ' density', 'density prefilled', base=as_pxyzc(dpre))


# ---- box march (DirectVoxGO) ----------------------------------------------------------------------------------------
BOX_LO, BOX_HI = [-1.0, -0.8, -1.1], [1.0, 0.9, 1.2]
BOX_SHAPE = (23, 37, 41)
BOX_SHIFT, BOX_INTERVAL = -2.0, 0.5
RUN_LENGTHS = (31, 32, 33, 64, 65)      # L = ceil(n / 32) = 1, 1, 2, 2, 3


def box_rays(stepdist, g):
    """x-rays starting inside the box with exactly n steps (n in RUN_LENGTHS); rays lying in a face (one sample, on the face)
    and along an edge; rays from the two extreme corners into the box; rays from outside through the box."""
    lo, hi = np.array(BOX_LO, np.float64), np.array(BOX_HI, np.float64)
    o, d = [], []
    for n in RUN_LENGTHS:
        for k in range(8):
            y, z = lo[1:] + (hi[1:] - lo[1:]) * (0.1 + 0.8 * torch.rand(2, generator=g).numpy())
            o.append([hi[0] - (n - 0.5) * stepdist, y, z])
            d.append([1.0, 0.0, 0.0])
    for k in range(8):
        x, z = 0.2 * k - 0.7, 0.13 * k - 0.5
        o.append([x, hi[1], z]); d.append([1.0, 0.0, 0.3])         # in the y = hi face
        o.append([x, lo[1], z]); d.append([-0.5, 0.0, 1.0])        # in the y = lo face
        o.append([x, hi[1], lo[2]]); d.append([1.0, 0.0, 0.0])     # along an edge
    o.append(list(lo)); d.append([1.0, 1.1, 0.9])
    o.append(list(hi)); d.append([-1.0, -0.9, -1.2])
    c = (lo + hi) / 2
    for k in range(64):
        dirn = torch.randn(3, generator=g).numpy()
        o.append(list(c - 3 * dirn / np.linalg.norm(dirn)))
        d.append(list(dirn + 0.3 * torch.randn(3, generator=g).numpy()))
    return torch.tensor(o, dtype=torch.float32, device=DEV), torch.tensor(d, dtype=torch.float32, device=DEV)


BOX = {'C12': dict(C=12, stepdist=0.02), 'C3': dict(C=3, stepdist=0.02),
       'C12-longS': dict(C=12, stepdist=0.0013), 'C3-longS': dict(C=3, stepdist=0.0013)}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(BOX))
def test_box_scatter_vs_fp64(case, selections):
    """BoxMarch: k0 scatter (C = 12 all red.v4, C = 3 red.v2 + scalar by address) and the density scatter through raw_alpha under
    both density scatters, with rays of different n_steps in one launch, on either side of the run scatter's limit."""
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import march, ops as O
    ops = selections
    C, sd = BOX[case]['C'], BOX[case]['stepdist']
    X, Y, Z = BOX_SHAPE
    g = _gen(C + int(1e4 * sd))
    dgrid = torch.randn(1, 1, X, Y, Z, generator=g).to(DEV)
    kvals = torch.randn(1, X, Y, Z, C, generator=g).to(DEV)
    ro, rd = box_rays(sd, g)
    cfg = march.make_box_cfg(BOX_LO, BOX_HI, 0.0, sd, BOX_SHIFT, BOX_INTERVAL, 0.0, None, None, None)
    S = cfg.s_max
    side = 'run scatter' if run_smem_ok(S) else 'per-sample fallback'
    assert run_smem_ok(S) == (not case.endswith('longS'))
    ddesc = G.grid_desc(dgrid, BOX_LO, BOX_HI, 0)
    kdesc = G.grid_desc(channels_last(kvals), BOX_LO, BOX_HI, 0)

    def run(g_feat=None, g_alpha=None):
        dg = dgrid.clone().requires_grad_(True)
        kg = channels_last(kvals).clone().requires_grad_(True)
        _, _, alpha, feat, rid, sid = march.BoxMarch.apply(dg, kg, ro, rd, None, cfg, ddesc, kdesc)
        if g_feat is not None:
            ((feat * g_feat).sum() + (alpha * g_alpha).sum()).backward()
        return feat.detach(), rid, sid, kg.grad, dg.grad

    feat0, ray_id, step_id, _, _ = run()
    M = ray_id.numel()
    lo_t, hi_t = torch.tensor(BOX_LO, device=DEV), torch.tensor(BOX_HI, device=DEV)
    pts, _, rid_all, _, n_steps = O.sample_pts_on_rays(ro, rd, lo_t, hi_t, 0.0, 1e9, np.float32(sd))[:5]
    p = pts[(torch.cumsum(n_steps, 0) - n_steps)[ray_id] + step_id]
    x0, f = cells(slab_coords(p, BOX_LO, BOX_HI, 0), BOX_SHAPE)
    # structure: every run length, and samples on faces, edges and corners of the grid
    per_ray = torch.bincount(ray_id, minlength=ro.shape[0])
    lens = set(per_ray.tolist())
    at = ((x0[0] == torch.tensor([X - 2, Y - 2, Z - 2], device=DEV)) & (f[0] == 1)) | ((x0[0] == 0) & (f[0] == 0))
    on = at.sum(1)
    faces = [int((on == k).sum()) for k in (1, 2, 3)]
    tag = f'box C={C} {_shape_str(BOX_SHAPE)} S_max={S}'
    print(f'[coverage] {tag}: {M} survivors; n_steps {sorted(set(n_steps.tolist()) & set(RUN_LENGTHS))} present; samples on '
          f'1 / 2 / 3 faces: {faces}; density scatter mode 1 -> {side}')
    assert set(RUN_LENGTHS) <= lens, f'{tag}: rays of {sorted(set(RUN_LENGTHS) - lens)} survivors missing'
    assert min(faces) > 0, f'{tag}: face / edge / corner samples {faces}'
    if C == 3:
        am = torch.bincount((x0[0, :, 0] * Y + x0[0, :, 1]) * Z + x0[0, :, 2], minlength=1)
        vv = torch.arange(am.numel(), device=DEV)[am > 0]
        mods = sorted(set(((vv * C) % 4).tolist()))
        print(f'[coverage] {tag}: (v * C) mod 4 of the base records: {mods}')
        assert mods == [0, 1, 2, 3]
    gen = torch.Generator(DEV).manual_seed(M)
    g_feat = torch.randn(M, C, device=DEV, generator=gen)
    g_alpha = torch.randn(M, device=DEV, generator=gen)
    raw = F.grid_sample(dgrid, (((p - lo_t) / (hi_t - lo_t)).flip((-1,)) * 2 - 1).reshape(1, 1, 1, -1, 3), mode='bilinear',
                        align_corners=True).reshape(-1)
    gd = raw2alpha_grad(raw, cfg.act_shift, cfg.interval, g_alpha)
    want_k, bound_k = ref_scatter(x0, f, g_feat, BOX_SHAPE)
    want_d, bound_d = ref_scatter(x0, f, gd[:, None], BOX_SHAPE)
    fw, fb = ref_gather(x0, f, kvals)
    dw, db = ref_gather(x0, f, as_pxyzc(dgrid))
    judge(feat0[:, :, None], fw[:, :, None], fb[:, :, None], tag + ' k0 forward self-check', 'forward self-check', tau=TAU_FWD)
    judge(raw[:, None, None], dw[:, :, None], db[:, :, None], tag + ' density (grid_sample) self-check', 'forward self-check',
          tau=TAU_FWD)
    fails = []
    for ds in (1, 0):
        ops.set_density_scatter(ds)
        _, rid, sid, gk, gdg = run(g_feat, g_alpha)
        try:
            assert torch.equal(rid, ray_id) and torch.equal(sid, step_id)
            judge(as_pxyzc(gk), want_k, bound_k, f'{tag} ds={ds} k0 scatter', f'box k0 C={C}')
            judge(as_pxyzc(gdg), want_d, bound_d, f'{tag} ds={ds} density scatter', f'box density ds={ds}')
        except AssertionError as e:
            fails.append(str(e))
    assert not fails, '\n'.join(fails)


# ---- NDC march (DirectMPIGO) ----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('C', [9, 3])
def test_ndc_scatter_vs_fp64(C, selections):
    """NdcMarch: the k0 scatter of 36- / 12-byte records (red.v4 / v2 / scalar chosen per corner from the address) and the
    density scatter through raw_alpha under both density scatters."""
    from tests.test_gpu_mpi import _ndc_scene
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import march, ops as O
    from oracle.cpu_ref import dense_grid_forward
    ops = selections
    m, ro, rd, _ = _ndc_scene(C)
    S = m._n_samples(0.5)
    lo, hi = m._host()
    cfg = march.make_ndc_cfg(lo, hi, S, 0.5 * m.voxel_size_ratio, 1e-3, m.mask_cache.mask, *m._mask_geometry())
    descs = [G.grid_desc(gr.grid, *gr._bounds(), 0) for gr in (m.density, m.k0, m.act_shift)]
    shape = tuple(m.density.grid.shape[2:])
    assert tuple(m.k0.grid.shape[2:]) == shape

    def run(g_feat=None, g_alpha=None):
        dg = m.density.grid.detach().clone().requires_grad_(True)
        kg = m.k0.grid.detach().clone().requires_grad_(True)
        _, _, alpha, feat, rid, sid = march.NdcMarch.apply(dg, kg, m.act_shift.grid, ro, rd, m.mask_cache.mask, cfg, *descs)
        if g_feat is not None:
            ((feat * g_feat).sum() + (alpha * g_alpha).sum()).backward()
        return feat.detach(), rid, sid, kg.grad, dg.grad

    feat0, ray_id, step_id, _, _ = run()
    M = ray_id.numel()
    assert M > 10000
    p = O.sample_ndc_pts_on_rays(ro, rd, m.xyz_min, m.xyz_max, S)[0][ray_id, step_id]
    dmn, dmx = m.density._bounds()
    kmn, kmx = m.k0._bounds()
    assert (dmn, dmx) == (kmn, kmx)
    x0, f = cells(slab_coords(p, kmn, kmx, 0), shape)
    X, Y, Z = shape
    vv = torch.unique((x0[0, :, 0] * Y + x0[0, :, 1]) * Z + x0[0, :, 2])
    mods = sorted(set(((vv * C) % 4).tolist()))
    tag = f'ndc C={C} {_shape_str(shape)} S={S}'
    print(f'[coverage] {tag}: {M} survivors; (v * C) mod 4 of the base records: {mods}; density scatter mode 1 -> '
          f'{"run scatter" if run_smem_ok(S) else "per-sample fallback"}')
    assert mods == [0, 1, 2, 3]
    gen = torch.Generator(DEV).manual_seed(M)
    g_feat = torch.randn(M, C, device=DEV, generator=gen)
    g_alpha = torch.randn(M, device=DEV, generator=gen)
    with torch.no_grad():
        raw = dense_grid_forward(m.density.grid, p, m.density.xyz_min, m.density.xyz_max) + \
            dense_grid_forward(m.act_shift.grid, p, m.act_shift.xyz_min, m.act_shift.xyz_max)
    gd = raw2alpha_grad(raw, 0.0, cfg.interval, g_alpha)
    want_k, bound_k = ref_scatter(x0, f, g_feat, shape)
    want_d, bound_d = ref_scatter(x0, f, gd[:, None], shape)
    fw, fb = ref_gather(x0, f, as_pxyzc(m.k0.grid.detach()))
    judge(feat0[:, :, None], fw[:, :, None], fb[:, :, None], tag + ' k0 forward self-check', 'forward self-check', tau=TAU_FWD)
    fails = []
    for ds in (1, 0):
        ops.set_density_scatter(ds)
        _, rid, sid, gk, gdg = run(g_feat, g_alpha)
        try:
            assert torch.equal(rid, ray_id) and torch.equal(sid, step_id)
            judge(as_pxyzc(gk), want_k, bound_k, f'{tag} ds={ds} k0 scatter', f'ndc k0 C={C}')
            judge(as_pxyzc(gdg), want_d, bound_d, f'{tag} ds={ds} density scatter', f'ndc density ds={ds}')
        except AssertionError as e:
            fails.append(str(e))
    assert not fails, '\n'.join(fails)


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    if WORST:
        print('\n[march-scatter] worst |got - want| / B: ' + ', '.join(f'{k} {v:.2e}' for k, v in sorted(WORST.items())))


# ---- CPU: the check is tight enough to see one misplaced sample ---------------------------------------------------------
def fp32_addends(x0, f, g, shape):
    """The scatter restated in the kernels' fp32 arithmetic: per (slab, corner, sample) the flat index and the addend
    (((wz * wy) * wx) / P) * g, with 1 / P as the fp32 reciprocal.  Returns (index, value, slab, sample) rows."""
    P, M = x0.shape[:2]
    X, Y, Z = shape
    rcp = torch.tensor(1.0, dtype=torch.float32) / P if P > 1 else torch.tensor(1.0)
    rows = []
    for s in range(P):
        fs = f[s]
        for corner in range(8):
            bx, by, bz = corner >> 2, (corner >> 1) & 1, corner & 1
            w = ((fs[:, 2] if bz else 1 - fs[:, 2]) * (fs[:, 1] if by else 1 - fs[:, 1])) * (fs[:, 0] if bx else 1 - fs[:, 0])
            idx = s * X * Y * Z + ((x0[s, :, 0] + bx) * Y + x0[s, :, 1] + by) * Z + x0[s, :, 2] + bz
            rows.append((idx, (w * rcp)[:, None] * g, torch.full((M,), s), torch.arange(M)))
    return [torch.cat(c) for c in zip(*rows)]


def accumulate(idx, val, P, shape):
    out = torch.zeros(P * int(np.prod(shape)), val.shape[1], dtype=torch.float32)
    out.index_add_(0, idx, val)
    return out.view(P, *shape, val.shape[1])


def test_checker_rejects_faults():
    """On a small CPU scene (P = 5, 7 x 9 x 11, 4 channels): the fp32 restatement of the scatter passes at TAU; one sample's
    contribution moved to the neighbouring x cell, one sample dropped, one sample added twice, one sample's sin- and cos-slab
    contributions swapped, and all samples whose slab-0 cell starts on an x-range boundary plane dropped each fail."""
    P, shape, C = 5, (7, 9, 11), 4
    X, Y, Z = shape
    g = _gen(3)
    pts = []
    for k in range(24):                        # rays along x at fixed (y, z), 5 samples per voxel, plus random points
        yz = (torch.rand(2, generator=g) * 2 - 1) * 0.9
        xs = torch.linspace(-0.98, 0.98, 5 * (X - 1))
        pts.append(torch.cat([xs[:, None], yz.expand(xs.numel(), 2)], 1))
    pts.append((torch.rand(400, 3, generator=g) * 2 - 1) * 0.99)
    pts = torch.cat(pts)
    M = pts.shape[0]
    x0, f = cells(slab_coords(pts, [-1.] * 3, [1.] * 3, (P - 1) // 2), shape)
    gr = torch.randn(M, C, generator=g)
    want, bound = ref_scatter(x0, f, gr, shape)
    idx, val, slab, smp = fp32_addends(x0, f, gr, shape)
    honest, stray = ratio(accumulate(idx, val, P, shape), want, bound)
    assert stray == 0 and honest <= TAU / 10, f'fp32 restatement: {honest:.2e} of B, {stray} stray writes'
    # the sample farthest inside its cells over all slabs and axes (no tiny corner weight), not on the last x cell of slab 0
    depth = torch.minimum(f, 1 - f).amin(2).amin(0) * (x0[0, :, 0] < X - 2)
    i = int(depth.argmax())
    assert float(depth[i]) > 0.05
    mine = smp == i
    faults = {}
    moved = idx.clone()
    moved[mine & (slab == 0)] += Y * Z
    faults['moved to the next x cell'] = (moved, val)
    faults['dropped'] = (idx[~mine], val[~mine])
    faults['added twice'] = (torch.cat([idx, idx[mine]]), torch.cat([val, val[mine]]))
    sw = idx.clone()
    XYZ = X * Y * Z
    sw[mine & (slab == 1)] += XYZ
    sw[mine & (slab == 2)] -= XYZ
    faults['sin / cos slabs swapped'] = (sw, val)
    b = part_bounds(X, 4)[1]
    plane = torch.cat([(x0[s, :, 0] == b) for s in range(P)]).view(P, M)[slab, smp] & (slab == 0)
    assert int(plane.sum()) > 0
    faults[f'slab-0 samples on boundary plane {b} dropped'] = (idx[~plane], val[~plane])
    margins = {}
    for name, (fi, fv) in faults.items():
        r, stray = ratio(accumulate(fi, fv, P, shape), want, bound)
        margins[name] = r / TAU
        assert r > 10 * TAU or stray > 0, f'{name}: only {r:.2e} of B'
    print(f'[march-scatter checker] fp32 restatement {honest:.2e} of B; fault / TAU: '
          + ', '.join(f'{k} {v:.1f}' for k, v in margins.items()) + f'; smallest {min(margins.values()):.1f}')
