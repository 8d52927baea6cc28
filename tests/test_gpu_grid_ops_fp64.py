"""The stand-alone grid read and its adjoint (csrc/trilinear.cu: ubn_grid_sample_fwd / _bwd behind grid.grid_sample) and the
grid-maintenance kernels (csrc/grid_utils.cu) against plain fp64 restatements, element by element.

Read and adjoint.  The yardstick is test_gpu_march_scatter's: every point's cells come from the reference's fp32 normalisation,
Fourier embedding and ATen's unnormalisation on the GPU; only the eight corner weights and the sums are fp64.  Points may lie
anywhere, so the cells are taken on the grid padded by one zero voxel per side (padded_cells): a corner outside the grid lands in
the padding and is dropped, which is what padding_mode='zeros' does, and a point with no corner inside -- far outside, or with a
NaN / inf coordinate, whose source index ATen's grid sampler replaces by -100 -- adds nothing.  Each gradient element must lie
within TAU = 1e-5 of its own bound B = sum |w| * |g| / P (elements without addends exactly 0.0 or exactly the prefill), each
forward value within TAU_FWD of the fp64 gather's bound, and the C = 1 read -- ATen's corner order and torch-CUDA's slab-mean
order (trilinear.cuh: trilerp1, SlabMean) -- must equal F.grid_sample(...).mean(0) on the GPU bit for bit.  The cases cover the
three kernels (k_grid_*_c1, k_grid_*_generic, k_grid_coop) at P = 1 .. 17, with the kernel each case takes asserted from the
dispatch conditions (route): the coop grid-stride wrap at 135 169 points and several trips at 10^6, the fallbacks at P = 17 and
for an output or upstream gradient one float off 16-byte alignment, odd non-cubic grids with a dimension of 2, and points on
lattice nodes, faces, edges and corners, one ulp inside and outside the box, at +-1e6, and inside and outside in one warp group.

Maintenance.  Each kernel's float part is held to fp64 and each discrete decision is then required to be exact wherever fp64
says it cannot go either way:
  * ubn_lattice_alpha: bit for bit Raw2Alpha of the C = 1 read at torch.linspace's lattice on the GPU, and within
    alpha_bound of 1 - (1 + e^(d64 + shift))^-interval, d64 the fp64 gather;
  * ubn_maxpool3_gt_and: exactly F.max_pool3d(alpha, 3, 1, 1) > thres AND the prior mask, NaN windows and ties included;
  * update_occupancy_cache: every cell outside the band the alpha bound leaves around fast_color_thres is exact;
  * ubn_view_scatter_ones: each view's buffer within TAU of the fp64 adjoint of the reference's fp32 sample points, counts
    exact outside the +-TAU * B band around 1;
  * ubn_maskout_near_cam(_lattice): exact wherever the fp64 distance is outside 8 u of near_clip;
  * ubn_resample_grid: within RESAMPLE_U u of the fp64 trilinear resample, and equal to F.interpolate where the blend is short.
test_checker_rejects_faults (CPU) shows the judges reject a moved, dropped or doubled addend, a missing 1/P, a dropped corner on
the last x face, a max-pool window without its z+1 plane and a window that drops its NaN."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_march_scatter import (TAU, TAU_FWD, accumulate, as_pxyzc, cells, channels_last, fp32_addends, judge,
                                          ratio, ref_gather, ref_scatter, slab_coords)
from tests.test_gpu_march_transmittance import U, c_alpha

DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
COOP_WARPS, MAX_SLABS, NUM_SMS = 4, 16, 132      # kCoopWarps, kMaxSlabs (trilinear.cu), kNumSMs (common.cuh)
MN, MX = [-1.3, -0.7, -2.1], [0.9, 1.6, 0.4]      # a non-cubic box; the kernels and torch both see its float32 rounding
WORST = {}
BANDS = {}


def check(got, want, bound, what, key, base=None, tau=TAU):
    r, _ = ratio(got, want, bound, base)
    WORST[key] = max(WORST.get(key, 0.0), r)
    judge(got, want, bound, what, key, base, tau)


def _seed(name):
    return sum(ord(c) * (i + 1) for i, c in enumerate(name)) % (2 ** 31)


# ---- fp64 reference for points anywhere -------------------------------------------------------------------------------------
def padded_cells(coords, shape):
    """(x0, f) of cells() on the grid padded by one voxel per side: x0 = floor(c) + 1 in padded indices, f = c - floor(c).  A
    point-slab with no corner inside the grid (floor(c) outside [-1, size - 1] on an axis, NaN or inf) gets x0 = 0, f = 0: its
    weight lands on the padding corner (0, 0, 0), i.e. nowhere."""
    x0, f = cells(coords, shape)
    c = x0.float() + f                      # cells()' unnormalised coordinate, recovered exactly
    fl = torch.floor(c)
    hi = torch.tensor(shape, dtype=torch.float32, device=c.device) - 1
    live = ((fl >= -1) & (fl <= hi)).all(-1, keepdim=True)
    return torch.where(live, fl + 1, 0).long(), torch.where(live, c - fl, 0)


def pad(vals):
    """[P, X, Y, Z, C] -> the same with a border of zero voxels."""
    P, X, Y, Z, C = vals.shape
    out = torch.zeros(P, X + 2, Y + 2, Z + 2, C, dtype=vals.dtype, device=vals.device)
    out[:, 1:-1, 1:-1, 1:-1] = vals
    return out


def crop(t):
    return t[:, 1:-1, 1:-1, 1:-1]


def fp64_read(pts, vals, mn, mx, n_freqs):
    """fp64 gather (value, bound) [M, C] of vals [P, X, Y, Z, C] at world points pts [M, 3]."""
    x0, f = padded_cells(slab_coords(pts, mn, mx, n_freqs), tuple(vals.shape[1:4]))
    return ref_gather(x0, f, pad(vals))


def fp64_adjoint(pts, g, shape, P, mn, mx, n_freqs):
    """fp64 adjoint (want, bound) [P, X, Y, Z, C] of the read at pts for upstream g [M, C]."""
    x0, f = padded_cells(slab_coords(pts, mn, mx, n_freqs), shape)
    assert x0.shape[0] == P
    want, bound = ref_scatter(x0, f, g, tuple(s + 2 for s in shape))
    return crop(want), crop(bound)


# ---- the kernel a call takes --------------------------------------------------------------------------------------------
def route(desc, grid_ptr, io_ptr):
    """The kernel ubn_grid_sample_fwd / _bwd launches for this descriptor, grid (or gradient) address and output (or upstream
    gradient) address: trilinear.cu's dispatch and coop_ok, restated."""
    if desc.C == 1:
        return 'c1'
    coop = (desc.stride_c == 1 and desc.stride_v == desc.C and desc.C in (4, 8, 12, 16) and desc.P <= MAX_SLABS
            and grid_ptr % 16 == 0 and io_ptr % 16 == 0 and desc.stride_p % 4 == 0)
    return 'coop' if coop else 'generic'


def coop_trips(n):
    """Trips the busiest warp of k_grid_coop makes around its grid-stride loop over the ceil(n / 32) point groups."""
    groups = -(-n // 32)
    blocks = min(-(-groups // COOP_WARPS), NUM_SMS * 8)
    return -(-groups // (blocks * COOP_WARPS))


def test_launch_constants_match_sources():
    """route() and coop_trips() restate constants of the CUDA sources; they must stay in step with them."""
    tri = open(os.path.join(CSRC, 'trilinear.cu')).read()
    com = open(os.path.join(CSRC, 'common.cuh')).read()
    assert int(re.search(r'constexpr int kCoopWarps = (\d+);', tri).group(1)) == COOP_WARPS
    assert int(re.search(r'constexpr int kMaxSlabs = (\d+);', tri).group(1)) == MAX_SLABS
    assert int(re.search(r'constexpr int kNumSMs = (\d+);', com).group(1)) == NUM_SMS
    assert tri.count('(int64_t)kNumSMs * 8') == 2
    assert coop_trips(135_168) == 1 and coop_trips(135_169) == 2 and coop_trips(1_000_000) == 8


def _abi(name, *args):
    from unboundednerfpytorch_b200 import ops
    from unboundednerfpytorch_b200._cabi import check as abi_check
    with ops._Guard(args[0]) as lib:
        abi_check(getattr(lib, name)(*args[1:]))


def abi_read(grid, desc, pts, out):
    """ubn_grid_sample_fwd into any fp32 buffer `out` (e.g. one float off alignment)."""
    from unboundednerfpytorch_b200._cabi import c_i64, ptr, stream_of
    _abi('ubn_grid_sample_fwd', grid, ptr(grid), desc, ptr(pts), c_i64(pts.shape[0]), ptr(out), stream_of(grid))


def abi_adjoint(grad_out, desc, pts, grad_grid):
    """ubn_grid_sample_bwd: adds the adjoint of grad_out into grad_grid as it is."""
    from unboundednerfpytorch_b200._cabi import c_i64, ptr, stream_of
    _abi('ubn_grid_sample_bwd', grad_grid, ptr(grad_out), desc, ptr(pts), c_i64(pts.shape[0]), ptr(grad_grid),
         stream_of(grad_grid))


# ---- point sets ------------------------------------------------------------------------------------------------------------
def box_points(n, shape, gen, mn=MN, mx=MX):
    """n fp32 world points, shuffled: lattice nodes (the linspace lattice) and the 8 box corners; points on 1 and 2 box faces;
    one ulp inside and outside a face and outside a corner; within one voxel outside a face; +-1e6 on one and on all axes; the
    rest uniform over the box grown by 10 % per side."""
    mn32 = torch.tensor(mn, dtype=torch.float32)
    mx32 = torch.tensor(mx, dtype=torch.float32)
    span = mx32 - mn32

    def inside(k):
        return mn32 + torch.rand(k, 3, generator=gen) * span

    parts = []
    lin = [torch.linspace(float(mn32[a]), float(mx32[a]), shape[a]) for a in range(3)]
    idx = [torch.randint(0, shape[a], (512,), generator=gen) for a in range(3)]
    parts.append(torch.stack([lin[a][idx[a]] for a in range(3)], 1))
    parts.append(torch.tensor([[float((mx32 if (c >> a) & 1 else mn32)[a]) for a in range(3)] for c in range(8)]))
    inf = torch.tensor(float('inf'))
    for k_faces in (1, 2):
        for rep in range(64):
            p = inside(8)
            axes = torch.randperm(3, generator=gen)[:k_faces]
            for j in range(8):
                for a in axes.tolist():
                    p[j, a] = (mx32 if (j >> a) & 1 else mn32)[a]
            parts.append(p)
    for a in range(3):
        for side, toward in ((mn32, -inf), (mn32, inf), (mx32, inf), (mx32, -inf)):
            p = inside(16)
            p[:, a] = torch.nextafter(side[a], toward)
            parts.append(p)
        p = inside(32)
        vox = span[a] / (shape[a] - 1)
        p[:16, a] = mn32[a] - torch.rand(16, generator=gen) * vox
        p[16:, a] = mx32[a] + torch.rand(16, generator=gen) * vox
        parts.append(p)
    parts.append(torch.stack([torch.nextafter(mn32, -inf), torch.nextafter(mx32, inf)]))
    for a in range(3):
        p = inside(8)
        p[:4, a], p[4:, a] = 1e6, -1e6
        parts.append(p)
    parts.append(torch.tensor([[1e6] * 3, [-1e6] * 3, [1e6, -1e6, 1e6]]))
    special = torch.cat(parts)
    fill = max(n - special.shape[0], 0)
    rest = mn32 - 0.1 * span + torch.rand(fill, 3, generator=gen) * 1.2 * span
    pts = torch.cat([special, rest])
    return pts[torch.randperm(pts.shape[0], generator=gen)[:n]].contiguous()


def placement(pts, shape):
    """Counts of the structural point classes (slab-0 source indices, as the kernels see them)."""
    x0, f = cells(slab_coords(pts, MN, MX, 0), shape)
    c = (x0.float() + f)[0]
    hi = torch.tensor(shape, dtype=torch.float32, device=c.device) - 1
    inb = ((c >= 0) & (c <= hi)).all(1)
    node = inb & (c == torch.floor(c)).all(1)
    faces = ((c == 0) | (c == hi)).sum(1) * inb
    fl = torch.floor(c)
    part = ~inb & ((fl >= -1) & (fl <= hi)).all(1)
    out = ~inb & ~part
    n = pts.shape[0]
    grp = torch.arange(n, device=c.device) // 32
    mixed = 0
    if n >= 32:
        has_in = torch.zeros(int(grp.max()) + 1, dtype=torch.bool, device=c.device).index_fill_(0, grp[inb], True)
        has_out = torch.zeros_like(has_in).index_fill_(0, grp[out], True)
        mixed = int((has_in & has_out).sum())
    return dict(node=int(node.sum()), face=int((faces == 1).sum()), edge=int((faces == 2).sum()),
                corner=int((faces == 3).sum()), partial=int(part.sum()), outside=int(out.sum()), mixed_groups=mixed)


def upstream(n, C, gen):
    """Seeded upstream gradient with 10 % zero entries and 5 % zero rows."""
    g = torch.randn(n, C, generator=gen)
    g[torch.rand(n, C, generator=gen) < 0.1] = 0
    g[torch.rand(n, generator=gen) < 0.05] = 0
    return g


# ---- read and adjoint ---------------------------------------------------------------------------------------------------
S_A, S_B, S_C, S_D, S_BIG = (23, 2, 17), (7, 13, 5), (2, 9, 31), (11, 19, 3), (41, 23, 37)
READS = {
    'c1-P1-cl': dict(C=1, P=1, layout='cl', shape=S_A, n=50_000, route='c1'),
    'c1-P1-ref': dict(C=1, P=1, layout='ref', shape=S_B, n=4099, route='c1', prefill=True),
    'c1-P9-ref': dict(C=1, P=9, layout='ref', shape=S_C, n=20_000, route='c1'),
    'c1-P17-cl': dict(C=1, P=17, layout='cl', shape=S_D, n=9000, route='c1', prefill=True),
    'generic-C3-P5-cl': dict(C=3, P=5, layout='cl', shape=S_A, n=30_000, route='generic'),
    'generic-C3-P1-ref': dict(C=3, P=1, layout='ref', shape=S_B, n=7000, route='generic'),
    'generic-C12-P7-ref': dict(C=12, P=7, layout='ref', shape=S_C, n=20_000, route='generic', prefill=True),
    'generic-C12-P17-cl': dict(C=12, P=17, layout='cl', shape=S_B, n=20_000, route='generic'),
    'C8-P11-cl-unaligned-out': dict(C=8, P=11, layout='cl', shape=S_D, n=5000, route='generic', bwd_route='coop',
                                    unaligned_out=True),
    'C16-P3-cl-unaligned-gout': dict(C=16, P=3, layout='cl', shape=S_A, n=5000, route='coop', trips=1, bwd_route='generic',
                                     unaligned_gout=True, prefill=True),
    'coop-C4-P1': dict(C=4, P=1, layout='cl', shape=S_A, n=135_167, route='coop', trips=1),
    'coop-C8-P3': dict(C=8, P=3, layout='cl', shape=S_B, n=135_168, route='coop', trips=1),
    'coop-C12-P15': dict(C=12, P=15, layout='cl', shape=S_C, n=135_169, route='coop', trips=2),
    'coop-C16-P9': dict(C=16, P=9, layout='cl', shape=S_D, n=135_169, route='coop', trips=2, prefill=True),
    'coop-C12-P9-1M': dict(C=12, P=9, layout='cl', shape=S_BIG, n=1_000_000, route='coop', trips=8),
}
for _n in (1, 31, 32, 33):
    READS[f'c1-P3-n{_n}'] = dict(C=1, P=3, layout='ref', shape=S_B, n=_n, route='c1')
    READS[f'coop-C12-P5-n{_n}'] = dict(C=12, P=5, layout='cl', shape=S_A, n=_n, route='coop', trips=1)
    READS[f'generic-C3-P7-n{_n}'] = dict(C=3, P=7, layout='ref', shape=S_D, n=_n, route='generic')


def make_grid(vals, layout):
    """[P, X, Y, Z, C] values -> a [P, C, X, Y, Z] tensor, channels-last ('cl') or contiguous ('ref')."""
    return channels_last(vals) if layout == 'cl' else vals.permute(0, 4, 1, 2, 3).contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(READS))
def test_grid_read_and_adjoint_vs_fp64(case, oracle):
    from unboundednerfpytorch_b200 import grid as G
    spec = READS[case]
    C, P, shape, n = spec['C'], spec['P'], spec['shape'], spec['n']
    nf = (P - 1) // 2
    gen = torch.Generator().manual_seed(_seed(case))
    vals = torch.randn(P, *shape, C, generator=gen).to(DEV)
    grid = make_grid(vals, spec['layout'])
    pts = box_points(n, shape, gen).to(DEV)
    g = upstream(n, C, gen).to(DEV)
    pre = torch.randn(vals.shape, generator=gen).to(DEV) if spec.get('prefill') else None
    desc = G.grid_desc(grid, MN, MX, nf)
    tag = f'{case} ({"x".join(map(str, shape))}, {n} points)'

    # forward: through grid.grid_sample, or into an output one float off 16-byte alignment through the C ABI
    gg = grid.clone().requires_grad_(True)
    if spec.get('unaligned_out'):
        buf = torch.full((n * C + 4,), float('nan'), device=DEV)
        out = buf[1:1 + n * C].view(n, C)
        abi_read(grid, desc, pts, out)
        assert out.data_ptr() % 16 == 4
        assert torch.isnan(buf[0]) and torch.isnan(buf[1 + n * C:]).all(), f'{tag}: write outside the output'
    else:
        if pre is not None:
            gg.grad = make_grid(pre, spec['layout']).clone()
        out = G.grid_sample(gg, pts, MN, MX, nf)
        assert out.shape == ((n,) if C == 1 else (n, C))
    got_route = route(desc, gg.data_ptr(), out.data_ptr())
    assert got_route == spec['route'], f'{tag}: takes {got_route}'
    if got_route == 'coop':
        assert coop_trips(n) == spec['trips']
    cov = placement(pts, shape)
    print(f'[coverage] {tag}: route {got_route}' + (f', {coop_trips(n)} grid-stride trips' if got_route == 'coop' else '')
          + f'; points {cov}; {int((g == 0).all(1).sum())} zero upstream rows')
    if n >= 4096:
        assert min(cov.values()) > 0, f'{tag}: a point class is missing: {cov}'

    fw, fb = fp64_read(pts, vals, MN, MX, nf)
    check(out.reshape(n, C), fw, fb, f'{tag} read', 'read', tau=TAU_FWD)
    if C == 1:      # ATen's corner order and torch-CUDA's slab mean: F.grid_sample(...).mean(0) on the GPU, bit for bit
        want = oracle.fourier_grid_forward(grid.detach(), pts, torch.tensor(MN, device=DEV), torch.tensor(MX, device=DEV), nf)
        diff = int((out.reshape(-1) != want.reshape(-1)).sum())
        assert diff == 0, f'{tag}: {diff} of {n} values differ from F.grid_sample on the GPU'

    # adjoint: through autograd (into a prefilled .grad where the case has one), or through the C ABI for the unaligned cases
    want, bound = fp64_adjoint(pts, g, shape, P, MN, MX, nf)
    bwd_route = spec.get('bwd_route', spec['route'])
    what = f'{tag} adjoint' + (' into a prefilled gradient' if pre is not None else '')
    if spec.get('unaligned_out') or spec.get('unaligned_gout'):
        gout = g
        if spec.get('unaligned_gout'):
            gout = torch.empty(n * C + 4, device=DEV)[1:1 + n * C].view(n, C).copy_(g)
            assert gout.data_ptr() % 16 == 4
        gsum = make_grid(pre, spec['layout']).clone() if pre is not None else torch.zeros_like(grid)
        assert route(desc, gsum.data_ptr(), gout.data_ptr()) == bwd_route
        abi_adjoint(gout, desc, pts, gsum)
    else:
        out.backward(g.view_as(out))
        gsum = gg.grad
        assert gsum.stride() == grid.stride()
        assert route(desc, gsum.data_ptr(), g.data_ptr()) == bwd_route
    check(as_pxyzc(gsum), want, bound, what, f'adjoint {bwd_route}', base=pre)
    if pre is not None and not spec.get('unaligned_gout'):     # the kernel itself adds into a prefilled buffer
        gsum = make_grid(pre, spec['layout']).clone()
        abi_adjoint(g, desc, pts, gsum)
        check(as_pxyzc(gsum), want, bound, f'{tag} adjoint added by the kernel into a prefilled buffer', f'adjoint {bwd_route}',
              base=pre)


NONFINITE = {
    'c1-P1': dict(C=1, P=1, layout='cl'),
    'c1-P5': dict(C=1, P=5, layout='ref'),
    'generic-C3-P1': dict(C=3, P=1, layout='cl'),
    'generic-C12-P3-ref': dict(C=12, P=3, layout='ref'),
    'coop-C12-P3': dict(C=12, P=3, layout='cl'),
    'coop-C4-P9': dict(C=4, P=9, layout='cl'),
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(NONFINITE))
def test_nonfinite_coordinates_match_torch(case, oracle):
    """A NaN, +inf or -inf in one coordinate (each axis, each value, in warp groups with finite points, with zero and nonzero
    upstream gradients): the read and the grid gradient equal torch-CUDA's F.grid_sample -- whose grid sampler replaces a
    non-finite source index by -100, so such a point reads 0 and scatters nothing -- NaN for NaN, and both are judged
    against the fp64 reference."""
    from unboundednerfpytorch_b200 import grid as G
    spec = NONFINITE[case]
    C, P, shape = spec['C'], spec['P'], S_B
    nf = (P - 1) // 2
    gen = torch.Generator().manual_seed(_seed(case))
    vals = torch.randn(P, *shape, C, generator=gen).to(DEV)
    grid = make_grid(vals, spec['layout'])
    n = 2048
    pts = box_points(n, shape, gen)
    bad = torch.zeros(n, dtype=torch.bool)
    rows = torch.randperm(n, generator=gen)[:36]
    for k, r in enumerate(rows.tolist()):
        pts[r, k % 3] = (float('nan'), float('inf'), -float('inf'))[(k // 3) % 3]
        bad[r] = True
    g = upstream(n, C, gen)
    g[rows[::2]] = 0                            # half of the non-finite rows have a zero upstream gradient
    pts, g, bad = pts.to(DEV), g.to(DEV), bad.to(DEV)

    gg = grid.clone().requires_grad_(True)
    out = G.grid_sample(gg, pts, MN, MX, nf).reshape(n, C)
    out.backward(g)
    tg = vals.permute(0, 4, 1, 2, 3).contiguous().requires_grad_(True)
    tout = oracle.fourier_grid_forward(tg, pts, torch.tensor(MN, device=DEV), torch.tensor(MX, device=DEV), nf).reshape(n, C)
    tout.backward(g)
    tag = f'non-finite {case}'
    print(f'[coverage] {tag}: route {route(G.grid_desc(grid, MN, MX, nf), gg.data_ptr(), out.data_ptr())}; {int(bad.sum())} '
          f'non-finite points; torch reads {int(torch.isnan(tout).sum())} NaN values, its gradient holds '
          f'{int(torch.isnan(tg.grad).sum())} NaN')
    assert torch.equal(torch.isnan(out), torch.isnan(tout)), f'{tag}: NaN reads differ from torch'
    assert torch.equal(torch.isnan(gg.grad), torch.isnan(tg.grad)), f'{tag}: NaN gradient elements differ from torch'
    assert torch.equal(out[bad], tout[bad]), f'{tag}: reads at non-finite points differ from torch'
    if C == 1:
        assert torch.equal(out, tout), f'{tag}: reads differ from torch bit for bit'
    fw, fb = fp64_read(pts, vals, MN, MX, nf)
    check(out, fw, fb, f'{tag} read', 'read', tau=TAU_FWD)
    want, bound = fp64_adjoint(pts, g, shape, P, MN, MX, nf)
    check(as_pxyzc(gg.grad), want, bound, f'{tag} adjoint', 'adjoint non-finite')
    check(as_pxyzc(tg.grad), want, bound, f'{tag} torch F.grid_sample adjoint (yardstick self-check)', 'torch adjoint')


# ---- maintenance: lattice alpha, max-pool mask, occupancy update ------------------------------------------------------
def lattice(lo, hi, shape):
    """[mX, mY, mZ, 3] torch.linspace lattice on the GPU, as the reference's meshgrid builds it."""
    axes = [torch.linspace(float(lo[a]), float(hi[a]), int(shape[a]), device=DEV) for a in range(3)]
    return torch.stack(torch.meshgrid(*axes, indexing='ij'), -1)


def alpha_fp64(vals, mn, mx, n_freqs, xyz, shift, interval):
    """(alpha64, bound, d64, d_bound) at lattice points xyz [.., 3] for a density [P, X, Y, Z, 1]: the fp64 gather d64 of the same
    cells, alpha64 = 1 - (1 + e^(d64 + shift))^-interval, and the bound on |alpha32 - alpha64|: c_alpha(interval) u for the fp32
    Raw2Alpha of a given fp32 x (test_gpu_march_transmittance), plus alpha'(x) times the error of x = fp32(d32 + shift):
    TAU_FWD of the gather's bound and u |x|, doubled for the change of alpha' over that interval."""
    d64, db = fp64_read(xyz.reshape(-1, 3), vals, mn, mx, n_freqs)
    d64, db = d64.view(xyz.shape[:-1]), db.view(xyz.shape[:-1])
    x = d64 + float(np.float32(shift))
    e = torch.exp(x)
    a64 = 1 - (1 + e).pow(-interval)
    slope = interval * e * (1 + e).pow(-interval - 1)
    return a64, c_alpha(interval) * U + 2 * slope * (TAU_FWD * db + U * x.abs()), d64, db


LATTICE = {
    'dense-P1-same': dict(P=1, shape=S_A, lattice=S_A),
    'dense-P1-other': dict(P=1, shape=S_B, lattice=(20, 3, 9)),
    'fourier-P9-same': dict(P=9, shape=S_D, lattice=S_D),
    'fourier-P9-other': dict(P=9, shape=S_D, lattice=(16, 5, 24)),
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(LATTICE))
def test_lattice_alpha_vs_torch_and_fp64(case, oracle):
    from unboundednerfpytorch_b200 import ops
    spec = LATTICE[case]
    P, shape, lat = spec['P'], spec['shape'], spec['lattice']
    nf = (P - 1) // 2
    gen = torch.Generator().manual_seed(_seed(case))
    vals = (torch.randn(P, *shape, 1, generator=gen) * 3).to(DEV)
    grid = make_grid(vals, 'ref')
    shift, interval = -4.0, 0.7
    alpha = ops.lattice_alpha(grid, MN, MX, nf, MN, MX, lat, shift, interval)
    xyz = lattice(MN, MX, lat)
    dens = oracle.fourier_grid_forward(grid, xyz, torch.tensor(MN, device=DEV), torch.tensor(MX, device=DEV), nf)
    want = ops.raw2alpha(dens.contiguous(), shift, interval)[1]
    diff = int((alpha != want).sum())
    assert diff == 0, f'{case}: {diff} alphas differ from Raw2Alpha(F.grid_sample) at torch.linspace lattice points'
    a64, bnd, d64, db = alpha_fp64(vals, MN, MX, nf, xyz, shift, interval)
    check(dens[..., None], d64[..., None], db[..., None], f'{case} lattice density', 'read', tau=TAU_FWD)
    r = float(((alpha.double() - a64).abs() / bnd).max())
    WORST['lattice alpha / alpha bound'] = max(WORST.get('lattice alpha / alpha bound', 0.0), r)
    print(f'[grid-ops] {case}: worst |alpha - alpha64| / alpha bound = {r:.2e}; alpha spans [{float(alpha.min()):.1e}, '
          f'{float(alpha.max()):.1e}]')
    assert r <= 1.0


def pool_want(alpha, prior, thres):
    """prior AND F.max_pool3d(alpha, 3, stride 1, padding 1) > thres, on alpha's device."""
    return prior & (F.max_pool3d(alpha[None, None], kernel_size=3, stride=1, padding=1)[0, 0] > thres)


def pool_scene(shape, gen, thres):
    """alpha on the lattice drawn from {-inf, 0, thres and its neighbours, 0.9}, one NaN in a window of live cells (a corner cell
    and, where the lattice has one, an interior cell), and a prior mask with 20 % False cells."""
    vals = torch.tensor([-float('inf'), 0.0, float(np.nextafter(np.float32(thres), np.float32(0))), thres, thres, thres,
                         float(np.nextafter(np.float32(thres), np.float32(1))), 0.9], dtype=torch.float32)
    alpha = vals[torch.randint(0, vals.numel(), shape, generator=gen)]
    for k in range(3):
        alpha[tuple(min(1, s - 1) if a == k else 0 for a, s in enumerate(shape))] = 0.9
    alpha[(0,) * 3] = float('nan')
    alpha[tuple(s // 2 for s in shape)] = float('nan')
    prior = torch.rand(shape, generator=gen) > 0.2
    return alpha, prior


POOL = [(1, 1, 1), (1, 1, 5), (2, 1, 3), (3, 2, 1), (2, 2, 2), (3, 3, 3), (1, 7, 4), (5, 3, 2), (9, 6, 13), (17, 23, 11)]


@pytest.mark.gpu
@pytest.mark.parametrize('shape', POOL, ids=lambda s: 'x'.join(map(str, s)))
def test_maxpool3_gt_and_matches_torch(shape):
    """Every cell, faces / edges / corners included, against torch's max_pool3d on the GPU with zero tolerance: ties with thres
    (strict >), NaN windows (NaN pools to NaN, so the cell clears), -inf cells and prior-False cells (stay False)."""
    from unboundednerfpytorch_b200 import ops
    gen = torch.Generator().manual_seed(_seed('pool' + str(shape)))
    thres = 0.375
    alpha, prior = pool_scene(shape, gen, thres)
    alpha, prior = alpha.to(DEV), prior.to(DEV)
    want = pool_want(alpha, prior, thres)
    got = prior.clone()
    ops.maxpool3_gt_and_(got, alpha, thres)
    pooled = F.max_pool3d(alpha[None, None], kernel_size=3, stride=1, padding=1)[0, 0]
    print(f'[coverage] max-pool {shape}: {int(torch.isnan(pooled).sum())} NaN windows, {int((pooled == thres).sum())} windows '
          f'whose max equals thres, {int((~prior).sum())} prior-False cells, {int(want.sum())} kept')
    bad = got != want
    assert not bool(bad.any()), f'{shape}: {int(bad.sum())} cells differ from max_pool3d, at {bad.nonzero()[:8].tolist()}'


def _occupancy_fg():
    from unboundednerfpytorch_b200 import models
    m = models.FourierGridModel([-1.] * 3, [1.] * 3, num_voxels_density=19 ** 3, num_voxels_base_density=19 ** 3,
                                num_voxels_rgb=12 ** 3, num_voxels_base_rgb=12 ** 3, num_voxels_viewdir=-1, alpha_init=1e-2,
                                fast_color_thres=1e-3, rgbnet_dim=12, fourier_freq_num=4, mask_cache_world_size=[23, 2, 17])
    return m.to(DEV)


def _occupancy_dcvgo():
    from unboundednerfpytorch_b200 import models
    m = models.DirectContractedVoxGO([-1.] * 3, [1.] * 3, num_voxels=21 ** 3, num_voxels_base=21 ** 3, alpha_init=1e-2,
                                     fast_color_thres=1e-3, rgbnet_dim=12, bg_len=0.2, mask_cache_world_size=[17, 30, 11])
    return m.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['fouriergrid', 'dcvgo'])
def test_update_occupancy_cache_vs_fp64(kind):
    """update_occupancy_cache end to end: every cell whose decision the fp64 alpha bound settles equals prior AND (max-pooled
    alpha > fast_color_thres); the cells the bound cannot settle are counted."""
    from unboundednerfpytorch_b200.functional import host_scalar
    torch.manual_seed(_seed(kind))
    m = (_occupancy_fg if kind == 'fouriergrid' else _occupancy_dcvgo)()
    with torch.no_grad():
        m.density.grid.normal_(-2.0, 3.0)
        m.mask_cache.mask.copy_(torch.rand(m.mask_cache.mask.shape, device=DEV) > 0.2)
    prior = m.mask_cache.mask.clone()
    mn, mx = m.density._bounds()
    vals = as_pxyzc(m.density.grid.detach())
    nf = m.density.num_freqs
    xyz = lattice(m.xyz_min.tolist(), m.xyz_max.tolist(), prior.shape)
    a64, bnd, _, _ = alpha_fp64(vals, mn, mx, nf, xyz, host_scalar(m._density_shift()), float(m._voxel_size_ratio()))
    thres = float(np.float32(m.fast_color_thres))

    def pool(t):
        return F.max_pool3d(t[None, None], kernel_size=3, stride=1, padding=1)[0, 0]

    sure_true, sure_false = pool(a64 - bnd) > thres, pool(a64 + bnd) <= thres
    band = ~(sure_true | sure_false)
    m.update_occupancy_cache()
    got = m.mask_cache.mask
    want = prior & sure_true
    BANDS[f'occupancy {kind}'] = int((band & prior).sum())
    print(f'[bands] update_occupancy_cache {kind} {tuple(prior.shape)}: {int((band & prior).sum())} of {prior.numel()} cells '
          f'in the band around fast_color_thres; {int(got.sum())} kept')
    assert int((got & ~prior).sum()) == 0
    assert 0.02 < float(want.float().mean()) < 0.98, 'degenerate occupancy scene'
    bad = (got != want) & ~band
    assert not bool(bad.any()), f'{kind}: {int(bad.sum())} cells outside the band differ'


# ---- maintenance: view counts ---------------------------------------------------------------------------------------------
def count_rays(n, mn, mx, gen):
    """Rays for voxel_count_views: origins inside the box (t_min clamped to near) and outside it, direction components exactly
    zero, one zero direction (its sample points are NaN and add nothing), rays that miss the box, and rays whose entry lies beyond
    `far` (t_min clamped to far when far is small)."""
    mn, mx = torch.tensor(mn), torch.tensor(mx)
    c, half = (mn + mx) / 2, (mx - mn) / 2
    o = c + (torch.rand(n, 3, generator=gen) * 2 - 1) * half * 2.5
    d = torch.randn(n, 3, generator=gen)
    d[::5, 0] = 0
    d[1::7, 1] = 0
    d[3::10, 1:] = 0
    k = n // 8                                    # origins outside, pointing away: the ray misses
    o[:k] = c + half * 3
    d[:k] = torch.rand(k, 3, generator=gen) + 0.1
    d[k] = 0
    return o, d


def count_points(o, d, mn, mx, n_samples, step, near, far):
    """The reference's sample points, in its fp32 torch ops (FourierGrid_model.py:408-415, dvgo.py:262-269), on the GPU."""
    mn_t, mx_t = torch.tensor(mn, device=DEV), torch.tensor(mx, device=DEV)
    rng = torch.arange(n_samples, device=DEV)[None].float()
    vec = torch.where(d == 0, torch.full_like(d, 1e-6), d)
    rate_a, rate_b = (mx_t - o) / vec, (mn_t - o) / vec
    t_min = torch.minimum(rate_a, rate_b).amax(-1).clamp(min=near, max=far)
    interpx = t_min[..., None] + (step * rng) / d.norm(dim=-1, keepdim=True)
    return (o[..., None, :] + d[..., None, :] * interpx[..., None]).reshape(-1, 3), t_min


def _count_model(kind):
    from unboundednerfpytorch_b200 import models
    if kind == 'fouriergrid':
        m = models.FourierGridModel([-1.] * 3, [1.] * 3, num_voxels_density=18 ** 3, num_voxels_base_density=18 ** 3,
                                    num_voxels_rgb=12 ** 3, num_voxels_base_rgb=12 ** 3, num_voxels_viewdir=-1, alpha_init=1e-2,
                                    rgbnet_dim=12, fourier_freq_num=2)
    elif kind == 'dvgo':
        m = models.DirectVoxGO(MN, MX, num_voxels=16 ** 3, num_voxels_base=16 ** 3, alpha_init=1e-2, rgbnet_dim=12,
                               rgbnet_direct=True)
    else:       # DirectContractedVoxGO has no voxel_count_views; its world [-1 - bg, 1 + bg] is counted through the op
        m = models.DirectContractedVoxGO([-1.] * 3, [1.] * 3, num_voxels=20 ** 3, num_voxels_base=20 ** 3, alpha_init=1e-2,
                                         rgbnet_dim=12, bg_len=0.2)
    return m.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['fouriergrid', 'dcvgo', 'dvgo'])
def test_voxel_count_views_vs_fp64(kind):
    """ubn_view_scatter_ones per view against the fp64 adjoint of the reference's fp32 sample points; ubn_count_gt's counts
    exact outside the band around 1; the model method's counts; and count_gt_ adding into existing counts."""
    from unboundednerfpytorch_b200 import ops
    m = _count_model(kind)
    ws = [int(v) for v in m.world_size]
    mn, mx = m.density._bounds()
    vsize = float(m._voxel_size())
    stepsize = 0.5
    n_samples = int(np.linalg.norm(np.array(ws) + 1) / stepsize) + 1
    step = float(stepsize * torch.tensor(vsize, dtype=torch.float32))
    gen = torch.Generator().manual_seed(_seed(kind))
    imsz = [611, 1, 96]
    o, d = count_rays(sum(imsz), mn, mx, gen)
    o, d = o.to(DEV), d.to(DEV)
    cnt_want, in_band = torch.zeros(ws, device=DEV), torch.zeros(ws, dtype=torch.bool, device=DEV)
    bufs, clamped = [], {'near': 0, 'far': 0}
    for far in (1e9, 0.6):
        for v, (ro, rd) in enumerate(zip(o.split(imsz), d.split(imsz))):
            near = 0.1
            pts, t_min = count_points(ro, rd, mn, mx, n_samples, step, near, far)
            buf = torch.zeros(ws, device=DEV)
            ops.view_scatter_ones(ro.contiguous(), rd.contiguous(), mn, mx, ws, n_samples, near, far, step, buf)
            want, bound = fp64_adjoint(pts, torch.ones(pts.shape[0], 1, device=DEV), tuple(ws), 1, mn, mx, 0)
            tag = f'view count {kind} far={far:g} view {v} ({ro.shape[0]} rays x {n_samples} samples)'
            clamped['near'] += int((t_min == near).sum())
            clamped['far'] += int((t_min == far).sum())
            check(buf[None, ..., None], want, bound, tag, f'view count {kind}')
            band = (want[0, ..., 0] - 1).abs() <= TAU * bound[0, ..., 0]
            bad = ((buf > 1) != (want[0, ..., 0] > 1)) & ~band
            assert not bool(bad.any()), f'{tag}: {int(bad.sum())} count decisions outside the band differ'
            if far == 1e9:
                cnt_want += want[0, ..., 0] > 1
                in_band |= band
                bufs.append(buf)
    print(f'[coverage] view count {kind}: t_min clamped to near on {clamped["near"]} rays, to far on {clamped["far"]}')
    assert min(clamped.values()) > 0
    BANDS[f'view count {kind}'] = int(in_band.sum())
    print(f'[bands] view count {kind} {ws}: {int(in_band.sum())} voxels with a view in the band around 1; max count '
          f'{int(cnt_want.max())}')
    assert int(cnt_want.max()) >= 2
    # count_gt_ adds into existing counts
    base = torch.randint(0, 5, ws, generator=gen).float().to(DEV)
    acc = base.clone()
    for buf in bufs:
        ops.count_gt_(acc, buf, 1.0)
    assert torch.equal(acc, base + sum((b > 1).float() for b in bufs))
    if kind != 'dcvgo':
        cnt = m.voxel_count_views(o, d, imsz, near=0.1, far=1e9, stepsize=stepsize, irregular_shape=True)
        assert torch.equal(cnt[0, 0], acc - base)
        bad = (cnt[0, 0] != cnt_want) & ~in_band
        assert not bool(bad.any()), f'{kind}: voxel_count_views differs outside the band at {int(bad.sum())} voxels'


# ---- maintenance: maskout near cameras ----------------------------------------------------------------------------------
MASK_LATTICES = {'slab': ((-1., -1., -1.), (1., 1., 1.), (13, 2, 9), 1), 'world': (tuple(MN), tuple(MX), (7, 11, 5), 3)}


@pytest.mark.gpu
@pytest.mark.parametrize('n_cams', [1, 10, 11, 1000])
@pytest.mark.parametrize('which', list(MASK_LATTICES))
def test_maskout_near_cam_vs_fp64(which, n_cams):
    """ubn_maskout_near_cam ([-1, 1] slab lattice) and ubn_maskout_near_cam_lattice (DVGO's world lattice): every voxel whose
    fp64 distance to the nearest camera is outside 8 u of near_clip is masked exactly when that distance <= near_clip; cameras on
    lattice nodes; near_clip = 0; a strided slab view (channel stride 3)."""
    from unboundednerfpytorch_b200 import ops
    lo, hi, shape, sv = MASK_LATTICES[which]
    gen = torch.Generator().manual_seed(_seed(which) + n_cams)
    xyz = lattice(lo, hi, shape)
    lo_t, hi_t = torch.tensor(lo), torch.tensor(hi)
    cams = lo_t + (torch.rand(n_cams, 3, generator=gen) * 1.4 - 0.2) * (hi_t - lo_t)
    k = min(n_cams, 3)
    nodes = torch.stack([torch.randint(0, s, (k,), generator=gen) for s in shape], 1)
    cams[:k] = xyz.cpu()[nodes[:, 0], nodes[:, 1], nodes[:, 2]]
    cams = cams.to(DEV)
    g64 = xyz.double().reshape(-1, 1, 3)
    dist = torch.cat([(g64 - c.double()[None]).pow(2).sum(-1).sqrt().amin(-1, keepdim=True) for c in cams.split(100)], 1).amin(1)
    dist = dist.view(shape)
    for near_clip in (0.0, 0.35):
        nc = float(np.float32(near_clip))
        store = torch.randn(*shape, sv, generator=gen).to(DEV)
        slab = store[..., 0]
        before = store.clone()
        ops.maskout_near_cam_(slab, cams, near_clip, -100.0, lattice=None if which == 'slab' else (lo, hi))
        band = (dist > 0) & ((dist - nc).abs() <= 8 * U * dist)
        masked = slab == -100.0
        want = dist <= nc
        key = f'maskout {which} cams={n_cams} near_clip={near_clip}'
        BANDS[key] = int(band.sum())
        print(f'[bands] {key} {shape}: {int(want.sum())} voxels within near_clip, {int(band.sum())} in the band')
        if near_clip == 0.0:
            assert int(want.sum()) >= len(set(map(tuple, nodes.tolist())))
        bad = (masked != want) & ~band
        assert not bool(bad.any()), f'{key}: {int(bad.sum())} voxels outside the band differ'
        assert torch.equal(store[..., 1:], before[..., 1:]) and torch.equal(slab[~masked], before[..., 0][~masked])


# ---- maintenance: resample ----------------------------------------------------------------------------------------------
RESAMPLE = [((1, 1, 1), (2, 3, 1)), ((2, 2, 2), (1, 1, 1)), ((2, 1, 3), (5, 2, 1)), ((7, 5, 9), (3, 2, 4)),
            ((3, 4, 2), (8, 9, 5)), ((5, 2, 7), (2, 7, 3)), ((1, 2, 1), (2, 1, 2))]
RESAMPLE_GRIDS = [(1, 1, 'ref'), (9, 1, 'ref'), (1, 3, 'cl'), (9, 12, 'cl'), (9, 12, 'ref')]
RESAMPLE_U = 16       # |got - want| <= RESAMPLE_U * u * sum |w| |v|: the nested blend rounds at most 3 products and 7 sums on a path,
                      # and lambda0 = 1 - lambda1 once more, each at most u of the magnitudes below it


def resample_fp64(vals, dst):
    """F.interpolate(trilinear, align_corners=True) of vals [P, X, Y, Z, C] in fp64 (value, bound), with ATen's fp32 source
    positions: scale = fp32((in - 1) / (out - 1)), src = fp32(scale * o), i0 = (int)src, lambda1 = src - i0 (exact)."""
    mats = []
    for n_in, n_out in zip(vals.shape[1:4], dst):
        scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
        src = np.float32(scale) * np.arange(n_out, dtype=np.float32)
        i0 = src.astype(np.int64)
        l1 = (src - i0.astype(np.float32)).astype(np.float64)
        w = np.zeros((n_out, n_in))
        np.add.at(w, (np.arange(n_out), i0), 1 - l1)
        np.add.at(w, (np.arange(n_out), np.minimum(i0 + 1, n_in - 1)), l1)
        mats.append(torch.tensor(w, device=vals.device))
    v = vals.double()
    want = torch.einsum('xi,yj,zk,pijkc->pxyzc', *mats, v)
    bound = torch.einsum('xi,yj,zk,pijkc->pxyzc', *[m.abs() for m in mats], v.abs())
    return want, bound


@pytest.mark.gpu
@pytest.mark.parametrize('sizes', RESAMPLE, ids=lambda s: '-'.join('x'.join(map(str, t)) for t in s))
@pytest.mark.parametrize('pcl', RESAMPLE_GRIDS, ids=lambda t: f'P{t[0]}-C{t[1]}-{t[2]}')
def test_resample_grid_vs_fp64_and_interpolate(pcl, sizes):
    """ubn_resample_grid within RESAMPLE_U u of the fp64 resample (sizes of 1 and 2, down- and up-sampling, non-cubic, P = 9
    in both layouts); its values are counted against F.interpolate on the GPU bit for bit, and must equal it where every output
    is a copy or a single-axis blend (no input dimension above 2)."""
    from unboundednerfpytorch_b200 import ops
    P, C, layout = pcl
    src, dst = sizes
    gen = torch.Generator().manual_seed(_seed(str(pcl) + str(sizes)))
    vals = torch.randn(P, *src, C, generator=gen).to(DEV)
    grid = make_grid(vals, layout)
    out = ops.resample_grid(grid, dst)
    want, bound = resample_fp64(vals, dst)
    r = float(((as_pxyzc(out).double() - want).abs() / (U * bound).clamp(min=1e-300)).max())
    WORST['resample / (u B)'] = max(WORST.get('resample / (u B)', 0.0), r)
    ref = F.interpolate(grid.contiguous(), size=dst, mode='trilinear', align_corners=True)
    diff = int((out != ref).sum())
    key = f'resample values differing from F.interpolate {src}->{dst}'
    BANDS[key] = BANDS.get(key, 0) + diff
    print(f'[grid-ops] resample P={P} C={C} {layout} {src} -> {dst}: worst {r:.2f} u of B; {diff} of {ref.numel()} values '
          f'differ from F.interpolate')
    assert r <= RESAMPLE_U
    if max(src) <= 2:
        assert diff == 0


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    if WORST:
        print('\n[grid-ops] worst |got - want| / B: ' + ', '.join(f'{k} {v:.2e}' for k, v in sorted(WORST.items())))
    if BANDS:
        print('[grid-ops] cells in ambiguity bands: ' + ', '.join(f'{k} {v}' for k, v in sorted(BANDS.items())))


# ---- CPU: the judges see one wrong addend and one wrong window ---------------------------------------------------------
def pool_restated(alpha, prior, thres, z_offsets=(0, 1, 2), keep_nan=True):
    """The max-pool mask restated in fp32: ATen's window maximum (v > m || isnan(v) takes v) over the -inf-padded lattice."""
    X, Y, Z = alpha.shape
    padded = F.pad(alpha, (1, 1, 1, 1, 1, 1), value=-float('inf'))
    m = torch.full_like(alpha, -float('inf'))
    for a in range(3):
        for b in range(3):
            for c in z_offsets:
                v = padded[a:a + X, b:b + Y, c:c + Z]
                take = (v > m) | (torch.isnan(v) if keep_nan else torch.zeros_like(prior))
                m = torch.where(take, v, m)
    return prior & (m > thres)


def test_checker_rejects_faults():
    """fp32 restatements of the adjoint (P = 9, 7 x 9 x 11, 4 channels) and of the max-pool mask pass the judges; one addend
    moved one voxel, dropped or doubled, the 1/P missing, one corner on the x = X - 1 face dropped, a window without its z+1 plane
    and a window that drops its NaN each fail them."""
    P, shape, C = 9, (7, 9, 11), 4
    X, Y, Z = shape
    g = torch.Generator().manual_seed(5)
    pts = []
    for k in range(24):                      # rays along x through every cell, the last one included, and random points
        yz = (torch.rand(2, generator=g) * 2 - 1) * 0.9
        xs = torch.linspace(-0.999, 0.999, 5 * (X - 1))
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
    depth = torch.minimum(f, 1 - f).amin(2).amin(0) * (x0[0, :, 0] < X - 2) * (gr.abs().amin(1) > 0.3)
    i = int(depth.argmax())
    assert float(depth[i]) > 0.05
    one = int(((smp == i) & (slab == 0)).nonzero()[0])          # sample i's corner (0, 0, 0) addend in slab 0
    keep = torch.ones(idx.numel(), dtype=torch.bool)
    keep[one] = False
    faults = {}
    moved = idx.clone()
    moved[one] += 1
    faults['one addend moved one voxel'] = (moved, val)
    faults['one addend dropped'] = (idx[keep], val[keep])
    faults['one addend doubled'] = (torch.cat([idx, idx[one:one + 1]]), torch.cat([val, val[one:one + 1]]))
    faults['1/P missing'] = (idx, val * P)
    last = (x0[0, :, 0] == X - 2) & (f[0, :, 0] > 0.5) & (gr.abs().amin(1) > 0.3)
    j = int(last.nonzero()[0])
    face = (smp == j) & (slab == 0) & ((idx % (X * Y * Z)) // (Y * Z) == X - 1)
    assert int(face.sum()) == 4
    drop = torch.ones(idx.numel(), dtype=torch.bool)
    drop[int(face.nonzero()[0])] = False
    faults['one corner on the x = X - 1 face dropped'] = (idx[drop], val[drop])
    margins = {}
    for name, (fi, fv) in faults.items():
        r, stray = ratio(accumulate(fi, fv, P, shape), want, bound)
        margins[name] = r / TAU
        assert r > 10 * TAU or stray > 0, f'{name}: only {r:.2e} of B'

    gp = torch.Generator().manual_seed(6)
    thres = 0.375
    for pshape in ((5, 4, 6), (3, 1, 2)):
        alpha, prior = pool_scene(pshape, gp, thres)
        want_mask = pool_want(alpha, prior, thres)
        assert torch.equal(pool_restated(alpha, prior, thres), want_mask)
    alpha, prior = pool_scene((5, 4, 6), gp, thres)
    want_mask = pool_want(alpha, prior, thres)
    pool_faults = {'window without its z+1 plane': pool_restated(alpha, prior, thres, z_offsets=(0, 1)),
                   'NaN dropped from the window': pool_restated(alpha, prior, thres, keep_nan=False)}
    for name, got in pool_faults.items():
        n_bad = int((got != want_mask).sum())
        margins[name] = n_bad
        assert n_bad > 0, f'{name}: the max-pool judge sees no difference'
    print(f'[grid-ops checker] fp32 restatement {honest:.2e} of B; scatter fault / TAU, max-pool fault cells: '
          + ', '.join(f'{k} {v:.1f}' for k, v in margins.items()))
