"""The TMA-staged render read (csrc/render_tma.cu: k_march_feature_tma, march.March with coherent=True under no_grad) against
the gather kernel, torch's F.grid_sample and an fp64 gather, at the step counts, ray groups and brick spans where its
bookkeeping changes.

Every case runs the march twice on the same scene, coherent=False (march_feature.cu's gather kernel) and coherent=True, and
holds the TMA read to four judges:
  1. every per-survivor record except the features -- ray_id, step_id, raw density, raw_alpha, weights, t, inner -- and
     alphainv_last equal the gather kernel's bit for bit (pass A is shared; a wrong output cursor moves records);
  2. the features equal F.grid_sample on the GPU bit for bit (the reference's DenseGrid.forward: .flip, align_corners=True)
     wherever every unnormalised coordinate lies in [0, size - 1].  Outside that range the kernel's clamped cell (cell_of,
     shared with march_feature.cu::make_cell) extrapolates from the last cell where ATen drops the corners beyond the face, so
     those samples are counted and left to judge 3;
  3. the features lie within TAU_FWD of the fp64 gather of the same cells (test_gpu_march_scatter.ref_gather's bound);
  4. the kernel's counters (march.TMA_STATS) equal (n_tma, n_fallback) predicted from the cells: a unit is one 32-ray group
     (ray_id // 32) x one 4-step block (step_id // 4) holding at least one survivor, served by TMA when the cell bases of its
     survivors span at most 6 on every axis (the 8-point brick then holds every corner) and by global loads otherwise.
The cases assert their structure from the survivors and the predicted cells: both ways the kernel counts a ray's earlier
survivors (16-byte popcounts when S % 16 == 0, a byte loop otherwise), S = 512 over 8 segments, S < 64 and a partial last
block, W = 53-pixel image rows, 1 / 31 / 32 / 33 rays, non-cubic grids, an axis shorter than 8 and an axis of 2, both contracted
norms, groups whose bases span exactly 6 and exactly 7 on each axis, bricks past the far faces and samples exactly on them,
empty blocks and empty segments, and the benchmark's 320^3 frame.  test_checker_rejects_faults (CPU) restates the kernel and
shows that the judges reject one broken line of it each."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_march_scatter import TAU_FWD, cells, judge, ragged_planes, ref_gather, slab_coords

DEV = 'cuda:0'
BG = 0.2                  # bg_len of DirectContractedVoxGO
T_BOUNDARY = 2.0          # dcvgo.py:243-244
LO, HI = -1.0 - BG, 1.0 + BG
GROUP, BLOCK, SEG = 32, 4, 64          # rays per warp, steps per block, steps per warp segment (render_tma.cu: rt::)
BOX = 8                   # lattice points per axis of a staged brick: bases may span BOX - 2 = 6
OUTS = ('weights', 'alphainv_last', 'raw_alpha', 'raw_density', 'feat', 'ray_id', 'step_id', 't', 'inner')
RECORDS = tuple(k for k in OUTS if k != 'feat')


# ---- the judges (shared with the CPU checker) ----------------------------------------------------------------------------
def grid_sample_ref(kgrid, pts, mn, mx):
    """The reference's DenseGrid.forward (grid.py:50-61) on [M, 3] world points: F.grid_sample on the normalised, flipped
    coordinates, align_corners=True.  [M, C]."""
    mn = torch.as_tensor(mn, dtype=torch.float32, device=pts.device)
    mx = torch.as_tensor(mx, dtype=torch.float32, device=pts.device)
    ind = ((pts - mn) / (mx - mn)).flip((-1,)) * 2 - 1
    out = F.grid_sample(kgrid, ind.reshape(1, 1, 1, -1, 3), mode='bilinear', align_corners=True)
    return out.reshape(kgrid.shape[1], -1).T


def outside_faces(coords, shape):
    """[M] bool: a sample with an unnormalised coordinate ((c + 1) / 2) * (size - 1) outside [0, size - 1] on some axis."""
    size = torch.tensor(shape, dtype=torch.float32, device=coords.device)
    c = ((coords + 1) / 2) * (size - 1)
    return ((c < 0) | (c > size - 1)).any(-1)


def predict_units(ray_id, step_id, x0, S):
    """The kernel's brick decisions from the survivors and their cell bases x0 [M, 3]: per unit (32-ray group, 4-step block)
    with a survivor, the smallest base and the span on each axis; a unit fits one brick when every span is <= BOX - 2."""
    key = (ray_id // GROUP) * -(-S // BLOCK) + step_id // BLOCK
    units, inv = torch.unique(key, return_inverse=True)
    idx = inv[:, None].expand(-1, 3)
    lo = torch.zeros(units.numel(), 3, dtype=x0.dtype, device=x0.device).scatter_reduce(0, idx, x0, 'amin', include_self=False)
    hi = torch.zeros_like(lo).scatter_reduce(0, idx, x0, 'amax', include_self=False)
    span = hi - lo
    fits = (span <= BOX - 2).all(1)
    return dict(units=units, inv=inv, lo=lo, span=span, fits=fits, n_tma=int(fits.sum()), n_fallback=int((~fits).sum()))


def judge_records(got, want, what):
    """Judge 1: the TMA read's records equal the gather kernel's bit for bit."""
    for k in RECORDS:
        if k in want:
            assert got[k].shape == want[k].shape and torch.equal(got[k], want[k]), f'{what}: {k} differs from the gather kernel'


def judge_grid_sample(feat, want, outside, what):
    """Judge 2: features bit for bit equal to F.grid_sample at every sample inside [0, size - 1]."""
    bad = ((feat != want).any(1) & ~outside).sum()
    assert int(bad) == 0, f'{what}: {int(bad)} of {int((~outside).sum())} in-range samples differ from F.grid_sample'


def judge_fp64(feat, x0, f, kvals, what):
    """Judge 3: every feature within TAU_FWD of the fp64 gather of the same cells."""
    want, bound = ref_gather(x0, f, kvals)
    judge(feat[:, :, None], want[:, :, None], bound[:, :, None], what + ' TMA features vs fp64', 'tma forward', tau=TAU_FWD)


def judge_counts(stats, pred, what):
    """Judge 4: the kernel's (blocks by TMA, blocks by the fallback) equal the prediction exactly."""
    assert tuple(stats) == (pred['n_tma'], pred['n_fallback']), \
        f'{what}: TMA_STATS {tuple(stats)} != predicted {(pred["n_tma"], pred["n_fallback"])}'


# ---- scenes --------------------------------------------------------------------------------------------------------------
def frame(H, W, c2w=((1., 0., 0., 0.15), (0., 1., 0., -0.10), (0., 0., 1., 0.35))):
    """Image-ordered rays of one pinhole view (focal = W, as bench.frame_rays) from inside the unit scene."""
    from unboundednerfpytorch_b200 import rays as R
    K = np.array([[float(W), 0., W / 2], [0., float(W), H / 2], [0., 0., 1.]])
    ro, rd, _ = R.get_rays_of_a_view(H, W, K, torch.tensor(c2w), False, False, False, False, 'center')
    return ro.reshape(-1, 3).float(), rd.reshape(-1, 3).float()


def random_rays(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, 3, generator=g) * 2 - 1) * 0.9, torch.randn(n, 3, generator=g)


def src_to_world(c, size):
    """World coordinate whose unnormalised index on a [LO, HI] grid axis of `size` points is (close to) c."""
    return LO + c / (size - 1) * (HI - LO)


def span_groups(shape):
    """Six 32-ray groups of parallel rays in the linear inner region: group 2a + k spreads its lanes along axis a so that the
    cell bases of every inner block span exactly 6 + k on axis a (k = 0: one brick; k = 1: the fallback), travelling along the
    next axis, with the third axis fixed."""
    o, d = [], []
    for a in range(3):
        t_ax, f_ax = (a + 1) % 3, (a + 2) % 3
        for span in (6, 7):
            base = shape[a] // 2 - 4
            for lane in range(GROUP):
                p = [0.0, 0.0, 0.0]
                p[a] = src_to_world(base + 0.5 + span * lane / (GROUP - 1), shape[a])
                p[t_ax] = -0.9
                p[f_ax] = 0.1
                o.append(p)
                dd = [0.0, 0.0, 0.0]
                dd[t_ax] = 1.0
                d.append(dd)
    return torch.tensor(o), torch.tensor(d)


def face_groups():
    """32-ray groups along +x, +y, +z and -x (inf norm) with the other two coordinates on a small patch: every lane of a group
    meets the same contracted coordinate along its axis at every step, so a grid bound set to one of them puts a whole block
    exactly on the far face."""
    o, d = [], []
    g = torch.Generator().manual_seed(11)
    for a, sign in ((0, 1.0), (1, 1.0), (2, 1.0), (0, -1.0)):
        patch = (torch.rand(GROUP, 2, generator=g) * 2 - 1) * 0.1
        for lane in range(GROUP):
            p = patch[lane].tolist()
            p.insert(a, 0.3 * sign)
            o.append(p)
            dd = [0.0, 0.0, 0.0]
            dd[a] = sign
            d.append(dd)
    return torch.tensor(o), torch.tensor(d)


def x_patch_groups(n_groups, seed):
    """Groups of 32 rays along +x from x = -1.19 on 4 x 8 patches of (y, z) at random places: they cross the ragged density's
    x planes together."""
    g = torch.Generator().manual_seed(seed)
    o = []
    for _ in range(n_groups):
        c = (torch.rand(2, generator=g) * 2 - 1) * 0.8
        for lane in range(GROUP):
            o.append([-1.19, float(c[0]) + 0.01 * (lane % 8), float(c[1]) + 0.01 * (lane // 8)])
    o = torch.tensor(o)
    d = torch.zeros_like(o)
    d[:, 0] = 1
    return o, d


class Scene:
    """A DirectContractedVoxGO-style scene on raw grids, driven through march.March.  k0 may have its own bounds (kmn, kmx)."""

    def __init__(self, shape, ro, rd, norm='inf', world_len=41, stepsize=0.5, thres=0.0, dens=None, mask=None, kmn=None,
                 kmx=None, seed=0):
        from unboundednerfpytorch_b200 import grid as G
        from unboundednerfpytorch_b200 import march
        X, Y, Z = self.shape = tuple(shape)
        g = torch.Generator().manual_seed(seed)
        self.dgrid = (dens if dens is not None else torch.randn(1, 1, X, Y, Z, generator=g)).to(DEV)
        self.kvals = torch.randn(1, X, Y, Z, 12, generator=g).to(DEV)
        self.kgrid = self.kvals.permute(0, 4, 1, 2, 3)              # channels-last [1, 12, X, Y, Z], as grid.zeros_grid
        self.ro, self.rd = ro.to(DEV).contiguous(), rd.to(DEV).contiguous()
        self.norm, self.world_len, self.stepsize, self.thres = norm, world_len, stepsize, thres
        self.t_table = march.t_schedule(world_len, stepsize, BG, T_BOUNDARY, DEV)
        self.S = self.t_table.numel()
        self.mask = mask.to(DEV) if mask is not None else None
        mscale = mshift = None
        if mask is not None:
            mscale = [(n - 1) / (HI - LO) for n in mask.shape]
            mshift = [-LO * s for s in mscale]
        self.cfg = march.make_cfg([0.] * 3, [1.] * 3, BG, norm, self.S, 0.0, 0.5, thres, mask=mask, mask_scale=mscale,
                                  mask_shift=mshift)
        self.kmn = list(kmn) if kmn is not None else [LO] * 3
        self.kmx = list(kmx) if kmx is not None else [HI] * 3
        self.ddesc = G.grid_desc(self.dgrid, [LO] * 3, [HI] * 3, 0)
        self.kdesc = G.grid_desc(self.kgrid, self.kmn, self.kmx, 0)

    def points_all(self):
        from unboundednerfpytorch_b200 import models
        ns = types.SimpleNamespace(scene_center=torch.zeros(3, device=DEV), scene_radius=torch.ones(3, device=DEV), bg_len=BG,
                                   T_BOUNDARY=T_BOUNDARY, contracted_norm=self.norm, _world_len=lambda: self.world_len)
        return models._ContractedBase._sample_dense(ns, self.ro, self.rd, self.stepsize)[0]

    def run(self, coherent):
        from unboundednerfpytorch_b200 import march
        return run_march(lambda: march.March.apply(self.dgrid, self.kgrid, self.ro, self.rd, self.t_table, self.mask, self.cfg,
                                                   self.ddesc, self.kdesc, self.thres <= 0 and self.mask is None, coherent))


def run_march(fn):
    """(the march's outputs by name, the TMA counters of this launch) with march.TMA_STATS restored afterwards."""
    from unboundednerfpytorch_b200 import march
    stats = torch.zeros(2, dtype=torch.int64, device=DEV)
    old = march.TMA_STATS
    march.TMA_STATS = stats
    try:
        with torch.no_grad():
            out = fn()
    finally:
        march.TMA_STATS = old
    return (out if isinstance(out, dict) else dict(zip(OUTS, out))), tuple(stats.tolist())


def judge_all(gat, tma, stats, pts, kmn, kmx, shape, kvals, kgrid, S, what):
    """The four judges on one launch pair.  pts: [M, 3] world points of the gather kernel's survivors.  Returns the prediction
    and the per-sample facts the coverage lines report."""
    judge_records(tma, gat, what)
    coords = slab_coords(pts, kmn, kmx, 0)
    x0, f = cells(coords, shape)
    outside = outside_faces(coords[0], shape)
    n_out = int(outside.sum())
    want = grid_sample_ref(kgrid, pts, kmn, kmx)
    diff = (tma['feat'] - want).abs()[outside]
    print(f'[tma] {what}: {n_out} of {outside.numel()} samples outside [0, size - 1] (judged against fp64 only); of these '
          f'{int((diff > 0).any(1).sum())} differ from F.grid_sample, by at most {float(diff.max()) if n_out else 0.0:.3g}')
    judge_grid_sample(tma['feat'], want, outside, what)
    judge_fp64(tma['feat'], x0, f, kvals, what)
    pred = predict_units(gat['ray_id'], gat['step_id'], x0[0], S)
    judge_counts(stats, pred, what)
    pred.update(x0=x0[0], f=f[0], n_out=n_out, coords=coords[0])
    return pred


def structure(ray_id, step_id, N, S, pred):
    """Units the kernel sees: empty (32-ray group, 4-step block) pairs and empty (group, 64-step segment) pairs."""
    n_groups, n_blk, n_seg = -(-N // GROUP), -(-S // BLOCK), -(-S // SEG)
    live_blk = pred['units'].numel()
    seg_key = torch.unique((ray_id // GROUP) * n_seg + step_id // SEG)
    return dict(n_groups=n_groups, n_seg=n_seg, empty_blocks=n_groups * n_blk - live_blk,
                empty_segments=n_groups * n_seg - seg_key.numel(), path='uint4' if S % 16 == 0 else 'byte')


def check_scene(sc, tag):
    gat, st_g = sc.run(False)
    tma, st_t = sc.run(True)
    assert st_g == (0, 0), f'{tag}: the gather kernel counted TMA blocks'
    ray_id, step_id = gat['ray_id'], gat['step_id']
    assert ray_id.numel() > 0, f'{tag}: no survivors'
    pts = sc.points_all()[ray_id, step_id]
    pred = judge_all(gat, tma, st_t, pts, sc.kmn, sc.kmx, sc.shape, sc.kvals, sc.kgrid, sc.S, tag)
    st = structure(ray_id, step_id, sc.ro.shape[0], sc.S, pred)
    spans = pred['span']
    print(f"[coverage] {tag}: S = {sc.S} ({st['path']} cursor, {st['n_seg']} segments, S % 4 = {sc.S % 4}), "
          f"{sc.ro.shape[0]} rays, {ray_id.numel()} survivors; units by TMA {pred['n_tma']} / fallback {pred['n_fallback']} "
          f"(= TMA_STATS); max span {spans.max(0).values.tolist()}; empty blocks {st['empty_blocks']}, empty segments "
          f"{st['empty_segments']}; {pred['n_out']} samples outside [0, size - 1]")
    return gat, tma, st_t, pred, st


# ---- GPU cases -----------------------------------------------------------------------------------------------------------
SHAPE = (41, 23, 37)
FRAME_HW = (37, 53)           # 1961 rays; W = 53 rows wrap inside warps
CASES = {
    # S = 144: 16-byte cursor popcounts over 3 segments
    'frame-S144': dict(shape=SHAPE, stepsize=0.48, want_S=144),
    # S = 512 (the benchmark's step count): 16-byte popcounts over 8 segments, l2 norm
    'frame-S512-l2': dict(shape=SHAPE, stepsize=0.1338, norm='l2', want_S=512),
    # S = 274: byte-loop cursor over 5 segments, a partial last block; X = 5 and Z = 3 are shorter than a brick
    'frame-S274-short': dict(shape=(5, 40, 3), stepsize=0.25, want_S=274),
    # S = 58 < 64: one segment, a partial last block; an axis of 2
    'frame-S58-X2-l2': dict(shape=(2, 29, 17), stepsize=1.2, norm='l2', want_S=58),
    # random rays: the fallback serves most blocks
    'random-S138': dict(shape=SHAPE, stepsize=0.5, want_S=138, rays='random'),
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(CASES))
def test_tma_read_frames(case):
    """Image-ordered 37 x 53 frames (and random rays) at each cursor path, step count and grid shape of CASES."""
    spec = dict(CASES[case])
    want_S, kind = spec.pop('want_S'), spec.pop('rays', 'frame')
    ro, rd = frame(*FRAME_HW) if kind == 'frame' else random_rays(3001, 5)
    sc = Scene(ro=ro, rd=rd, seed=len(case), **spec)
    assert sc.S == want_S
    _, _, _, pred, st = check_scene(sc, f"{case} {'x'.join(map(str, sc.shape))} {sc.norm}")
    if kind == 'random':
        assert pred['n_fallback'] > pred['n_tma'], 'random rays: the fallback should serve most blocks'
    else:
        assert pred['n_tma'] > 0
    if want_S % 4:
        assert int((pred['units'] % -(-want_S // BLOCK)).max()) == want_S // BLOCK, 'the partial last block has no survivor'
    assert st['path'] == ('uint4' if want_S % 16 == 0 else 'byte')
    if want_S >= SEG:
        assert st['n_seg'] > 1


@pytest.mark.gpu
def test_tma_read_ray_counts():
    """1, 31, 32 and 33 image-ordered rays: a lone lane, a warp short of one lane, one full warp, one lane over a warp."""
    ro, rd = frame(*FRAME_HW)
    for n in (1, 31, 32, 33):
        sc = Scene(SHAPE, ro[700:700 + n], rd[700:700 + n], world_len=32, stepsize=0.5, seed=n)
        assert sc.S == 108 and sc.S % 16 and not sc.S % 4
        _, _, _, pred, st = check_scene(sc, f'{n} rays')
        assert st['n_groups'] == -(-n // GROUP) and pred['n_tma'] > 0


@pytest.mark.gpu
def test_tma_read_brick_spans():
    """Groups whose cell bases span exactly 6 (one brick) and exactly 7 (the fallback) on each axis in turn."""
    ro, rd = span_groups(SHAPE)
    sc = Scene(SHAPE, ro, rd, stepsize=0.48, seed=3)
    _, _, _, pred, _ = check_scene(sc, 'span groups')
    group = pred['units'] // -(-sc.S // BLOCK)
    other = lambda a: [b for b in range(3) if b != a]
    for a in range(3):
        for k, span in enumerate((6, 7)):
            g = 2 * a + k
            sel = (group == g) & (pred['span'][:, a] == span) & (pred['span'][:, other(a)] <= BOX - 2).all(1)
            n = int(sel.sum())
            print(f'[coverage] span groups: axis {"xyz"[a]} span {span}: {n} units, by TMA {int(pred["fits"][sel].sum())}')
            assert n > 0, f'axis {a}: no unit spans exactly {span}'
            assert bool((pred['fits'][sel] == (span == 6)).all())


@pytest.mark.gpu
def test_tma_read_far_faces():
    """k0 bounds set to contracted coordinates of the face groups: a whole block lies exactly on each far face (unnormalised
    coordinate size - 1, base clamped to size - 2), later samples beyond it, and bricks run past the faces into TMA's zero
    fill.  The lower bound sits inside the domain too, so some samples lie below 0."""
    ro, rd = face_groups()
    probe = Scene(SHAPE, ro, rd, stepsize=0.48, seed=4)
    pts = probe.points_all()
    # the first contracted coordinate beyond 1.1 along each group's axis (outer shell)
    kmx = [float(pts[GROUP * a, int((pts[GROUP * a, :, a] > 1.1).nonzero()[0]), a]) for a in range(3)]
    assert all(1.1 < v < HI for v in kmx)
    sc = Scene(SHAPE, ro, rd, stepsize=0.48, seed=4, kmn=[-1.15] * 3, kmx=kmx)
    gat, _, _, pred, _ = check_scene(sc, 'far faces')
    size = torch.tensor(SHAPE, device=DEV)
    c = ((pred['coords'] + 1) / 2) * (size - 1).float()
    on_face = (c == (size - 1).float()) & (pred['x0'] == size - 2)
    n_face = [int(on_face[:, a].sum()) for a in range(3)]
    past = ((pred['lo'] + BOX - 1) > (size - 1)).any(1) & pred['fits']
    below = int((c < 0).any(1).sum())
    print(f'[coverage] far faces: samples exactly on the x / y / z far face {n_face}; {int(past.sum())} TMA bricks run past a far '
          f'face; {below} samples below 0')
    assert min(n_face) >= GROUP and int(past.sum()) > 0 and below > 0 and pred['n_out'] > 0


@pytest.mark.gpu
@pytest.mark.parametrize('stepsize,want_S', [(0.48, 144), (0.5, 138)])
def test_tma_read_sparse_survivors(stepsize, want_S):
    """fast_color_thres > 0 on a striped density plus a mask cache: blocks where no lane keeps a sample (the warp-uniform
    skip), whole segments without survivors and rays without any, under both cursor counts."""
    X = SHAPE[0]
    g = torch.Generator().manual_seed(9)
    dens = (ragged_planes(X)[:, None, None] + 0.3 * torch.randn(X, *SHAPE[1:], generator=g))[None, None]
    mask = torch.ones(24, 24, 24, dtype=torch.bool)
    mask[:, 16:, :] = False                        # y > ~0.47: masked out
    ro, rd = x_patch_groups(24, 10)
    sc = Scene(SHAPE, ro, rd, stepsize=stepsize, thres=1e-4, dens=dens, mask=mask, seed=5)
    assert sc.S == want_S
    gat, _, _, pred, st = check_scene(sc, f'sparse S={want_S}')
    empty_rays = sc.ro.shape[0] - int(torch.unique(gat['ray_id']).numel())
    print(f'[coverage] sparse S={want_S}: {empty_rays} rays without survivors')
    assert st['empty_blocks'] > 0 and st['empty_segments'] > 0 and empty_rays > 0 and st['n_seg'] > 1
    assert st['path'] == ('uint4' if want_S % 16 == 0 else 'byte')


@pytest.mark.gpu
def test_tma_read_at_benchmark_size():
    """The garden frame's model: DirectContractedVoxGO at bench.workload_kwargs('bicycle') (320^3, 12 channels, l2 norm),
    stepsize 1.045 (S = 512), the first, middle and last 8192-ray chunk of the 1600 x 1067 frame, every sample judged."""
    import bench
    from unboundednerfpytorch_b200 import march
    m, stepsize = bench.block_model(bench.SEED, DEV)
    kgrid = m.k0.grid.detach()
    assert tuple(kgrid.shape) == (1, 12, 320, 320, 320) and stepsize == 1.045
    S = march.t_schedule(m._world_len(), stepsize, m.bg_len, m.T_BOUNDARY, DEV).numel()
    assert S == 512
    H, W = bench.FRAME_HW
    ro, rd, _ = bench.frame_rays(DEV, H, W)
    chunk = 8192
    n_chunks = -(-ro.shape[0] // chunk)
    kmn, kmx = m.k0._bounds()
    kvals = kgrid.permute(0, 2, 3, 4, 1)
    for i in (0, n_chunks // 2, n_chunks - 1):
        a, b = ro[i * chunk:(i + 1) * chunk], rd[i * chunk:(i + 1) * chunk]
        gat, _ = run_march(lambda: m._march(a, b, stepsize, coherent=False)[0])
        tma, stats = run_march(lambda: m._march(a, b, stepsize, coherent=True)[0])
        with torch.no_grad():
            pts = m._sample_dense(a, b, stepsize)[0][gat['ray_id'], gat['step_id']]
        M = gat['ray_id'].numel()
        tag = f'garden chunk {i} of {n_chunks}'
        pred = judge_all(gat, tma, stats, pts, kmn, kmx, (320, 320, 320), kvals, kgrid, S, tag)
        st = structure(gat['ray_id'], gat['step_id'], a.shape[0], S, pred)
        print(f"[coverage] {tag}: {a.shape[0]} rays, S = {S} ({st['path']} cursor, {st['n_seg']} segments), {M} survivors; "
              f"units by TMA {pred['n_tma']} / fallback {pred['n_fallback']} (= TMA_STATS); {pred['n_out']} samples outside "
              f"[0, size - 1]")
        assert st['path'] == 'uint4' and st['n_seg'] == 8 and pred['n_tma'] > 4 * max(pred['n_fallback'], 1)


@pytest.mark.gpu
def test_coherent_render_matches_gather_and_forward_ops():
    """The model path: DirectContractedVoxGO.forward with render_kwargs['coherent_rays'] on an image-ordered frame and on random
    rays gives the gather kernel's records and its colours to fp32 rounding after the rgbnet, and the op-by-op composition's."""
    from tests.test_gpu_render import _model
    from tests.util import assert_close, seeded_rays
    from unboundednerfpytorch_b200 import rays as R
    m = _model(7)
    H, W = 48, 64
    K = np.array([[float(W), 0., W / 2], [0., float(W), H / 2], [0., 0., 1.]])
    c2w = torch.tensor([[1., 0., 0., 0.1], [0., 1., 0., -0.2], [0., 0., 1., 0.3]])
    ro, rd, vd = (t.view(-1, 3) for t in R.get_rays_of_a_view(H, W, K, c2w, False, False, False, False))
    rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, render_depth=True)
    ro2, rd2, vd2 = seeded_rays(3001, 5, DEV)
    res = {}
    for nm, (o, d, v) in (('coherent', (ro, rd, vd)), ('random', (ro2, rd2, vd2))):
        a, stats = run_march(lambda: m(o, d, v, coherent_rays=True, **rk))
        b, _ = run_march(lambda: m(o, d, v, **rk))
        res[nm] = stats
        assert torch.equal(a['ray_id'], b['ray_id']) and torch.equal(a['step_id'], b['step_id']), nm
        for k in ('weights', 'raw_alpha', 'raw_density', 't', 'alphainv_last'):
            assert torch.equal(a[k], b[k]), f'{nm} {k}'
        for k in ('raw_rgb', 'rgb_marched', 'depth'):
            assert_close(a[k], b[k], rtol=1e-5, atol=2e-6, what=f'{nm} {k}')
        if nm == 'coherent':
            with torch.no_grad():
                e = m.forward_ops(o, d, v, global_step=None, **rk)
            assert torch.equal(a['ray_id'], e['ray_id'])
            assert_close(a['rgb_marched'], e['rgb_marched'], rtol=1e-5, atol=2e-6, what='tma vs ops')
    print(f'[coverage] model path: blocks by TMA / fallback: coherent {res["coherent"]}, random {res["random"]}')
    assert res['coherent'][0] > 4 * max(res['coherent'][1], 1) and res['random'][1] > res['random'][0]


# ---- CPU: the judges reject each broken line of the kernel ---------------------------------------------------------------
def emulate_tma(ray_id, step_id, x0, f, kvals, S, fault=None):
    """k_march_feature_tma restated on the CPU for survivors sorted by (ray, step) with cells (x0, f): per unit the brick
    decision; the corners read from the zero-filled 8 x 8 x 8 brick at the unit's smallest base or from the grid; the sum in
    ATen's corner order; the record written at the ray's cursor.  Products and sums are rounded separately, as torch-CPU's grid
    sampler rounds them (the GPU kernel and torch-CUDA both fuse them), so the honest output is F.grid_sample on the CPU bit
    for bit.  fault breaks one line of the kernel.  Returns (records, (n_tma, n_fallback))."""
    _, X, Y, Z, C = kvals.shape
    M = ray_id.numel()
    pred = predict_units(ray_id, step_id, x0, S)
    lo, inv = pred['lo'], pred['inv']
    fits_u = (pred['span'] <= (BOX - 1 if fault == 'fits threshold off by one' else BOX - 2)).all(1)
    fits = fits_u[inv]
    grid = kvals[0]
    pad = torch.zeros(X + BOX, Y + BOX, Z + BOX, C)                    # TMA's zero fill beyond the far faces
    pad[:X, :Y, :Z] = grid
    r = torch.arange(BOX)
    brick = pad[lo[:, 0, None, None, None] + r[:, None, None], lo[:, 1, None, None, None] + r[None, :, None],
                lo[:, 2, None, None, None] + r[None, None, :]].reshape(-1, BOX ** 3, C)
    brick = torch.cat([brick, torch.zeros(brick.shape[0], 4 * BOX ** 3, C)], 1)     # what lies beyond one brick: not its data
    acc = torch.zeros(M, C)
    for corner in range(8):
        bx, by, bz = corner >> 2, (corner >> 1) & 1, corner & 1
        w = ((f[:, 2] if bz else 1 - f[:, 2]) * (f[:, 1] if by else 1 - f[:, 1])) * (f[:, 0] if bx else 1 - f[:, 0])
        dx, dy, dz = x0[:, 0] - lo[inv, 0] + bx, x0[:, 1] - lo[inv, 1] + by, x0[:, 2] - lo[inv, 2] + bz
        if fault == 'one corner one voxel off' and corner == 5:
            dz = dz + 1
        idx = (dx * BOX + dz) * BOX + dy if fault == 'y and z swapped in the brick index' else (dx * BOX + dy) * BOX + dz
        v_brick = brick[inv, idx]
        v_glob = grid[x0[:, 0] + bx, x0[:, 1] + by, x0[:, 2] + bz]
        acc = acc + torch.where(fits[:, None], v_brick, v_glob) * w[:, None]
    slot = torch.arange(M)
    if fault == 'survivor written to the next cursor slot':
        i = int(torch.nonzero(ray_id[1:] == ray_id[:-1])[M // 3 // 2])       # not its ray's last survivor
        slot[i] = i + 1
    out = dict(feat=torch.full((M, C), float('nan')), ray_id=torch.full((M,), -1), step_id=torch.full((M,), -1))
    for k, v in (('feat', acc), ('ray_id', ray_id), ('step_id', step_id)):
        for j in range(M):                    # in the kernel's order: a later survivor of the ray overwrites a stray write
            out[k][slot[j]] = v[j]
    if fault == "features in a neighbouring ray's slot":
        key = ray_id * S + step_id
        has_next = torch.nonzero(torch.isin(key + S, key))[:, 0]        # survivors whose next ray keeps the same step
        i = int(has_next[has_next.numel() // 2])
        j = int(torch.nonzero(key == key[i] + S)[0])
        out['feat'][j] = acc[i]
    return out, (int(fits_u.sum()), int((~fits_u).sum()))


def checker_scene():
    """A small CPU scene (12 x 10 x 14 grid, 4 channels, 70 rays x S = 22 steps) of survivors in image-like groups: group 0's
    lanes spread over exactly 6 + 1 y bases (one brick), group 1's over 7 + 1 z bases (the fallback), a ragged group of 6
    random rays; a quarter of the samples dropped and one of group 0's blocks empty."""
    shape, C, N, S = (12, 10, 14), 4, 70, 22
    g = torch.Generator().manual_seed(21)
    lane = torch.arange(N) % GROUP
    s = torch.arange(S, dtype=torch.float32)
    c = torch.empty(N, S, 3)
    l0 = lane[:GROUP, None].float() / (GROUP - 1)
    c[:GROUP] = torch.stack(torch.broadcast_tensors(1.3 + 0.35 * s, 1.5 + 6.0 * l0, 3.2 + 0.1 * s), -1)
    c[GROUP:2 * GROUP] = torch.stack(torch.broadcast_tensors(2.4 + 0.3 * s, torch.full_like(l0, 4.2), 1.5 + 7.0 * l0), -1)
    c[2 * GROUP:] = torch.rand(N - 2 * GROUP, S, 3, generator=g) * (torch.tensor(shape) - 1)
    keep = torch.rand(N, S, generator=g) < 0.75
    keep[:GROUP, 8:12] = False
    ray_id, step_id = torch.nonzero(keep, as_tuple=True)
    pts = (c / (torch.tensor(shape) - 1) * 2 - 1)[ray_id, step_id]           # world = normalised coordinates on [-1, 1]
    kvals = torch.randn(1, *shape, C, generator=g)
    return shape, S, ray_id, step_id, pts, kvals


def test_checker_rejects_faults():
    """The CPU restatement of the kernel passes all four judges; each broken line fails the judge written for it: a y / z swap
    in the brick index and one corner read one voxel off (judges 2 and 3), a survivor written to the next cursor slot (judge 1),
    the fits threshold off by one so that a span of 7 takes a brick (judge 4), one sample's features in the neighbouring ray's
    slot (judges 2 and 3)."""
    shape, S, ray_id, step_id, pts, kvals = checker_scene()
    mn, mx = [-1.0] * 3, [1.0] * 3
    coords = slab_coords(pts, mn, mx, 0)
    x0, f = cells(coords, shape)
    x0, f = x0[0], f[0]
    pred = predict_units(ray_id, step_id, x0, S)
    span6 = int(((pred['span'] == 6).any(1) & pred['fits']).sum())
    span7 = int(((pred['span'] == 7).any(1) & (pred['span'] <= 7).all(1)).sum())
    n_units = -(-70 // GROUP) * -(-S // BLOCK)
    assert span6 > 0 and span7 > 0 and pred['units'].numel() < n_units and pred['n_tma'] > 0
    kgrid = kvals.permute(0, 4, 1, 2, 3).contiguous()
    want_gs = grid_sample_ref(kgrid, pts, mn, mx)
    outside = outside_faces(coords[0], shape)
    honest = dict(ray_id=ray_id, step_id=step_id)
    judges = {
        1: lambda got, st: judge_records(got, honest, 'checker'),
        2: lambda got, st: judge_grid_sample(got['feat'], want_gs, outside, 'checker'),
        3: lambda got, st: judge_fp64(got['feat'], x0[None], f[None], kvals, 'checker'),
        4: lambda got, st: judge_counts(st, pred, 'checker'),
    }

    def failing(fault):
        got, st = emulate_tma(ray_id, step_id, x0, f, kvals, S, fault)
        bad = []
        for k, fn in judges.items():
            try:
                fn(got, st)
            except AssertionError:
                bad.append(k)
        return bad

    assert failing(None) == [], 'the honest restatement fails a judge'
    expect = {'y and z swapped in the brick index': {2, 3}, 'one corner one voxel off': {2, 3},
              'survivor written to the next cursor slot': {1}, 'fits threshold off by one': {4},
              "features in a neighbouring ray's slot": {2, 3}}
    seen = {}
    for fault, want in expect.items():
        seen[fault] = failing(fault)
        assert want <= set(seen[fault]), f'{fault}: judges {seen[fault]} fail, expected {sorted(want)}'
    print('[tma checker] ' + '; '.join(f'{k}: judges {v} fail' for k, v in seen.items()))
