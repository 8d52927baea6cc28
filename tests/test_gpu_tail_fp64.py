"""The training-step tail (csrc/grid_sweep.cu): the total-variation gradient (k_total_variation_stream<dense>,
k_total_variation<dense, false>), the three Adam kernels (k_adam_vec4 / k_adam_scalar<mode>), the fused two-sweep tail
(k_adam_zero_*<mode, zero>), the ping-pong sweep (k_tv_adam_stream<dense, mode, write_grad>) and the multi-GPU peer sweep
(k_tv_adam_peer<dense, mode, N>), at the benchmarked grid shapes and, for the peer sweep, with 1, 2, 4 and 8 "ranks" on one GPU.

Every case has two judges.
  (a) Bit for bit against the reference's own CUDA (oracle/_ref: total_variation_cuda, adam_upd_cuda) on contiguous copies of the
      same fp32 inputs.  For the ping-pong and peer sweeps the expected result is the rank-ordered fp32 mean
      ((g0 + g1) + ...) * (1/N) (what k_tv_adam_peer computes), then the reference TV, then the reference (masked) Adam.  Params,
      both moments and, where the kernel writes it, the gradient are compared; NaN positions must match.  Non-finite inputs (a
      diverged step: +-inf and NaN in params and gradients, -0.0 and denormal gradients in masked mode) are judged by (a) only.
  (b) Within a per-element bound of an fp64 restatement of the reference's formulas, with the fp32 inputs b1, b2, lr, eps and the
      TV weights taken as exact.  u = 2^-24, gamma_k = k u / (1 - k u).
      TV.  t = sum of w clamp(p - q, -1, 1) over the six neighbours, weights wz / 6 on k, wy / 6 on j and wz / 6 on i
      (total_variation_kernel.cu; wx is unused).  Per term: fl(p - q) is u of |p - q|, and clamp never enlarges that (a
      difference beyond +-1 rounds to at least 1 in magnitude and clamps exactly), the fp32 w / 6 is u, the product u: gamma_3 of
      |term|.  The six adds into 0 and the add to g are recursive summation, gamma_6 of |g| + sum|terms|.  Bound:
          B_tv = gamma_7 (|g| + A) + gamma_3 A,   A = sum |terms|.
      Contraction into an FMA only removes a rounding.  In sparse mode an element with g == 0 (either sign) must keep its bits.
      Peer mean.  N - 1 rank-ordered adds and an exact power-of-two scale: within (N - 1) u sum_r |g_r| / N of the fp64 mean.
      This error eg and B_tv (where TV applies) are carried into Adam as the gradient's error.
      Adam.  m* = b1 m + (1 - b1) g, v* = b2 v + (1 - b2) g^2, s* = lr sqrt(1 - b2^t) / (1 - b1^t), p* = p - s* m* / (sqrt(v*) +
      eps) (times perlr in the per-voxel-lr mode).  The kernel's m is fma(m, b1, fl(fl(1 - b1) g)): gamma_3 of A_m = |b1 m| +
      |(1 - b1) g|, plus (1 - b1) eg; v is fma(v, b2, fl(fl(fl(1 - b2) g) g)): gamma_4 of A_v = |b2 v| + (1 - b2) g^2, plus
      (1 - b2)(2 |g| eg + eg^2).  These are magnitudes of the addends, not of m* and v*, which can cancel.  The host step size
      (powf and sqrtf in fp32, make_hyper) is within E_s = 1.01 u (b2^t / (1 - b2^t) + 2 b1^t / (1 - b1^t) + 4.5) relative: one
      ulp (2u) per powf amplified by b^t / (1 - b^t) in 1 - b^t, a half for the square root, and four roundings; at t = 1 with
      b2 = 0.99 that is 121 u.  The update is bounded by interval arithmetic over m in [m* - em, m* + em], v in [v* - ev, v* + ev],
      s in s* [1 - E_s, 1 + E_s], with gamma_2 more on the denominator (sqrt, + eps) and gamma_3 of the result (products, divide):
      ed = max distance of s m / den over that box from s* m* / den* + gamma_3 max|d|, and p within ed + u (|p| + |d*| + ed).
      Masked mode: the skip decision must equal "the fp32 TV-augmented gradient == 0", -0.0 included (skipped elements keep the
      bits of p, m and v; the fp32 augmented gradient is the reference's).  Elements where fp64 and fp32 disagree on zero-ness
      are judged by (a) only.

Worst ratios seen on an H100 80GB HBM3, |got - fp64| over the bound (1.0 = at the bound), over all cases: TV
gradient 0.43; ping-pong p 0.96, m 0.33, v 0.34, gradient 0.34; peer p 0.93, m 0.34, v 0.36; Adam p 0.996, m 0.63, v 0.70;
fused tail p 0.83, m 0.39, v 0.52, gradient 0.24; slab slices p 0.50, m 0.27, v 0.24, gradient 0.18.  The p ratios near 1 are
the last rounding, fl(p - d) within u |p - d|, which is sharp for a result just above a power of two when d is small.  Every
(a) comparison was bit-identical.  The file ran in 19 s (H100 80GB HBM3, 700 W power limit); the truck peer
cases peaked at 19.1 GiB of device memory.

Cases.  The kernel each call takes is named by grid_sweep.cu's dispatch conditions restated here (tv_route, adam_route and the
template arguments of the ping-pong and peer launchers); test_launch_constants_match_sources keeps the restated constants and
gates in step with the sources, and test_zz_every_instantiation_ran requires every one of the 42 instantiations listed in
EXPECTED to be taken by some case.
  * streaming TV: row4 = Z C / 4 at 31 (falls back), 32, 33, 459, 960, 1024, 1025 (falls back); C in {1, 3, 4, 9, 12, 15, 16}
    (C = 1, 3, 9, 15 take the element kernel); sz_i in {7 (falls back), 8, 15, 16, 17, 153, 320}, so 1 to 20 i-segments with a
    ragged last one; ragged last j-tiles; lead 1 and 9; a 4-byte-misaligned view (falls back); dense and sparse; the full
    bicycle k0 grid [1, 12, 320, 320, 320] (two columns per thread, 7 ragged i-segments).
  * ping-pong: all 8 (dense, masked, write_grad) combinations at row4 32, 459, 512, steps 1, 2, 3, 50, 20 000; row4 31 and
    513 refused by tv_adam_pingpong_supported and by ubn_tv_adam_pingpong; MaskedAdam.step_fused_tv(write_grad=False), the
    benchmark's ping-pong leg, bit-identical to TV + step() with .grad still the raw gradient.
  * peer sweep on one GPU: N distinct gradient buffers, N distinct output buffers pre-filled with a NaN sentinel, per-rank
    moments, every rank's range launched on one stream (also in reverse rank order).  Every output buffer must equal the
    single-process mean-gradient step on the union of the ranges, each rank's moments change only on its own planes, and no
    plane outside the ranges changes.  Ranges: dist.shard_range, single planes, a range starting at i = sz_i - 1, one ending
    at i = 0 of the next slab, ranges shorter than 8 planes, an empty range, the whole grid.  Truck's k0 grid
    [9, 12, 153, 153, 153] (row4 459, one row per tile, odd sz_i, segments across slab boundaries) at N = 1 and N = 4, with
    the gradient and output buffers repeated across ranks and one moment pair shared by the four disjoint ranges, judged slab
    by slab; and dist.PeerTail at world 1 through its real step() on the truck-shaped FourierGridModel.
  * Adam: n = 1, n mod 4 in {0, 1, 2, 3}, truck's density element count 9 * 153^3 (vec4 body + a one-element scalar tail);
    storage offsets 0 to 3 and a misaligned perlr alone; the three modes, per-voxel lr through set_pervoxel_lr counts;
    tv_adam_fused for every tv_mode x adam_mode x zero_grad; the slab slices dist.reduce_tv_step passes for an odd X Y Z.

test_checker_rejects_faults (CPU) runs judge (b) on an fp32 CPU emulation of the tail (accepted) and on nine faults injected
into it, each rejected: wy on the i axis, the halo plane dropped at a segment start, an i neighbour read from the
already-updated buffer, bias correction at t + 1, eps inside the square root, the masked skip keyed on the raw gradient, the
rank sum without 1/N, a peer range one plane short, and -0.0 treated as non-zero."""
import itertools
import math
import os
import re

import numpy as np
import pytest
import torch

DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'unboundednerfpytorch_b200', 'csrc')
U = 2.0 ** -24
TVS_THREADS, TVS_COLS, TA_THREADS = 512, 2, 512          # kTvsThreads, kTvsCols, kTaThreads (grid_sweep.cu)
W = (0.05, 0.02, 0.03)                                   # wx (unused), wy, wz
B1, B2, LR, EPS = 0.9, 0.99, 0.1, 1e-8
SENTINEL = 0x7FC0DEAD                                    # a quiet NaN no kernel produces
CHUNK = 12_000_000                                       # elements per fp64 block of the judge
TRUCK_K0 = (9, 12, 153, 153, 153)
BICYCLE_K0 = (1, 12, 320, 320, 320)
TF = ('true', 'false')
EXPECTED = ({f'k_total_variation_stream<{d}>' for d in TF}
            | {f'k_total_variation<{d}, false>' for d in TF}
            | {f'k_tv_adam_stream<{d}, {m}, {w}>' for d in TF for m in (0, 1) for w in TF}
            | {f'k_tv_adam_peer<{d}, {m}, {n}>' for d in TF for m in (0, 1) for n in (1, 2, 4, 8)}
            | {f'k_adam_{k}<{m}>' for k in ('vec4', 'scalar') for m in (0, 1, 2)}
            | {f'k_adam_zero_{k}<{m}, {z}>' for k in ('vec4', 'scalar') for m in (0, 1) for z in TF})
RAN = set()
WORST = {}


def f32(x):
    return float(np.float32(x))


def gam(k):
    return k * U / (1 - k * U)


def _cl(b):
    return 'true' if b else 'false'


# ---- layouts and data --------------------------------------------------------------------------------------------------------
def mem(t, layout):
    """The memory-order (contiguous) view of a logical [P,C,X,Y,Z] grid."""
    return t.permute(0, 2, 3, 4, 1) if layout == 'cl' else t


def alloc(shape, layout, device, offset=0):
    """Empty fp32 [P,C,X,Y,Z] grid, channels-last ('cl': memory [P,X,Y,Z,C]) or contiguous ('c'), `offset` floats into its
    storage."""
    P, C, X, Y, Z = shape
    n = P * C * X * Y * Z
    buf = torch.empty(n + offset, dtype=torch.float32, device=device)[offset:]
    if layout == 'cl':
        return buf.view(P, X, Y, Z, C).permute(0, 4, 1, 2, 3)
    return buf.view(shape)


def sentinel_like(t):
    out = torch.empty_like(t, memory_format=torch.preserve_format)
    out.view(torch.int32).fill_(SENTINEL)
    return out


def make(kind, shape, layout, seed, device=DEV, offset=0, specials=False):
    """Seeded fp32 data in the given layout.
    param: N(0, 0.6^2) (neighbour differences beyond +-1 are common, so the clamp binds), with constant patches where the TV
           term is exactly 0; grad: 1e-2 N(0, 1) on half the elements, 0 elsewhere, -0.0 on some of the zeros;
    m: 1e-2 N(0, 1); v: 1e-4 U(0, 1)^2 (small v makes eps matter); perlr: U(0, 1).
    specials: +-inf and NaN in params, +-inf, NaN, -0.0 and denormals in gradients."""
    t = alloc(shape, layout, device, offset)
    tm = mem(t, layout)
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(tm.shape, generator=g, device=device)
    if kind == 'param':
        P, C, X, Y, Z = shape
        ax = [torch.arange(s, device=device) for s in (X, Y, Z)]
        ix, iy, iz = ax[0].view(1, X, 1, 1), ax[1].view(1, 1, Y, 1), ax[2].view(1, 1, 1, Z)
        flat = ((ix // 3 + iy // 2 + iz // 3) % 5 == 0)
        flat = flat.unsqueeze(-1) if layout == 'cl' else flat.unsqueeze(1)
        x = torch.where(flat, torch.tensor(0.375, device=device), x * 0.6)
    elif kind == 'grad':
        r = torch.rand(tm.shape, generator=g, device=device)
        x = torch.where(r > 0.5, x * 1e-2, torch.where(r < 0.05, torch.tensor(-0.0, device=device), torch.tensor(0.0, device=device)))
    elif kind == 'm':
        x = x * 1e-2
    elif kind == 'v':
        x = torch.rand(tm.shape, generator=g, device=device) ** 2 * 1e-4
    elif kind == 'perlr':
        x = torch.rand(tm.shape, generator=g, device=device)
    if specials:
        r = torch.rand(tm.shape, generator=g, device=device)
        vals = ([math.inf, -math.inf, math.nan] if kind == 'param' else
                [math.inf, -math.inf, math.nan, -0.0, 1e-40, -3e-42] if kind == 'grad' else [])
        for k, val in enumerate(vals):
            x = torch.where((r >= k * 2e-3) & (r < (k + 1) * 2e-3), torch.tensor(val, device=device), x)
    tm.copy_(x)
    return t


def mismatches(a, b):
    """Elements whose fp32 bits differ (any NaN equals any NaN), for logical tensors of any layout."""
    same = (a.view(torch.int32) == b.view(torch.int32)) | (torch.isnan(a) & torch.isnan(b))
    return int((~same).sum())


def is_sentinel(a):
    return a.view(torch.int32) == SENTINEL


# ---- which kernel a call takes ----------------------------------------------------------------------------------------------
def launched(fn, expect):
    """Run fn, which by the restated dispatch conditions below launches exactly the grid_sweep.cu kernels `expect`
    (e.g. 'k_tv_adam_peer<true, 1, 4>'), and record them for test_zz_every_instantiation_ran."""
    fn()
    RAN.update(expect)


def sweep_layout(shape, layout):
    """(lead, inner) ops._sweep_layout passes for a [P,C,X,Y,Z] grid (a C = 1 grid is contiguous in either layout)."""
    P, C = shape[:2]
    return (P, C) if layout == 'cl' and C > 1 else (P * C, 1)


def tv_route(shape, layout, *tensors):
    """ubn_total_variation_add_grad's choice: launch_tv_stream's gates, else the 32-bit element kernel."""
    X, Z = shape[2], shape[4]
    _, inner = sweep_layout(shape, layout)
    aligned = all(t.data_ptr() % 16 == 0 for t in tensors)
    row4 = Z * inner // 4
    return 'stream' if (inner % 4 == 0 and X >= 8 and aligned and 32 <= row4 <= TVS_THREADS * TVS_COLS) else 'element'


def tv_kernel(route, dense):
    return f'k_total_variation_stream<{_cl(dense)}>' if route == 'stream' else f'k_total_variation<{_cl(dense)}, false>'


def adam_route(n, tensors, prefix, tmpl):
    """launch_adam / launch_adam_zero: a float4 body when every operand is 16-byte aligned, a scalar kernel for the rest."""
    n4 = n // 4 if all(t.data_ptr() % 16 == 0 for t in tensors) else 0
    out = set()
    if n4:
        out.add(f'{prefix}_vec4<{tmpl}>')
    if n4 * 4 < n:
        out.add(f'{prefix}_scalar<{tmpl}>')
    return out


# ---- the reference's CUDA ---------------------------------------------------------------------------------------------------
def ref_tv(p, g, w, dense):
    from tests.util import ref_cuda
    out = g.contiguous().clone()
    ref_cuda('total_variation_cuda').total_variation_add_grad(p.contiguous(), out, *w, bool(dense))
    return out


def ref_adam(p, g, m, v, t, mode, perlr=None):
    from tests.util import ref_cuda
    mod = ref_cuda('adam_upd_cuda')
    pc, mc, vc = (x.contiguous().clone() for x in (p, m, v))
    gc = g.contiguous()
    if mode == 0:
        mod.adam_upd(pc, gc, mc, vc, t, B1, B2, LR, EPS)
    elif mode == 1:
        mod.masked_adam_upd(pc, gc, mc, vc, t, B1, B2, LR, EPS)
    else:
        mod.adam_upd_with_perlr(pc, gc, mc, vc, perlr.contiguous(), t, B1, B2, LR, EPS)
    return pc, mc, vc


def rank_mean(grads):
    """The fp32 mean in k_tv_adam_peer's order: ((g0 + g1) + ...) * (1/N)."""
    s = grads[0].clone()
    for g in grads[1:]:
        s = s + g
    return s * (1.0 / len(grads)) if len(grads) > 1 else s


# ---- judge (b): fp64 restatement with per-element bounds ----------------------------------------------------------------------
def tv64(p, wy, wz):
    """fp64 TV term and sum of |terms| of a [C, nI, Y, Z] fp64 block (faces of the block have no neighbour)."""
    t, a = torch.zeros_like(p), torch.zeros_like(p)
    for dim, w in ((1, f32(wz) / 6), (2, f32(wy) / 6), (3, f32(wz) / 6)):
        n = p.shape[dim]
        if n < 2:
            continue
        c = (p.narrow(dim, 1, n - 1) - p.narrow(dim, 0, n - 1)).clamp(-1, 1) * w
        t.narrow(dim, 0, n - 1).sub_(c)
        t.narrow(dim, 1, n - 1).add_(c)
        a.narrow(dim, 0, n - 1).add_(c.abs())
        a.narrow(dim, 1, n - 1).add_(c.abs())
    return t, a


def adam64(p, g, m, v, eg, t, perlr=None):
    """fp64 Adam step and the bounds (ep, em, ev) of the fp32 kernel's p, m, v; eg = error bound of the fp32 gradient."""
    b1, b2, lr, eps = f32(B1), f32(B2), f32(LR), f32(EPS)
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    P1, P2 = b1 ** t, b2 ** t
    s = lr * math.sqrt(1 - P2) / (1 - P1)
    es = 1.01 * U * (P2 / (1 - P2) + 2 * P1 / (1 - P1) + 4.5)
    se = s if perlr is None else s * perlr
    em = gam(3) * ((b1 * m).abs() + ((1 - b1) * g).abs()) + (1 - b1) * eg
    ev = gam(4) * ((b2 * v).abs() + (1 - b2) * g * g) + (1 - b2) * (2 * g.abs() * eg + eg * eg)
    d = se * m1 / (v1.sqrt() + eps)
    m_lo, m_hi = m1 - em, m1 + em
    den_lo = ((v1 - ev).clamp_min(0).sqrt() + eps) * (1 - gam(2))
    den_hi = ((v1 + ev).sqrt() + eps) * (1 + gam(2))
    s_lo, s_hi = se * (1 - es), se * (1 + es)
    d_hi = torch.where(m_hi >= 0, s_hi * m_hi / den_lo, s_lo * m_hi / den_hi)
    d_lo = torch.where(m_lo <= 0, s_hi * m_lo / den_lo, s_lo * m_lo / den_hi)
    ed = torch.maximum(d_hi - d, d - d_lo) + gam(3) * torch.maximum(d_lo.abs(), d_hi.abs())
    ep = ed + U * (p.abs() + d.abs() + ed)
    return p - d, m1, v1, ep, em, ev


def _ratio(got, want, bound, sel):
    err = (got.double() - want).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    r = torch.where(sel, r, torch.zeros_like(r))
    return float(r.max()) if r.numel() else 0.0


def judge_tail(fails, key, inp, got, planes=None, zero32=None):
    """Judge (b) of one tail call on a logical [P,C,X,Y,Z] grid, block by block.
    inp: p, grads (list, rank order), w (None: no TV), dense, mode (None: TV only; 0 plain, 1 masked, 2 per-voxel lr), t, m, v,
         perlr.  got: g (written gradient) and / or p, m, v.  planes: bool [P*X] of the (slab, i) planes the call updated
         (default all).  zero32: bool grid, the fp32 TV-augmented gradient == 0 (masked mode)."""
    p, grads = inp['p'], inp['grads']
    N = len(grads)
    P, C, X, Y, Z = p.shape
    w, mode, dense = inp.get('w'), inp.get('mode'), inp.get('dense', True)
    ni = max(1, CHUNK // (C * Y * Z))
    for l in range(P):
        for i0 in range(0, X, ni):
            i1 = min(X, i0 + ni)
            if planes is not None:
                keep = planes[l * X + i0:l * X + i1].view(1, -1, 1, 1)
                if not bool(keep.any()):
                    continue
            else:
                keep = torch.ones(1, i1 - i0, 1, 1, dtype=torch.bool, device=p.device)
            blk = lambda x: x[l, :, i0:i1]
            gs = [blk(g) for g in grads]
            mean32 = rank_mean(gs)
            g64 = sum(g.double() for g in gs) / N
            gabs = sum(g.double().abs() for g in gs) / N
            eg = (N - 1) * U * gabs
            if w is not None:
                h0, h1 = max(i0 - 1, 0), min(i1 + 1, X)
                tv, a = tv64(p[l, :, h0:h1].double(), w[1], w[2])
                tv, a = tv[:, i0 - h0:i1 - h0], a[:, i0 - h0:i1 - h0]
                gate = torch.ones_like(keep) if dense else mean32 != 0
                aug = g64 + torch.where(gate, tv, torch.zeros_like(tv))
                eg = eg + torch.where(gate, gam(7) * (gabs + a) + gam(3) * a, torch.zeros_like(a))
            else:
                gate = torch.zeros_like(keep)
                aug = g64
            sel = keep.expand(aug.shape)

            def J(what, g_, want, bound, s):
                r = _ratio(g_, want, bound, s)
                WORST[f'{key} {what}'] = max(WORST.get(f'{key} {what}', 0.0), r)
                if r > 1:
                    fails.append(f'{key} {what} (slab {l}, i {i0}..{i1}): {r:.3e} of its bound')

            if got.get('g') is not None:
                gg = blk(got['g'])
                J('grad', gg, aug, eg, sel & gate)
                n_bad = int((sel & ~gate & ~(gg.view(torch.int32) == mean32.view(torch.int32))).sum())
                if n_bad:
                    fails.append(f'{key} grad: {n_bad} elements outside the TV gate changed (slab {l}, i {i0}..{i1})')
            if mode is None:
                continue
            pp, mm, vv = blk(p), blk(inp['m']), blk(inp['v'])
            lr_e = blk(inp['perlr']).double() if inp.get('perlr') is not None else None
            pw, mw, vw, ep, em, ev = adam64(pp.double(), aug, mm.double(), vv.double(), eg, inp['t'], lr_e)
            upd = sel
            if mode == 1:
                z = blk(zero32)
                still = sel & z
                for what, a_, b_ in (('p', blk(got['p']), pp), ('m', blk(got['m']), mm), ('v', blk(got['v']), vv)):
                    n_bad = int((still & ~(a_.view(torch.int32) == b_.view(torch.int32))).sum())
                    if n_bad:
                        fails.append(f'{key} {what}: {n_bad} skipped elements changed (slab {l}, i {i0}..{i1})')
                upd = sel & ~z & (aug != 0)
            J('p', blk(got['p']), pw, ep, upd)
            J('m', blk(got['m']), mw, em, upd)
            J('v', blk(got['v']), vw, ev, upd)


# ---- CPU emulation of the tail (for the checker self-test) ----------------------------------------------------------------------
def _neighbour(p, dim, side):
    n = p.shape[dim]
    q = torch.zeros_like(p)
    ex = torch.zeros(n, dtype=torch.bool)
    if side < 0:
        q.narrow(dim, 1, n - 1).copy_(p.narrow(dim, 0, n - 1))
        ex[1:] = True
    else:
        q.narrow(dim, 0, n - 1).copy_(p.narrow(dim, 1, n - 1))
        ex[:-1] = True
    shape = [1] * p.dim()
    shape[dim] = n
    return q, ex.view(shape)


def step_size32(t):
    f = np.float32
    return float(f(LR) * np.sqrt(f(1) - np.power(f(B2), f(t))) / (f(1) - np.power(f(B1), f(t))))


def emulate(inp, fault=None, seg_starts=(), ranges=None):
    """fp32 CPU restatement of the peer / ping-pong tail (TV on the rank-ordered mean, then (masked) Adam) with one fault."""
    p, m, v = inp['p'], inp['m'], inp['v']
    s = inp['grads'][0].clone()
    for g in inp['grads'][1:]:
        s = s + g
    if len(inp['grads']) > 1 and fault != 'no_inv_n':
        s = s * (1.0 / len(inp['grads']))
    wy, wz = (torch.tensor(x, dtype=torch.float32) / 6 for x in inp['w'][1:])
    upd_p = emulate(inp, ranges=ranges)['p'] if fault == 'updated' else None
    add = torch.zeros_like(p)
    for dim, w in ((4, wz), (3, wy), (2, wy if fault == 'wy_on_i' else wz)):
        for side in (-1, 1):
            q, ex = _neighbour(p, dim, side)
            if dim == 2 and side < 0 and fault == 'updated':
                q, _ = _neighbour(upd_p, dim, side)
            if dim == 2 and side < 0 and fault == 'halo':
                q[:, :, list(seg_starts)] = 0
            add = add + torch.where(ex, w * (p - q).clamp(-1, 1), torch.zeros_like(p))
    nz = (s != 0) | (torch.signbit(s) if fault == 'neg_zero' else torch.zeros_like(s, dtype=torch.bool))
    gate = torch.ones_like(nz) if inp['dense'] else nz
    aug = torch.where(gate, s + add, s)
    h = step_size32(inp['t'] + (1 if fault == 'bias_t1' else 0))
    b1, b2, eps = (torch.tensor(x, dtype=torch.float32) for x in (B1, B2, EPS))
    m1 = m * b1 + (1 - b1) * aug
    v1 = v * b2 + ((1 - b2) * aug) * aug
    den = torch.sqrt(v1 + eps) if fault == 'eps_in_sqrt' else torch.sqrt(v1) + eps
    p1 = p - (h * m1) / den
    if inp['mode'] == 1:
        key = s if fault == 'mask_raw' else aug
        skip = (key == 0) & ~(torch.signbit(key) if fault == 'neg_zero' else torch.zeros_like(key, dtype=torch.bool))
        p1, m1, v1 = torch.where(skip, p, p1), torch.where(skip, m, m1), torch.where(skip, v, v1)
    if ranges is not None:
        P, C, X = p.shape[:3]
        planes = torch.zeros(P * X, dtype=torch.bool)
        for k, (lo, hi) in enumerate(ranges):
            planes[lo:hi - (1 if fault == 'range_short' and k == len(ranges) - 1 else 0)] = True
        pm = planes.view(P, 1, X, 1, 1)
        p1 = torch.where(pm, p1, sentinel_like(p))
        m1, v1 = torch.where(pm, m1, m), torch.where(pm, v1, v)
    return dict(p=p1, m=m1, v=v1, g=aug)


# ---- CPU tests --------------------------------------------------------------------------------------------------------------
def test_launch_constants_match_sources():
    """The routes above restate grid_sweep.cu's launch constants and gates and ops.tv_adam_pingpong_supported; they must stay in
    step with the sources, and EXPECTED must list exactly the instantiations the launchers can reach."""
    src = open(os.path.join(CSRC, 'grid_sweep.cu')).read()
    ops_src = open(os.path.join(ROOT, 'unboundednerfpytorch_b200', 'ops.py')).read()
    assert int(re.search(r'constexpr int kTvsThreads = (\d+);', src).group(1)) == TVS_THREADS
    assert int(re.search(r'constexpr int kTvsCols = (\d+);', src).group(1)) == TVS_COLS
    assert int(re.search(r'constexpr int kTaThreads = (\d+);', src).group(1)) == TA_THREADS
    assert "if (!tv_stream_enabled() || inner % 4 != 0 || sz_i < 8) return false;" in src
    assert 'if ((((uintptr_t)param) | ((uintptr_t)grad)) & 15) return false;' in src
    assert 'if (row4 > kTvsThreads * kTvsCols || row4 < 32) return false;' in src
    assert src.count('if (row4 > kTaThreads || row4 < 32) return finish(cudaErrorInvalidValue);') == 2
    assert src.count('const int64_t n4 = aligned ? n / 4 : 0;') == 2
    assert 'const bool wide = g.n >= (1ll << 31);' in src
    assert 'return C % 4 == 0 and X >= 8 and 32 <= Z * C // 4 <= 512' in ops_src
    assert len(re.findall(r'UBN_TA\((true|false), [01], (true|false)\)', src)) == 8
    assert len(re.findall(r'case [1248]: UBN_TP\(D, M, [1248]\)|default: UBN_TP\(D, M, 8\)', src)) == 4
    assert len(EXPECTED) == 2 + 2 + 8 + 16 + 6 + 8


def _cpu_case(fault):
    """A small CPU grid [2, 4, 20, 5, 6] (sz_i = 20, segments of 8 planes) and the tail inputs the fault needs to show."""
    shape = (2, 4, 20, 5, 6)
    N = 2 if fault in ('no_inv_n', 'range_short') else 1
    mk = lambda kind, s: make(kind, shape, 'c', s, device='cpu')
    inp = dict(p=mk('param', 1), grads=[mk('grad', 2 + r) for r in range(N)], m=mk('m', 7), v=mk('v', 8), w=W,
               dense=fault not in ('neg_zero',), mode=1, t=2 if fault != 'bias_t1' else 1)
    ranges = [(0, 13), (13, 40)] if N == 2 else None
    return inp, ranges


@pytest.mark.parametrize('fault', [None, 'wy_on_i', 'halo', 'updated', 'bias_t1', 'eps_in_sqrt', 'mask_raw', 'no_inv_n',
                                   'range_short', 'neg_zero'])
def test_checker_rejects_faults(fault):
    """Judge (b) accepts the CPU emulation of the tail and rejects each injected fault."""
    inp, ranges = _cpu_case(fault)
    good = emulate(inp, ranges=ranges)
    got = emulate(inp, fault, seg_starts=(8, 16), ranges=ranges)
    if ranges is not None:
        planes = torch.zeros(inp['p'].shape[0] * inp['p'].shape[2], dtype=torch.bool)
        for lo, hi in ranges:
            planes[lo:hi] = True
        got = dict(p=got['p'], m=got['m'], v=got['v'])
    else:
        planes = None
    fails = []
    judge_tail(fails, 'cpu', inp, got, planes=planes, zero32=good['g'] == 0)
    if fault is None:
        assert not fails, fails
    else:
        assert fails, f'fault {fault} was accepted'


# ---- GPU: streaming and element TV ----------------------------------------------------------------------------------------------
TV_CASES = [  # (shape, layout, offset, route)
    ((1, 4, 9, 5, 31), 'cl', 0, 'element'),        # row4 31
    ((1, 4, 9, 5, 32), 'cl', 0, 'stream'),         # row4 32, one i-segment
    ((9, 12, 8, 40, 11), 'cl', 0, 'stream'),       # row4 33, lead 9, sz_i 8, tj 31: ragged last j-tile
    ((1, 12, 17, 41, 153), 'cl', 0, 'stream'),     # row4 459 (truck), tj 2, ragged last j-tile (1 row), sz_i 17
    ((9, 12, 153, 2, 153), 'cl', 0, 'stream'),     # truck's row4 and sz_i, lead 9: 9 segments of 17 planes
    ((1, 12, 16, 3, 320), 'cl', 0, 'stream'),      # row4 960 (bicycle): two columns per thread, one segment
    ((1, 12, 320, 2, 320), 'cl', 0, 'stream'),     # row4 960, sz_i 320: 20 segments of 16
    ((1, 16, 15, 5, 256), 'cl', 0, 'stream'),      # row4 1024, sz_i 15
    ((1, 16, 16, 7, 8), 'cl', 0, 'stream'),        # C 16, row4 32, sz_i 16
    ((9, 4, 17, 6, 40), 'cl', 0, 'stream'),        # lead 9, sz_i 17: 1 segment
    ((1, 4, 8, 3, 1025), 'cl', 0, 'element'),      # row4 1025
    ((2, 1, 153, 20, 33), 'c', 0, 'element'),      # C 1 (density)
    ((1, 3, 20, 9, 41), 'cl', 0, 'element'),       # C 3 (DirectMPIGO / narrow k0)
    ((1, 9, 12, 7, 30), 'cl', 0, 'element'),       # C 9
    ((1, 15, 10, 6, 20), 'cl', 0, 'element'),      # C 15
    ((1, 12, 7, 5, 40), 'cl', 0, 'element'),       # sz_i 7
    ((1, 12, 16, 5, 40), 'cl', 1, 'element'),      # 4-byte-misaligned view
]


def _tv_case(shape, layout, offset, route, dense, specials, seed):
    from unboundednerfpytorch_b200 import ops
    p = make('param', shape, layout, seed, offset=offset, specials=specials)
    g = make('grad', shape, layout, seed + 1, offset=offset, specials=specials)
    assert tv_route(shape, layout, p, g) == route
    gk = g.clone(memory_format=torch.preserve_format) if offset == 0 else alloc(shape, layout, DEV, offset).copy_(g)
    launched(lambda: ops.total_variation_add_grad(p, gk, *W, dense), {tv_kernel(route, dense)})
    want = ref_tv(p, g, W, dense)
    assert mismatches(gk, want) == 0, f'{shape} dense={dense}: TV differs from the reference CUDA'
    if not specials:
        fails = []
        judge_tail(fails, 'tv', dict(p=p, grads=[g], w=W, dense=dense, mode=None), dict(g=gk))
        assert not fails, fails


@pytest.mark.gpu
@pytest.mark.parametrize('shape,layout,offset,route', TV_CASES, ids=[f'{"x".join(map(str, c[0]))}-{c[1]}{c[2]}' for c in TV_CASES])
def test_total_variation(shape, layout, offset, route):
    for k, (dense, specials) in enumerate(itertools.product((True, False), (False, True))):
        _tv_case(shape, layout, offset, route, dense, specials, 10 * k + sum(shape))


@pytest.mark.gpu
def test_total_variation_bicycle_k0():
    for k, dense in enumerate((True, False)):
        _tv_case(BICYCLE_K0, 'cl', 0, 'stream', dense, False, 31 + k)
        torch.cuda.empty_cache()


# ---- GPU: ping-pong sweep -------------------------------------------------------------------------------------------------------
PP_SHAPES = [(2, 4, 9, 5, 32), (1, 12, 17, 5, 153), (2, 16, 20, 3, 128)]    # row4 32, 459, 512


def _pingpong_case(shape, dense, masked, write_grad, t, seed, specials=False):
    from unboundednerfpytorch_b200 import ops
    p = make('param', shape, 'cl', seed, specials=specials)
    g = make('grad', shape, 'cl', seed + 1, specials=specials)
    m, v = make('m', shape, 'cl', seed + 2), make('v', shape, 'cl', seed + 3)
    p0, g0, m0, v0 = (x.clone(memory_format=torch.preserve_format) for x in (p, g, m, v))
    po = sentinel_like(p)
    launched(lambda: ops.tv_adam_pingpong(p, po, g, m, v, *W, dense, t, B1, B2, LR, EPS, skip_zero_grad=masked,
                                          write_grad=write_grad), {f'k_tv_adam_stream<{_cl(dense)}, {int(masked)}, {_cl(write_grad)}>'})
    aug = ref_tv(p0, g0, W, dense)
    pr, mr, vr = ref_adam(p0, aug, m0, v0, t, int(masked))
    tag = f'{shape} dense={dense} masked={masked} write_grad={write_grad} t={t}'
    assert mismatches(p, p0) == 0, tag + ': the input parameters changed'
    for what, a, b in (('p', po, pr), ('m', m, mr), ('v', v, vr), ('grad', g, aug if write_grad else g0)):
        assert mismatches(a, b) == 0, f'{tag}: {what} differs from the reference CUDA'
    if not specials:
        fails = []
        judge_tail(fails, 'pingpong', dict(p=p0, grads=[g0], w=W, dense=dense, mode=int(masked), t=t, m=m0, v=v0),
                   dict(p=po, m=m, v=v, g=g if write_grad else None), zero32=aug == 0)
        assert not fails, fails


@pytest.mark.gpu
@pytest.mark.parametrize('shape', PP_SHAPES, ids=['row4_32', 'row4_459', 'row4_512'])
def test_tv_adam_pingpong(shape):
    from unboundednerfpytorch_b200 import ops
    assert ops.tv_adam_pingpong_supported(alloc(shape, 'cl', DEV))
    for k, (dense, masked, wg) in enumerate(itertools.product((True, False), repeat=3)):
        for t in (1, 2, 3, 50, 20000):
            _pingpong_case(shape, dense, masked, wg, t, 100 * k + t)
        _pingpong_case(shape, dense, masked, wg, 3, 7 + k, specials=True)


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(1, 4, 9, 5, 31), (1, 4, 9, 5, 513)], ids=['row4_31', 'row4_513'])
def test_tv_adam_pingpong_refuses(shape):
    from unboundednerfpytorch_b200 import _cabi, ops
    from unboundednerfpytorch_b200._cabi import c_f, c_i64, c_int, ptr, stream_of
    p, g, m, v = (make(k, shape, 'cl', 5) for k in ('param', 'grad', 'm', 'v'))
    assert not ops.tv_adam_pingpong_supported(p)
    po = sentinel_like(p)
    with pytest.raises(RuntimeError):
        ops.tv_adam_pingpong(p, po, g, m, v, *W, True, 1, B1, B2, LR, EPS)
    keep = [x.clone(memory_format=torch.preserve_format) for x in (g, m, v)]
    P, C, X, Y, Z = shape
    lib = _cabi.load()
    errs = []
    launched(lambda: errs.append(lib.ubn_tv_adam_pingpong(
        ptr(p), ptr(po), ptr(g), ptr(m), ptr(v), c_f(W[0]), c_f(W[1]), c_f(W[2]), c_i64(P), c_i64(X), c_i64(Y), c_i64(Z),
        c_i64(C), c_int(1), c_int(1), c_f(B1), c_f(B2), c_f(LR), c_f(EPS), c_int(1), c_int(1), stream_of(p))), set())
    assert errs == [1]                                   # cudaErrorInvalidValue
    assert bool(is_sentinel(po).all()) and all(mismatches(a, b) == 0 for a, b in zip((g, m, v), keep))


@pytest.mark.gpu
def test_step_fused_tv_without_grad_write_is_tv_then_step():
    """bench.py's ping-pong leg: MaskedAdam.step_fused_tv(write_grad=False) == total_variation_add_grad + step() for params and
    moments, bit for bit, and .grad still holds the raw gradient."""
    from unboundednerfpytorch_b200 import ops
    from unboundednerfpytorch_b200.masked_adam import MaskedAdam
    shape = (1, 12, 17, 5, 153)
    for skip in (True, False):
        init = make('param', shape, 'cl', 40 + skip)
        pa = torch.nn.Parameter(init.clone(memory_format=torch.preserve_format))
        pb = torch.nn.Parameter(init.clone(memory_format=torch.preserve_format))
        oa = MaskedAdam([dict(params=[pa], lr=LR, skip_zero_grad=skip)])
        ob = MaskedAdam([dict(params=[pb], lr=LR, skip_zero_grad=skip)])
        for it in range(3):
            grad = make('grad', shape, 'cl', 50 + it)
            pa.grad = grad.clone(memory_format=torch.preserve_format)
            pb.grad = grad.clone(memory_format=torch.preserve_format)
            dense = it != 1
            launched(lambda: oa.step_fused_tv({pa: (*W, dense)}, write_grad=False), {f'k_tv_adam_stream<{_cl(dense)}, {int(skip)}, false>'})
            ops.total_variation_add_grad(pb, pb.grad, *W, dense)
            ob.step()
            assert mismatches(pa.data, pb.data) == 0, f'param step {it} skip={skip}'
            assert mismatches(oa.state[pa]['exp_avg'], ob.state[pb]['exp_avg']) == 0
            assert mismatches(oa.state[pa]['exp_avg_sq'], ob.state[pb]['exp_avg_sq']) == 0
            assert mismatches(pa.grad, grad) == 0, 'step_fused_tv(write_grad=False) changed .grad'


# ---- GPU: peer sweep on one GPU -------------------------------------------------------------------------------------------------
PEER_SHAPE = (3, 8, 10, 5, 17)       # row4 34, 30 planes of sz_i 10


def _shard(n, world):
    from unboundednerfpytorch_b200.dist import shard_range
    return [shard_range(n, r, world) for r in range(world)]


PEER_SETS = [  # (N, ranges in rank order, launch in reverse rank order)
    (1, [(0, 30)], False),
    (1, [(9, 10)], False),                                    # one plane, i = sz_i - 1
    (1, [(3, 21)], False),                                    # across two slab boundaries
    (2, _shard(30, 2), False),
    (2, [(9, 14), (2, 9)], True),                             # starts at i = sz_i - 1 / ends before it; reverse order
    (4, _shard(30, 4), False),
    (4, [(0, 1), (9, 10), (10, 11), (29, 30)], False),        # single planes at the slab edges
    (4, [(5, 11), (11, 12), (19, 26), (26, 30)], True),       # ends at i = 0 of the next slab; short ranges; reverse order
    (8, _shard(30, 8), False),
    (8, [(0, 2), (2, 3), (9, 10), (10, 16), (16, 20), (20, 29), (29, 30), (30, 30)], True),   # an empty range
]


def _plane_mask(ranges, n_planes, device=DEV):
    mask = torch.zeros(n_planes, dtype=torch.bool, device=device)
    for lo, hi in ranges:
        mask[lo:hi] = True
    return mask


def _peer_case(shape, N, ranges, reverse, dense, masked, t, seed, specials=False, grads=None, outs=None, shared=False):
    """Run ops.tv_adam_peer for every rank's range on one stream and judge the result.  grads / outs: the ranks' buffers
    (default: N distinct seeded gradients, N distinct sentinel-filled outputs); shared: one moment pair for all ranks."""
    from unboundednerfpytorch_b200 import ops
    P, C, X = shape[:3]
    p = make('param', shape, 'cl', seed, specials=specials)
    if grads is None:
        grads = [make('grad', shape, 'cl', seed + 1 + r, specials=specials) for r in range(N)]
    if outs is None:
        outs = [sentinel_like(p) for _ in range(N)]
    m0, v0 = make('m', shape, 'cl', seed + 20), make('v', shape, 'cl', seed + 21)
    mean = rank_mean(grads)
    aug = ref_tv(p, mean, W, dense)
    del mean
    pr, mr, vr = ref_adam(p, aug, m0, v0, t, int(masked))
    zero32 = aug == 0
    del aug
    if shared:
        ms, vs = [m0] * N, [v0] * N
    else:
        ms = [m0.clone(memory_format=torch.preserve_format) for _ in range(N)]
        vs = [v0.clone(memory_format=torch.preserve_format) for _ in range(N)]
    order = list(range(N))[::-1] if reverse else list(range(N))

    def run():
        for r in order:
            ops.tv_adam_peer(p, [o.data_ptr() for o in outs], [g.data_ptr() for g in grads], ms[r], vs[r], *W, dense, ranges[r][0],
                             ranges[r][1], t, B1, B2, LR, EPS, skip_zero_grad=masked)
    launched(run, {f'k_tv_adam_peer<{_cl(dense)}, {int(masked)}, {N}>'})
    tag = f'{shape} N={N} {ranges} dense={dense} masked={masked} t={t}'
    union = _plane_mask(ranges, P * X).view(P, 1, X, 1, 1)
    for o in {id(o): o for o in outs}.values():
        on = union.expand(shape)
        bad = int((on & ~((o.view(torch.int32) == pr.view(torch.int32)) | (torch.isnan(o) & torch.isnan(pr)))).sum())
        assert bad == 0, f'{tag}: {bad} output elements differ from the reference CUDA'
        assert bool(is_sentinel(o)[~on].all()), f'{tag}: a plane outside the ranges was written'
    if not shared:
        for r in range(N):
            own = _plane_mask(ranges[r:r + 1], P * X).view(P, 1, X, 1, 1).expand(shape)
            for what, a, want, before in (('m', ms[r], mr, m0), ('v', vs[r], vr, v0)):
                assert mismatches(torch.where(own, want, before), a) == 0, f'{tag}: rank {r} {what} wrong on or off its planes'
    else:
        on = union.expand(shape)
        for what, a, want in (('m', m0, mr), ('v', v0, vr)):
            assert mismatches(torch.where(on, want, a), a) == 0, f'{tag}: {what} differs from the reference CUDA'
    if specials:
        return
    if shared:
        m_got, v_got = m0, v0
        m_in, v_in = None, None
    else:
        m_got = m0.clone(memory_format=torch.preserve_format)
        v_got = v0.clone(memory_format=torch.preserve_format)
        for r in range(N):
            own = _plane_mask(ranges[r:r + 1], P * X).view(P, 1, X, 1, 1).expand(shape)
            m_got = torch.where(own, ms[r], m_got)
            v_got = torch.where(own, vs[r], v_got)
        m_in, v_in = m0, v0
    if shared:                      # the inputs were updated in place: restate them from the seed for the judge
        m_in, v_in = make('m', shape, 'cl', seed + 20), make('v', shape, 'cl', seed + 21)
    fails = []
    judge_tail(fails, 'peer', dict(p=p, grads=grads, w=W, dense=dense, mode=int(masked), t=t, m=m_in, v=v_in),
               dict(p=outs[0], m=m_got, v=v_got), planes=_plane_mask(ranges, P * X), zero32=zero32)
    assert not fails, fails


@pytest.mark.gpu
@pytest.mark.parametrize('k', range(len(PEER_SETS)), ids=[f'N{s[0]}-{i}' for i, s in enumerate(PEER_SETS)])
def test_tv_adam_peer_one_gpu(k):
    N, ranges, reverse = PEER_SETS[k]
    for j, (dense, masked) in enumerate(itertools.product((True, False), repeat=2)):
        _peer_case(PEER_SHAPE, N, ranges, reverse, dense, masked, (1, 2, 3, 50)[j], 1000 * k + 10 * j)
    _peer_case(PEER_SHAPE, N, ranges, reverse, True, True, 3, 1000 * k + 77, specials=True)


@pytest.mark.gpu
@pytest.mark.parametrize('N', [1, 4])
def test_tv_adam_peer_truck_k0(N):
    """Truck's k0 grid, the geometry of the 4-GPU runs.  The gradient and output buffers repeat across ranks (the kernel only
    reads the former; the same thread stores identical values into every copy of the latter) and the four disjoint ranges
    share one moment pair, to hold device memory down."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    P, X = TRUCK_K0[0], TRUCK_K0[2]
    g = make('grad', TRUCK_K0, 'cl', 501)
    o = sentinel_like(g)
    _peer_case(TRUCK_K0, N, _shard(P * X, N), False, True, True, 2, 500, grads=[g] * N, outs=[o] * N, shared=True)
    print(f'\n[tail-fp64] truck k0 peer N={N}: peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB')
    del g, o
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_peer_tail_world1_truck_step():
    """dist.PeerTail at world 1 through its real step() on the truck-shaped FourierGridModel: the k0 grid takes
    k_tv_adam_peer<true, 1, 1>, the density grid the classic route; both bit-identical to the reference's TV + masked Adam."""
    from unboundednerfpytorch_b200 import dist as D, models
    from unboundednerfpytorch_b200.masked_adam import create_optimizer_or_freeze_model
    torch.cuda.empty_cache()
    kw = dict(xyz_min=[-1.] * 3, xyz_max=[1.] * 3, num_voxels_density=153 ** 3, num_voxels_base_density=153 ** 3,
              num_voxels_rgb=153 ** 3, num_voxels_base_rgb=153 ** 3, num_voxels_viewdir=-1, alpha_init=1e-4, fast_color_thres=0,
              rgbnet_dim=12, fourier_freq_num=4)
    torch.manual_seed(0)
    model = models.FourierGridModel(**kw).to(DEV)
    assert tuple(model.k0.grid.shape) == TRUCK_K0
    with torch.no_grad():
        mem(model.k0.grid, 'cl').copy_(mem(make('param', TRUCK_K0, 'cl', 600), 'cl'))
        model.density.grid.copy_(make('param', tuple(model.density.grid.shape), 'c', 601))
    opt = create_optimizer_or_freeze_model(model, dict(lrate_density=0.1, lrate_k0=0.1, lrate_rgbnet=1e-3, lrate_decay=20,
                                                       skip_zero_grad_fields=['density', 'k0']), 0)
    tail = D.PeerTail(opt)
    k0, dens = model.k0.grid, model.density.grid
    assert k0 in tail.grids and dens not in tail.grids
    gk = make('grad', TRUCK_K0, 'cl', 602)
    gd = make('grad', tuple(dens.shape), 'c', 603)
    k0._ubn_grad_buffer.copy_(gk)
    k0.grad = k0._ubn_grad_buffer
    dens.grad = gd.clone()
    tv = model.tv_terms(1e-3, 1e-4, True)
    want = {}
    for prm, gr in ((k0, gk), (dens, gd)):
        aug = ref_tv(prm.detach(), gr, tv[prm][:3], tv[prm][3])
        z = torch.zeros_like(aug)
        want[prm] = ref_adam(prm.detach(), aug, z, z, 1, 1)
        del aug, z
    launched(lambda: tail.step(tv), {'k_tv_adam_peer<true, 1, 1>'})
    for prm in (k0, dens):
        st = opt.state[prm]
        for what, a, b in (('param', prm.detach(), want[prm][0]), ('exp_avg', st['exp_avg'], want[prm][1]),
                           ('exp_avg_sq', st['exp_avg_sq'], want[prm][2])):
            assert mismatches(a, b) == 0, f'{tuple(prm.shape)} {what} differs from the reference CUDA'
    assert k0.grad is None and float(k0._ubn_grad_buffer.abs().max()) == 0.0
    del model, opt, tail, want, gk, gd
    torch.cuda.empty_cache()


# ---- GPU: Adam kernels ---------------------------------------------------------------------------------------------------------
ADAM_N = [1, 4, 5, 6, 7, 1000, 1003, 9 * 153 ** 3]


def _adam_case(n, mode, offset, seed, perlr_offset=None, specials=False):
    from unboundednerfpytorch_b200 import ops
    shape = (1, 1, n, 1, 1)
    p = make('param', shape, 'c', seed, offset=offset, specials=specials).view(-1)
    g = make('grad', shape, 'c', seed + 1, offset=offset, specials=specials).view(-1)
    m, v = make('m', shape, 'c', seed + 2, offset=offset).view(-1), make('v', shape, 'c', seed + 3, offset=offset).view(-1)
    lr = make('perlr', shape, 'c', seed + 4, offset=offset if perlr_offset is None else perlr_offset).view(-1) if mode == 2 else None
    p0, m0, v0 = p.clone(), m.clone(), v.clone()
    t = 1 + seed % 3
    if mode == 0:
        fn = lambda: ops.adam_upd(p, g, m, v, t, B1, B2, LR, EPS)
    elif mode == 1:
        fn = lambda: ops.masked_adam_upd(p, g, m, v, t, B1, B2, LR, EPS)
    else:
        fn = lambda: ops.adam_upd_with_perlr(p, g, m, v, lr, t, B1, B2, LR, EPS)
    expect = adam_route(n, [p, g, m, v] + ([lr] if lr is not None else []), 'k_adam', mode)
    launched(fn, expect)
    pr, mr, vr = ref_adam(p0, g, m0, v0, t, mode, lr)
    tag = f'adam n={n} mode={mode} offset={offset} perlr_offset={perlr_offset}'
    for what, a, b in (('p', p, pr), ('m', m, mr), ('v', v, vr)):
        assert mismatches(a, b) == 0, f'{tag}: {what} differs from the reference CUDA'
    if not specials:
        fails = []
        v5 = lambda x: x.view(shape)
        judge_tail(fails, 'adam', dict(p=v5(p0), grads=[v5(g)], w=None, mode=mode, t=t, m=v5(m0), v=v5(v0),
                                       perlr=v5(lr) if lr is not None else None),
                   dict(p=v5(p), m=v5(m), v=v5(v)), zero32=v5(g) == 0)
        assert not fails, fails


@pytest.mark.gpu
@pytest.mark.parametrize('n', ADAM_N)
def test_adam_kernels(n):
    for mode in (0, 1, 2):
        for offset in (0, 1, 2, 3):
            _adam_case(n, mode, offset, 7 * n + 3 * mode + offset)
        if n <= 1003:
            _adam_case(n, mode, 0, 11 * n + mode, specials=True)
    _adam_case(n, 2, 0, 5 * n + 1, perlr_offset=1)                # a misaligned perlr alone


@pytest.mark.gpu
def test_masked_adam_pervoxel_lr_counts():
    """MaskedAdam.set_pervoxel_lr(count) -> per_lr = count / count.max() -> adam_upd_with_perlr, over three steps."""
    from unboundednerfpytorch_b200.masked_adam import MaskedAdam
    shape = (1, 1, 21, 13, 11)
    prm = torch.nn.Parameter(make('param', shape, 'c', 70))
    opt = MaskedAdam([dict(params=[prm], lr=LR, skip_zero_grad=True)])
    count = torch.randint(0, 50, shape, generator=torch.Generator(device=DEV).manual_seed(71), device=DEV)
    opt.set_pervoxel_lr(count)
    p_ref = prm.detach().clone()
    m_ref, v_ref = torch.zeros_like(p_ref), torch.zeros_like(p_ref)
    for t in (1, 2, 3):
        g = make('grad', shape, 'c', 72 + t)
        prm.grad = g.clone()
        p0 = prm.detach().clone()
        m0, v0 = m_ref.clone(), v_ref.clone()
        launched(opt.step, adam_route(prm.numel(), [prm, g, opt.per_lr], 'k_adam', 2))
        p_ref, m_ref, v_ref = ref_adam(p_ref, g, m_ref, v_ref, t, 2, opt.per_lr)
        st = opt.state[prm]
        for what, a, b in (('p', prm.detach(), p_ref), ('m', st['exp_avg'], m_ref), ('v', st['exp_avg_sq'], v_ref)):
            assert mismatches(a, b) == 0, f'step {t}: {what} differs from the reference CUDA'
        fails = []
        judge_tail(fails, 'adam', dict(p=p0, grads=[g], w=None, mode=2, t=t, m=m0, v=v0, perlr=opt.per_lr),
                   dict(p=prm.detach(), m=st['exp_avg'], v=st['exp_avg_sq']))
        assert not fails, fails


@pytest.mark.gpu
@pytest.mark.parametrize('tv_mode', [0, 1, 2])
def test_tv_adam_fused(tv_mode):
    """ops.tv_adam_fused: TV (none / dense / sparse) then (masked) Adam that may clear the gradient it consumed; n = 1134 is
    2 mod 4, so both the float4 body and the scalar tail run."""
    from unboundednerfpytorch_b200 import ops
    shape = (3, 1, 7, 6, 9)
    for k, (masked, zero) in enumerate(itertools.product((True, False), repeat=2)):
        for specials in (False, True):
            seed = 90 + 10 * tv_mode + k + 50 * specials
            p, g = make('param', shape, 'c', seed, specials=specials), make('grad', shape, 'c', seed + 1, specials=specials)
            m, v = make('m', shape, 'c', seed + 2), make('v', shape, 'c', seed + 3)
            p0, g0, m0, v0 = p.clone(), g.clone(), m.clone(), v.clone()
            t = 4
            expect = adam_route(p.numel(), [p, g, m, v], 'k_adam_zero', f'{int(masked)}, {_cl(zero)}')
            if tv_mode:
                expect.add(tv_kernel(tv_route(shape, 'c', p, g), tv_mode == 1))
            launched(lambda: ops.tv_adam_fused(p, g, m, v, *W, tv_mode, t, B1, B2, LR, EPS, skip_zero_grad=masked,
                                               zero_grad=zero), expect)
            aug = ref_tv(p0, g0, W, tv_mode == 1) if tv_mode else g0.clone()
            pr, mr, vr = ref_adam(p0, aug, m0, v0, t, int(masked))
            tag = f'fused tv_mode={tv_mode} masked={masked} zero={zero} specials={specials}'
            for what, a, b in (('p', p, pr), ('m', m, mr), ('v', v, vr)):
                assert mismatches(a, b) == 0, f'{tag}: {what} differs from the reference CUDA'
            if zero:
                assert bool((g == 0).all()), f'{tag}: gradient not cleared'
            else:
                assert mismatches(g, aug) == 0, f'{tag}: gradient is not the TV-augmented one'
            if not specials:
                fails = []
                judge_tail(fails, 'fused', dict(p=p0, grads=[g0], w=W if tv_mode else None, dense=tv_mode == 1,
                                                mode=int(masked), t=t, m=m0, v=v0),
                           dict(p=p, m=m, v=v, g=None if zero else g), zero32=aug == 0)
                assert not fails, fails


@pytest.mark.gpu
def test_reduce_tv_step_slab_slices():
    """The per-slab calls dist.reduce_tv_step makes on several ranks: TV and masked Adam on grid[p:p+1] of a contiguous
    [4, 1, 7, 5, 9] grid, X Y Z = 315 odd, so slabs 1 to 3 start off 16-byte alignment and take the scalar Adam kernel."""
    from unboundednerfpytorch_b200 import ops
    shape = (4, 1, 7, 5, 9)
    p, g = make('param', shape, 'c', 80), make('grad', shape, 'c', 81)
    m, v = make('m', shape, 'c', 82), make('v', shape, 'c', 83)
    for s in range(4):
        sl = slice(s, s + 1)
        ps, gs, ms, vs = p[sl], g[sl], m[sl], v[sl]
        p0, g0, m0, v0 = ps.clone(), gs.clone(), ms.clone(), vs.clone()
        assert tv_route(tuple(ps.shape), 'c', ps, gs) == 'element'
        expect = adam_route(ps.numel(), [ps, gs, ms, vs], 'k_adam', 1) | {tv_kernel('element', True)}
        assert (s == 0) == ('k_adam_vec4<1>' in expect), (s, expect)
        launched(lambda: (ops.total_variation_add_grad(ps, gs, *W, True),
                          ops.masked_adam_upd(ps, gs, ms, vs, 2, B1, B2, LR, EPS)), expect)
        aug = ref_tv(p0, g0, W, True)
        pr, mr, vr = ref_adam(p0, aug, m0, v0, 2, 1)
        for what, a, b in (('grad', gs, aug), ('p', ps, pr), ('m', ms, mr), ('v', vs, vr)):
            assert mismatches(a, b) == 0, f'slab {s}: {what} differs from the reference CUDA'
        fails = []
        judge_tail(fails, 'slab', dict(p=p0, grads=[g0], w=W, dense=True, mode=1, t=2, m=m0, v=v0),
                   dict(p=ps, m=ms, v=vs, g=gs), zero32=aug == 0)
        assert not fails, fails


@pytest.mark.gpu
def test_zz_every_instantiation_ran():
    """Runs last: every instantiation EXPECTED lists was launched by a case above."""
    print('\n[tail-fp64] worst ratio per judge: ' + ', '.join(f'{k} {v:.3g}' for k, v in sorted(WORST.items())))
    missing = sorted(EXPECTED - RAN)
    assert not missing, f'never launched: {missing}'
