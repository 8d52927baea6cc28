"""The fused march's transmittance adjoint -- g_weight and g_last through the reverse scan of k_march_density_bwd (csrc/march.cu) back
to each sample's density -- against an exact fp32 emulation of the reference's recurrences and an fp64 adjoint, sample by sample,
in all four geometries (contracted March, NDC NdcMarch, box BoxMarch, box-TensoRF BoxTensorfMarch), and the op path's
Alphas2Weights kernels (ops.alpha2weight / alpha2weight_backward) against the same emulation.

Two references, for two different questions:
  (a) emulation.  numpy restates the reference's sequential recurrences in the kernels' own fp32 / fp64 operations, fed with the
      kernel's own fp32 alphas: T <- fp32(f64(T) * (1 - f64(a))), w = fp32(T * a), stop at f64(T) < 1e-3; back = fp32(g_last * last),
      then back = fmaf(gw_j, w_j, back) from the last scanned sample to the first (gw_j = 0 unless KEEP);
      ga = fp32([KEEP] g_alpha + fp32(f64(fp32(gw * T)) - f64(back) / (f64(fp32(1 - a)) + 1e-10))).  Every one of these operations
      is IEEE-rounded, and fmaf is emulated exactly (the product is exact in fp64, TwoSum gives the exact sum as s + e, and rounding
      s to fp32 is correct unless s lies exactly halfway between two fp32 values, where the sign of e decides).  So the emulation
      is the bit-exact expectation of the kernel's T, weight, last, flags, compaction and of its intermediate ga.
  (b) fp64.  The same formulas in fp64 (T and w as fp64 products of the kernel's fp32 alphas, the chain in fp64), which shows the
      emulation -- and with it the kernel -- computes the adjoint of the real thing: T and w within gamma_k of the fp64 products,
      ga_emul within gamma_(2n+6) * (sum of the magnitudes of its terms) of ga64.

The kernel's per-sample density gradient gd is observable: launch 1 of the run scatter writes it, already divided by the slab
count P, to gd_scratch (contracted P in {1, 3, 5, 7, 9} under ubn_set_density_scatter(1), every NDC / box / TensoRF call).  The
entries are called directly on the forward's own dense records with a NaN-filled gd_scratch, and gd is judged against
([KEEP] g_density + r'64(d) * ga_emul) / P, r'(d) = interval * min(e, 1e10) * (1 + e)^(-interval - 1), e = exp(f64(fp32(d + shift))),
within C_GD = c_gd(interval) = 22 + 5 interval units of 2^-24 of (|[KEEP] g_density| + |r'64 * ga_emul|) / P, plus absolute
floors for fp32 underflow (expf / powf results below FLT_MIN, a subnormal final rounding).  C_GD does not grow with the ray length, so one dropped chain term is caught even on a
4096-step ray, where the fp64 comparison of ga alone could not see it.  The paths where launch 1 does not write gd_scratch
(generic P = 11, the per-sample scatter) are judged at the grid with test_gpu_march_scatter's fp64 scatter at 1e-5 of each
element's bound, each sample contributing its per-sample bound.

Worst ratios seen on an H100 80GB HBM3 (700 W power limit), |got - want| over the bound (1.0 = at the bound), over all cases:
  T / w / last vs the fp64 products: 0.64 of gamma_k;  alpha vs fp64 raw2alpha: 0.15 of c_alpha * 2^-24;
  ga_emul vs the fp64 chain: 0.25 of gamma_(2n+6);  per-sample gd: 0.24 of its bound (C_GD = 24.5 at interval 0.5);
  grid level (of B, judged at 1e-5): P = 11 run-scatter mode 5.6e-7, P = 9 per-sample scatter 1.8e-6, P = 1 per-sample 2.3e-7.
Every forward record, flag and compacted output equalled the emulation bit for bit, and so did the op path's alpha2weight and
alpha2weight_backward.
test_checker_rejects_faults (CPU) feeds the judges emulated results with one injected fault each and shows each is rejected."""
import numpy as np
import pytest
import torch

from tests.test_gpu_march_scatter import (C_SHAPE, C_SHAPE4, Contracted, cells, judge, ref_scatter, selections,  # noqa: F401
                                          slab_coords)

DEV = 'cuda:0'
F32, F64 = np.float32, np.float64
U = 2.0 ** -24
U1 = 2.0 ** -24 + 2.0 ** -50      # one T step: fp64 product rounded to fp32 (and the fp64 reference's own rounding)
QUERIED, LISTED, SCANNED, KEEP = 1, 2, 4, 8
WORST = {}


def gamma(k):
    k = np.asarray(k, F64)
    return k * U1 / (1 - k * U1)


def c_gd(interval):
    """gd's relative bound in units of 2^-24.  expf: 2 ulp (CUDA's documented bound) = 4 u in min(e, 1e10); 1 + e: 4 u + u = 5 u,
    raised to the power interval + 1; powf: 4 ulp = 8 u; fp32 rounding of the fp64 product with ga: u; the fp32 add of
    [KEEP] g_density: u of the magnitudes; times fp32(1 / P): 2 u; one more u for the second-order terms."""
    return 4 + 5 * (1 + interval) + 8 + 1 + 1 + 2 + 1


def c_alpha(interval):
    """alpha = 1 - powf(1 + expf(x), -interval), absolute: 1 + e carries 5 u (above), the power interval * 5 u on q; powf 8 u on q
    (q <= 1); fp32(1 - q) u; one u for second-order terms."""
    return 5 * interval + 8 + 1 + 1


# ---- emulation ------------------------------------------------------------------------------------------------------------
def fmaf(a, b, c):
    """fp32 fmaf(a, b, c) elementwise, exactly."""
    a, b, c = (np.asarray(v, F32) for v in (a, b, c))
    p = a.astype(F64) * b.astype(F64)                       # exact: 24 x 24 bits
    c64 = c.astype(F64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)                         # TwoSum: p + c = s + e exactly
    with np.errstate(over='ignore', invalid='ignore'):
        r = s.astype(F32)
        other = np.nextafter(r, np.where(s > r.astype(F64), F32(np.inf), F32(-np.inf)).astype(F32))
        mid = (r.astype(F64) != s) & np.isfinite(r) & (np.abs(s - r.astype(F64)) == np.abs(other.astype(F64) - s))
        up = np.where(e > 0, np.maximum(r, other), np.where(e < 0, np.minimum(r, other), r))
    return np.where(mid, up, r).astype(F32)


def emulate_forward(alpha, queried, valid, thres, late_stop=False):
    """The reference's sequential scan over [N, S] fp32 alphas: (T, w, flags, last, stop) with T = 1, w = 0 where not scanned;
    thres per ray.  late_stop (a fault for the checker) stops one listed sample after the real stop."""
    N, S = alpha.shape
    thres = np.broadcast_to(np.asarray(thres, F32), (N,))
    listed = queried & valid & np.where(thres[:, None] > 0, alpha > thres[:, None], True)
    T = np.ones((N, S), F32)
    w = np.zeros((N, S), F32)
    scanned = np.zeros((N, S), bool)
    Tc = np.ones(N, F32)
    done = np.zeros(N, bool)
    pend = np.zeros(N, bool)
    stop = np.full(N, -1)
    for s in range(S):
        act = listed[:, s] & ~done
        T[act, s] = Tc[act]
        w[act, s] = Tc[act] * alpha[act, s]
        scanned[act, s] = True
        Tc = np.where(act, (Tc.astype(F64) * (1.0 - alpha[:, s].astype(F64))).astype(F32), Tc)
        hit = act & (Tc.astype(F64) < 1e-3)
        if late_stop:
            now = act & pend
            pend |= hit
            hit = now
        stop = np.where(hit, s, stop)
        done |= hit
    keep = listed & np.where(thres[:, None] > 0, w > thres[:, None], True)
    flags = (queried & valid) * QUERIED + listed * LISTED + scanned * SCANNED + keep * KEEP
    return dict(T=T, w=w, flags=flags.astype(np.uint8), last=Tc, stop=stop, keep=keep, scanned=scanned)


def emulate_backward(alpha, T, w, last, scanned, keep, gw, ga_up, gl, fault=None, fault_at=None):
    """ga [N, S] fp32 of the reverse scan: gw / ga_up [N, S] are the upstream g_weight / g_alpha at KEEP samples (0 elsewhere),
    gl [N] g_last.  fault (checker only): 'drop' (the chain term of sample fault_at = (ray, s) dropped), 'neighbour' (my_back
    taken after the sample's own term), 'next_T' (T of the next sample), 'no_glast' (g_last term missing)."""
    N, S = alpha.shape
    back = (np.asarray(gl, F32) * last).astype(F32)
    if fault == 'no_glast':
        back = np.zeros(N, F32)
    ga = np.where(keep, ga_up, F32(0)).astype(F32)
    den = (F32(1) - alpha).astype(F32).astype(F64) + 1e-10
    Tn = np.concatenate([T[:, 1:], np.ones((N, 1), F32)], 1) if fault == 'next_T' else T
    for s in range(S - 1, -1, -1):
        sc = scanned[:, s]
        g = np.where(keep[:, s], gw[:, s], F32(0)).astype(F32)
        nb = fmaf(g, w[:, s], back)
        if fault == 'drop':
            nb[fault_at[0]] = back[fault_at[0]] if s == fault_at[1] else nb[fault_at[0]]
        my_back = nb if fault == 'neighbour' else back
        term = ((g * Tn[:, s]).astype(F32).astype(F64) - my_back.astype(F64) / den[:, s]).astype(F32)
        ga[:, s] = np.where(sc, (ga[:, s] + term).astype(F32), ga[:, s])
        back = np.where(sc, nb, back).astype(F32)
    return ga


# ---- fp64 references ------------------------------------------------------------------------------------------------------
def fp64_forward(alpha, scanned):
    """T64, w64, last64 as fp64 products of the fp32 alphas over the scanned samples, and the rounding counts k of T / w / last."""
    a = alpha.astype(F64)
    fac = np.where(scanned, 1 - a, 1.0)
    cp = np.cumprod(fac, 1)
    T64 = np.concatenate([np.ones((a.shape[0], 1)), cp[:, :-1]], 1)
    k = np.cumsum(scanned, 1) - scanned
    return T64, T64 * a, cp[:, -1], k, scanned.sum(1)


def fp64_chain(alpha, scanned, keep, T64, w64, last64, T, w, last, gw, ga_up, gl):
    """ga64 of the fp64 chain and the magnitude of its terms (for ga_emul's bound)."""
    a = alpha.astype(F64)
    g = np.where(keep, gw, 0).astype(F64)
    gl = np.asarray(gl, F64)

    def suffix(x):                      # sum over j > s
        c = np.cumsum(x[:, ::-1], 1)[:, ::-1]
        return c - x
    den = 1 - a + 1e-10
    back64 = gl[:, None] * last64[:, None] + suffix(np.where(scanned, g * w64, 0))
    mback = np.abs(gl[:, None] * last.astype(F64)[:, None]) + suffix(np.where(scanned, np.abs(g * w.astype(F64)), 0))
    up = np.where(keep, ga_up, 0).astype(F64)
    ga64 = up + np.where(scanned, g * T64 - back64 / den, 0)
    mag = np.abs(up) + np.where(scanned, np.abs(g * T.astype(F64)) + mback / den, 0)
    return ga64, mag


def raw2alpha_d(dens, shift, interval):
    """(e64, r'64, alpha64) at the fp32 densities: e = exp(f64(fp32(d + shift))); the exponent -interval - 1 is the kernel's fp32."""
    x = (dens.astype(F32) + F32(shift)).astype(F32).astype(F64)
    iv = F64(F32(interval))
    y = F64(F32(-F32(interval)) - F32(1))
    with np.errstate(over='ignore'):
        e = np.exp(x)
        r = iv * np.minimum(e, 1e10) * (1 + e) ** y
        a = 1 - (1 + e) ** (-iv)
    return e, r, a


def gd_expect(dens, shift, interval, P, keep, gdens, ga):
    """(want, bound) of the kernel's per-sample gd: ([KEEP] g_density + r'64 * ga) / P."""
    e, r, _ = raw2alpha_d(dens, shift, interval)
    kd = np.where(keep, gdens, 0).astype(F64)
    g = ga.astype(F64)
    want = (kd + r * g) / P
    iv = F64(F32(interval))
    bound = (c_gd(iv) * U * (np.abs(kd) + np.abs(r * g)) + iv * (2.0 ** -147 + np.minimum(e, 1e10) * 2.0 ** -125) * np.abs(g)) / P \
        + 2.0 ** -148
    return want, bound


def fp32_gd(dens, shift, interval, P, keep, gdens, ga):
    """gd restated in fp32 with correctly rounded expf / powf (an implementation within the documented bounds): the checker's
    honest kernel."""
    x = (dens.astype(F32) + F32(shift)).astype(F32)
    with np.errstate(over='ignore'):
        e = np.exp(x.astype(F64)).astype(F32)
        p = np.power((F32(1) + e).astype(F64), F64(F32(-F32(interval)) - F32(1))).astype(F32)
    r = (np.minimum(e.astype(F64), 1e10) * p.astype(F64) * F64(F32(interval)) * ga.astype(F64)).astype(F32)
    gd = np.where(ga != 0, (np.where(keep, gdens, 0).astype(F32) + r).astype(F32), np.where(keep, gdens, 0).astype(F32))
    return (gd * (F32(1) / F32(P))).astype(F32) if P > 1 else gd


# ---- judges -----------------------------------------------------------------------------------------------------------------
def _note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), float(r))


def judge_forward(what, rec, emu, alpha, valid):
    """Records of pass A (dense, [N, S]) against the emulation bit for bit on s < n, and T / w / last against fp64."""
    fails = []
    for k in ('T', 'w'):
        bad = int(((rec[k] != emu[k]) & valid).sum())
        if bad:
            fails.append(f'{k}: {bad} samples differ from the emulation')
    badf = int((((rec['flags'] & 15) != emu['flags']) & valid).sum())
    if badf:
        fails.append(f'flags: {badf} samples differ')
    if not np.array_equal(rec['last'], emu['last']):
        fails.append(f"last: {int((rec['last'] != emu['last']).sum())} rays differ")
    T64, w64, last64, k, ns = fp64_forward(alpha, emu['scanned'])
    sc = emu['scanned'] & valid
    rT = np.abs(rec['T'].astype(F64) - T64)[sc] / np.maximum(gamma(k)[sc] * T64[sc], 1e-300)
    rw = np.abs(rec['w'].astype(F64) - w64)[sc] / np.maximum(gamma(k + 1)[sc] * w64[sc], 1e-300)
    rl = np.abs(rec['last'].astype(F64) - last64) / np.maximum(gamma(ns) * last64, 1e-300)
    worst = max([float(v.max()) for v in (rT, rw, rl) if v.size] + [0.0])
    _note('T / w / last vs fp64 products / gamma_k', worst)
    print(f'[transmittance] {what}: T / w / last vs fp64 worst {worst:.2e} of gamma_k')
    if worst > 1:
        fails.append(f'T / w / last beyond gamma_k of the fp64 products ({worst:.2e})')
    return fails


def judge_gd(what, gd, want, bound, queried, valid):
    """Per-sample gd (fp32 [N, S] as written to gd_scratch) against (want, bound); s >= n untouched (NaN), non-QUERIED 0.0."""
    fails = []
    live = valid & queried
    if np.isnan(gd[valid]).any():
        fails.append(f'{int(np.isnan(gd[valid]).sum())} slots with s < n were not written')
    if (~np.isnan(gd[~valid])).any():
        fails.append(f'{int((~np.isnan(gd[~valid])).sum())} slots with s >= n were written')
    dead = valid & ~queried
    if (gd[dead] != 0).any() or np.signbit(gd[dead]).any():
        fails.append(f'{int((gd[dead] != 0).sum())} non-QUERIED slots are not 0.0')
    err = np.abs(gd.astype(F64) - want)[live]
    r = float((err / bound[live]).max()) if live.any() else 0.0
    if not np.isfinite(r):
        r = float('inf')
    _note('gd vs ([KEEP] g_density + r\'64 ga_emul) / P', r)
    print(f'[transmittance] {what}: gd worst {r:.2e} of its bound')
    if r > 1:
        fails.append(f'gd beyond its bound: {r:.2e}')
    return fails


def judge_chain(what, ga, ga64, mag, ns):
    """ga_emul against the fp64 chain within gamma_(2n+6) of its terms' magnitudes."""
    lim = gamma(2 * ns + 6)[:, None] * mag
    live = mag > 0
    r = float((np.abs(ga.astype(F64) - ga64)[live] / lim[live]).max()) if live.any() else 0.0
    _note('ga_emul vs fp64 chain / gamma_(2n+6)', r)
    print(f'[transmittance] {what}: ga_emul vs fp64 chain worst {r:.2e} of gamma_(2n+6)')
    return [] if r <= 1 else [f'ga_emul beyond gamma_(2n+6) of the fp64 chain: {r:.2e}']


# ---- structure ----------------------------------------------------------------------------------------------------------------
def structure(flags, n, alpha, stop):
    """Counts of the bookkeeping cases present, from the flags ([N, S]) and per-ray n / stop (records at s >= n are not data)."""
    N, S = flags.shape
    valid = np.arange(S)[None] < n[:, None]
    flags, alpha = np.where(valid, flags, 0), np.where(valid, alpha, 0)
    q, lst, sc, kp = ((flags & b) != 0 for b in (QUERIED, LISTED, SCANNED, KEEP))
    stopped = stop >= 0
    first_sc = np.where(sc.any(1), sc.argmax(1), -1)
    idx = np.arange(S)[None]
    nk = kp.sum(1)
    # a listed-but-not-kept sample between two kept ones of the same ray
    kc = np.cumsum(kp, 1)
    between = lst & ~kp & (kc > 0) & (kc < nk[:, None])
    qprefix = (q & (idx < n[:, None])).sum(1) == np.where(q.any(1), S - np.argmax(q[:, ::-1], 1), 0)
    gap = q.any(1) & ~qprefix & (q[:, :1].sum(1) >= 0)
    return dict(
        rays=N, stop_lane0=int((stopped & (stop % 32 == 0) & (stop > 0)).sum()), stop_lane31=int((stopped & (stop % 32 == 31)).sum()),
        stop_last=int((stopped & (stop == n - 1)).sum()), stop_first=int((stopped & (stop == first_sc)).sum()),
        never=int((~stopped & sc.any(1)).sum()), alpha1=int((sc & (alpha == 1)).sum()),
        one_minus_a_ulps=int((sc & (alpha < 1) & (alpha >= 1 - 8 * U)).sum()),
        listed_not_kept_between=int(between.sum()), nothing_queried=int((~q.any(1)).sum()),
        scanned_none_kept=int((sc.any(1) & (nk == 0)).sum()), not_prefix=int(gap.sum()),
        lengths=sorted(set(n.tolist()) & {1, 31, 32, 33, 63, 64, 65}), max_n=int(n.max()))


# ---- running the kernels --------------------------------------------------------------------------------------------------
def _records(out, n):
    rays_o, rays_d, dens, alpha, weight, T, flags, last, offsets = out[0].grad_fn.saved_tensors[:9]
    N = rays_o.shape[0]
    S = dens.numel() // N
    h = lambda t: t.detach().cpu().numpy()          # noqa: E731
    rec = dict(dens=h(dens).reshape(N, S), alpha=h(alpha).reshape(N, S), w=h(weight).reshape(N, S), T=h(T).reshape(N, S),
               flags=h(flags).reshape(N, S), last=h(last), offsets=h(offsets))
    dev = dict(rays_o=rays_o, rays_d=rays_d, args=(dens, alpha, weight, T, flags, last, offsets))
    return rec, dev, N, S


class Geo:
    """One forward of a geometry: its dense records, the kernel's compact outputs, and a call of its density_bwd C entry."""

    def __init__(self, name, out, n, shift, interval, thres, P, call, ray_id_at, has_gdens=False):
        self.name, self.shift, self.interval, self.thres, self.P, self.call = name, shift, interval, thres, P, call
        self.rec, self.dev, self.N, self.S = _records(out, n)
        self.n = np.broadcast_to(np.asarray(n), (self.N,)).astype(np.int64)
        self.valid = np.arange(self.S)[None] < self.n[:, None]
        self.compact = dict(weights=out[0].detach().cpu().numpy(), last=out[1].detach().cpu().numpy(),
                            raw_alpha=out[2].detach().cpu().numpy(), ray_id=out[ray_id_at].cpu().numpy(),
                            step_id=out[ray_id_at + 1].cpu().numpy())
        self.has_gdens = has_gdens


def check_forward(geo):
    rec, valid = geo.rec, geo.valid
    queried = (rec['flags'] & QUERIED) != 0
    emu = emulate_forward(rec['alpha'], queried, valid, geo.thres)
    fails = judge_forward(geo.name, rec, emu, rec['alpha'], valid)
    kp = emu['keep']
    cnt = kp.sum(1)
    if not np.array_equal(np.diff(rec['offsets']), cnt) or rec['offsets'][0] != 0:
        fails.append('offsets / n_keep differ from the emulation')
    r, s = np.nonzero(kp)
    c = geo.compact
    for k, v in (('ray_id', r), ('step_id', s), ('weights', emu['w'][kp]), ('raw_alpha', rec['alpha'][kp]), ('last', emu['last'])):
        if not np.array_equal(c[k], v):
            fails.append(f'compact {k} differs from the emulation')
    # alpha of every queried sample within c_alpha u of fp64 1 - (1 + e)^-interval at the kernel's own density
    _, _, a64 = raw2alpha_d(rec['dens'], geo.shift, geo.interval)
    live = queried & valid
    ra = float((np.abs(rec['alpha'].astype(F64) - a64)[live]).max() / (c_alpha(F64(F32(geo.interval))) * U)) if live.any() else 0
    _note('alpha vs fp64 raw2alpha / c_alpha u', ra)
    print(f'[transmittance] {geo.name}: alpha worst {ra:.2e} of c_alpha 2^-24')
    if ra > 1:
        fails.append(f'alpha beyond c_alpha 2^-24: {ra:.2e}')
    dead = valid & ~queried
    if (rec['alpha'][dead] != 0).any() or (rec['dens'][dead] != 0).any():
        fails.append('non-QUERIED records are not 0')
    return emu, fails


UPSTREAMS = ('all', 'g_weight', 'g_last', 'g_alpha', 'g_density')


def upstream(geo, kind, seed):
    g = torch.Generator().manual_seed(seed)
    M = geo.compact['ray_id'].size
    on = lambda name: kind in ('all', name)          # noqa: E731
    mk = lambda n, name: (torch.randn(n, generator=g).numpy() if on(name) else np.zeros(n, F32)).astype(F32)   # noqa: E731
    return dict(g_weight=mk(M, 'g_weight'), g_alpha=mk(M, 'g_alpha'), g_density=mk(M, 'g_density') if geo.has_gdens else None,
                g_last=mk(geo.N, 'g_last'))


def dense_of(geo, keep, v):
    out = np.zeros((geo.N, geo.S), F32)
    out[keep] = v
    return out


def run_bwd(geo, ups, nulls=False):
    """gd_scratch [N, S] after the geometry's density_bwd C entry (NaN where it wrote nothing)."""
    t = lambda a: (None if a is None or (nulls and not np.any(a)) else torch.from_numpy(np.ascontiguousarray(a)).to(DEV))  # noqa
    gd = torch.full((geo.N * geo.S,), float('nan'), device=DEV)
    geo.call(t(ups['g_weight']), t(ups['g_alpha']), t(ups['g_density']), t(ups['g_last']), gd)
    torch.cuda.synchronize()
    return gd.cpu().numpy().reshape(geo.N, geo.S)


def check_backward(geo, emu, kinds=UPSTREAMS, seed=0):
    """Every upstream configuration: gd per sample, zero buffers == null pointers, ga_emul vs the fp64 chain."""
    rec, valid = geo.rec, geo.valid
    queried = ((rec['flags'] & QUERIED) != 0) & valid
    kp, sc = emu['keep'], emu['scanned']
    T64, w64, last64, _, ns = fp64_forward(rec['alpha'], sc)
    fails = []
    for i, kind in enumerate(kinds):
        if kind == 'g_density' and not geo.has_gdens:
            continue
        ups = upstream(geo, kind, seed * 100 + i)
        gw, gal = dense_of(geo, kp, ups['g_weight']), dense_of(geo, kp, ups['g_alpha'])
        gdn = dense_of(geo, kp, ups['g_density']) if geo.has_gdens else np.zeros_like(gw)
        ga = emulate_backward(rec['alpha'], rec['T'], rec['w'], rec['last'], sc, kp, gw, gal, ups['g_last'])
        want, bound = gd_expect(rec['dens'], geo.shift, geo.interval, geo.P, kp, gdn, ga)
        gd = run_bwd(geo, ups)
        what = f'{geo.name} upstream={kind}'
        fails += [f'{what}: {m}' for m in judge_gd(what, gd, want, bound, queried, valid)]
        ga64, mag = fp64_chain(rec['alpha'], sc, kp, T64, w64, last64, rec['T'], rec['w'], rec['last'], gw, gal, ups['g_last'])
        fails += [f'{what}: {m}' for m in judge_chain(what, ga, ga64, mag, ns)]
        if kind != 'all':
            gdn_null = run_bwd(geo, ups, nulls=True)
            if not np.array_equal(gd, gdn_null, equal_nan=True):
                fails.append(f'{what}: null upstream pointers give a different gd than zero buffers')
    return fails


# ---- geometries -------------------------------------------------------------------------------------------------------------
def _lib():
    from unboundednerfpytorch_b200 import _cabi
    return _cabi.load()


def contracted_geo(name, sc, retune=None):
    """March on a test_gpu_march_scatter.Contracted scene; retune(dgrid) may reshape its density."""
    from unboundednerfpytorch_b200 import march
    from unboundednerfpytorch_b200._cabi import c_i64, check, ptr, stream_of
    if retune is not None:
        sc.dgrid = retune(sc.dgrid)
    dg = sc.dgrid.clone().requires_grad_(True)
    kg = sc.kvals.contiguous().permute(0, 4, 1, 2, 3).clone().requires_grad_(True)
    out = march.March.apply(dg, kg, sc.ro, sc.rd, sc.t_table, None, sc.cfg, sc.ddesc, sc.kdesc, False, False)
    grad = torch.zeros_like(sc.dgrid)

    def call(gw, ga, gdn, gl, gd):
        d = geo.dev
        check(_lib().ubn_march_density_bwd(ptr(d['rays_o']), ptr(d['rays_d']), ptr(sc.t_table), sc.ddesc, sc.cfg, c_i64(geo.N),
                                           *map(ptr, d['args']), ptr(gw), ptr(ga), ptr(gdn), ptr(gl), ptr(grad), ptr(gd),
                                           stream_of(d['rays_o'])))
    geo = Geo(name, out, sc.S, sc.cfg.act_shift, sc.cfg.interval, sc.cfg.fast_color_thres, sc.P, call, 5, has_gdens=True)
    geo.grad, geo.scene = grad, sc
    return geo


def ndc_geo(name):
    from tests.test_gpu_mpi import _ndc_scene
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import march
    from unboundednerfpytorch_b200._cabi import c_i64, check, ptr, stream_of
    m, ro, rd, _ = _ndc_scene(3, thres=1e-3, mask_p=0.8, n=2047)
    with torch.no_grad():
        m.act_shift.grid.copy_(torch.randn(m.act_shift.grid.shape, generator=torch.Generator().manual_seed(2)).to(DEV) * 2 - 1)
    S = m._n_samples(0.5)
    lo, hi = m._host()
    cfg = march.make_ndc_cfg(lo, hi, S, 0.5 * m.voxel_size_ratio, 1e-3, m.mask_cache.mask, *m._mask_geometry())
    descs = [G.grid_desc(gr.grid, *gr._bounds(), 0) for gr in (m.density, m.k0, m.act_shift)]
    dg = m.density.grid.detach().clone().requires_grad_(True)
    kg = m.k0.grid.detach().clone().requires_grad_(True)
    out = march.NdcMarch.apply(dg, kg, m.act_shift.grid, ro, rd, m.mask_cache.mask, cfg, *descs)
    grad = torch.zeros_like(dg)

    def call(gw, ga, gdn, gl, gd):
        d = geo.dev
        check(_lib().ubn_march_ndc_density_bwd(ptr(d['rays_o']), ptr(d['rays_d']), descs[0], cfg, c_i64(geo.N), *map(ptr, d['args']),
                                               ptr(gw), ptr(ga), ptr(gl), ptr(grad), ptr(gd), stream_of(d['rays_o'])))
    geo = Geo(name, out, S, 0.0, cfg.interval, cfg.fast_color_thres, 1, call, 4)
    return geo


BOX_LO, BOX_HI = [-1.0, -0.8, -1.1], [1.0, 0.9, 1.2]
BOX_SHIFT, BOX_INTERVAL = -2.0, 0.5


def box_n_steps(ro, rd, cfg):
    from unboundednerfpytorch_b200 import ops as O
    lo, hi = torch.tensor(list(cfg.xyz_min), device=DEV), torch.tensor(list(cfg.xyz_max), device=DEV)
    n = O.sample_pts_on_rays(ro, rd, lo, hi, cfg.near, 1e9, F32(cfg.stepdist))[4]
    return np.minimum(n.cpu().numpy(), cfg.s_max)


def exact_rays(lengths, sd, g):
    """x-rays starting inside the box with exactly n steps each."""
    o, d = [], []
    for n in lengths:
        y, z = (np.array(BOX_LO[1:]) + (np.array(BOX_HI[1:]) - np.array(BOX_LO[1:])) * (0.1 + 0.8 * g.random(2)))
        o.append([BOX_HI[0] - (n - 0.5) * sd, y, z])
        d.append([1.0, 0.0, 0.0])
    return o, d


def diagonal_rays(k, g):
    """Rays from just outside the lo corner towards the hi corner: the longest chords of the box."""
    lo, hi = np.array(BOX_LO), np.array(BOX_HI)
    d = hi - lo
    o = [lo - 0.01 * d + 0.002 * g.standard_normal(3) for _ in range(k)]
    return o, [d + 0.003 * g.standard_normal(3) for _ in range(k)]


def box_cfg_s_max(target, thres, mask=None):
    """A box cfg whose s_max is exactly target."""
    from unboundednerfpytorch_b200 import march
    diag = float(np.linalg.norm(np.array(BOX_HI) - np.array(BOX_LO)))
    sd = float(F32(diag / (target - 4 - 0.5)))
    ms = (None, None, None) if mask is None else mask
    cfg = march.make_box_cfg(BOX_LO, BOX_HI, 0.0, sd, BOX_SHIFT, BOX_INTERVAL, thres, *ms)
    assert cfg.s_max == target, (cfg.s_max, target)
    return cfg


def _box_call(geo_ref, grad, ddesc, cfg):
    from unboundednerfpytorch_b200._cabi import c_i64, check, ptr, stream_of

    def call(gw, ga, gdn, gl, gd):
        d = geo_ref[0].dev
        check(_lib().ubn_march_box_density_bwd(ptr(d['rays_o']), ptr(d['rays_d']), ddesc, cfg, c_i64(geo_ref[0].N), *map(ptr, d['args']),
                                               ptr(gw), ptr(ga), ptr(gl), ptr(grad), ptr(gd), stream_of(d['rays_o'])))
    return call


def box_geo(name, n_rand, s_max, thres, dens_fn, lengths=(1, 31, 32, 33, 63, 64, 65), n_diag=0, holes=False, seed=0):
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import march
    g = np.random.default_rng(seed)
    shape = (23, 37, 41)
    mask = None
    if holes:
        mk = torch.from_numpy(g.random(shape) > 0.2).to(DEV)
        scale = (torch.tensor(shape, dtype=torch.float32) - 1) / (torch.tensor(BOX_HI) - torch.tensor(BOX_LO))
        mask = (mk, scale.tolist(), (-torch.tensor(BOX_LO) * scale).tolist())
    cfg = box_cfg_s_max(s_max, thres, mask)
    o, d = exact_rays([n for n in lengths for _ in range(4)], cfg.stepdist, g)
    o2, d2 = diagonal_rays(n_diag, g)
    c = (np.array(BOX_LO) + np.array(BOX_HI)) / 2
    o3 = [c - 3 * v / np.linalg.norm(v) + 0.3 * g.standard_normal(3) for v in g.standard_normal((n_rand, 3))]
    d3 = [c - oo + 0.4 * g.standard_normal(3) for oo in o3]
    ro = torch.tensor(np.array(o + o2 + o3, F64), dtype=torch.float32, device=DEV)
    rd = torch.tensor(np.array(d + d2 + d3, F64), dtype=torch.float32, device=DEV)
    dgrid = dens_fn(g, shape).to(DEV)
    kvals = torch.randn(1, 3, *shape, generator=torch.Generator().manual_seed(seed)).to(DEV)
    kg = kvals.permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3).requires_grad_(True)
    ddesc = G.grid_desc(dgrid, BOX_LO, BOX_HI, 0)
    kdesc = G.grid_desc(kg, BOX_LO, BOX_HI, 0)
    dg = dgrid.clone().requires_grad_(True)
    out = march.BoxMarch.apply(dg, kg, ro, rd, mask[0] if mask else None, cfg, ddesc, kdesc)
    grad = torch.zeros_like(dgrid)
    ref = [None]
    geo = Geo(name, out, box_n_steps(ro, rd, cfg), BOX_SHIFT, BOX_INTERVAL, cfg.fast_color_thres, 1, _box_call(ref, grad, ddesc, cfg), 4)
    ref[0] = geo
    return geo


def tensorf_geo(name, R, Rxy):
    from tests.test_gpu_tensorf_march import _box_cfg, _model, _rays
    from unboundednerfpytorch_b200 import grid as G
    from unboundednerfpytorch_b200 import march
    from unboundednerfpytorch_b200._cabi import c_i64, c_int, check, ptr, stream_of
    from unboundednerfpytorch_b200.grid import _factor_array
    m = _model('TensoRFGrid', 'TensoRFGrid', R=R, Rxy=Rxy, kR=R, thres=1e-4)
    ro, rd, _ = _rays(1023, seed=13)
    cfg = _box_cfg(m)
    fs = m.density.factors()
    desc = G.tensorf_desc(fs, 1, *m.density._bounds())
    out = march.BoxTensorfMarch.apply(ro, rd, m.mask_cache.mask, cfg, desc, True, 1, *fs)
    grads = [torch.zeros_like(p) for p in fs]
    vec = torch.empty(desc.X * desc.R + desc.Y * desc.R + desc.Z * desc.Rxy, device=DEV)

    def call(gw, ga, gdn, gl, gd):
        d = geo.dev
        check(_lib().ubn_march_box_tensorf_density_bwd(
            ptr(d['rays_o']), ptr(d['rays_d']), _factor_array(fs), desc, cfg, c_i64(geo.N), *map(ptr, d['args']), ptr(gw), ptr(ga),
            ptr(gl), _factor_array(grads), c_int(1), ptr(gd), ptr(vec), stream_of(d['rays_o'])))
    geo = Geo(name, out, box_n_steps(ro, rd, cfg), float(m.act_shift), cfg.interval, cfg.fast_color_thres, 1, call, 4)
    return geo


def _dens_box(g, shape, scale=3.0, offset=0.0):
    return torch.from_numpy((g.standard_normal(shape) * scale + offset).astype(F32))[None, None]


def _dens_box_edges(g, shape):
    """Random densities, one x-slab block where expf overflows (alpha = 1.0 exactly) and one at d + shift ~ 30.5 (1 - alpha a few
    ulps) for the rays that start in them."""
    d = g.standard_normal(shape) * 2.5 - 1.0
    d[:, :12, :12] = 400.0
    d[:, -12:, -12:] = 32.5
    return torch.from_numpy(d.astype(F32))[None, None]


def _tiny(dgrid):
    return dgrid * 1.5 - 7.0


GEOMETRIES = {
    'contracted-P1-inf': lambda: contracted_geo('contracted P=1 inf', Contracted(P=1, shape=C_SHAPE, n_x=96, n_rand=64),
                                                lambda d: d * 2.5 - 5.0),
    'contracted-P9-l2-ragged': lambda: contracted_geo('contracted P=9 l2 thres=1e-4', Contracted(
        P=9, shape=C_SHAPE4, norm='l2', thres=1e-4, stepsize=0.5, n_x=384, n_rand=64, n_far=16)),
    'contracted-P5-cumdist': lambda: _cumdist_geo(),
    'contracted-P1-S4096': lambda: contracted_geo('contracted P=1 S=4096', Contracted(
        P=1, shape=C_SHAPE4, stepsize=0.01669, n_x=24, n_rand=16), _tiny),
    'ndc': lambda: ndc_geo('ndc act_shift grid'),
    'box-edges': lambda: box_geo('box edges', 509, 160, 0.0, _dens_box_edges),
    'box-thres-holes': lambda: box_geo('box thres=1e-4 mask holes', 509, 160, 1e-4,
                                       lambda g, s: _dens_box(g, s, 2.0, -2.5), holes=True, seed=1),
    'box-S4096': lambda: box_geo('box S_max=4096', 13, 4096, 0.0, lambda g, s: _dens_box(g, s, 0.05, -4.9), n_diag=16, seed=2),
    'box-8191': lambda: box_geo('box 8191 rays', 8191 - 28, 160, 1e-4, lambda g, s: _dens_box(g, s, 3.0, -1.0), seed=3),
    'tensorf-R8': lambda: tensorf_geo('tensorf R=8 (4-wide records)', 8, 8),
    'tensorf-R5-7': lambda: tensorf_geo('tensorf R=5 Rxy=7 (scalar records)', 5, 7),
}


def _cumdist_geo():
    from unboundednerfpytorch_b200 import march
    sc = Contracted(P=5, shape=C_SHAPE, n_x=64, n_rand=64, n_far=64)
    sc.cfg = march.make_cfg([0.] * 3, [1.] * 3, 0.2, 'inf', sc.S, 0.0, 0.5, 0.0, cumdist_thres=0.3)
    return contracted_geo('contracted P=5 cumdist', sc, lambda d: d * 2.0 - 4.0)


# what each geometry must show (asserted from the kernel's own flags)
NEEDS = {
    'contracted-P1-inf': ('stop_lane31', 'never'),
    'contracted-P9-l2-ragged': ('listed_not_kept_between', 'never'),
    'contracted-P5-cumdist': ('not_prefix',),
    'contracted-P1-S4096': ('never',),
    'ndc': ('listed_not_kept_between', 'not_prefix'),
    'box-edges': ('alpha1', 'one_minus_a_ulps', 'stop_first', 'stop_last', 'stop_lane0', 'stop_lane31', 'never'),
    'box-thres-holes': ('listed_not_kept_between', 'not_prefix', 'never'),
    'box-S4096': ('never',),
    'box-8191': ('stop_lane0', 'stop_lane31', 'stop_last'),
    'tensorf-R8': ('listed_not_kept_between', 'nothing_queried', 'not_prefix'),
    'tensorf-R5-7': ('listed_not_kept_between', 'nothing_queried', 'not_prefix'),
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(GEOMETRIES))
def test_transmittance_adjoint_per_sample(case, selections):
    """Pass A's records and compaction equal the emulation bit for bit; launch 1's per-sample gd matches the emulated chain
    through the fp64 raw2alpha' within C_GD 2^-24, under every upstream configuration and with null upstream pointers."""
    ops = selections
    ops.set_density_scatter(1)
    geo = GEOMETRIES[case]()
    emu, fails = check_forward(geo)
    st = structure(geo.rec['flags'], geo.n, geo.rec['alpha'], emu['stop'])
    print(f'[coverage] {geo.name}: N={geo.N} S={geo.S} {st}')
    if geo.n.max() == geo.S and geo.S > 32:
        assert st['max_n'] == geo.S
    if case.startswith('box') and case != 'box-S4096':
        assert st['lengths'] == [1, 31, 32, 33, 63, 64, 65], st['lengths']
    if case.endswith('S4096'):
        assert geo.S == 4096 and st['max_n'] > 4000, (geo.S, st['max_n'])
    missing = [k for k in NEEDS[case] if st[k] == 0]
    assert not missing, f'{geo.name}: no {missing}'
    fails += check_backward(geo, emu)
    assert not fails, '\n'.join(fails)


# ---- crafted records: every stop position the backward's bookkeeping distinguishes ------------------------------------------
def crafted(n, S, g):
    """alpha / queried / thres rows [R, S] for rays of lengths n: each length gets every kind below."""
    kinds = ['never', 'stop_lane0_c2', 'stop_lane31_c2', 'stop_last', 'alpha1_first', 'ulps', 'straddle', 'nothing', 'holes',
             'scanned_none_kept']
    rows = []
    for L in n:
        for k in kinds:
            a = (g.uniform(0.5, 1.5, S) * 5e-4).astype(F32)
            q = np.arange(S) < L
            th = 0.0
            at = {'stop_lane0_c2': 64, 'stop_lane31_c2': 95, 'stop_last': L - 1}.get(k)
            if at is not None:
                if at >= L:
                    continue
                a[at] = F32(0.9995)
            elif k == 'alpha1_first':
                a[0] = F32(1.0)
            elif k == 'ulps':
                s = min(L - 1, 40)
                a[s] = F32(1 - 3 * U)
            elif k == 'straddle':
                a = (g.uniform(0.3, 3.0, S) * 1e-4).astype(F32)
                a[3] = F32(0.5)              # halves T: later alphas just above thres give weights below it
                th = 1e-4
            elif k == 'nothing':
                q[:] = False
            elif k == 'holes':
                q &= g.random(S) > 0.3
                th = 1e-4
            rows.append((k, L, a, q, th))
    return rows


@pytest.mark.gpu
def test_transmittance_adjoint_crafted_records(selections):
    """The box march's launch 1 on records emulated from chosen alphas: stops on lane 0 and lane 31 of chunk 2, on a ray's last
    sample, at alpha = 1.0 on the first sample, with 1 - alpha = 3 ulps; never on ~4090-step rays with S_max = 4096 (the chunk
    table full); listed-but-not-kept samples between kept ones; rays with nothing queried, with holes, and with everything
    scanned and nothing kept (KEEP cleared: only g_last reaches them)."""
    from unboundednerfpytorch_b200._cabi import FLAG_KEEP
    ops = selections
    ops.set_density_scatter(1)
    g = np.random.default_rng(5)
    cfg = box_cfg_s_max(4096, 0.0)
    S = cfg.s_max
    lengths = [1, 31, 32, 33, 63, 64, 65, 96, 200]
    o, d = exact_rays(lengths, cfg.stepdist, g)
    o2, d2 = diagonal_rays(4, g)
    ro = torch.tensor(np.array(o + o2, F64), dtype=torch.float32, device=DEV)
    rd = torch.tensor(np.array(d + d2, F64), dtype=torch.float32, device=DEV)
    n_ray = box_n_steps(ro, rd, cfg)
    assert list(n_ray[:len(lengths)]) == lengths and (n_ray[len(lengths):] > 4080).all(), n_ray
    rows = crafted(n_ray, S, g)
    N = len(rows)
    pick = {L: i for i, L in enumerate(n_ray)}
    idx = np.array([pick[r[1]] for r in rows])
    alpha = np.stack([r[2] for r in rows])
    queried = np.stack([r[3] for r in rows])
    thres = np.array([r[4] for r in rows], F32)
    n = np.array([r[1] for r in rows])
    valid = np.arange(S)[None] < n[:, None]
    alpha = np.where(queried & valid, alpha, F32(0))
    emu = emulate_forward(alpha, queried, valid, thres)
    none_kept = np.array([r[0] == 'scanned_none_kept' for r in rows])
    emu['keep'] &= ~none_kept[:, None]
    emu['flags'] = np.where(none_kept[:, None], emu['flags'] & ~np.uint8(FLAG_KEEP), emu['flags']).astype(np.uint8)
    with np.errstate(divide='ignore'):
        dens = np.where(alpha >= 1, F32(400), np.log(np.power(1 - alpha.astype(F64), -1 / BOX_INTERVAL) - 1) - BOX_SHIFT)
    dens = np.where(queried & valid, dens, 0).astype(F32)
    st = structure(emu['flags'], n, alpha, emu['stop'])
    print(f'[coverage] crafted box records: N={N} S={S} {st}')
    for k in ('stop_lane0', 'stop_lane31', 'stop_last', 'stop_first', 'never', 'alpha1', 'one_minus_a_ulps', 'listed_not_kept_between',
              'nothing_queried', 'scanned_none_kept', 'not_prefix'):
        assert st[k] > 0, k
    assert st['lengths'] == [1, 31, 32, 33, 63, 64, 65] and st['max_n'] > 4080
    assert ((emu['stop'] == 64) | (emu['stop'] == 95)).sum() >= 2
    from unboundednerfpytorch_b200 import grid as G
    dgrid = torch.zeros(1, 1, 5, 5, 5, device=DEV)
    ddesc = G.grid_desc(dgrid, BOX_LO, BOX_HI, 0)
    keep = emu['keep']
    offsets = np.concatenate([[0], np.cumsum(keep.sum(1))]).astype(np.int64)
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)          # noqa: E731
    dev_args = (tt(dens.ravel()), tt(alpha.ravel()), tt(np.where(valid, emu['w'], 0).ravel()), tt(emu['T'].ravel()),
                tt(emu['flags'].ravel()), tt(emu['last']), tt(offsets))
    rays_o, rays_d = ro[idx].contiguous(), rd[idx].contiguous()

    class Crafted:
        pass
    geo = Crafted()
    geo.name, geo.N, geo.S, geo.n, geo.valid, geo.shift, geo.interval, geo.P, geo.has_gdens = \
        'crafted box', N, S, n, valid, BOX_SHIFT, BOX_INTERVAL, 1, False
    geo.rec = dict(dens=dens, alpha=alpha, w=emu['w'], T=emu['T'], flags=emu['flags'], last=emu['last'], offsets=offsets)
    geo.compact = dict(ray_id=np.nonzero(keep)[0])
    geo.dev = dict(rays_o=rays_o, rays_d=rays_d, args=dev_args)
    geo.call = _box_call([geo], torch.zeros_like(dgrid), ddesc, cfg)
    fails = check_backward(geo, emu, seed=9)
    assert not fails, '\n'.join(fails)


# ---- grid level: the paths where launch 1 scatters itself ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('case,scatter', [('P11', 1), ('P9', 0), ('P1', 0)])
def test_transmittance_adjoint_grid_level(case, scatter, selections):
    """Generic P = 11 (launch 1 scatters every sample itself) and the per-sample scatter: the density-grid gradient against the
    fp64 scatter of the per-sample gd, at 1e-5 of each element's bound (each sample contributing its per-sample bound)."""
    ops = selections
    ops.set_density_scatter(scatter)
    P = int(case[1:])
    sc = Contracted(P=P, shape=C_SHAPE, n_x=96, n_rand=48)
    geo = contracted_geo(f'contracted P={P} scatter={scatter}', sc, lambda d: d * 2.5 - 4.0)
    emu, fails = check_forward(geo)
    assert not fails, '\n'.join(fails)
    rec = geo.rec
    queried = (rec['flags'] & QUERIED) != 0
    ups = upstream(geo, 'all', 17)
    kp, scn = emu['keep'], emu['scanned']
    gw, gal, gdn = (dense_of(geo, kp, ups[k]) for k in ('g_weight', 'g_alpha', 'g_density'))
    ga = emulate_backward(rec['alpha'], rec['T'], rec['w'], rec['last'], scn, kp, gw, gal, ups['g_last'])
    want, bound = gd_expect(rec['dens'], geo.shift, geo.interval, 1, kp, gdn, ga)     # P applied by ref_scatter
    geo.grad.zero_()
    gd = run_bwd(geo, ups)
    if scatter == 0 or P == 11:
        assert np.isnan(gd).all(), 'launch 1 of the per-sample scatter wrote gd_scratch'
    r, s = np.nonzero(queried & (want != 0))
    x0, f = cells(slab_coords(sc.points(torch.from_numpy(r).to(DEV), torch.from_numpy(s).to(DEV)), sc.mn, sc.mx, sc.n_freqs),
                  sc.shape)
    w_t = torch.from_numpy(want[r, s]).to(DEV)
    b_t = torch.from_numpy(np.abs(want[r, s]) + bound[r, s]).to(DEV)
    want_g, _ = ref_scatter(x0, f, w_t[:, None], sc.shape)
    _, bound_g = ref_scatter(x0, f, b_t[:, None], sc.shape)
    got = geo.grad.permute(0, 2, 3, 4, 1)
    judge(got, want_g, bound_g, f'{geo.name} density grid', f'transmittance grid P={P} ds={scatter}')


# ---- the op path: Alphas2Weights ----------------------------------------------------------------------------------------------
def ragged_long(n_rays, seed):
    """Rays of 0 .. 4096 samples in one 32-ray tile, tiny alphas (no stop over 4096 samples) and rays that stop on the first / last
    sample of a 32-sample tile column (31, 32, 63, 64) and at alpha = 1.0."""
    g = np.random.default_rng(seed)
    lens = np.array(([0, 1, 31, 32, 33, 63, 64, 65, 4095, 4096] + list(g.integers(0, 4097, n_rays)))[:n_rays])
    alphas = []
    for i, L in enumerate(lens):
        a = (g.uniform(0.5, 1.5, L) * 5e-4).astype(F32)
        stop = [None, 31, 32, 63, 64, 0][i % 6] if L < 4000 else None
        if stop is not None and stop < L:
            a[stop] = F32(1.0) if stop == 0 else F32(0.9995)
        alphas.append(a)
    alpha = np.concatenate(alphas) if alphas else np.zeros(0, F32)
    ray_id = np.repeat(np.arange(n_rays), lens)
    return torch.from_numpy(alpha), torch.from_numpy(ray_id), lens


@pytest.mark.gpu
@pytest.mark.parametrize('n_rays', [32, 45])
def test_alpha2weight_op_path_vs_emulation(n_rays):
    """ops.alpha2weight / alpha2weight_backward (what _compose and forward_ops run) bit for bit against the emulation, and
    against the fp64 products / chain within gamma, on ragged rays up to 4096 samples."""
    from unboundednerfpytorch_b200 import ops
    alpha, ray_id, lens = ragged_long(n_rays, n_rays)
    w, T, last, i_s, i_e = ops.alpha2weight(alpha.to(DEV), ray_id.to(DEV), n_rays)
    S = int(lens.max())
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    valid = np.arange(S)[None] < lens[:, None]
    A = np.zeros((n_rays, S), F32)
    A[valid] = alpha.numpy()
    emu = emulate_forward(A, valid, valid, 0.0)
    h = lambda t: t.cpu().numpy()          # noqa: E731
    Wd, Td = np.zeros((n_rays, S), F32), np.ones((n_rays, S), F32)
    Wd[valid], Td[valid] = h(w), h(T)
    fails = judge_forward(f'alpha2weight {n_rays} rays', dict(T=Td, w=Wd, flags=emu['flags'], last=h(last)), emu, A, valid)
    n_sc = emu['scanned'].sum(1)
    assert np.array_equal(h(i_s)[lens > 0], starts[lens > 0]) and np.array_equal((h(i_e) - h(i_s))[lens > 0], n_sc[lens > 0])
    stop = emu['stop']
    assert ((stop == 31) | (stop == 63)).any() and ((stop == 32) | (stop == 64)).any() and (stop == 0).any()
    assert (lens == 4096).any() and (stop[lens == 4096] < 0).any()
    g = torch.Generator().manual_seed(n_rays)
    gw, gl = torch.randn(alpha.numel(), generator=g), torch.randn(n_rays, generator=g)
    ga = ops.alpha2weight_backward(alpha.to(DEV), w, T, last, i_s, i_e, n_rays, gw.to(DEV), gl.to(DEV))
    GW = np.zeros((n_rays, S), F32)
    GW[valid] = gw.numpy()
    sc = emu['scanned']
    want = emulate_backward(A, Td, Wd, h(last), sc, sc, GW, np.zeros_like(GW), gl.numpy())
    got = np.zeros((n_rays, S), F32)
    got[valid] = h(ga)
    if not np.array_equal(got[valid], np.where(sc, want, 0)[valid]):
        fails.append(f'alpha2weight_backward: {int((got != np.where(sc, want, 0))[valid].sum())} elements differ from the emulation')
    T64, w64, last64, _, ns = fp64_forward(A, sc)
    ga64, mag = fp64_chain(A, sc, sc, T64, w64, last64, Td, Wd, h(last), GW, np.zeros_like(GW), gl.numpy())
    fails += judge_chain(f'alpha2weight {n_rays} rays', got, ga64, mag, ns)
    assert not fails, '\n'.join(fails)


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    if WORST:
        print('\n[transmittance] worst ratios: ' + ', '.join(f'{k} {v:.2e}' for k, v in sorted(WORST.items())))


# ---- CPU: the judges reject one injected fault each -------------------------------------------------------------------------
def _checker_scene():
    """Rays of 4096, 100 and 70 samples: tiny alphas on the long ray (no stop), a stop at 71 on the second, thres = 1e-4 with
    listed-but-not-kept samples on the third."""
    g = np.random.default_rng(1)
    S = 4096
    n = np.array([4096, 100, 70])
    alpha = (g.uniform(0.5, 1.5, (3, S)) * 5e-4).astype(F32)
    alpha[1, 71] = F32(0.9995)
    alpha[2] = (g.uniform(0.3, 3.0, S) * 1e-4).astype(F32)
    alpha[2, 5] = F32(0.5)
    valid = np.arange(S)[None] < n[:, None]
    alpha = np.where(valid, alpha, F32(0))
    thres = np.array([0, 0, 1e-4], F32)
    with np.errstate(divide='ignore'):
        dens = np.where(valid, np.log(np.power(1 - alpha.astype(F64), -2.0) - 1) - BOX_SHIFT, 0).astype(F32)
    return alpha, valid, thres, dens, n


def test_checker_rejects_faults():
    """An honest fp32 restatement passes every judge; one dropped chain term on the 4096-step ray, my_back from the neighbouring
    sample, T of the next sample, the missing g_last term, the stop one sample late, g_weight read at a scanned-but-not-kept
    sample and the missing 1/P at P = 9 are each rejected."""
    seen = dict(WORST)                  # the faults' ratios are not measurements of the kernels
    try:
        _check_faults()
    finally:
        WORST.clear()
        WORST.update(seen)


def _check_faults():
    alpha, valid, thres, dens, n = _checker_scene()
    emu = emulate_forward(alpha, valid, valid, thres)
    assert emu['stop'][0] < 0 and emu['stop'][1] == 71
    kp, sc = emu['keep'], emu['scanned']
    lnk = sc & ~kp
    assert lnk[2].any() and kp[2].any()
    g = np.random.default_rng(2)
    gw = np.where(kp, g.standard_normal(alpha.shape), 0).astype(F32)
    gal = np.where(kp, g.standard_normal(alpha.shape), 0).astype(F32)
    gl = g.standard_normal(3).astype(F32)
    zeros = np.zeros_like(gw)
    T, w, last = emu['T'], emu['w'], emu['last']
    ga = emulate_backward(alpha, T, w, last, sc, kp, gw, gal, gl)
    rec = dict(T=T, w=w, flags=emu['flags'], last=last)
    assert not judge_forward('checker honest', rec, emu, alpha, valid)
    T64, w64, last64, _, ns = fp64_forward(alpha, sc)
    ga64, mag = fp64_chain(alpha, sc, kp, T64, w64, last64, T, w, last, gw, gal, gl)
    assert not judge_chain('checker honest', ga, ga64, mag, ns)

    def gd_fails(ga_got, P=1, P_got=None):
        want, bound = gd_expect(dens, BOX_SHIFT, BOX_INTERVAL, P, kp, zeros, ga)
        got = fp32_gd(dens, BOX_SHIFT, BOX_INTERVAL, P if P_got is None else P_got, kp, zeros, ga_got)
        got = np.where(valid, got, np.nan)
        return judge_gd('checker', got, want, bound, valid, valid)
    assert not gd_fails(ga) and not gd_fails(ga, P=9)
    # on the 4096-step ray, the chain term of a sample in the middle: every sample before it sees it
    faults = {
        'chain term dropped (4096-step ray)': gd_fails(emulate_backward(alpha, T, w, last, sc, kp, gw, gal, gl, 'drop', (0, 2048))),
        'my_back of the neighbouring sample': gd_fails(emulate_backward(alpha, T, w, last, sc, kp, gw, gal, gl, 'neighbour')),
        'T of the next sample': gd_fails(emulate_backward(alpha, T, w, last, sc, kp, gw, gal, gl, 'next_T')),
        'g_last term missing': gd_fails(emulate_backward(alpha, T, w, last, sc, kp, gw, gal, gl, 'no_glast')),
        'g_weight read at a scanned-but-not-kept sample': gd_fails(emulate_backward(
            alpha, T, w, last, sc, kp | lnk, np.where(lnk, F32(1.0), gw), np.where(lnk, F32(0), gal), gl)),
        '1/P missing at P = 9': gd_fails(ga, P=9, P_got=1),
    }
    late = emulate_forward(alpha, valid, valid, thres, late_stop=True)
    assert late['stop'][1] == 72
    faults['stop one sample late'] = judge_forward('checker late stop', dict(T=late['T'], w=late['w'], flags=late['flags'],
                                                                            last=late['last']), emu, alpha, valid)
    print('[transmittance checker] ' + '; '.join(f'{k}: {v[0] if v else "ACCEPTED"}' for k, v in faults.items()))
    accepted = [k for k, v in faults.items() if not v]
    assert not accepted, f'faults the judges accept: {accepted}'
