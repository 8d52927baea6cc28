"""The per-ray composite and segment sums (csrc/alpha_ops.cu: k_composite_fwd / _bwd, k_segment_sum<K>, SegmentSum.backward,
segment_coo), the training losses of run_train.py:254-279 (csrc/loss.cu: k_render_loss + k_render_loss_finish behind
functional.render_loss) and the distortion loss (k_distortion_loss, flatten_eff_distloss) against plain fp64 restatements, element
by element.  The fp64 references restate run_train.py:254-279, FourierMSELoss (FourierGrid_model.py:114-130, through
torch.fft.fft in fp64) and the distortion maths of dcvgo.py:387-409 in torch float64, on fp64 copies of the fp32 inputs.

Notation: u = 2^-24; n_r = a ray's sample count; k_r = ceil(n_r / 32) + 5 (the lane chain plus five butterfly levels); N = the
batch size (rows of rgb_marched); R = ray_id.max() + 1.  Every bound is first order in u plus one u for the second-order terms,
and holds whether or not nvcc contracts a product and an add into an FMA: a fused product is exact, so contraction only removes
a rounding.  The loss weights reach the kernels as fp32 (one u each against the Python floats the reference uses).

Sums (exact emulation).  k_composite_fwd and k_segment_sum use __fmul_rn and plain fp32 adds only: lane L of the ray's warp adds
samples s+L, s+L+32, ... in order into +0.0, then the 32 lane sums are combined by an xor butterfly (o = 16, 8, 4, 2, 1) and lane
0 writes.  emulate_warp_sum restates that order with IEEE fp32 torch ops, so each output must equal it bit for bit; an empty ray
is +0.0.  Against fp64, the product (composite) is one u, the lane chain ceil(n_r/32) - 1 adds and the butterfly 5 adds, each u
of at most the sum of the magnitudes: |got - fp64| <= (k_r + 1) u sum|addends|.  The emulation is what catches an addend too small
for that bound (a dropped 1e-7 addend on a 4 096-sample ray).  k_composite_bwd must equal torch fp32 on the GPU bit for bit:
grad_rgb = g[rid] * w[:, None] and grad_w = (g0 r0 + g1 r1) + g2 r2 as separate ops; SegmentSum.backward is g[ray_id].

render_loss values (out = {loss, mse, entropy_last, rgbper, freq}).  The kernel forms each per-ray or per-sample term in fp32 and
adds the terms in double; with at most 2^22 double adds that accumulation is below u/128 of the magnitudes, counted as one u.
The finish divides in double and rounds to fp32: one u.
  mse:  d = fl(a - b) is u, d*d 2u + u:          C_MSE  = 2 + 1 + 1 + 1 = 5,  of sum d^2 / (3 N).
  freq: with D = sum_c |d_c| and X1a = |d0| + (|d1| + |d2|)/2, x0 = (d0 + d1) + d2 is within 3u D (u per d, two adds) and
        x1 = d0 - (d1 + d2)/2 within 3u X1a; x0^2 + 2 x1^2 then carries 6u D^2 + 12u X1a^2, two products and an add 2u:
                                                  C_FREQ = 6 + 2 + 1 + 1 = 10, of sum (D^2 + 2 X1a^2) / (3 N).
  entropy_last, p = clamp(a) (exact), lp = logf(p), lq = logf(fl(1 - p)): CUDA's logf is within 1 ulp <= 2u of the result; 1 - p
        is exact for p >= 1/2 (Sterbenz) and otherwise rounded by at most u/2 absolute, which moves lq by at most u absolute, and
        (1 - p) lq by at most u absolute.  Products u, (1 - p) recomputed u, the add 2u of the magnitudes:
                                                  C_ENT  = 2 + 1 + 1 + 2 + 1 + 1 = 8, of sum (|p lp| + |(1-p) lq|) / N, plus
        u * #{p < 1/2} / N absolute.
  rgbper: d u (2u on d^2), three fmaf 3u, times w u:  C_PER = 2 + 3 + 1 + 1 + 1 = 8, of sum |w| sum_c d^2 / N.
  loss = w_main mse + w_ent ent + w_per per + w_freq freq in fp32: sum_k |W_k| B_k + C_SUM u sum_k |W_k T_k|, C_SUM = 5 (weight
        rounding, product, three adds); with distortion, render_loss adds W_d * dl in torch fp32: |W_d| B_dist + 3u |W_d dl| + u |loss|.

render_loss gradients, element by element (the backward multiplies by the fp32 upstream scale: 2u more, folded into every C):
  g_rgb_marched: g_mse = fl(fl(2 W_main) / (3 N)) is 2u (3 N is exact below 2^24), g_frq likewise.  With A = g_mse d_c, A is within
        2u + u (d) + 2u (product, add); B = g_frq y, y = x0 + 2 x1 (channel 0) or x0 - x1 (channels 1, 2), y is within 4u (D + 2 X1a),
        B within 2u + 4u + 2u:                    C_GRGB = 8 + 1 + 2 = 11, of g_mse |d_c| + g_frq (D + 2 X1a).
  g_alphainv_last = W_e * (1/N) * (lq - lp) where the clamp passes: lp 2u |lp|, lq 2u |lq| + u <= 2u |lq| + 1.45u |lp| (p < 1/2
        means |lp| >= ln 2), the subtraction u, W_e / N three roundings, the product u:
                                                  C_GLAST = 3.45 + 1 + 3 + 1 + 0.55 + 2 = 11, of (W_e / N)(|lp| + |lq|).
        Its zero / non-zero mask must be torch's fp32 clamp backward mask (bounds rounded to fp32, [min, max] inclusive, NaN -> 0).
  g_raw_rgb = fl(fl(2 W_per) * fl(1/N)) * w * d: 3u + 2u + u (d):  C_GRAW = 6 + 1 + 2 = 9, of (2 W_per / N) |w| |d|.
  g_raw_density: bit-identical to (t < near_thres).float() * w_nearclip, t the fp32 tensor as torch compares it.

Distortion (L = sum_rays [sum_i iota/3 w_i^2 + 2 sum_i w_i (s_i W_<i - WS_<i)] / R).  The exclusive prefix is formed as
cw + (iw - w_i): iw is a 5-level Hillis-Steele scan (5u of the chunk's magnitudes up to and including i), cw the chain of chunk
totals (u per chunk), so W_<i is within (k_r + 2) u W_<=i and WS_<i within (k_r + 3) u WS_<=i (ws = fl(w s) adds u), both
INCLUSIVE of sample i because iw contains it.  The term adds s*pw, the subtraction, 2 w (.), the uniform part: 3u more; the double
sum is exact enough and the finish (fp32 1/R, rounding) is 2u: (k_r + 8) u <= C_DV k_r u with
  C_DV = 3 (k_r >= 6), of m_i = iota/3 w_i^2 + 2 |w_i| (|s_i| W_<=i + WS_<=i), summed and divided by R.
The gradient dL/dw_i = (1/R)(2/3 iota w_i + 2 (s_i W_<i - WS_<i) + 2 (WS_>i - s_i W_>i)) takes the strictly-after sums as
total - (cw + iw): the total and cw + iw are each within (k_r + 1) u W_r, so W_>i is within (2k_r + 2) u W_r and WS_>i within
(2k_r + 4) u WS_r; the prefixes add (k_r + 2) u and (k_r + 3) u, together (3k_r + 7) u of 2|s_i| W_r + 2 WS_r; the products, the
four adds, the uniform part and 1/R are 8u, the upstream scale 3u: (3k_r + 18) u <= C_DG k_r u with
  C_DG = 6 (k_r >= 6), of B_i = (2/3 iota |w_i| + 2 |s_i| W_r + 2 WS_r) / R,  W_r, WS_r the ray's totals of |w|, |w s|.
R must be ray_id.max() + 1: a batch whose last rays are empty would otherwise be divided by its size.

Wiring through the models: the fused forward of FourierGridModel, DirectContractedVoxGO (bg = 1), DirectMPIGO and DirectVoxGO,
render_loss with the bicycle weights, and each retained .grad (weights, raw_rgb, alphainv_last, raw_density) against fp64 autograd
of composite + alphainv_last * bg + the loss over fp64 copies of the returned tensors.  The composite's own error
delta_c <= (k_r + 2) u (sum |w rgb_c| + |last bg|) reaches g_rgb_marched through the linear loss gradient, |dg0| <= (g_mse +
3 g_frq) delta_0, |dg1| <= g_mse delta_1 + 1.5 g_frq (delta_1 + delta_2); the composite backward adds u (grad_rgb) or 3u (grad_w)
of its products, and torch's accumulation of two gradient contributions u of their magnitudes.

Worst ratios seen on an H100 80GB HBM3, |got - fp64| over the bound (1.0 = at the bound), over all cases: sums 0.40; values mse
0.16, freq 0.038, entropy_last 0.22, rgbper 0.093, distortion 0.0069, loss 0.15; gradients g_rgb_marched 0.22, g_alphainv_last
0.33, g_raw_rgb 0.31, distortion 0.089; through the models weights 0.13, raw_rgb 0.19, alphainv_last 0.22.  Into a pre-filled .grad
(1e-4, well above the gradients) the fp32 accumulate's own rounding, u of the sum, dominates and the ratios reach 0.99.  Every
emulated sum, composite / SegmentSum backward, entropy mask and nearclip gradient was bit-identical.

test_checker_rejects_faults (CPU) feeds the judges fp64 results rounded to fp32 (accepted) and eight injected faults (each
rejected): the distortion loss divided by the batch size, an inclusive prefix of w in the distortion gradient, an exclusive entropy mask,
t <= near_thres, coefficient 1 on X1 in the FourierMSE gradient, a chunk-edge sample credited to the next ray, a dropped 1e-7
addend on a 4 096-sample ray (caught by the emulation, accepted by fp64) and a missing 1/N on rgbper."""
import math

import numpy as np
import pytest
import torch

DEV = 'cuda:0'
U = 2.0 ** -24
F32 = np.float32
C_MSE, C_FREQ, C_ENT, C_PER, C_SUM = 5, 10, 8, 8, 5
C_GRGB, C_GLAST, C_GRAW = 11, 11, 9
C_DV, C_DG = 3, 6
LO32 = float(F32(1e-6))
HI32 = float(F32(1) - F32(1e-6))
NEAR = 0.7
N_MAX = 512
BICYCLE = dict(main=1.0, freq=5.0, ent=1e-3, clip=1.0, dist=0.05, per=1e-2)     # bicycle_single.py
DEFAULT = dict(main=1.0, freq=0.0, ent=0.01, clip=0.0, dist=0.0, per=0.1)       # default.py
WORST = {}


def _note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), float(r))


def _ratio(got, want, bound):
    """max |got - want| / bound (0 / 0 = 0, x / 0 = inf), NaN in got or want = inf."""
    err = (got.double() - want.double()).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound.double())
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    return float(r.max()) if r.numel() else 0.0


def _t64(x):
    return torch.tensor([x], dtype=torch.float64)


def _judge(fails, what, key, got, want, bound):
    r = _ratio(got, want, bound)
    _note(key, r)
    if r > 1:
        fails.append(f'{what}: {r:.3e} of its bound')


# ---- ray structure ------------------------------------------------------------------------------------------------------------
HEAD = [0, 0, 1, 2, 31, 32, 0, 33, 63, 64, 65, 1000, 0, 4096, 4097]


def ray_lengths(n_rays, seed):
    """Sample counts per ray: empty rays first, in the middle and as the last three rays, every 32-lane chunk edge, 1 000 and
    4 096 / 4 097 samples; the rest 0..7 samples."""
    if n_rays == 1:
        return np.array([4097])
    if n_rays == 3:
        return np.array([0, 65, 0])
    if n_rays == 5:
        return np.array([33, 0, 4096, 0, 0])
    g = np.random.default_rng(seed)
    mid = g.integers(0, 8, n_rays - len(HEAD) - 3)
    return np.concatenate([HEAD, mid, [0, 0, 0]]).astype(np.int64)


def layout(rid, n_rays):
    """(counts [n_rays], pos [n]: index of each sample inside its ray, k [n_rays] = ceil(n_r / 32) + 5)."""
    counts = torch.bincount(rid, minlength=n_rays)
    start = torch.cumsum(counts, 0) - counts
    pos = torch.arange(rid.numel(), device=rid.device) - start[rid]
    return counts, pos, (counts + 31) // 32 + 5


def make_batch(n_rays, seed, s_kind='contracted', device=DEV):
    """Crafted fp32 batch: w in [0, 0.1) with runs of zeros and an opaque sample near 1, raw_rgb / target / rgb_marched in [0, 1),
    alphainv_last with the clamp's boundary values and their neighbours, t with fp32(NEAR) and its neighbours, and s monotone
    per ray (contracted 1 - 1/(1 + t), or DirectMPIGO's (step_id + 0.5) / N_samples), or random (non-monotone)."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.from_numpy(ray_lengths(n_rays, seed))
    rid = torch.repeat_interleave(torch.arange(n_rays), lens)
    n = rid.numel()
    _, pos, _ = layout(rid, n_rays)
    w = torch.rand(n, generator=g) * 0.1
    w[(pos % 97) < 6] = 0.0                                          # runs of zero weights inside rays
    big = ((lens[rid] == 4096) & (pos == 100)) | ((lens[rid] == 33) & (pos == 32)) | ((lens[rid] == 65) & (pos == 0))
    w[big] = 0.9995
    raw = torch.rand(n, 3, generator=g)
    tgt = torch.rand(n_rays, 3, generator=g)
    rgbm = torch.rand(n_rays, 3, generator=g)
    t = (pos.float() + torch.rand(n, generator=g)) * (2.0 / 64)      # increasing along the ray, crosses NEAR
    nt = torch.tensor(NEAR, dtype=torch.float32)
    edge = torch.stack([nt, torch.nextafter(nt, torch.tensor(0.)), torch.nextafter(nt, torch.tensor(2.))])
    if s_kind == 'contracted':
        s = 1 - 1 / (1 + t)
    elif s_kind == 'mpi':
        step = pos * 2 + (torch.rand(n, generator=g) < 0.5).long()
        s = (step + 0.5) / 8200
    else:
        s = torch.rand(n, generator=g)
    if n >= 6:
        t[:6] = edge.repeat(2)                                       # after s: s stays monotone along the ray
    last = torch.rand(n_rays, generator=g)
    lo, hi = torch.tensor(LO32), torch.tensor(HI32)
    zero, two = torch.tensor(0.), torch.tensor(2.)
    special = torch.stack([zero, lo, torch.nextafter(lo, zero), torch.nextafter(lo, two), hi, torch.nextafter(hi, zero),
                           torch.nextafter(hi, two), torch.tensor(1.), torch.tensor(1.5), torch.tensor(2e-6)])
    k = min(n_rays, special.numel())
    last[:k] = special[:k]
    dens = torch.randn(n, generator=g)
    d = dict(rgb_marched=rgbm, alphainv_last=last, raw_rgb=raw, weights=w, ray_id=rid, raw_density=dens, t=t, s=s, n_max=N_MAX)
    return {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}, tgt.to(device)


# ---- sums: exact emulation and fp64 -------------------------------------------------------------------------------------------
def emulate_warp_sum(src, rid, n_rays, drop=None):
    """[n, K] fp32 -> [n_rays, K] fp32 in the kernels' order: lane L adds samples s+L, s+L+32, ... into +0.0, then
    acc += acc[lane ^ o] for o = 16 .. 1 and lane 0 is the result.  drop (checker): a sample index whose addend is skipped."""
    _, pos, _ = layout(rid, n_rays)
    lane, chunk = pos % 32, pos // 32
    K = src.shape[1]
    acc = torch.zeros(n_rays, 32, K, dtype=torch.float32, device=src.device)
    keep = torch.ones(rid.numel(), dtype=torch.bool, device=src.device)
    if drop is not None:
        keep[drop] = False
    order = torch.argsort(chunk, stable=True)
    sizes = torch.bincount(chunk).tolist() if chunk.numel() else []
    off = 0
    for c in sizes:
        idx = order[off:off + c]
        off += c
        idx = idx[keep[idx]]
        r, l = rid[idx], lane[idx]
        acc[r, l] = acc[r, l] + src[idx]
    lanes = torch.arange(32, device=src.device)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lanes ^ o]
    return acc[:, 0]


def fp64_warp_sum(src64, rid, n_rays):
    """(sum, sum of |addends|) per ray in fp64."""
    K = src64.shape[1]
    z = torch.zeros(n_rays, K, dtype=torch.float64, device=src64.device)
    return z.index_add(0, rid, src64), z.clone().index_add(0, rid, src64.abs())


def judge_sum(fails, what, got, emu, want, mag, counts, k):
    """Bit for bit against the emulation, empty rays +0.0, and within (k_r + 1) u sum|addends| of fp64."""
    if not torch.equal(got, emu):
        bad = int((got != emu).any(-1).sum())
        fails.append(f'{what}: {bad} rays differ from the fp32 emulation')
    empty = counts == 0
    if empty.any() and ((got[empty] != 0).any() or torch.signbit(got[empty]).any()):
        fails.append(f'{what}: empty rays are not +0.0')
    _judge(fails, what + ' vs fp64', 'sums vs fp64 / ((k_r + 1) u sum|addends|)', got, want,
           ((k + 1).double() * U)[:, None] * mag)


# ---- fp64 distortion (dcvgo.py:387-409) ---------------------------------------------------------------------------------------
def seg_excl_prefix(x, rid, counts, pos):
    """Exclusive prefix sums of x [n] (fp64) inside each ray, cumulated per ray (rays bucketed by length into dense rows)."""
    out = torch.zeros_like(x)
    n_rays = counts.numel()
    for lo, hi in ((0, 8), (8, 64), (64, 1 << 40)):
        rays = ((counts > lo) & (counts <= hi)).nonzero().squeeze(1)
        if not rays.numel():
            continue
        row = torch.full((n_rays,), -1, dtype=torch.long, device=x.device)
        row[rays] = torch.arange(rays.numel(), device=x.device)
        sel = (row[rid] >= 0).nonzero().squeeze(1)
        dense = torch.zeros(rays.numel(), int(counts[rays].max()), dtype=x.dtype, device=x.device)
        rr, pp = row[rid[sel]], pos[sel]
        dense[rr, pp] = x[sel]
        out[sel] = (torch.cumsum(dense, 1) - dense)[rr, pp]
    return out


def distortion_parts(w, s, rid, interval, fault=None):
    """fp64 value, gradient (per unit upstream), value magnitudes m_i and gradient magnitudes B_i.  fault (checker): 'batch_R'
    divides by the batch size, 'inclusive' takes the prefix of w inclusive in the gradient (pw = cw + iw; inclusive prefixes of
    both w and w s would cancel exactly: s_i w_i - w_i s_i = 0)."""
    n_rays = int(rid.max()) + 1
    counts, pos, _ = layout(rid, n_rays)
    w, s = w.double(), s.double()
    ws = w * s
    wp, wsp = seg_excl_prefix(w, rid, counts, pos), seg_excl_prefix(ws, rid, counts, pos)
    z = torch.zeros(n_rays, dtype=torch.float64, device=w.device)
    wt, wst = z.index_add(0, rid, w)[rid], z.clone().index_add(0, rid, ws)[rid]
    R = float(n_rays)
    value = ((interval / 3) * w * w + 2 * w * (s * wp - wsp)).sum() / R
    gp = wp + w if fault == 'inclusive' else wp
    grad = ((2 / 3) * interval * w + 2 * (s * (gp - (wt - wp - w)) + ((wst - wsp - ws) - wsp))) / R
    aw, aws = w.abs(), ws.abs()
    wpa, wspa = seg_excl_prefix(aw, rid, counts, pos) + aw, seg_excl_prefix(aws, rid, counts, pos) + aws
    m = (interval / 3) * w * w + 2 * aw * (s.abs() * wpa + wspa)
    Wr, WSr = z.clone().index_add(0, rid, aw)[rid], z.clone().index_add(0, rid, aws)[rid]
    B = ((2 / 3) * interval * aw + 2 * s.abs() * Wr + 2 * WSr) / R
    return value, grad, m, B, R


class Distortion64(torch.autograd.Function):
    """flatten_eff_distloss in fp64 with dcvgo.py's explicit backward."""

    @staticmethod
    def forward(ctx, w, s, interval, rid):
        value, grad, _, _, _ = distortion_parts(w, s, rid, interval)
        ctx.save_for_backward(grad)
        return value

    @staticmethod
    def backward(ctx, g):
        return ctx.saved_tensors[0] * g, None, None, None


# ---- fp64 loss (run_train.py:254-279) -----------------------------------------------------------------------------------------
def fp64_terms(rgbm, last, raw, w, rid, tgt, dens, t, s, W, near=NEAR, n_max=N_MAX):
    """The reference's loss composition in fp64 on fp64 tensors: (loss, dict of terms).  rgbper takes weights.detach(); the
    nearclip mask is taken on the fp32 t as the reference compares it."""
    tgt = tgt.double()
    mse = torch.nn.functional.mse_loss(rgbm, tgt)
    freq = torch.nn.functional.mse_loss(torch.fft.fft(rgbm, dim=-1).real, torch.fft.fft(tgt, dim=-1).real)
    loss = W['main'] * mse + W['freq'] * freq
    terms = dict(mse=mse, freq=freq)
    if W['ent'] > 0:
        pout = last.clamp(LO32, HI32)         # torch clamps an fp32 tensor with its bounds rounded to fp32
        terms['entropy_last'] = -(pout * torch.log(pout) + (1 - pout) * torch.log(1 - pout)).mean()
        loss = loss + W['ent'] * terms['entropy_last']
    if W['clip'] > 0:
        d = dens[t < near]
        loss = loss + W['clip'] * (d - d.detach()).sum()
    if W['dist'] > 0:
        terms['distortion'] = Distortion64.apply(w, s, 1 / n_max, rid)
        loss = loss + W['dist'] * terms['distortion']
    if W['per'] > 0:
        per = (raw - tgt[rid]).pow(2).sum(-1)
        terms['rgbper'] = (per * w.detach()).sum() / len(rgbm)
        loss = loss + W['per'] * terms['rgbper']
    return loss, terms


def loss_bounds(rgbm, last, raw, w, rid, tgt, s, W, scale=1.0, n_max=N_MAX):
    """Value bounds of each term and of the loss, and the per-element gradient bounds (before any prefill), all fp64."""
    N = rgbm.shape[0]
    d = rgbm.double() - tgt.double()
    D = d.abs().sum(1)
    X1a = d[:, 0].abs() + 0.5 * (d[:, 1].abs() + d[:, 2].abs())
    T, B = {}, {}
    T['mse'] = float((d * d).sum()) / (3 * N)
    B['mse'] = C_MSE * U * T['mse']
    B['freq'] = C_FREQ * U * float((D * D + 2 * X1a * X1a).sum()) / (3 * N)
    T['freq'] = float(((D * D + 2 * X1a * X1a)).sum()) / (3 * N)
    p = last.double().clamp(LO32, HI32)
    lp, lq = torch.log(p), torch.log(1 - p)
    ent_mag = (p * lp).abs() + ((1 - p) * lq).abs()
    fin = torch.isfinite(ent_mag)
    B['entropy_last'] = U * (C_ENT * float(ent_mag[fin].sum()) + float((p[fin] < 0.5).sum())) / N
    T['entropy_last'] = float(ent_mag[fin].sum()) / N
    dm = raw.double() - tgt.double()[rid]
    per_mag = w.double().abs() * (dm * dm).sum(1)
    B['rgbper'] = C_PER * U * float(per_mag.sum()) / N
    T['rgbper'] = float(per_mag.sum()) / N
    wk = dict(mse=W['main'], freq=W['freq'], entropy_last=W['ent'], rgbper=W['per'])
    B['loss'] = sum(abs(wk[k]) * B[k] for k in wk) + C_SUM * U * sum(abs(wk[k]) * T[k] for k in wk)
    G = {}
    g_mse, g_frq = W['main'] * 2 / (3 * N), W['freq'] * 2 / (3 * N)
    G['rgb'] = C_GRGB * U * abs(scale) * (g_mse * d.abs() + g_frq * (D + 2 * X1a)[:, None])
    G['last'] = C_GLAST * U * abs(scale) * (W['ent'] / N) * (lp.abs() + lq.abs())
    G['raw'] = C_GRAW * U * abs(scale) * (2 * W['per'] / N) * w.double().abs()[:, None] * dm.abs()
    if W['dist'] > 0:
        n_rays = int(rid.max()) + 1
        _, _, k = layout(rid, n_rays)
        _, _, m, Bd, R = distortion_parts(w, s, rid, float(F32(1 / n_max)))
        B['distortion'] = C_DV * U * float((k[rid].double() * m).sum()) / R
        G['w'] = C_DG * U * abs(scale * W['dist']) * k[rid].double() * Bd
    return B, G, (g_mse, g_frq)


def clamp_mask(last):
    """torch's fp32 clamp backward mask (on the tensor's device)."""
    a = last.detach().clone().requires_grad_(True)
    a.clamp(1e-6, 1 - 1e-6).backward(torch.ones_like(a))
    return a.grad != 0


def judge_loss(fails, tag, got_vals, want_vals, B, W, got_grads, want_grads, G, batch, prefill=None, scale=1.0, R_got=None):
    """Values and element-by-element gradients of render_loss against fp64 (keys of got_grads: rgb, last, raw, dens, w)."""
    on = dict(mse=True, freq=W['freq'] != 0, entropy_last=W['ent'] != 0, rgbper=W['per'] != 0, distortion=W['dist'] > 0)
    for k, bk in B.items():
        if k != 'loss' and on[k]:
            _judge(fails, f'{tag} {k}', f'value {k} / bound', _t64(got_vals[k]), _t64(want_vals[k]), _t64(bk))
    pre = prefill or {}
    sfx = ' (prefilled: the fp32 accumulate dominates)' if pre else ''

    def with_prefill(key, want, bound):
        if key not in pre:
            return want, bound
        p = pre[key].double()
        return p + want, bound + U * (p.abs() + want.abs())
    if 'rgb' in got_grads:
        want, bound = with_prefill('rgb', want_grads['rgb'], G['rgb'])
        _judge(fails, f'{tag} g_rgb_marched', 'g_rgb_marched / bound' + sfx, got_grads['rgb'], want, bound)
    if 'last' in got_grads:
        gl = got_grads['last']
        base = gl - pre['last'] if 'last' in pre else gl
        tm = clamp_mask(batch['alphainv_last'])
        wl = want_grads['last']
        if not torch.equal(base != 0, tm & (wl != 0)):
            fails.append(f'{tag} g_alphainv_last: zero / non-zero mask differs from torch clamp ('
                         f'{int(((base != 0) != (tm & (wl != 0))).sum())} elements)')
        want, bound = with_prefill('last', wl, G['last'])
        _judge(fails, f'{tag} g_alphainv_last', 'g_alphainv_last / bound' + sfx, gl, want, bound)
    if 'raw' in got_grads:
        want, bound = with_prefill('raw', want_grads['raw'], G['raw'])
        _judge(fails, f'{tag} g_raw_rgb', 'g_raw_rgb / bound' + sfx, got_grads['raw'], want, bound)
    if 'dens' in got_grads:
        exp = (batch['t'] < NEAR).float() * W['clip']
        if scale != 1.0:
            exp = exp * torch.tensor(scale, dtype=torch.float32, device=exp.device)
        if 'dens' in pre:
            exp = pre['dens'] + exp
        if not torch.equal(got_grads['dens'], exp):
            fails.append(f'{tag} g_raw_density: {int((got_grads["dens"] != exp).sum())} elements differ from '
                         f'(t < near_thres).float() * w_nearclip')
    if 'w' in got_grads:
        want, bound = with_prefill('w', want_grads['w'], G['w'])
        _judge(fails, f'{tag} distortion grad', 'distortion grad / (C_DG k_r u B_i)' + sfx, got_grads['w'], want, bound)
    return fails


def fp64_reference(batch, tgt, W, scale=1.0):
    """fp64 autograd of the loss over fp64 copies of the fp32 inputs: (values, grads)."""
    leaves = {k: batch[k].double().requires_grad_(True) for k in ('rgb_marched', 'alphainv_last', 'raw_rgb', 'weights',
                                                                  'raw_density')}
    loss, terms = fp64_terms(leaves['rgb_marched'], leaves['alphainv_last'], leaves['raw_rgb'], leaves['weights'],
                             batch['ray_id'], tgt, leaves['raw_density'], batch['t'], batch['s'].double(), W)
    (loss * scale).backward()
    vals = {k: float(v.detach()) for k, v in terms.items()}
    vals['loss'] = float(loss.detach())
    z = lambda k: leaves[k].grad if leaves[k].grad is not None else torch.zeros_like(leaves[k])   # noqa: E731
    grads = dict(rgb=z('rgb_marched'), last=z('alphainv_last'), raw=z('raw_rgb'), w=z('weights'), dens=z('raw_density'))
    return vals, grads


# ---- GPU: sums -----------------------------------------------------------------------------------------------------------------
N_RAYS = [1, 3, 5, 8192, 151_553, 1 << 20]


@pytest.mark.gpu
@pytest.mark.parametrize('n_rays', N_RAYS)
def test_composite_and_segment_sums_vs_emulation_and_fp64(n_rays):
    """k_composite_fwd and k_segment_sum<K> (K = 1..4) bit for bit against the emulation and within (k_r + 1) u of fp64;
    k_composite_bwd, SegmentSum.backward and segment_coo's out + form bit-identical to torch fp32; and wsum_mid's sparse ids."""
    from unboundednerfpytorch_b200.functional import composite_rgb, segment_coo, segment_sum
    batch, _ = make_batch(n_rays, 11 + n_rays)
    rid, w, rgb = batch['ray_id'], batch['weights'], batch['raw_rgb']
    counts, _, k = layout(rid, n_rays)
    fails = []
    wl, rl = w.clone().requires_grad_(True), rgb.clone().requires_grad_(True)
    out = composite_rgb(wl, rl, rid, n_rays)
    emu = emulate_warp_sum(w[:, None] * rgb, rid, n_rays)
    want, mag = fp64_warp_sum(w.double()[:, None] * rgb.double(), rid, n_rays)
    judge_sum(fails, f'composite ({n_rays} rays)', out.detach(), emu, want, mag, counts, k)
    g = torch.randn(n_rays, 3, device=DEV, generator=torch.Generator(DEV).manual_seed(n_rays))
    out.backward(g)
    gr = g[rid]
    if not torch.equal(rl.grad, gr * w[:, None]):
        fails.append('k_composite_bwd: grad_rgb != g[rid] * w[:, None]')
    gw = (gr[:, 0] * rgb[:, 0] + gr[:, 1] * rgb[:, 1]) + gr[:, 2] * rgb[:, 2]
    if not torch.equal(wl.grad, gw):
        fails.append(f'k_composite_bwd: grad_w differs from (g0*r0 + g1*r1) + g2*r2 at {int((wl.grad != gw).sum())} samples')
    gen = torch.Generator(DEV).manual_seed(7 * n_rays)
    for K in (1, 2, 3, 4):
        src = (torch.rand(rid.numel(), K, device=DEV, generator=gen) - 0.3) * 2
        src[::7] = 0.0
        sl = (src[:, 0] if K == 1 else src).clone().requires_grad_(True)
        got = segment_sum(sl, rid, n_rays)
        judge_sum(fails, f'segment_sum K={K} ({n_rays} rays)', got.detach().reshape(n_rays, K), emulate_warp_sum(src, rid, n_rays),
                  *fp64_warp_sum(src.double(), rid, n_rays), counts, k)
        go = torch.randn(got.shape, device=DEV, generator=gen)
        got.backward(go)
        if not torch.equal(sl.grad, go[rid]):
            fails.append(f'SegmentSum.backward K={K} != g[ray_id]')
    # segment_coo(src, index, out): out + the segment sums, gradients g and g[index]
    base = torch.randn(n_rays, 3, device=DEV, generator=gen).requires_grad_(True)
    src = rgb.clone().requires_grad_(True)
    res = segment_coo(src, rid, base)
    if not torch.equal(res.detach(), base.detach() + emulate_warp_sum(rgb, rid, n_rays)):
        fails.append('segment_coo: out + sums differs from the emulation')
    go = torch.randn(n_rays, 3, device=DEV, generator=gen)
    res.backward(go)
    if not (torch.equal(base.grad, go) and torch.equal(src.grad, go[rid])):
        fails.append('segment_coo backward: not (g, g[index])')
    # wsum_mid = segment_sum(weights[inner_mask], ray_id[inner_mask], N): sparse sorted ids, K = 1
    inner = torch.rand(rid.numel(), device=DEV, generator=gen) < 0.6
    inner[counts[rid] == 33] = False                  # whole rays drop out
    sid, sw = rid[inner], w[inner]
    if sid.numel():
        c2, _, k2 = layout(sid, n_rays)
        judge_sum(fails, f'wsum_mid ({n_rays} rays)', segment_sum(sw, sid, n_rays).reshape(n_rays, 1),
                  emulate_warp_sum(sw[:, None], sid, n_rays), *fp64_warp_sum(sw.double()[:, None], sid, n_rays), c2, k2)
    assert not fails, '\n'.join(fails)


# ---- GPU: losses ---------------------------------------------------------------------------------------------------------------
def _alone(term):
    W = dict(main=0.0, freq=0.0, ent=0.0, clip=0.0, dist=0.0, per=0.0)
    W[term] = {'main': 1.0, 'freq': 5.0, 'ent': 1e-3, 'clip': 1.0, 'dist': 0.05, 'per': 1e-2}[term]
    return W


LOSS_CASES = {
    'main_alone_5': (5, 'contracted', _alone('main'), 1.0, False),
    'freq_alone_3': (3, 'contracted', _alone('freq'), 1.0, False),
    'entropy_alone_8192': (8192, 'contracted', _alone('ent'), 1.0, False),
    'nearclip_alone_8192': (8192, 'contracted', _alone('clip'), 1.0, False),
    'distortion_alone_8192': (8192, 'contracted', _alone('dist'), 1.0, False),
    'rgbper_alone_8192': (8192, 'contracted', _alone('per'), 1.0, False),
    'bicycle_1': (1, 'contracted', BICYCLE, 1.0, False),
    'bicycle_5_nonmonotone_s': (5, 'random', BICYCLE, 1.0, False),
    'bicycle_8192_mpi_s': (8192, 'mpi', BICYCLE, 1.0, False),
    'bicycle_151553': (151_553, 'contracted', BICYCLE, 1.0, False),
    'bicycle_1M': (1 << 20, 'contracted', BICYCLE, 1.0, False),
    'default_151553': (151_553, 'contracted', DEFAULT, 1.0, False),
    'bicycle_8192_scaled': (8192, 'contracted', BICYCLE, 3.7, False),
    'bicycle_8192_prefilled': (8192, 'contracted', BICYCLE, 1.0, True),
}


def _run_render_loss(batch, tgt, W, scale=1.0, prefill=False, seed=0):
    """render_loss on leaf copies of the batch; returns (values, grads, prefill values)."""
    from unboundednerfpytorch_b200.functional import render_loss
    leaves = {k: batch[k].clone().requires_grad_(True) for k in ('rgb_marched', 'alphainv_last', 'raw_rgb', 'raw_density')}
    leaves['weights'] = batch['weights'].clone().requires_grad_(W['dist'] > 0)
    pre = {}
    if prefill:
        gen = torch.Generator(DEV).manual_seed(seed)
        for key, name in (('rgb', 'rgb_marched'), ('last', 'alphainv_last'), ('raw', 'raw_rgb'), ('dens', 'raw_density'),
                          ('w', 'weights')):
            if leaves[name].requires_grad:
                pre[key] = torch.randn(leaves[name].shape, device=DEV, generator=gen) * 1e-4
                leaves[name].grad = pre[key].clone()
    ret = dict(batch, **leaves)
    loss, terms = render_loss(ret, tgt, W['main'], W['ent'], W['per'], weight_freq=W['freq'], weight_nearclip=W['clip'],
                              near_thres=NEAR, weight_distortion=W['dist'])
    (loss * scale if scale != 1.0 else loss).backward()
    vals = {k: float(v) for k, v in terms.items()}
    vals['loss'] = float(loss.detach())
    grads = {}
    for key, name in (('rgb', 'rgb_marched'), ('last', 'alphainv_last'), ('raw', 'raw_rgb'), ('dens', 'raw_density'),
                      ('w', 'weights')):
        if leaves[name].grad is not None:
            grads[key] = leaves[name].grad
    return vals, grads, pre


def _loss_fails(tag, batch, tgt, W, scale, vals, grads, pre):
    want_vals, want_grads = fp64_reference(batch, tgt, W, scale)
    B, G, _ = loss_bounds(batch['rgb_marched'], batch['alphainv_last'], batch['raw_rgb'], batch['weights'], batch['ray_id'], tgt,
                          batch['s'], W, scale)
    if W['dist'] > 0:
        B['loss'] += W['dist'] * B['distortion'] + U * (3 * abs(W['dist'] * want_vals['distortion']) + abs(want_vals['loss']))
    fails = []
    _judge(fails, f'{tag} loss', 'value loss / bound', _t64(vals['loss']), _t64(want_vals['loss']), _t64(B['loss']))
    return judge_loss(fails, tag, vals, want_vals, B, W, grads, want_grads, G, batch, pre, scale)


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(LOSS_CASES))
def test_render_loss_vs_fp64(case):
    """render_loss: each term's value within C u of fp64, every gradient element within its own bound, the entropy mask and the
    nearclip gradient exact, R = ray_id.max() + 1 (the structured batches end in empty rays)."""
    n_rays, s_kind, W, scale, prefill = LOSS_CASES[case]
    batch, tgt = make_batch(n_rays, 101 + n_rays, s_kind)
    vals, grads, pre = _run_render_loss(batch, tgt, W, scale, prefill, seed=n_rays)
    for key, on in (('last', W['ent'] > 0), ('raw', W['per'] > 0), ('dens', W['clip'] > 0), ('w', W['dist'] > 0)):
        assert (key in grads) == on, f'{case}: gradient of {key} present = {key in grads}, term weight {W}'
    if W['dist'] > 0:
        counts = torch.bincount(batch['ray_id'], minlength=n_rays)
        R = int(batch['ray_id'].max()) + 1
        assert n_rays == 1 or R < n_rays, 'the batch must end in empty rays'
        assert R == int((counts > 0).nonzero().max()) + 1
    fails = _loss_fails(case, batch, tgt, W, scale, vals, grads, pre)
    assert not fails, '\n'.join(fails)


@pytest.mark.gpu
def test_entropy_nan_propagates_like_clamp():
    """A NaN alphainv_last makes entropy_last and the loss NaN, as torch's clamp does in the reference; its gradient element is
    0 (clamp's mask), and every other term and gradient element is still within its bound."""
    batch, tgt = make_batch(8192, 5)
    batch['alphainv_last'][20] = float('nan')
    W = BICYCLE
    seen = dict(WORST)                  # the NaN terms' ratios are not measurements
    vals, grads, pre = _run_render_loss(batch, tgt, W)
    want_vals, _ = fp64_reference(batch, tgt, W)
    assert math.isnan(want_vals['entropy_last']) and math.isnan(want_vals['loss'])
    assert math.isnan(vals['entropy_last']), f'entropy_last = {vals["entropy_last"]} for a NaN alphainv_last'
    assert math.isnan(vals['loss'])
    gl = grads['last']
    assert gl[20] == 0 and not torch.signbit(gl[20])
    assert torch.isfinite(gl).all() and torch.isfinite(grads['rgb']).all()
    fails = [f for f in _loss_fails('nan entropy', batch, tgt, W, 1.0, vals, grads, pre)
             if not f.startswith('nan entropy loss') and 'entropy_last:' not in f]
    WORST.clear()
    WORST.update(seen)
    assert not fails, '\n'.join(fails)


@pytest.mark.gpu
def test_zero_weights_give_no_gradient():
    """Zero entropy / rgbper / nearclip / distortion weights leave alphainv_last, raw_rgb, raw_density and weights without
    .grad and add no 'distortion' term; zero main and freq weights give an all-zero rgb_marched gradient."""
    batch, tgt = make_batch(8192, 17)
    W = dict(main=0.0, freq=0.0, ent=0.0, clip=0.0, dist=0.0, per=0.0)
    from unboundednerfpytorch_b200.functional import render_loss
    leaves = {k: batch[k].clone().requires_grad_(True) for k in ('rgb_marched', 'alphainv_last', 'raw_rgb', 'raw_density',
                                                                 'weights')}
    loss, terms = render_loss(dict(batch, **leaves), tgt, W['main'], W['ent'], W['per'], weight_freq=W['freq'],
                              weight_nearclip=W['clip'], near_thres=NEAR, weight_distortion=W['dist'])
    loss.backward()
    assert 'distortion' not in terms and float(loss) == 0.0
    for k in ('alphainv_last', 'raw_rgb', 'raw_density', 'weights'):
        assert leaves[k].grad is None, k
    assert (leaves['rgb_marched'].grad == 0).all()


@pytest.mark.gpu
def test_losses_deterministic_across_calls_and_streams():
    """Two calls give bit-identical values and gradients, on the default stream and on a side stream."""
    batch, tgt = make_batch(151_553, 23)
    runs = [_run_render_loss(batch, tgt, BICYCLE) for _ in range(2)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        runs.append(_run_render_loss(batch, tgt, BICYCLE))
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for v, g, _ in runs[1:]:
        for k in runs[0][0]:
            assert v[k] == runs[0][0][k] or (math.isnan(v[k]) and math.isnan(runs[0][0][k])), k
        for k in runs[0][1]:
            assert torch.equal(g[k], runs[0][1][k]), k


@pytest.mark.gpu
def test_distortion_R_from_ray_ids_not_batch_size():
    """flatten_eff_distloss divides by ray_id.max() + 1 whether or not the batch size is passed, with the last rays empty."""
    from unboundednerfpytorch_b200.functional import flatten_eff_distloss
    batch, _ = make_batch(8192, 31)
    w, s, rid = batch['weights'], batch['s'], batch['ray_id']
    value, grad, m, Bd, R = distortion_parts(w, s, rid, 1 / N_MAX)
    assert R < 8192
    k = layout(rid, int(R))[2][rid].double()
    for n_rays in (8192, None):
        wl = w.clone().requires_grad_(True)
        out = flatten_eff_distloss(wl, s, 1 / N_MAX, rid, n_rays=n_rays)
        out.backward()
        fails = []
        _judge(fails, f'distortion value (n_rays={n_rays})', 'value distortion / bound', out.detach().reshape(1),
               value.reshape(1), (C_DV * U * (k * m).sum() / R).reshape(1))
        _judge(fails, f'distortion grad (n_rays={n_rays})', 'distortion grad / (C_DG k_r u B_i)', wl.grad, grad, C_DG * U * k * Bd)
        assert not fails, '\n'.join(fails)


# ---- GPU: wiring through the models --------------------------------------------------------------------------------------------
def _model(name):
    """(model, rays_o, rays_d, viewdirs, render kwargs, bg or None) from the helpers the model tests use."""
    from tests.util import seeded_rays
    if name in ('fouriergrid', 'dcvgo'):
        from tests.test_gpu_models import _fresh_model
        m, _ = _fresh_model(name, 40 if name == 'fouriergrid' else 48, 3 if name == 'fouriergrid' else 0, 1e-4, 321,
                            dens_mean=6.0, dens_std=3.0, norm='l2')
        ro, rd, vd = (x.to(DEV) for x in seeded_rays(1024, 322))
        rk = dict(near=0., far=1e9, bg=1, rand_bkgd=False, stepsize=0.5, render_depth=False)
        return m.to(DEV), ro, rd, vd, rk, (None if name == 'fouriergrid' else 1.0)
    if name == 'mpi':
        from tests.test_gpu_mpi import RK, _ndc_scene
        m, ro, rd, vd = _ndc_scene(9, n=1024, seed=41)
        return m, ro, rd, vd, dict(RK, render_depth=False), float(RK['bg'])
    from tests.test_gpu_dvgo import RK, _scene, _vd
    m, ro, rd = _scene(3, n=1024, seed=43)
    return m, ro, rd, _vd(rd), dict(RK, render_depth=False), float(RK['bg'])


def _g_rgbm(rgbm64, tgt, W):
    """d(main * mse + freq * FourierMSE) / d rgb_marched in fp64."""
    r = rgbm64.clone().requires_grad_(True)
    loss, _ = fp64_terms(r, None, None, None, None, tgt, None, None, None, dict(W, ent=0.0, clip=0.0, dist=0.0, per=0.0))
    return torch.autograd.grad(loss, r)[0]


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['fouriergrid', 'dcvgo', 'mpi', 'dvgo'])
def test_model_forward_loss_gradients_vs_fp64(name):
    """The fused forward + render_loss (bicycle weights; DirectVoxGO without distortion and nearclip): each retained .grad of
    weights, raw_rgb, alphainv_last and raw_density against fp64 autograd of composite + alphainv_last * bg + the loss."""
    from unboundednerfpytorch_b200.functional import render_loss
    m, ro, rd, vd, rk, bg = _model(name)
    ret = m(ro, rd, vd, global_step=None, is_train=False, **rk)
    N = ro.shape[0]
    W = dict(BICYCLE)
    if 't' not in ret:
        W['clip'] = 0.0
    if 's' not in ret:
        W['dist'] = 0.0
    keys = [k for k in ('weights', 'raw_rgb', 'alphainv_last', 'raw_density') if k in ret and ret[k].requires_grad]
    assert {'weights', 'raw_rgb', 'alphainv_last'} <= set(keys)
    for k in keys:
        ret[k].retain_grad()
    tgt = torch.rand(N, 3, device=DEV, generator=torch.Generator(DEV).manual_seed(9))
    loss, terms = render_loss(ret, tgt, W['main'], W['ent'], W['per'], weight_freq=W['freq'], weight_nearclip=W['clip'],
                              near_thres=NEAR, weight_distortion=W['dist'])
    loss.backward()
    rid = ret['ray_id']
    assert rid.numel() > 10 * N
    w, rgb, last = ret['weights'].detach(), ret['raw_rgb'].detach(), ret['alphainv_last'].detach()
    # fp64 autograd of the composition over fp64 copies
    L = {k: ret[k].detach().double().requires_grad_(True) for k in keys}
    rgbm64 = torch.zeros(N, 3, dtype=torch.float64, device=DEV).index_add(0, rid, L['weights'][:, None] * L['raw_rgb'])
    if bg is not None:
        rgbm64 = rgbm64 + L['alphainv_last'][:, None] * bg
    dens64 = L.get('raw_density', torch.zeros(rid.numel(), dtype=torch.float64, device=DEV))
    t32 = ret.get('t')
    s64 = ret['s'].double() if 's' in ret else torch.zeros_like(dens64)
    loss64, _ = fp64_terms(rgbm64, L['alphainv_last'], L['raw_rgb'], L['weights'], rid, tgt, dens64, t32, s64, W, NEAR,
                           ret.get('n_max', N_MAX))
    loss64.backward()
    # bounds: the loss's own, plus the composite's error carried through the linear loss gradient
    batch = dict(rgb_marched=ret['rgb_marched'].detach(), alphainv_last=last, raw_rgb=rgb, weights=w, ray_id=rid,
                 s=ret.get('s', s64.float()), t=ret.get('t'))
    _, G, (g_mse, g_frq) = loss_bounds(batch['rgb_marched'], last, rgb, w, rid, tgt, batch['s'], W, 1.0, ret.get('n_max', N_MAX))
    _, _, k = layout(rid, N)
    cmag = torch.zeros(N, 3, dtype=torch.float64, device=DEV).index_add(0, rid, (w[:, None] * rgb).double().abs())
    if bg is not None:
        cmag = cmag + (last.double() * bg).abs()[:, None]
    delta = (k + 2).double()[:, None] * U * cmag
    dg = torch.stack([(g_mse + 3 * g_frq) * delta[:, 0], g_mse * delta[:, 1] + 1.5 * g_frq * (delta[:, 1] + delta[:, 2]),
                      g_mse * delta[:, 2] + 1.5 * g_frq * (delta[:, 1] + delta[:, 2])], 1)
    gm = _g_rgbm(rgbm64.detach(), tgt, W)                 # fp64 upstream gradient of rgb_marched
    Eg = G['rgb'] + dg                                   # bound on the kernel's g_rgb_marched per ray and channel
    fails = []
    # raw_rgb: fl(g[rid] * w) + rgbper's gradient, accumulated in fp32
    gr_c = gm[rid] * w.double()[:, None]
    b_raw = w.double().abs()[:, None] * Eg[rid] + U * gr_c.abs() + G['raw']
    b_raw = b_raw + U * (gr_c.abs() + L['raw_rgb'].grad.abs())
    _judge(fails, f'{name} raw_rgb.grad', 'model raw_rgb.grad / bound', ret['raw_rgb'].grad, L['raw_rgb'].grad, b_raw)
    # weights: (g0 r0 + g1 r1) + g2 r2 + the distortion term
    gw_c = (gm[rid] * rgb.double()).abs().sum(1)
    b_w = (rgb.double().abs() * Eg[rid]).sum(1) + 3 * U * gw_c
    if W['dist'] > 0:
        b_w = b_w + G['w']
    b_w = b_w + U * (gw_c + L['weights'].grad.abs())
    _judge(fails, f'{name} weights.grad', 'model weights.grad / bound', ret['weights'].grad, L['weights'].grad, b_w)
    # alphainv_last: bg * sum_c g_c (torch: product, then a 3-term sum) + the entropy term
    b_l = G['last'].clone()
    if bg is not None:
        b_l = b_l + abs(bg) * Eg.sum(1) + 3 * U * abs(bg) * gm.abs().sum(1)
    b_l = b_l + U * L['alphainv_last'].grad.abs()
    _judge(fails, f'{name} alphainv_last.grad', 'model alphainv_last.grad / bound', ret['alphainv_last'].grad,
           L['alphainv_last'].grad, b_l)
    if 'raw_density' in keys:
        exp = (ret['t'] < NEAR).float() * W['clip'] if W['clip'] > 0 else None
        got = ret['raw_density'].grad
        if exp is None:
            assert got is None
        else:
            assert (exp != 0).any() and (exp == 0).any()
            if not torch.equal(got, exp):
                fails.append(f'{name} raw_density.grad differs from (t < near_thres).float() * w_nearclip')
    assert not fails, '\n'.join(fails)


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    if WORST:
        print('\n[loss fp64] worst ratios: ' + ', '.join(f'{k} {v:.2e}' for k, v in sorted(WORST.items())))


# ---- CPU: the judges reject one injected fault each -------------------------------------------------------------------------
def test_checker_rejects_faults():
    """fp64 results rounded to fp32 pass every judge; each of the eight injected faults is rejected."""
    seen = dict(WORST)                  # the faults' ratios are not measurements of the kernels
    try:
        _check_faults()
    finally:
        WORST.clear()
        WORST.update(seen)


def _check_faults():
    assert F32(1) - F32(1e-6) == F32(1 - 1e-6)          # the kernel's 1.f - 1e-6f is torch's fp32 bound
    n_rays = 5                                             # rays of 33, 0, 4 096, 0 and 0 samples: R = 3
    batch, tgt = make_batch(n_rays, 3, device='cpu')
    rid, w, rgb = batch['ray_id'], batch['weights'], batch['raw_rgb']
    W = BICYCLE
    vals64, grads64 = fp64_reference(batch, tgt, W)
    honest_vals = {k: float(F32(v)) for k, v in vals64.items()}
    honest_grads = {k: v.float() for k, v in grads64.items()}
    honest_grads['dens'] = (batch['t'] < NEAR).float() * W['clip']
    assert torch.equal(honest_grads['dens'], grads64['dens'].float())

    def loss_fails(vals=None, **grads):
        return _loss_fails('checker', batch, tgt, W, 1.0, dict(honest_vals, **(vals or {})), dict(honest_grads, **grads), {})
    assert not loss_fails(), loss_fails()

    counts, pos, k = layout(rid, n_rays)
    prod = w[:, None] * rgb
    emu = emulate_warp_sum(prod, rid, n_rays)
    want, mag = fp64_warp_sum(w.double()[:, None] * rgb.double(), rid, n_rays)

    def sum_fails(got, wnt=want, mg=mag, em=emu):
        f = []
        judge_sum(f, 'checker sum', got, em, wnt, mg, counts, k)
        return f
    assert not sum_fails(emu) and not sum_fails(want.float())[1:]     # fp64 rounded: within the fp64 bound

    faults = {}
    # 1. the distortion loss divided by the batch size (the last two rays are empty)
    R = int(rid.max()) + 1
    assert R == 3 < n_rays
    dist_b = vals64['distortion'] * R / n_rays
    faults['distortion / batch size'] = loss_fails(dict(distortion=float(F32(dist_b)),
                                                        loss=float(F32(vals64['loss'] + W['dist'] * (dist_b - vals64['distortion'])))))
    # 2. an inclusive prefix of w in the distortion gradient
    _, g_incl, _, _, _ = distortion_parts(w, batch['s'], rid, 1 / N_MAX, fault='inclusive')
    faults['inclusive distortion prefix'] = loss_fails(w=(W['dist'] * g_incl).float())
    # 3. an exclusive entropy mask: no gradient at exactly 1e-6f and 1.f - 1e-6f
    a = batch['alphainv_last']
    assert (a == LO32).any() and (a == HI32).any()
    faults['exclusive entropy mask'] = loss_fails(last=torch.where((a == LO32) | (a == HI32), 0.0, honest_grads['last']))
    # 4. t <= near_thres
    assert (batch['t'] == F32(NEAR)).any()
    faults['t <= near_thres'] = loss_fails(dens=(batch['t'] <= NEAR).float() * W['clip'])
    # 5. coefficient 1 instead of 2 on X1 in the FourierMSE gradient (channel 0: g_frq (x0 + x1) instead of g_frq (x0 + 2 x1))
    d = batch['rgb_marched'].double() - tgt.double()
    x1 = d[:, 0] - 0.5 * (d[:, 1] + d[:, 2])
    g_rgb = grads64['rgb'].clone()
    g_rgb[:, 0] -= W['freq'] * 2 / (3 * n_rays) * x1
    faults['FourierMSE X1 coefficient 1'] = loss_fails(rgb=g_rgb.float())
    # 6. the chunk-edge sample (index 32 of the 33-sample ray) credited to the next ray
    edge = int(((counts[rid] == 33) & (pos == 32)).nonzero()[0])
    rid_f = rid.clone()
    rid_f[edge] += 1
    faults['chunk-edge sample in the next ray'] = sum_fails(emulate_warp_sum(prod, rid_f, n_rays))
    # 7. a dropped 1e-7 addend on the 4 096-sample ray: within the fp64 bound, not the emulation
    # (ray total ~0.25: a 1e-7 change is a few ulps of it, (k_r + 1) u sum|src| ~ 2e-6 is far above it)
    src = torch.rand(rid.numel(), 1, generator=torch.Generator().manual_seed(4)) * 1.2e-4
    s0 = int(((counts[rid] == 4096) & (pos == 5)).nonzero()[0])
    src[s0] = 1e-7
    em7 = emulate_warp_sum(src, rid, n_rays)
    w7, m7 = fp64_warp_sum(src.double(), rid, n_rays)
    assert not sum_fails(em7, w7, m7, em7)
    dropped = emulate_warp_sum(src, rid, n_rays, drop=s0)
    f7 = sum_fails(dropped, w7, m7, em7)
    assert f7 and all('emulation' in f for f in f7), f7         # the fp64 judge alone would accept it
    faults['dropped 1e-7 addend (4 096 samples)'] = f7
    # 8. rgbper without its 1/N
    faults['rgbper without 1/N'] = loss_fails(dict(rgbper=float(F32(vals64['rgbper'] * n_rays))),
                                              raw=(grads64['raw'] * n_rays).float())
    print('[loss fp64 checker] ' + '; '.join(f'{k}: {" | ".join(v) if v else "ACCEPTED"}' for k, v in faults.items()))
    accepted = [k for k, v in faults.items() if not v]
    assert not accepted, f'faults the judges accept: {accepted}'
