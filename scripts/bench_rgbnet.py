"""The rgbnet alone (shade.shade forward + backward, csrc/shade_tc.cu) at one of two shapes, seeded inputs:

* ``--shape truck`` (default): 12 -> 128 -> 128 -> 3 (27 view-embedding columns), M = 4,194,304 samples, 8192 rays with sorted
  ray_id (512 consecutive samples per ray);
* ``--shape llff``: DirectMPIGO of llff_default, 9 -> 64 -> 64 -> 3 (3 view-direction columns), M = the survivor count
  scripts/bench_mpi.py reports for its 4096 rays (override with --samples), in rays of 255 consecutive samples (mpi_depth 128 at
  stepsize 0.5).

Prints one JSON line:

* ms             -- CUDA events around the forward launch (``rgbnet_fwd``) and around the two backward launches
                    (``rgbnet_bwd``), mean over --iters steps after --warmup;
* kernels_ms     -- with --profile DIR: per-kernel mean times from a torch.profiler run of its own (trace written to DIR);
* rates          -- per kernel (or the backward pair from the events): HMMA-equivalent TFLOP/s, counting every issued
                    mma.m16n8k8 TF32 as 16 * 8 * 8 * 2 FLOP (3xTF32 issues three per product), and algorithmic HBM GB/s
                    (the bytes each kernel must read and write, computed from the shapes below), with the share of the H100 SXM
                    data-sheet peaks (495 TFLOP/s dense TF32, 3.35 TB/s);
* max_err        -- every gradient (k0, W1, b1, W2, b2, W3, b3) at the timed size against an fp64 evaluation, as a fraction of
                    the largest element of the fp64 gradient (samples whose fp64 pre-activations come within 1e-5 of zero are
                    dropped for this check, as in tests/test_gpu_models.py);
* dw2            -- with --dw2 mma,wgmma (width 128): the dW2 engines timed alternately in this one run, --rounds times each
                    (a torch.profiler pass per round), with the rates of the fastest round and max_err for each engine;
* fwd            -- with --fwd mma,wgmma (width 128): the same for the forward engines (k_shade_fwd_tc, k_shade_fwd_wgmma);
* gpu / power_limit_w -- where it ran, read in the same run.

    python scripts/bench_rgbnet.py [--shape truck|llff] [--iters 20] [--warmup 3] [--profile DIR] [--no-check]
                                   [--dw2 mma,wgmma] [--fwd mma,wgmma] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TF32_PEAK = 495e12          # H100 SXM data sheet, dense
HBM_PEAK = 3.35e12
MMA_FLOP = 16 * 8 * 8 * 2
LLFF_SURVIVORS = 412_419     # outputs.survivors of scripts/bench_mpi.py at its 4096 rays (seeded scene, before training)
# issued mma.m16n8k8 per sample in the default 3xTF32 build (read off the SASS of the kernels)
HMMA_PER_SAMPLE = {'k_shade_fwd_tc': 864 / 16,      # layer 1 (2 k-steps) + layer 2 (16 k-steps), 16 column tiles, 3 passes
                   'k_shade_bwd_tc': 1120 / 16,     # dH1 768 + dX 96 + dW1k/view bias 96 + dW3 96 + E 64, per 16-sample unit
                   'k_shade_dw2_tc': 1536 / 32,     # 8 warps x 4 k-steps x 16 column tiles x 3 passes per 32-sample chunk
                   'k_shade_dw2_wgmma': 1536 / 32,  # the same products as 2 warpgroups x 4 k-steps x 3 wgmma.m64n128k8
                   'k_shade_fwd_wgmma': 864 / 16,   # the same products as 18 k-steps x 3 wgmma.m64n128k8 per 64-sample tile
                   # width 64, 9 features
                   'k_shade_fwd_tc_w': 240 / 16,    # layer 1 (2 k-steps) + layer 2 (8 k-steps), 8 column tiles, 3 passes
                   'k_shade_bwd_tc_w': 368 / 16,    # dH1 192 + dX 48 + dW1k/view bias 48 + dW3 48 + E 32, per 16-sample unit
                   'k_shade_dw2_tc_w': 384 / 32}    # 8 warps x 4 k-steps x 4 column tiles x 3 passes per 32-sample chunk
# bytes each kernel must move per sample (fp32 unless noted)
BYTES_PER_SAMPLE = {'k_shade_fwd_tc': 48 + 8 + 12 + 512 + 512 + 16,          # feat, ray_id, rgb, H1 + H2 saves, H1 masks
                    'k_shade_bwd_tc': 512 + 48 + 12 + 12 + 8 + 16 + 48 + 16,  # H2, feat, rgb, grad_rgb, ray_id, H1 masks; grad_feat, H2 masks
                    'k_shade_dw2_tc': 512 + 16 + 12 + 12,                     # H1, H2 masks, rgb, grad_rgb
                    'k_shade_dw2_wgmma': 512 + 16 + 12 + 12,
                    'k_shade_fwd_wgmma': 48 + 8 + 12 + 512 + 512 + 16,
                    'k_shade_fwd_tc_w': 36 + 8 + 12 + 256 + 256 + 8,          # the same at width 64 with 9 features
                    'k_shade_bwd_tc_w': 256 + 36 + 12 + 12 + 8 + 8 + 36 + 8,
                    'k_shade_dw2_tc_w': 256 + 8 + 12 + 12}
# shape -> feature columns, hidden width, view-embedding columns, kernel-name suffix, default samples and rays
# --dw2 engine name -> ubn_set_dw2_engine value and the kernel it runs at width 128
DW2_ENGINES = {'mma': (0, 'k_shade_dw2_tc'), 'wgmma': (1, 'k_shade_dw2_wgmma')}
# --fwd engine name -> ubn_set_fwd_engine value and the forward kernel it runs at width 128
FWD_ENGINES = {'mma': (0, 'k_shade_fwd_tc'), 'wgmma': (1, 'k_shade_fwd_wgmma')}
SHAPES = {'truck': dict(K=12, W=128, E=27, sfx='', samples=4_194_304, rays=8192),
          'llff': dict(K=9, W=64, E=3, sfx='_w', samples=LLFF_SURVIVORS, rays=None)}


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def _inputs(M, n_rays, K, W, E, seed=0):
    """n_rays = None: rays of 255 consecutive samples (the last one shorter)"""
    from unboundednerfpytorch_b200 import models
    torch.manual_seed(seed)
    net = models._make_rgbnet(K + E, W, 3).cuda()
    g = torch.Generator().manual_seed(seed)
    k0 = torch.randn(M, K, generator=g).cuda()
    if n_rays is None:
        ray_id = (torch.arange(M) // 255).cuda()
        n_rays = -(-M // 255)
    else:
        ray_id = torch.arange(n_rays).repeat_interleave(M // n_rays).cuda()
    emb = torch.randn(n_rays, E, generator=g).cuda()
    gr = torch.randn(M, 3, generator=g).cuda()
    return net, k0, emb, ray_id, gr


def _step(shade, net, k0, emb, ray_id, gr):
    net.zero_grad(set_to_none=True)
    k0.grad = None
    out = shade.shade(net, k0, emb, ray_id)
    out.backward(gr)


def _rates(name, ms, M):
    flop = HMMA_PER_SAMPLE[name] * MMA_FLOP * M
    byt = BYTES_PER_SAMPLE[name] * M
    return dict(ms=round(ms, 3), tflops_hmma_equiv=round(flop / ms / 1e9, 1), share_of_tf32_datasheet=round(flop / ms / 1e9 / (TF32_PEAK / 1e12), 3),
                hbm_gbs=round(byt / ms / 1e6, 1), share_of_hbm_datasheet=round(byt / ms * 1e3 / HBM_PEAK, 3))


def _kernel_ms(shade, inputs, iters, names, trace=None):
    """per-kernel mean device time (ms) over iters steps, from a torch.profiler pass of its own"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            _step(shade, *inputs)
        torch.cuda.synchronize()
    if trace:
        prof.export_chrome_trace(trace)
    kms = {}
    for ev in prof.key_averages():
        for kname in names:
            if kname + '<' in ev.key:
                t = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0.0)
                kms[kname] = kms.get(kname, 0.0) + t / 1e3 / iters
    return kms


def _check(shade, net, k0, emb, ray_id, gr, chunk=200_000):
    """max |grad - grad_fp64| / max |grad_fp64| for k0 and every parameter, at the full size, ReLU-ambiguous samples dropped"""
    from unboundednerfpytorch_b200 import models
    W1, b1, W2, b2 = (p.double() for p in (net[0].weight, net[0].bias, net[2][0].weight, net[2][0].bias))
    ok = torch.empty(k0.shape[0], dtype=torch.bool, device=k0.device)
    with torch.no_grad():
        for lo in range(0, k0.shape[0], chunk):
            sl = slice(lo, lo + chunk)
            z1 = torch.cat([k0[sl], emb[ray_id[sl]]], -1).double() @ W1.t() + b1
            z2 = torch.relu(z1) @ W2.t() + b2
            ok[sl] = torch.minimum(z1.abs().amin(1), z2.abs().amin(1)) > 1e-5
    k0, ray_id, gr = k0[ok].clone().requires_grad_(True), ray_id[ok].contiguous(), gr[ok].contiguous()
    net64 = models._make_rgbnet(net[0].weight.shape[1], net[0].weight.shape[0], 3).cuda().double()
    net64.load_state_dict({k: v.double() for k, v in net.state_dict().items()})
    k64 = k0.detach().double().requires_grad_(True)
    for lo in range(0, k0.shape[0], chunk):
        sl = slice(lo, lo + chunk)
        out64 = torch.sigmoid(net64(torch.cat([k64[sl], emb[ray_id[sl]].double()], -1)))
        (out64 * gr[sl].double()).sum().backward()
    want = [k64.grad] + [p.grad for p in net64.parameters()]
    _step(shade, net, k0, emb, ray_id, gr)
    got = [k0.grad] + [p.grad for p in net.parameters()]
    err = {}
    for a, b, nm in zip(got, want, ['k0', 'W1', 'b1', 'W2', 'b2', 'W3', 'b3']):
        err[nm] = float((a.double() - b).abs().max() / b.abs().max())
    return err, int(k0.shape[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--shape', choices=sorted(SHAPES), default='truck')
    ap.add_argument('--samples', type=int, default=None)
    ap.add_argument('--rays', type=int, default=None)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--profile', default=None, help='also run a torch.profiler pass and write its trace under this directory')
    ap.add_argument('--no-check', action='store_true')
    ap.add_argument('--dw2', default=None, help='comma list of dW2 engines (mma, wgmma) to time alternately, width 128 only')
    ap.add_argument('--fwd', default=None, help='comma list of forward engines (mma, wgmma) to time alternately, width 128 only')
    ap.add_argument('--rounds', type=int, default=3, help='rounds of the --dw2 / --fwd alternation')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_rgbnet.py needs a GPU')
    from unboundednerfpytorch_b200 import _cabi, shade
    name, power = _gpu_info()
    sh = SHAPES[args.shape]
    M = args.samples or sh['samples']
    assert M > 0, '--samples is required at this shape'
    net, k0, emb, ray_id, gr = _inputs(M, args.rays or sh['rays'], sh['K'], sh['W'], sh['E'])
    assert shade.supported(net, sh['K'])
    k0.requires_grad_(True)
    from unboundednerfpytorch_b200 import ops
    fwd_k, bwd_k = (f'k_shade_{n}_tc{sh["sfx"]}' for n in ('fwd', 'bwd'))
    if sh['W'] == 128 and shade.MODE in ('tc3', 'tc1') and ops.get_fwd_engine() == FWD_ENGINES['wgmma'][0]:
        fwd_k = FWD_ENGINES['wgmma'][1]     # the 8-warp forward's engine; tc3w4 runs the 4-warp k_shade_fwd_tc
    dw2_k = DW2_ENGINES['wgmma'][1] if sh['W'] == 128 else 'k_shade_dw2_tc_w'
    engines = args.dw2.split(',') if args.dw2 else []
    assert all(e in DW2_ENGINES for e in engines) and (not engines or sh['W'] == 128), '--dw2 takes mma / wgmma at width 128'
    fwd_engines = args.fwd.split(',') if args.fwd else []
    assert all(e in FWD_ENGINES for e in fwd_engines) and (not fwd_engines or sh['W'] == 128), '--fwd takes mma / wgmma at width 128'
    res = dict(metric=f'rgbnet forward + backward, {args.shape} shape', gpu=name, power_limit_w=power, samples=M,
               rays=emb.shape[0], features=sh['K'], width=sh['W'], mode=shade.MODE, bwd_mode=shade.BWD_MODE)
    for _ in range(args.warmup):
        _step(shade, net, k0, emb, ray_id, gr)
    torch.cuda.synchronize()
    _cabi.TIMER = _cabi.KernelTimer()
    for _ in range(args.iters):
        _step(shade, net, k0, emb, ray_id, gr)
    summ = _cabi.TIMER.summary()
    _cabi.TIMER = None
    res['ms'] = {k: round(v[0], 3) for k, v in summ.items()}
    res['rates'] = {fwd_k: _rates(fwd_k, summ['rgbnet_fwd'][0], M)}
    bwd = summ['rgbnet_bwd'][0]
    pair_flop = (HMMA_PER_SAMPLE[bwd_k] + HMMA_PER_SAMPLE[dw2_k]) * MMA_FLOP * M
    res['rates']['backward_pair'] = dict(ms=round(bwd, 3), tflops_hmma_equiv=round(pair_flop / bwd / 1e9, 1),
                                         share_of_tf32_datasheet=round(pair_flop / bwd / 1e9 / (TF32_PEAK / 1e12), 3))
    if args.profile:
        os.makedirs(args.profile, exist_ok=True)
        kms = _kernel_ms(shade, (net, k0, emb, ray_id, gr), args.iters, (fwd_k, bwd_k, dw2_k),
                         os.path.join(args.profile, 'bench_rgbnet.pt.trace.json'))
        res['kernels_ms'] = {k: round(v, 3) for k, v in kms.items()}
        for k, v in kms.items():
            res['rates'][k] = _rates(k, v, M)
    for key, names, table, setter in (('dw2', engines, DW2_ENGINES, ops.set_dw2_engine),
                                      ('fwd', fwd_engines, FWD_ENGINES, ops.set_fwd_engine)):
        if not names:
            continue
        runs = {e: [] for e in names}
        try:
            for _ in range(args.rounds):
                for e in names:
                    value, kname = table[e]
                    setter(value)
                    for _ in range(args.warmup):
                        _step(shade, net, k0, emb, ray_id, gr)
                    torch.cuda.synchronize()
                    runs[e].append(_kernel_ms(shade, (net, k0, emb, ray_id, gr), args.iters, (kname,))[kname])
            res[key] = {}
            for e in names:
                value, kname = table[e]
                res[key][e] = dict(kernel=kname, ms_rounds=[round(v, 3) for v in runs[e]], **_rates(kname, min(runs[e]), M))
                if not args.no_check:
                    setter(value)
                    err, _ = _check(shade, net, k0.detach(), emb, ray_id, gr)
                    res[key][e]['max_err_of_scale'] = {k: float(f'{v:.3g}') for k, v in err.items()}
        finally:
            setter(1)
    if not args.no_check:
        err, n = _check(shade, net, k0.detach(), emb, ray_id, gr)
        res['max_err_of_scale'] = {k: float(f'{v:.3g}') for k, v in err.items()}
        res['check_samples'] = n
        res['check_ok'] = all(v <= 1e-5 for v in err.values())
    print(json.dumps(res))


if __name__ == '__main__':
    main()
