"""Time metrics.rgb_ssim (csrc/metrics.cu) against the reference's scipy utils.rgb_ssim on the same frames and print one JSON line.

    python scripts/bench_ssim.py [--steps 20] [--warmup 3]

Frames: 1008 x 756 (llff), 1237 x 822 (bicycle_single), 1600 x 1067 (garden) and 1920 x 1080, a seeded near-identical pair (a
textured frame and the same frame plus 1e-4 noise, oracle.ssim_ref.ssim_frames).  Per frame: CUDA-event time of the kernel pair
on device-resident images, mean only and with the map written; host-clock time of a call on numpy arrays (upload included);
the scipy time of the reference's own function (staged into oracle/_ref/py by __graft_entry__.build()) on the same frame in the
same run; the map and the mean against scipy's; algorithmic bytes and fp64 FLOPs, and which of the two bounds the kernel at
the H100 SXM data-sheet peaks (3.35 TB/s HBM3, 34 TFLOP/s FP64 without tensor cores, both for a 700 W card).  The card's name and
power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_dvgo import _gpu, _time  # noqa: E402

FRAMES = [(1008, 756), (1237, 822), (1600, 1067), (1920, 1080)]
PEAK_BYTES, PEAK_FP64 = 3.35e12, 34e12


def _reference_ssim():
    """utils.rgb_ssim from the staged reference (its imports: cv2, and adam_upd_cuda through masked_adam.py)."""
    import types
    from unboundednerfpytorch_b200 import legacy
    py = os.path.join(ROOT, 'oracle', '_ref', 'py')
    if not os.path.exists(os.path.join(py, 'FourierGrid', 'utils.py')):
        raise SystemExit('oracle/_ref/py/FourierGrid/utils.py is missing: run __graft_entry__.build() where the reference exists')
    legacy.install()
    try:
        import cv2  # noqa: F401
    except ImportError:
        sys.modules['cv2'] = types.ModuleType('cv2')
    sys.path.insert(0, py)
    try:
        from FourierGrid import utils
    finally:
        sys.path.remove(py)
    return utils.rgb_ssim


def _work(H, W, f, with_map):
    """Least bytes and fp64 FLOPs of separable 'valid' SSIM: both images read once (and the map written once); per channel the
    horizontal pass filters 5 moments over H x Wo positions and the vertical pass over Ho x Wo, f FMAs (2 FLOPs) each, plus ~23
    FLOPs of epilogue per map element (the kernel also refilters the f - 1 halo rows of each 32-row tile, not counted here)."""
    Ho, Wo = H - f + 1, W - f + 1
    nbytes = 2 * H * W * 3 * 4 + (Ho * Wo * 3 * 8 if with_map else 0)
    flops = 3 * (5 * 2 * f * (H * Wo + Ho * Wo) + 23 * Ho * Wo)
    return nbytes, flops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    from oracle.ssim_ref import ssim_frames
    from unboundednerfpytorch_b200 import metrics
    ref_ssim = _reference_ssim()
    name, power = _gpu()
    out = {'bench': 'rgb_ssim', 'gpu': name, 'power_limit': power, 'steps': args.steps, 'frames': {}}
    for W, H in FRAMES:
        a, b = ssim_frames('near', H, W, seed=W)
        ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        ms_mean = _time(lambda i: metrics.rgb_ssim(ta, tb, 1), args.steps, args.warmup)
        ms_map = _time(lambda i: metrics.rgb_ssim(ta, tb, 1, return_map=True), args.steps, args.warmup)
        metrics.rgb_ssim(a, b, 1)
        t0 = time.perf_counter()
        for _ in range(5):
            ours_mean = metrics.rgb_ssim(a, b, 1)
        ms_numpy = (time.perf_counter() - t0) / 5 * 1e3
        ours_map = metrics.rgb_ssim(ta, tb, 1, return_map=True).cpu().numpy()
        t0 = time.perf_counter()
        ref_map = ref_ssim(a, b, max_val=1, return_map=True)
        s_scipy = time.perf_counter() - t0
        rec = {'ssim_ms': round(ms_mean, 4), 'ssim_with_map_ms': round(ms_map, 4), 'numpy_call_ms': round(ms_numpy, 3),
               'scipy_s': round(s_scipy, 3), 'speedup_vs_scipy': round(s_scipy * 1e3 / ms_mean, 1),
               'map_max_abs_err': float(np.abs(ours_map - ref_map).max()),
               'mean_abs_err': abs(float(ours_mean) - float(np.mean(ref_map))), 'mean': float(ours_mean)}
        for tag, ms, with_map in (('mean', ms_mean, False), ('map', ms_map, True)):
            nbytes, flops = _work(H, W, 11, with_map)
            t_bytes, t_flops = nbytes / PEAK_BYTES, flops / PEAK_FP64
            rec[f'{tag}_bytes'] = nbytes
            rec[f'{tag}_fp64_flops'] = flops
            rec[f'{tag}_bound'] = 'fp64' if t_flops > t_bytes else 'hbm'
            rec[f'{tag}_share_of_peak'] = round(max(t_bytes, t_flops) / (ms * 1e-3), 3)
            rec[f'{tag}_fp64_tflops'] = round(flops / (ms * 1e-3) / 1e12, 2)
        out['frames'][f'{W}x{H}'] = rec
    print(json.dumps(out))


if __name__ == '__main__':
    main()
