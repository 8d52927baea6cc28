"""Time the ARF colour transfer (arf.ARF, csrc/color.cu) against the reference's ARF on the same GPU and print one JSON line.

    python scripts/bench_arf.py [--steps 20] [--warmup 3] [--frames 16,64,256] [--reps 2]

Sets of 16, 64 and 256 frames at 1152 x 864 and 1920 x 1080 (uniform pixels, generated on the device).  Per set:

* device time of ubn_color_moments and of ubn_color_affine (CUDA events around each launch pair, warmed up, the two kernels
  alternating in one loop), and their effective HBM bandwidth against the 12 B/px they must read and the 12 + 12 B/px the
  transform must read and write (36 B/px in all), as a share of the H100 SXM data-sheet 3.35 TB/s;
* the call on a numpy set (what render_viewpoints returns) end to end, host clock around a synchronised call, with the
  host-to-device upload of the same array timed on its own;
* the reference's match_colors_for_image_set (its staged arf.py over oracle/_ref/py, imageio stubbed with cv2) on the same
  numpy set and GPU, end to end;
* the peak device memory of both calls (torch.cuda.max_memory_allocated above what was allocated before), and the largest
  pixel difference between the two results;
* the card's name and power limit, read in the same run."""
import argparse
import importlib.util
import json
import os
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_dvgo import _gpu  # noqa: E402

SIZES = [(1152, 864), (1920, 1080)]
PEAK_BYTES = 3.35e12


class _Imageio:
    @staticmethod
    def imread(path):
        return np.ascontiguousarray(cv2.imread(path, cv2.IMREAD_UNCHANGED)[..., ::-1])

    @staticmethod
    def imwrite(path, a):
        cv2.imwrite(path, np.ascontiguousarray(np.asarray(a)[..., ::-1]))


def _reference_arf():
    path = os.path.join(ROOT, 'oracle', '_ref', 'py', 'FourierGrid', 'arf.py')
    if not os.path.exists(path):
        raise SystemExit('oracle/_ref/py/FourierGrid/arf.py is missing: run __graft_entry__.build() where the reference exists')
    spec = importlib.util.spec_from_file_location('_staged_reference_arf', path)
    mod = importlib.util.module_from_spec(spec)
    saved = sys.modules.get('imageio')
    sys.modules['imageio'] = _Imageio()
    try:
        spec.loader.exec_module(mod)
    finally:
        if saved is None:
            del sys.modules['imageio']
        else:
            sys.modules['imageio'] = saved
    return mod.ARF


class _Cfg(dict):
    def __getattr__(self, k):
        return self[k]


def _device_times(x, steps, warmup):
    """(moments ms, affine ms) per call: both kernels alternate in one loop, each bracketed by its own events."""
    import ctypes
    from unboundednerfpytorch_b200 import _cabi
    lib = _cabi.load()
    n = x.numel() // 3
    scratch = torch.empty(9 * _cabi.COLOR_MAX_CTAS, dtype=torch.float64, device=x.device)
    out9 = torch.empty(9, dtype=torch.float64, device=x.device)
    y = torch.empty_like(x)
    T = (ctypes.c_float * 9)(0.9, 0.05, 0.05, 0.05, 0.9, 0.05, 0.05, 0.05, 0.9)
    b = (ctypes.c_float * 3)(0.01, 0.01, 0.01)
    stream = _cabi.stream_of(x)

    def moments():
        _cabi.check(lib.ubn_color_moments(_cabi.ptr(x), _cabi.c_i64(n), _cabi.ptr(scratch), _cabi.ptr(out9), stream))

    def affine():
        _cabi.check(lib.ubn_color_affine(_cabi.ptr(x), _cabi.ptr(y), _cabi.c_i64(n), T, b, stream))
    for _ in range(warmup):
        moments()
        affine()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(steps)]
    for e in ev:
        e[0].record()
        moments()
        e[1].record()
        e[2].record()
        affine()
        e[3].record()
    torch.cuda.synchronize()
    del y
    return (sum(e[0].elapsed_time(e[1]) for e in ev) / steps, sum(e[2].elapsed_time(e[3]) for e in ev) / steps)


def _peak_and_time(fn, reps):
    """(result of the last call, mean host-clock ms of a synchronised call, peak device bytes above the starting allocation)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ms = []
    res = None
    for _ in range(reps):
        res = None
        t0 = time.perf_counter()
        res = fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return res, float(np.mean(ms)), torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--frames', default='16,64,256')
    ap.add_argument('--reps', type=int, default=2)
    args = ap.parse_args()
    from oracle import arf_ref
    from unboundednerfpytorch_b200.arf import ARF
    RefARF = _reference_arf()
    name, power = _gpu()
    out = {'bench': 'arf_match_colors', 'gpu': name, 'power_limit': power, 'steps': args.steps, 'sets': {}}
    dev = torch.device('cuda', 0)
    with tempfile.TemporaryDirectory() as tmp:
        ok, buf = cv2.imencode('.png', arf_ref.style_source('landscape', 5)[..., ::-1].copy())
        assert ok
        buf.tofile(os.path.join(tmp, '34.jpg'))
        for W, H in SIZES:
            cfg = _Cfg(arf=_Cfg(style_root=tmp, style_id=34))
            data_dict = {'HW': np.array([[H, W]])}
            ours, ref = ARF(cfg, data_dict, dev), RefARF(cfg, data_dict, dev)
            for F in (int(f) for f in args.frames.split(',')):
                n_px = F * H * W
                g = torch.Generator(device=dev).manual_seed(F + W)
                x = torch.rand(F, H, W, 3, device=dev, generator=g)
                ms_mom, ms_aff = _device_times(x, args.steps, args.warmup)
                x_np = x.cpu().numpy()
                del x
                torch.cuda.empty_cache()
                _, ms_up, _ = _peak_and_time(lambda: torch.from_numpy(x_np).to(dev), args.reps)
                torch.cuda.empty_cache()
                ours.match_colors_for_image_set(x_np[:1], tmp)                                     # warm up
                res_o, ms_ours, peak_ours = _peak_and_time(lambda: ours.match_colors_for_image_set(x_np, tmp), args.reps)
                o = res_o[0]
                del res_o
                torch.cuda.empty_cache()
                ref.match_colors_for_image_set(x_np[:1], tmp)
                res_r, ms_ref, peak_ref = _peak_and_time(lambda: ref.match_colors_for_image_set(x_np, tmp), args.reps)
                diff = float((o - res_r[0]).abs().max())
                del res_r, o, x_np
                torch.cuda.empty_cache()
                set_bytes = n_px * 12
                out['sets'][f'{F}x{W}x{H}'] = {
                    'pixels': n_px, 'set_bytes': set_bytes,
                    'moments_ms': round(ms_mom, 4), 'affine_ms': round(ms_aff, 4),
                    'moments_GBps': round(12 * n_px / (ms_mom * 1e-3) / 1e9, 1),
                    'affine_GBps': round(24 * n_px / (ms_aff * 1e-3) / 1e9, 1),
                    'kernels_share_of_hbm_peak': round(36 * n_px / PEAK_BYTES / ((ms_mom + ms_aff) * 1e-3), 3),
                    'numpy_call_ms': round(ms_ours, 2), 'upload_ms': round(ms_up, 2),
                    'reference_call_ms': round(ms_ref, 2),
                    'peak_bytes_ours': int(peak_ours), 'peak_bytes_reference': int(peak_ref),
                    'peak_over_set_ours': round(peak_ours / set_bytes, 3),
                    'peak_over_set_reference': round(peak_ref / set_bytes, 3),
                    'max_abs_diff_vs_reference': diff,
                }
    print(json.dumps(out))


if __name__ == '__main__':
    main()
