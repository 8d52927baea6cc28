"""ctypes binding of libubnerf_b200.so (C ABI declared in include/ubnerf_b200.h).

PyTorch is used here only as the owner of device memory and streams: every call passes raw device
pointers, sizes and the current CUDA stream handle across the C boundary.  There is NO fallback: if the
shared library has not been built, importing any op of this package raises.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libubnerf_b200.so')

c_i64 = ctypes.c_int64
c_i32 = ctypes.c_int32
c_int = ctypes.c_int
c_f = ctypes.c_float
c_p = ctypes.c_void_p


class UbnGridDesc(ctypes.Structure):
    _fields_ = [('P', c_i32), ('C', c_i32), ('X', c_i32), ('Y', c_i32), ('Z', c_i32), ('num_freqs', c_i32),
                ('stride_p', c_i64), ('stride_c', c_i64), ('stride_v', c_i64),
                ('xyz_min', c_f * 3), ('xyz_max', c_f * 3)]


class UbnTensorfDesc(ctypes.Structure):
    _fields_ = [('X', c_i32), ('Y', c_i32), ('Z', c_i32), ('R', c_i32), ('Rxy', c_i32), ('C', c_i32),
                ('stride_r', c_i64 * 6), ('stride_a', c_i64 * 6), ('stride_b', c_i64 * 6),
                ('xyz_min', c_f * 3), ('xyz_max', c_f * 3)]


TENSORF_BWD_MAX_CTAS = 528   # UBN_TENSORF_BWD_MAX_CTAS of include/ubnerf_b200.h
SSIM_MAX_TAPS = 32           # UBN_SSIM_MAX_TAPS
SSIM_MAX_CTAS = 1056         # UBN_SSIM_MAX_CTAS
COLOR_MAX_CTAS = 1056        # UBN_COLOR_MAX_CTAS


class UbnMarchCfg(ctypes.Structure):
    _fields_ = [('scene_center', c_f * 3), ('scene_radius', c_f * 3),
                ('contract_B', c_f), ('contract_A', c_f),
                ('contracted_norm', c_i32), ('n_samples', c_i32),
                ('act_shift', c_f), ('interval', c_f), ('fast_color_thres', c_f),
                ('use_cumdist', c_i32), ('cumdist_thres', c_f),
                ('use_maskcache', c_i32), ('mask_sz', c_i32 * 3), ('mask_scale', c_f * 3), ('mask_shift', c_f * 3)]


class UbnNdcMarchCfg(ctypes.Structure):
    _fields_ = [('xyz_min', c_f * 3), ('xyz_max', c_f * 3), ('n_samples', c_i32), ('interval', c_f), ('fast_color_thres', c_f),
                ('use_maskcache', c_i32), ('mask_sz', c_i32 * 3), ('mask_scale', c_f * 3), ('mask_shift', c_f * 3)]


class UbnBoxMarchCfg(ctypes.Structure):
    _fields_ = [('xyz_min', c_f * 3), ('xyz_max', c_f * 3), ('near', c_f), ('stepdist', c_f), ('s_max', c_i32), ('act_shift', c_f),
                ('interval', c_f), ('fast_color_thres', c_f), ('use_maskcache', c_i32), ('mask_sz', c_i32 * 3),
                ('mask_scale', c_f * 3), ('mask_shift', c_f * 3)]


ABI_VERSION = 3          # UBN_ABI_VERSION of include/ubnerf_b200.h this binding was written against
FLAG_QUERIED, FLAG_LISTED, FLAG_SCANNED, FLAG_KEEP, FLAG_INNER = 1, 2, 4, 8, 16

# name -> argtypes (all functions return int unless listed in _RESTYPE)
_SIGNATURES = {
    'ubn_abi_version': [],
    'ubn_last_error_string': [],
    'ubn_launch_count': [],
    'ubn_reset_launch_count': [],
    'ubn_infer_t_minmax': [c_p, c_p, c_p, c_p, c_f, c_f, c_i64, c_p, c_p, c_p],
    'ubn_infer_n_samples': [c_p, c_p, c_p, c_f, c_i64, c_p, c_p],
    'ubn_infer_ray_start_dir': [c_p, c_p, c_p, c_i64, c_p, c_p, c_p],
    'ubn_sample_pts_count': [c_p, c_p, c_p, c_p, c_f, c_f, c_f, c_i64, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_sample_pts_emit': [c_p, c_p, c_p, c_p, c_p, c_p, c_f, c_i64, c_i64, c_p, c_p, c_p, c_p, c_p],
    'ubn_sample_ndc_pts_on_rays': [c_p, c_p, c_p, c_p, c_i64, c_i64, c_p, c_p, c_p],
    'ubn_sample_bg_pts_on_rays': [c_p, c_p, c_p, c_f, c_i64, c_i64, c_p, c_p],
    'ubn_maskcache_lookup': [c_p, c_p, c_p, c_p, c_i64, c_i64, c_i64, c_i64, c_p, c_p],
    'ubn_raw2alpha': [c_p, c_f, c_f, c_p, c_i64, c_p, c_p, c_p],
    'ubn_raw2alpha_backward': [c_p, c_p, c_f, c_p, c_i64, c_p, c_p],
    'ubn_alpha2weight': [c_p, c_p, c_i64, c_i64, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_alpha2weight_backward': [c_p, c_p, c_p, c_p, c_p, c_p, c_i64, c_i64, c_p, c_p, c_p, c_p],
    'ubn_segment_sum': [c_p, c_i64, c_p, c_i64, c_i64, c_p, c_p, c_p, c_p],
    'ubn_rgbnet_fwd': [c_p] * 8 + [c_i64] + [c_p] * 4,
    'ubn_rgbnet_fwd_tc': [c_p] * 8 + [c_i64] + [c_p] * 4 + [c_int, c_p],
    'ubn_rgbnet_bwd_tc_data': [c_p] * 6 + [c_i64] + [c_p] * 3,
    'ubn_rgbnet_bwd_small': [c_p] * 8 + [c_i64] + [c_p] * 7,
    'ubn_rgbnet_bwd': [c_p] * 9 + [c_i64] + [c_p] * 8,
    'ubn_rgbnet_bwd_tc_fused': [c_p] * 9 + [c_i64] + [c_p] * 9 + [c_int, c_p],
    'ubn_rgbnet_fwd_tc_k': [c_int] + [c_p] * 8 + [c_i64] + [c_p] * 4 + [c_int, c_p],
    'ubn_rgbnet_bwd_tc_fused_k': [c_int] + [c_p] * 9 + [c_i64] + [c_p] * 9 + [c_int, c_p],
    'ubn_rgbnet_fwd_tc_kw': [c_int, c_int] + [c_p] * 8 + [c_i64] + [c_p] * 4 + [c_int, c_p],
    'ubn_rgbnet_bwd_tc_fused_kw': [c_int, c_int] + [c_p] * 9 + [c_i64] + [c_p] * 9 + [c_int, c_p],
    'ubn_set_dw2_engine': [c_int],
    'ubn_set_fwd_engine': [c_int],
    'ubn_get_fwd_engine': [],
    'ubn_total_variation_add_grad': [c_p, c_p, c_f, c_f, c_f, c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_p],
    'ubn_adam_upd': [c_p, c_p, c_p, c_p, c_p, c_i64, c_int, c_f, c_f, c_f, c_f, c_int, c_p],
    'ubn_tv_adam_fused': [c_p, c_p, c_p, c_p, c_f, c_f, c_f, c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_int,
                          c_f, c_f, c_f, c_f, c_int, c_int, c_p],
    'ubn_tv_adam_pingpong': [c_p, c_p, c_p, c_p, c_p, c_f, c_f, c_f, c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_int,
                             c_f, c_f, c_f, c_f, c_int, c_int, c_p],
    'ubn_tv_adam_peer': [c_p, c_p, c_p, c_int, c_p, c_p, c_f, c_f, c_f, c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_i64, c_i64,
                         c_int, c_f, c_f, c_f, c_f, c_int, c_p],
    'ubn_lattice_alpha': [c_p, ctypes.POINTER(UbnGridDesc), c_p, c_p, c_i64, c_i64, c_i64, c_f, c_f, c_p, c_p],
    'ubn_maxpool3_gt_and': [c_p, c_i64, c_i64, c_i64, c_f, c_p, c_p],
    'ubn_resample_grid': [c_p, ctypes.POINTER(UbnGridDesc), c_p, ctypes.POINTER(UbnGridDesc), c_p],
    'ubn_view_scatter_ones': [c_p, c_p, c_i64, c_i64, c_f, c_f, c_f, ctypes.POINTER(UbnGridDesc), c_p, c_p],
    'ubn_view_scatter_ones_contracted': [c_p, c_p, c_i64, c_p, ctypes.POINTER(UbnMarchCfg), ctypes.POINTER(UbnGridDesc), c_p,
                                         c_p],
    'ubn_count_gt': [c_p, c_f, c_i64, c_p, c_p],
    'ubn_maskout_near_cam': [c_p, c_i64, c_i64, c_i64, c_i64, c_p, c_i64, c_f, c_f, c_p],
    'ubn_maskout_near_cam_lattice': [c_p, c_i64, c_i64, c_i64, c_i64, c_p, c_p, c_p, c_i64, c_f, c_f, c_p],
    'ubn_cumdist_thres': [c_p, c_f, c_i64, c_i64, c_p, c_p],
    'ubn_get_rays_of_a_view': [c_int, c_int, c_p, c_p, c_int, c_int, c_int, c_int, c_int, c_int, c_p, c_p, c_p, c_p, c_p],
    'ubn_gather_rays': [c_p, c_p, c_int, c_p, c_i64, c_i64, c_p, c_p],
    'ubn_composite_fwd': [c_p, c_p, c_p, c_i64, c_i64, c_p, c_p, c_p, c_p],
    'ubn_composite_bwd': [c_p, c_p, c_p, c_p, c_i64, c_p, c_p, c_p],
    'ubn_distortion_loss': [c_p, c_p, c_p, c_i64, c_i64, c_f, c_p, c_p, c_p, c_p, c_p, c_i64, c_p],
    'ubn_render_loss': [c_p] * 7 + [c_i64, c_i64] + [c_f] * 6 + [c_p] * 6 + [c_i64, c_p],
    'ubn_grid_sample_fwd': [c_p, ctypes.POINTER(UbnGridDesc), c_p, c_i64, c_p, c_p],
    'ubn_grid_sample_bwd': [c_p, ctypes.POINTER(UbnGridDesc), c_p, c_i64, c_p, c_p],
    'ubn_march_density_fwd': [c_p, c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), c_p, ctypes.POINTER(UbnMarchCfg), c_i64,
                              c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_exclusive_scan_i32': [c_p, c_i64, c_p, c_p, c_p],
    'ubn_march_feature_fwd': [c_p, c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), ctypes.POINTER(UbnMarchCfg), c_i64,
                              c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_march_feature_fwd_tma': [c_p, c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), ctypes.POINTER(UbnMarchCfg), c_i64,
                                  c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_render_contracted': [c_p, c_p, c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), c_p, ctypes.POINTER(UbnGridDesc), c_p,
                              ctypes.POINTER(UbnMarchCfg), c_i64] + [c_p] * 6 + [c_int, c_int, c_int, c_f] + [c_p] * 6,
    'ubn_render_fourier': [c_p, c_p, c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), c_p, ctypes.POINTER(UbnGridDesc), c_p,
                           ctypes.POINTER(UbnMarchCfg), c_i64] + [c_p] * 6 + [c_int, c_int, c_int, c_f] + [c_p] * 6,
    'ubn_set_feature_kernel': [c_int],
    'ubn_get_feature_kernel': [],
    'ubn_set_density_scatter': [c_int],
    'ubn_get_density_scatter': [],
    'ubn_march_feature_bwd': [c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), ctypes.POINTER(UbnMarchCfg), c_i64,
                              c_p, c_p, c_p, c_p, c_p],
    'ubn_march_density_bwd': [c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), ctypes.POINTER(UbnMarchCfg), c_i64,
                              c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_march_ndc_density_fwd': [c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), c_p, ctypes.POINTER(UbnGridDesc), c_p,
                                  ctypes.POINTER(UbnNdcMarchCfg), c_i64, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_march_ndc_feature_fwd': [c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), ctypes.POINTER(UbnNdcMarchCfg), c_i64,
                                  c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_march_ndc_feature_bwd': [c_p, c_p, ctypes.POINTER(UbnGridDesc), ctypes.POINTER(UbnNdcMarchCfg), c_i64,
                                  c_p, c_p, c_p, c_p, c_p],
    'ubn_march_ndc_density_bwd': [c_p, c_p, ctypes.POINTER(UbnGridDesc), ctypes.POINTER(UbnNdcMarchCfg), c_i64,
                                  c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_march_box_density_fwd': [c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), c_p, ctypes.POINTER(UbnBoxMarchCfg), c_i64,
                                  c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_march_box_feature_fwd': [c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), ctypes.POINTER(UbnBoxMarchCfg), c_i64,
                                  c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_march_box_feature_bwd': [c_p, c_p, ctypes.POINTER(UbnGridDesc), ctypes.POINTER(UbnBoxMarchCfg), c_i64,
                                  c_p, c_p, c_p, c_p, c_p],
    'ubn_render_ndc': [c_p, c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), c_p, ctypes.POINTER(UbnGridDesc), c_p,
                       ctypes.POINTER(UbnGridDesc), c_p, ctypes.POINTER(UbnNdcMarchCfg), c_i64] + [c_p] * 6 + [c_int, c_int, c_f]
                      + [c_p] * 6,
    'ubn_render_box': [c_p, c_p, c_p, c_p, ctypes.POINTER(UbnGridDesc), c_p, ctypes.POINTER(UbnGridDesc), c_p,
                       ctypes.POINTER(UbnBoxMarchCfg), c_i64] + [c_p] * 6 + [c_int, c_int, c_f] + [c_p] * 7,
    'ubn_march_box_density_bwd': [c_p, c_p, ctypes.POINTER(UbnGridDesc), ctypes.POINTER(UbnBoxMarchCfg), c_i64,
                                  c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_tensorf_fwd': [c_p, c_p, ctypes.POINTER(UbnTensorfDesc), c_p, c_i64, c_p, c_p],
    'ubn_tensorf_bwd': [c_p, c_p, ctypes.POINTER(UbnTensorfDesc), c_p, c_i64, c_p, c_p, c_p, c_int, c_p, c_p],
    'ubn_tensorf_tv_add_grad': [c_p, c_p, ctypes.POINTER(UbnTensorfDesc), c_f, c_f, c_f, c_p],
    'ubn_tensorf_dense': [c_p, c_p, ctypes.POINTER(UbnTensorfDesc), c_p, c_p],
    'ubn_march_box_tensorf_density_fwd': [c_p, c_p, c_p, ctypes.POINTER(UbnTensorfDesc), c_p, ctypes.POINTER(UbnBoxMarchCfg), c_i64,
                                          c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_march_box_tensorf_density_bwd': [c_p, c_p, c_p, ctypes.POINTER(UbnTensorfDesc), ctypes.POINTER(UbnBoxMarchCfg), c_i64,
                                          c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_int, c_p, c_p, c_p],
    'ubn_march_box_points_fwd': [c_p, c_p, ctypes.POINTER(UbnBoxMarchCfg), c_i64, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    'ubn_frustum_bounds': [c_p, c_p, c_p, c_i64, c_i64, c_int, c_int, c_int, c_int, c_int, c_f, c_f, c_p, c_p],
    'ubn_lattice_points': [c_p, c_p, c_i64, c_i64, c_i64, c_p, c_p],
    'ubn_lattice_bounds': [c_p, ctypes.POINTER(UbnGridDesc), c_p, c_p, c_i64, c_i64, c_i64, c_f, c_f, c_f, c_p, c_p, c_p],
    'ubn_lattice_bounds_alpha': [c_p, c_p, c_p, c_i64, c_i64, c_i64, c_f, c_p, c_p, c_p],
    'ubn_rgb_ssim': [c_p, c_p, c_i64, c_i64, c_int, ctypes.POINTER(ctypes.c_double), ctypes.c_double, ctypes.c_double,
                     c_p, c_p, c_p, c_p],
    'ubn_color_moments': [c_p, c_i64, c_p, c_p, c_p],
    'ubn_color_affine': [c_p, c_p, c_i64, ctypes.POINTER(c_f), ctypes.POINTER(c_f), c_p],
}
_RESTYPE = {'ubn_last_error_string': ctypes.c_char_p, 'ubn_launch_count': c_i64, 'ubn_reset_launch_count': None}

_lib = None


def exported_symbols():
    """Names every entry point include/ubnerf_b200.h declares (used by the CPU symbol test)."""
    return sorted(_SIGNATURES)


def load():
    """dlopen the in-tree shared library; fail loudly (no CPU / eager fallback exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f'{LIB_PATH} is missing: the CUDA library has not been built. Run '
            '`python -m unboundednerfpytorch_b200.build` (or __graft_entry__.build()). '
            'This package has no CPU or eager-PyTorch fallback by design.')
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = _RESTYPE.get(name, c_int)
    if lib.ubn_abi_version() != ABI_VERSION:
        raise RuntimeError('libubnerf_b200.so ABI version mismatch')
    _lib = lib
    return lib


def check(err):
    if err:
        msg = load().ubn_last_error_string()
        raise RuntimeError(f'libubnerf_b200: CUDA error {err}: {msg.decode() if msg else "?"}')


def ptr(t):
    return c_p(t.data_ptr()) if t is not None else c_p(0)


def stream_of(t):
    return c_p(torch.cuda.current_stream(t.device).cuda_stream)


def launch_count():
    return int(load().ubn_launch_count())


def reset_launch_count():
    load().ubn_reset_launch_count()


# ---- optional per-kernel CUDA-event timing (bench.py's roofline line) -------------------------------------
class KernelTimer:
    """Records CUDA events on the launching stream around selected C-ABI calls; near-zero overhead, no sync until
    ``summary()``."""

    def __init__(self):
        self.records = {}

    class _Range:
        def __init__(self, timer, name):
            self.timer, self.name = timer, name

        def __enter__(self):
            self.s = torch.cuda.Event(enable_timing=True)
            self.e = torch.cuda.Event(enable_timing=True)
            self.s.record()
            return self

        def __exit__(self, *a):
            self.e.record()
            self.timer.records.setdefault(self.name, []).append((self.s, self.e))
            return False

    def range(self, name):
        return KernelTimer._Range(self, name)

    def summary(self):
        torch.cuda.synchronize()
        return {k: (sum(s.elapsed_time(e) for s, e in v) / len(v), len(v)) for k, v in self.records.items()}


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


TIMER = None


def timed(name):
    return TIMER.range(name) if TIMER is not None else _Null()
