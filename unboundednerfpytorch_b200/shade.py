"""rgbnet (feature -> RGB MLP) as one fused kernel per direction (csrc/shade.cu) behind an autograd.Function.

rgb = sigmoid(rgbnet(cat[k0, viewdirs_emb[ray_id]]))   (FourierGrid_model.py:631-637, dcvgo.py:337-342)

The view-direction half of the first Linear is constant along a ray, so the host folds it into a per-ray bias table
``vb = emb(viewdirs) @ W1[:, K:].T + b1`` ([N,W], one tiny GEMM that torch differentiates for dW1[:,K:], db1) and the
kernel runs the per-sample part: K -> W -> W -> 3 with the activations resident on chip, fp32 arithmetic.  W = 128 with K = 12
(every 12-channel config) has every engine below; K = 3 (rgbnet_dim = 3: the Waymo / Mega-NeRF FourierGrid configs), K = 15
(Tanks&Temples Train) and W = 64 with K = 9 (DirectMPIGO of llff_default; FourierGridModel and DirectVoxGO of the free-dataset
grass and lab configs) run the tensor-core forward and the fused backward with ReLU masks, at the precision UBN_RGBNET_MODE picks.
"""
import torch

import os

from . import _cabi, ops
from ._cabi import c_i64, c_int, check, ptr, stream_of

# engine: 'tc3' = tensor-core (mma.sync) 3xTF32 (fp32-grade, the default and the only mode the 1e-5 parity tests accept), 'tc1' = tensor cores with a
# single TF32 pass per product in the forward AND (with BWD_MODE 'fused') the backward -- the opt-in reduced-precision training
# mode, ~1e-3 relative error, gated by the PSNR test in tests/test_gpu_models.py --, 'simt' = fp32 FFMA
MODE = os.environ.get('UBN_RGBNET_MODE', 'tc3')
# backward engine: 'fused' = tensor-core 3xTF32, dZ2 -> dH1 -> dZ1 -> dX chained through registers + all sample reductions in one
# kernel of 8 warps, dW2 in a second launch; no intermediate in HBM; 'fused4' = the same with 4 warps per CTA (A/B); 'tc3' = the
# three-launch form (dZ1 round trip + CUDA-core kernel for the small gradients; kept for A/B); 'simt' = fp32 FFMA
BWD_MODE = os.environ.get('UBN_RGBNET_BWD_MODE', 'fused')
# ReLU masks instead of activation re-reads in the fused backward (default on): the forward leaves the masks of H1 (16 B per sample)
# so that launch 1 gates dH1 without loading the H1 rows; launch 1 ballots the masks of H2 so that the dW2 launch rebuilds dZ2 (and
# sums db2) without reading H2 a second time.  Off = both launches re-read the saves (A/B; tests cover both).
USE_MASKS = os.environ.get('UBN_RGBNET_MASKS', '1') == '1'


class _ShadeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, vb, ray_id, W1k, W2, b2, W3, b3, need_grad):
        feat, vb, ray_id = feat.contiguous(), vb.contiguous(), ray_id.contiguous()
        W1k, W2, b2, W3, b3 = (t.contiguous() for t in (W1k, W2, b2, W3, b3))
        M, K = feat.shape
        W = W2.shape[0]
        dev = feat.device
        rgb = torch.empty(M, 3, dtype=torch.float32, device=dev)
        # need_grad comes from the caller (shade()): inside Function.forward grad mode is always off, and needs_input_grad
        # mirrors requires_grad of the inputs even under torch.no_grad() -- render / eval forwards must not allocate and stream
        # the two [M,W] activation saves
        need_grad = bool(need_grad) and any(ctx.needs_input_grad)
        # panel-layout saves ([tile][W/4 column quads][128 rows][4], ceil(M/128)*128 rows): every 8-sample x 16-byte piece of a
        # tensor-core fragment is one contiguous 128-byte line; only the tensor-core forward writes it and only the fused backward reads it
        # K != 12: the tensor-core forward and the fused backward with masks only (the A/B engines are 12-column, 128-wide kernels)
        panel = need_grad and ((MODE in ('tc3', 'tc1', 'tc3w4') and BWD_MODE == 'fused') or K != 12)
        rows = -(-M // 128) * 128 if panel else M
        h1 = torch.empty(rows, W, dtype=torch.float32, device=dev) if need_grad else None
        h2 = torch.empty(rows, W, dtype=torch.float32, device=dev) if need_grad else None
        # ReLU masks of H1 (W/8 B per sample): the first backward launch gates dH1 with them instead of loading the H1 rows
        m1 = torch.empty(rows * W // 32, dtype=torch.int32, device=dev) if (panel and (USE_MASKS or K != 12)) else None
        with ops._Guard(feat) as lib:
            with _cabi.timed('rgbnet_fwd'):
                if K != 12:
                    check(lib.ubn_rgbnet_fwd_tc_kw(c_int(K), c_int(W), ptr(feat), ptr(vb), ptr(ray_id), ptr(W1k), ptr(W2), ptr(b2), ptr(W3),
                                                  ptr(b3), c_i64(M), ptr(rgb), ptr(h1), ptr(h2), ptr(m1),
                                                  c_int((1 if MODE == 'tc1' else 0) | (4 if panel else 0)), stream_of(feat)))
                elif MODE in ('tc3', 'tc1', 'tc3w4'):      # 'tc3w4': the 4-warp form of the forward kernel (A/B of the 8-warp default)
                    check(lib.ubn_rgbnet_fwd_tc(ptr(feat), ptr(vb), ptr(ray_id), ptr(W1k), ptr(W2), ptr(b2), ptr(W3), ptr(b3),
                                                c_i64(M), ptr(rgb), ptr(h1), ptr(h2), ptr(m1),
                                                c_int((1 if MODE == 'tc1' else 0) | (2 if MODE == 'tc3w4' else 0) | (4 if panel else 0)),
                                                stream_of(feat)))
                else:
                    check(lib.ubn_rgbnet_fwd(ptr(feat), ptr(vb), ptr(ray_id), ptr(W1k), ptr(W2), ptr(b2), ptr(W3), ptr(b3),
                                             c_i64(M), ptr(rgb), ptr(h1), ptr(h2), stream_of(feat)))
        if need_grad:
            ctx.save_for_backward(feat, ray_id, W1k, W2, W3, rgb, h1, h2)
            ctx.m1 = m1
            ctx.n_rays = vb.shape[0]
            ctx.panel = panel
            ctx.bwd_mode = BWD_MODE if K == 12 else 'fused'
        return rgb

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_rgb):
        feat, ray_id, W1k, W2, W3, rgb, h1, h2 = ctx.saved_tensors
        dev = feat.device
        M, K = feat.shape
        W = W2.shape[0]
        g_rgb = g_rgb.contiguous()
        g_feat = torch.empty_like(feat)
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        g_vb, gW1k, gW2, gb2, gW3, gb3 = z(ctx.n_rays, W), z(W, K), z(W, W), z(W), z(3, W), z(3)
        with ops._Guard(feat) as lib:
            bwd_mode = ctx.bwd_mode                      # as chosen in forward (the save layout depends on it)
            if K != 12:
                masks = torch.empty(-(-M // 128) * 128 * W // 32, dtype=torch.int32, device=dev)
                with _cabi.timed('rgbnet_bwd'):
                    check(lib.ubn_rgbnet_bwd_tc_fused_kw(c_int(K), c_int(W), ptr(feat), ptr(ray_id), ptr(W1k), ptr(W2), ptr(W3), ptr(rgb), ptr(h1),
                                                        ptr(h2), ptr(g_rgb), c_i64(M), ptr(g_feat), ptr(g_vb), ptr(gW1k), ptr(gW2),
                                                        ptr(gb2), ptr(gW3), ptr(gb3), ptr(masks), ptr(ctx.m1),
                                                        c_int((1 if MODE == 'tc1' else 0) | 4), stream_of(feat)))
                return g_feat, g_vb, None, gW1k, gW2, gb2, gW3, gb3, None
            if bwd_mode in ('fused', 'fused4'):          # 'fused4': the same kernels with 4 warps per CTA (A/B)
                # panel saves: launch 1 leaves the ReLU masks of H2 (2 KB per 128-sample tile) in this scratch and the dW2 launch
                # rebuilds dZ2 from them instead of reading the 512 B/sample of H2 again
                masks = torch.empty(-(-M // 128) * 512, dtype=torch.int32, device=dev) if (ctx.panel and ctx.m1 is not None) else None
                with _cabi.timed('rgbnet_bwd'):
                    check(lib.ubn_rgbnet_bwd_tc_fused(ptr(feat), ptr(ray_id), ptr(W1k), ptr(W2), ptr(W3), ptr(rgb), ptr(h1), ptr(h2),
                                                      ptr(g_rgb), c_i64(M), ptr(g_feat), ptr(g_vb), ptr(gW1k), ptr(gW2), ptr(gb2),
                                                      ptr(gW3), ptr(gb3), ptr(masks), ptr(ctx.m1 if bwd_mode == 'fused' else None), c_int((1 if MODE == 'tc1' else 0) | (2 if bwd_mode == 'fused4' else 0) | (4 if ctx.panel else 0)),
                                                      stream_of(feat)))
                return g_feat, g_vb, None, gW1k, gW2, gb2, gW3, gb3, None
            if bwd_mode == 'tc3':
                dz1 = torch.empty(M, 128, dtype=torch.float32, device=dev)
                with _cabi.timed('rgbnet_bwd'):
                    check(lib.ubn_rgbnet_bwd_tc_data(ptr(W2), ptr(W3), ptr(rgb), ptr(h1), ptr(h2), ptr(g_rgb), c_i64(M),
                                                     ptr(dz1), ptr(gW2), stream_of(feat)))
                with _cabi.timed('rgbnet_bwd_small'):
                    check(lib.ubn_rgbnet_bwd_small(ptr(feat), ptr(ray_id), ptr(W1k), ptr(W3), ptr(rgb), ptr(h2), ptr(g_rgb),
                                                   ptr(dz1), c_i64(M), ptr(g_feat), ptr(g_vb), ptr(gW1k), ptr(gb2), ptr(gW3),
                                                   ptr(gb3), stream_of(feat)))
                return g_feat, g_vb, None, gW1k, gW2, gb2, gW3, gb3, None
            with _cabi.timed('rgbnet_bwd'):
                check(lib.ubn_rgbnet_bwd(ptr(feat), ptr(ray_id), ptr(W1k), ptr(W2), ptr(W3), ptr(rgb), ptr(h1), ptr(h2),
                                         ptr(g_rgb), c_i64(M), ptr(g_feat), ptr(g_vb), ptr(gW1k), ptr(gW2), ptr(gb2),
                                         ptr(gW3), ptr(gb3), stream_of(feat)))
        return g_feat, g_vb, None, gW1k, gW2, gb2, gW3, gb3, None


# (features, hidden width) pairs with kernels: rgbnet_dim 3 / 12 / 15 at width 128, and (9, 64): llff_default, free-dataset grass / lab
KERNEL_SHAPES = {(3, 128), (12, 128), (15, 128), (9, 64)}


def supported(rgbnet, k0_dim):
    """3-layer rgbnet (rgbnet_depth=3) of width 128 on 3, 12 or 15 features, or of width 64 on 9 features (rgbnet_dim)."""
    try:
        l1, l2, l3 = rgbnet[0], rgbnet[2][0], rgbnet[3]
    except Exception:
        return False
    W = l1.weight.shape[0]
    return (len(rgbnet) == 4 and (k0_dim, W) in KERNEL_SHAPES and tuple(l2.weight.shape) == (W, W)
            and tuple(l3.weight.shape) == (3, W) and l1.weight.is_cuda and l1.weight.dtype == torch.float32)


def shade(rgbnet, k0, view_emb, ray_id):
    """k0 [M,K], view_emb [N,E] (cat[v, sin, cos]), ray_id [M] sorted -> rgb [M,3]; (K, width) as in supported()."""
    l1, l2, l3 = rgbnet[0], rgbnet[2][0], rgbnet[3]
    kd = k0.shape[1]
    vb = torch.addmm(l1.bias, view_emb, l1.weight[:, kd:].t())
    return _ShadeFn.apply(k0, vb, ray_id, l1.weight[:, :kd], l2.weight, l2.bias, l3.weight, l3.bias, torch.is_grad_enabled())
