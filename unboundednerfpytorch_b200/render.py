"""Frame rendering with the reference's driver surface (FourierGrid/run_render.py:15-114) plus the two multi-GPU render modes of
SURVEY.md 8e:

* ``render_viewpoints``         -- same signature / returns as run_render.render_viewpoints: per pose, rays of the view on the
                                   device (one launch), 8192-ray chunks through ``model(...)`` (run_render.py:56-63), numpy
                                   (rgbs, depths, bgmaps).  With torch.distributed initialised every rank renders a contiguous
                                   shard of each frame's rays and the frame is assembled with one all-gather (BASELINE config 4).
* ``render_rays``               -- flat ray arrays: one fused launch for the contracted models models.render_fused
                                   covers (and, with ``fused_frame=True``, for DirectVoxGO / DirectMPIGO where theirs
                                   does), otherwise the chunk loop.
* ``render_frame_sharded``      -- one frame: contiguous ray shard per rank + ``dist.gather_frame``.
* ``render_blocks_idw``         -- Block-NeRF style (eval_block_nerf.py:95-133, :215-216): one spatial block per rank, every rank
                                   renders the same frame, blocks that do not see the view are gated out, the frame is the
                                   inverse-distance-weighted mean of the visible blocks' images (one all-reduce).
``eval_ssim`` scores each frame on the device (metrics.rgb_ssim); LPIPS raises (it needs pretrained network weights)."""
import os

import numpy as np
import torch

from . import dist as D
from . import metrics as M
from . import rays as R

KEYS = ('rgb_marched', 'depth', 'alphainv_last')


@torch.no_grad()
def render_rays(model, rays_o, rays_d, viewdirs, render_kwargs, chunk=8192, keys=KEYS, fused_frame=False):
    """[n,3] ray arrays -> {key: [n, K]} (K = 3 for rgb_marched, 1 otherwise), in ``chunk``-ray calls like run_render.py:56-63.

    fused_frame: also take the fused whole-frame render of the models whose fused render is opt-in (DirectVoxGO, DirectMPIGO:
    ``FUSED_FRAME_BY_DEFAULT = False``) where their render_fused_ok holds.  Off by default: their chunk loop's frames are what
    forward computes bit for bit, the fused frames agree with it to about 1e-6 (forward's view bias is a cuBLAS addmm).

    render_kwargs keys read here besides the model's own: ``coherent_rays`` (TMA-staged feature reads of image-ordered chunks) and
    ``fused_slabs`` (FourierGridModel with 7, 9 or 11 Fourier slabs in one fused launch, models._ContractedBase.render_fused_ok);
    both off by default and passed on to every call, so render_frame_sharded, render_blocks_idw and render_viewpoints take them
    too."""
    rk = dict(render_kwargs)
    rk.setdefault('render_depth', True)
    # render_kwargs['coherent_rays']=True routes DenseGrid feature reads of image-ordered chunks through the TMA-staged brick
    # kernel (csrc/render_tma.cu).  Opt-in: the lane-per-sample gather stays the default (the TMA kernel was slower on a full
    # garden frame when it was last compared; not re-measured on the H100).
    rk.setdefault('coherent_rays', False)
    # render_kwargs['fused_slabs']=True extends the fused render to FourierGridModel with Fourier slabs (7, 9 or 11 slabs, the
    # (12, 4) rgbnet: csrc/render_fourier.cu).  Opt-in like fused_frame: its frames agree with the chunk loop to about 1e-6, and
    # on dense scenes it is not always the faster path (DESIGN.md §7).
    # contracted models the fused render covers (models._ContractedBase.render_fused_ok) take the whole ray array in one launch
    # (memory O(n), no per-sample buffers), and so do DirectVoxGO / DirectMPIGO with fused_frame=True; every other model or
    # configuration keeps the chunk loop
    opted_in = fused_frame or getattr(model, 'FUSED_FRAME_BY_DEFAULT', True)
    if hasattr(model, 'render_fused_ok') and opted_in and model.render_fused_ok(rays_o, rk):
        ret = model.render_fused(rays_o, rays_d, viewdirs, **rk)
        return {k: ret[k].reshape(rays_o.shape[0], -1) for k in keys}
    outs = {k: [] for k in keys}
    for ro, rd, vd in zip(rays_o.split(chunk, 0), rays_d.split(chunk, 0), viewdirs.split(chunk, 0)):
        ret = model(ro, rd, vd, **rk)
        for k in keys:
            outs[k].append(ret[k].reshape(ro.shape[0], -1))
    return {k: torch.cat(v) if v else torch.empty(0, 1, device=rays_o.device) for k, v in outs.items()}


@torch.no_grad()
def render_frame_sharded(model, rays_o, rays_d, viewdirs, render_kwargs, chunk=8192, keys=KEYS, fused_frame=False):
    """All ranks hold the same [n,3] rays; rank r renders the contiguous shard dist.shard_range(n, r, world) (contiguous keeps
    the image-space coherence of a chunk) and every rank receives the assembled {key: [n, K]}.  fused_frame: as render_rays."""
    world = torch.distributed.get_world_size() if (torch.distributed.is_available() and torch.distributed.is_initialized()) else 1
    rank = torch.distributed.get_rank() if world > 1 else 0
    n = rays_o.shape[0]
    lo, hi = D.shard_range(n, rank, world)
    local = render_rays(model, rays_o[lo:hi], rays_d[lo:hi], viewdirs[lo:hi], render_kwargs, chunk, keys, fused_frame)
    if world == 1:
        return local
    packed = torch.cat([local[k] for k in keys], -1)                       # one collective for all keys
    full = D.gather_frame(packed, n, rank, world)
    out, c = {}, 0
    for k in keys:
        w = local[k].shape[1]
        out[k] = full[:, c:c + w]
        c += w
    return out


@torch.no_grad()
def render_blocks_idw(model, rays_o, rays_d, viewdirs, render_kwargs, centroid, cam_origin=None, power=4, vis_thres=0.05,
                      chunk=8192, fused_frame=False):
    """One block model per rank, same frame on every rank -> IDW composite of the visible blocks on every rank.

    eval_block_nerf.py:215-216 keeps a block only when the mean transmittance its visibility network predicts for the view exceeds
    0.05; the grid models have no visibility network, so the gate uses what they do produce: the mean accumulated opacity of
    the block's own render (1 - alphainv_last).mean() > vis_thres -- a block that renders (almost) nothing for this view is
    dropped.  Weight of a kept block: ||cam_origin - centroid||^-power (DistanceWeight, :95-98), normalised over the kept
    blocks (:123-127).  Composited in fp32 (the reference composites uint8 images on the CPU).
    fused_frame: as render_rays.
    Returns (rgb [n,3], {'weight': this block's weight, 'visible': bool, 'den': sum of weights})."""
    out = render_rays(model, rays_o, rays_d, viewdirs, render_kwargs, chunk, ('rgb_marched', 'alphainv_last'), fused_frame)
    rgb = out['rgb_marched']
    origin = cam_origin if cam_origin is not None else rays_o[0]
    origin = torch.as_tensor(origin, dtype=torch.float32, device=rgb.device)
    cen = torch.as_tensor(centroid, dtype=torch.float32, device=rgb.device)
    visible = (1.0 - out['alphainv_last']).mean() > vis_thres                # device bool: no host sync before the collective
    w = (origin - cen).norm().clamp_min(1e-8).pow(-power) * visible.float()
    num = torch.cat([rgb * w, w.reshape(1, 1).expand(1, 3)], 0)              # [n + 1, 3]: numerator rows + the denominator
    if torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
        torch.distributed.all_reduce(num)
    den = num[-1, 0]
    return num[:-1] / den.clamp_min(1e-30), {'weight': w, 'visible': visible, 'den': den}


def render_viewpoints(cfg, model, render_poses, HW, Ks, ndc, render_kwargs, gt_imgs=None, savedir=None, dump_images=False,
                      render_factor=0, render_video_flipy=False, render_video_rot90=0, eval_ssim=False, eval_lpips_alex=False,
                      eval_lpips_vgg=False, verbose=True, chunk=8192, fused_frame=False):
    """run_render.py:15-114.  ``cfg`` only supplies cfg.data.flip_x / flip_y (None -> False).  Returns (rgbs, depths, bgmaps) as
    numpy arrays [n_views, H, W, K] like the reference; prints the average PSNR when ``gt_imgs`` is given.

    ``eval_ssim`` scores each frame against its ``gt_imgs`` entry with metrics.rgb_ssim(max_val=1) while the frame is still on
    the device, and prints ``Ssim <mean> (avg)`` after the Psnr line.  The reference scores only where it computes PSNR -- with
    ``gt_imgs`` and ``render_factor == 0`` -- and silently skips SSIM elsewhere; here ``eval_ssim`` outside that case raises
    NotImplementedError, so a requested score is never dropped without notice.  LPIPS raises: it needs pretrained networks.
    fused_frame: as render_rays (DirectVoxGO / DirectMPIGO frames in one fused launch where it applies)."""
    if eval_lpips_alex or eval_lpips_vgg:
        raise NotImplementedError('LPIPS evaluation needs pretrained network weights, which this package does not ship')
    if eval_ssim and (gt_imgs is None or render_factor != 0):
        raise NotImplementedError('eval_ssim scores rendered frames against gt_imgs at render_factor 0 only (as run_render.py '
                                  'does); here there is nothing to score')
    assert len(render_poses) == len(HW) and len(HW) == len(Ks)
    HW, Ks = np.asarray(HW), np.asarray(Ks, dtype=np.float64)
    if render_factor != 0:
        HW = (np.copy(HW) / render_factor).astype(int)
        Ks = np.copy(Ks)
        Ks[:, :2, :3] /= render_factor
    data = getattr(cfg, 'data', None)
    flip_x, flip_y = bool(getattr(data, 'flip_x', False)), bool(getattr(data, 'flip_y', False))
    dev = next(model.parameters()).device
    rgbs, depths, bgmaps, psnrs, ssims = [], [], [], [], []
    rk = {k: v for k, v in render_kwargs.items() if k != 'indexs'}
    for i, c2w in enumerate(render_poses):
        H, W = int(HW[i][0]), int(HW[i][1])
        c2w = torch.as_tensor(np.asarray(c2w), dtype=torch.float32)
        ro, rd, vd = R._rays_of_a_view(H, W, Ks[i], c2w, ndc, rk.get('inverse_y', False), flip_x, flip_y, 'center', device=dev)
        res = render_frame_sharded(model, ro.view(-1, 3), rd.view(-1, 3), vd.view(-1, 3), rk, chunk, fused_frame=fused_frame)
        frame = res['rgb_marched'].reshape(H, W, -1)
        if eval_ssim:
            ssims.append(M.rgb_ssim(frame, torch.as_tensor(gt_imgs[i], device=dev), max_val=1))
        rgb = frame.cpu().numpy()
        rgbs.append(rgb)
        depths.append(res['depth'].reshape(H, W, -1).cpu().numpy())
        bgmaps.append(res['alphainv_last'].reshape(H, W, -1).cpu().numpy())
        if gt_imgs is not None and render_factor == 0:
            psnrs.append(-10. * np.log10(np.mean(np.square(rgb - gt_imgs[i]))))
    if len(psnrs) and verbose:
        print('Psnr', np.mean(psnrs), '(avg)')
        if eval_ssim:
            print('Ssim', np.mean(torch.stack(ssims).cpu().numpy()), '(avg)')
    if render_video_flipy:
        rgbs, depths, bgmaps = ([np.flip(x, axis=0) for x in xs] for xs in (rgbs, depths, bgmaps))
    if render_video_rot90 != 0:
        rgbs, depths, bgmaps = ([np.rot90(x, k=render_video_rot90, axes=(0, 1)) for x in xs] for xs in (rgbs, depths, bgmaps))
    if savedir is not None and dump_images:
        import cv2
        os.makedirs(savedir, exist_ok=True)
        for i, rgb in enumerate(rgbs):
            rgb8 = (255 * np.clip(rgb, 0, 1)).astype(np.uint8)
            cv2.imwrite(os.path.join(savedir, '{:03d}.png'.format(i)), rgb8[..., ::-1])
    return np.array(rgbs), np.array(depths), np.array(bgmaps)
