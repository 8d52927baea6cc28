/*
 * ubnerf_b200.h -- C ABI of libubnerf_b200.so: the H100-native (sm_90a) replacement for the native
 * layer of sjtuytc/UnboundedNeRFPytorch's FourierGrid / DVGO rendering hot path.
 *
 * Boundary contract
 *   - Plain C: raw DEVICE pointers + sizes + scalars; no torch / ATen types anywhere.
 *   - Every entry point enqueues its kernels on `stream` (a cudaStream_t passed as void*; NULL = the
 *     legacy default stream) of the CURRENT device and returns immediately (asynchronous), exactly
 *     like the reference's launches, except that the reference always used the legacy default stream
 *     of the current device (no CUDAGuard, no getCurrentCUDAStream -- SURVEY.md 2a).
 *   - Return value: 0 on success, otherwise the cudaError_t of the failed launch / API call
 *     (the reference never checks; ubn_last_error_string() gives the text).
 *   - All float tensors are fp32, ids are int64, masks are 1-byte bools (torch.bool), all densely
 *     packed ("contiguous") unless a stride argument says otherwise.  Inputs are borrowed for the
 *     duration of the enqueued work; outputs are caller-allocated.
 *   - Unlike the reference (outputs pre-filled with zeros_like/ones_like), every output element is
 *     written by the kernels themselves, so callers may pass uninitialised (torch.empty) buffers.
 *
 * Each declaration cites the reference interface it replaces (paths relative to the reference repo).
 * The Python binding a maintainer would add is in INTEGRATION.md; this repo's own binding is
 * unboundednerfpytorch_b200/_cabi.py (ctypes).
 */
#ifndef UBNERF_B200_H_
#define UBNERF_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

#define UBN_ABI_VERSION 3

/* ---- library introspection ------------------------------------------------------------------ */
int ubn_abi_version(void);
/* Text of the last non-zero return value on this thread's device ("no error" if none). */
const char* ubn_last_error_string(void);
/* Number of kernel launches issued by this library since load / last reset (bench.py's gpu_launches). */
int64_t ubn_launch_count(void);
void ubn_reset_launch_count(void);

/* ---- render_utils_cuda (FourierGrid/cuda/render_utils.cpp:170-184) --------------------------- */

/* render_utils_cuda.infer_t_minmax            render_utils.cpp:50-57  / render_utils_kernel.cu:12-35,82-104 */
int ubn_infer_t_minmax(const float* rays_o, const float* rays_d, const float* xyz_min, const float* xyz_max,
                       float near, float far, int64_t n_rays, float* t_min, float* t_max, void* stream);

/* render_utils_cuda.infer_n_samples           render_utils.cpp:59-64  / render_utils_kernel.cu:38-55,106-121 */
int ubn_infer_n_samples(const float* rays_d, const float* t_min, const float* t_max, float stepdist,
                        int64_t n_rays, int64_t* n_samples, void* stream);

/* render_utils_cuda.infer_ray_start_dir       render_utils.cpp:66-71  / render_utils_kernel.cu:58-79,123-139 */
int ubn_infer_ray_start_dir(const float* rays_o, const float* rays_d, const float* t_min, int64_t n_rays,
                            float* rays_start, float* rays_dir, void* stream);

/* render_utils_cuda.sample_pts_on_rays        render_utils.cpp:73-83  / render_utils_kernel.cu:144-242.
 * The reference needs the ragged total on the host (N_steps.sum().item(), :212); the replacement
 * splits the call so the caller owns that single D2H read:
 *   ubn_sample_pts_count : fills t_min[n], t_max[n], n_steps[n] and offsets[n+1] (exclusive scan of
 *                          n_steps; offsets[n] == total_len).  scan_scratch: >= n/1024+2 int64.
 *   ubn_sample_pts_emit  : fills rays_pts[total,3], mask_outbbox[total], ray_id[total], step_id[total]. */
int ubn_sample_pts_count(const float* rays_o, const float* rays_d, const float* xyz_min, const float* xyz_max,
                         float near, float far, float stepdist, int64_t n_rays,
                         float* t_min, float* t_max, int64_t* n_steps, int64_t* offsets,
                         int64_t* scan_scratch, void* stream);
int ubn_sample_pts_emit(const float* rays_o, const float* rays_d, const float* xyz_min, const float* xyz_max,
                        const float* t_min, const int64_t* offsets, float stepdist, int64_t n_rays,
                        int64_t total_len, float* rays_pts, uint8_t* mask_outbbox, int64_t* ray_id,
                        int64_t* step_id, void* stream);

/* render_utils_cuda.sample_ndc_pts_on_rays    render_utils.cpp:85-94  / render_utils_kernel.cu:245-293 */
int ubn_sample_ndc_pts_on_rays(const float* rays_o, const float* rays_d, const float* xyz_min,
                               const float* xyz_max, int64_t n_samples, int64_t n_rays,
                               float* rays_pts, uint8_t* mask_outbbox, void* stream);

/* render_utils_cuda.sample_bg_pts_on_rays     render_utils.cpp:96-103 / render_utils_kernel.cu:301-360 (no live caller) */
int ubn_sample_bg_pts_on_rays(const float* rays_o, const float* rays_d, const float* t_max, float bg_preserve,
                              int64_t n_samples, int64_t n_rays, float* rays_pts, void* stream);

/* render_utils_cuda.maskcache_lookup          render_utils.cpp:105-117 / render_utils_kernel.cu:367-424 */
int ubn_maskcache_lookup(const uint8_t* world, const float* xyz, const float* xyz2ijk_scale,
                         const float* xyz2ijk_shift, int64_t sz_i, int64_t sz_j, int64_t sz_k,
                         int64_t n_pts, uint8_t* out, void* stream);

/* render_utils_cuda.raw2alpha / raw2alpha_nonuni          render_utils.cpp:119-131 / render_utils_kernel.cu:431-504
 * interval_arr == NULL -> uniform `interval`; else per-point interval_arr[n_pts] (nonuni). */
int ubn_raw2alpha(const float* density, float shift, float interval, const float* interval_arr,
                  int64_t n_pts, float* exp_d, float* alpha, void* stream);

/* render_utils_cuda.raw2alpha_backward / _nonuni_backward  render_utils.cpp:133-147 / render_utils_kernel.cu:507-574 */
int ubn_raw2alpha_backward(const float* exp_d, const float* grad_back, float interval,
                           const float* interval_arr, int64_t n_pts, float* grad, void* stream);

/* render_utils_cuda.alpha2weight              render_utils.cpp:149-154 / render_utils_kernel.cu:577-651.
 * ray_id must be sorted.  Writes weight[n_pts], T[n_pts], alphainv_last[n_rays], i_start/i_end[n_rays]. */
int ubn_alpha2weight(const float* alpha, const int64_t* ray_id, int64_t n_pts, int64_t n_rays,
                     float* weight, float* T, float* alphainv_last, int64_t* i_start, int64_t* i_end,
                     void* stream);

/* render_utils_cuda.alpha2weight_backward     render_utils.cpp:156-167 / render_utils_kernel.cu:654-707 */
int ubn_alpha2weight_backward(const float* alpha, const float* weight, const float* T,
                              const float* alphainv_last, const int64_t* i_start, const int64_t* i_end,
                              int64_t n_pts, int64_t n_rays, const float* grad_weights,
                              const float* grad_last, float* grad, void* stream);

/* torch_scatter.segment_coo(src, index, out=zeros, reduce='sum') on a sorted index, as the reference uses it for
 * the composite (dvgo.py:401,418; dcvgo.py:345,354,377; FourierGrid_model.py:640,666): out[r, 0:k] = sum of the
 * rows src[i, 0:k] with ray_id[i] == r (k <= 4).  Deterministic (no atomics).  i_start / i_end: int64[n_rays] scratch
 * that receives the segment bounds.  out[n_rays, k] is fully written (0 for rays without points). */
int ubn_segment_sum(const float* src, int64_t k, const int64_t* ray_id, int64_t n_pts, int64_t n_rays,
                    int64_t* i_start, int64_t* i_end, float* out, void* stream);

/* The colour composite itself, rgb_marched = segment_coo(weights[:,None] * rgb, ray_id, zeros[n_rays,3], 'sum')
 * (FourierGrid_model.py:640-644, dcvgo.py:345-349, dvgo.py:401-405), without materialising the [n_pts,3] product, and its
 * adjoint in one pass: grad_rgb_i = w_i * g[ray_i], grad_weights_i = sum_c g[ray_i,c] * rgb_i[c] (either may be NULL).
 * Same rounding as the two-op form (product rounded before the sum). */
int ubn_composite_fwd(const float* weights, const float* rgb, const int64_t* ray_id, int64_t n_pts, int64_t n_rays,
                      int64_t* i_start, int64_t* i_end, float* out, void* stream);
int ubn_composite_bwd(const float* weights, const float* rgb, const int64_t* ray_id, const float* grad_out, int64_t n_pts,
                      float* grad_weights, float* grad_rgb, void* stream);

/* ---- total_variation_cuda (FourierGrid/cuda/total_variation.cpp:22-24) ----------------------- */
/* total_variation_cuda.total_variation_add_grad   total_variation.cpp:13-20 / total_variation_kernel.cu:14-67.
 * param/grad: logical [lead, sz_i, sz_j, sz_k, inner] row-major in MEMORY.  Reference layout
 * [P,C,X,Y,Z] contiguous -> lead=P*C, inner=1;  channels-last storage [P,X,Y,Z,C] -> lead=P, inner=C.
 * Keeps the reference's axis-weight quirk (i-axis uses wz; wx unused, :31-32) and the /6 (:45-47). */
int ubn_total_variation_add_grad(const float* param, float* grad, float wx, float wy, float wz,
                                 int64_t lead, int64_t sz_i, int64_t sz_j, int64_t sz_k, int64_t inner,
                                 int dense_mode, void* stream);

/* ---- adam_upd_cuda (FourierGrid/cuda/adam_upd.cpp:79-86) -------------------------------------- */
/* adam_upd_cuda.adam_upd (mode 0) / masked_adam_upd (mode 1) / adam_upd_with_perlr (mode 2, needs perlr)
 * adam_upd.cpp:31-77 / adam_upd_kernel.cu:9-132.  Elementwise over n floats (any common layout). */
int ubn_adam_upd(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, const float* perlr,
                 int64_t n, int step, float beta1, float beta2, float lr, float eps, int mode, void* stream);

/* Fused training-step tail (SURVEY.md 8f rank 1): total-variation add + (masked) Adam + grad zeroing in
 * ONE sweep over the grid; same per-element arithmetic as ubn_total_variation_add_grad followed by
 * ubn_adam_upd.  tv_mode: 0 = no TV, 1 = dense TV, 2 = sparse TV (only where grad != 0). */
int ubn_tv_adam_fused(float* param, float* grad, float* exp_avg, float* exp_avg_sq,
                      float wx, float wy, float wz, int64_t lead, int64_t sz_i, int64_t sz_j, int64_t sz_k,
                      int64_t inner, int tv_mode, int step, float beta1, float beta2, float lr, float eps,
                      int adam_mode, int zero_grad, void* stream);

/* Single-pass tail with ping-pong parameters: total_variation_add_grad + (masked) adam_upd in ONE walk that reads param,
 * grad, exp_avg, exp_avg_sq once and writes the updated parameters to `param_out` (a second buffer of the same layout; the
 * caller swaps the two afterwards), so the TV stencil never sees a half-updated neighbourhood.  Channels-last grids only
 * (inner % 4 == 0, sz_k * inner / 4 <= 512).  Bit-identical to ubn_total_variation_add_grad followed by ubn_adam_upd
 * (adam_mode 0 / 1).  write_grad = 0 skips storing the TV-augmented gradient. */
int ubn_tv_adam_pingpong(const float* param, float* param_out, float* grad, float* exp_avg, float* exp_avg_sq, float wx,
                         float wy, float wz, int64_t lead, int64_t sz_i, int64_t sz_j, int64_t sz_k, int64_t inner,
                         int dense_mode, int step, float beta1, float beta2, float lr, float eps, int adam_mode,
                         int write_grad, void* stream);

/* Multi-GPU training-step tail in one sweep over NVLink peer memory (SURVEY.md 8e; no reference counterpart -- the reference has
 * no distributed code): for the planes [plane_begin, plane_end) of the flattened (lead, sz_i) axis that this rank OWNS,
 *   g = mean over the n_peers ranks of grad_peers[q]   (P2P loads = reduce-scatter),  g += TV(param)  (K20, as above),
 *   (masked) Adam on this rank's exp_avg / exp_avg_sq   (K17 / K18),
 *   param_out_peers[q] <- updated parameters for EVERY rank q  (P2P stores = all-gather; ping-pong buffer, != param).
 * param: this rank's replica (old values, read with halos).  grad_peers / param_out_peers: HOST arrays of n_peers DEVICE pointers
 * to whole-grid buffers that are peer-mapped into this process (n_peers in {1, 2, 4, 8}; entry order = rank order = summation
 * order).  Channels-last layout and limits as ubn_tv_adam_pingpong.  The caller provides the two cross-rank barriers (all
 * gradients complete before the launch, all stores complete before anyone reads param_out) and re-zeroes its own gradient.
 * n_peers = 1 gives bit-identical parameters and moments to ubn_total_variation_add_grad + ubn_adam_upd. */
int ubn_tv_adam_peer(const float* param, float* const* param_out_peers, const float* const* grad_peers, int n_peers,
                     float* exp_avg, float* exp_avg_sq, float wx, float wy, float wz, int64_t lead, int64_t sz_i, int64_t sz_j,
                     int64_t sz_k, int64_t inner, int dense_mode, int64_t plane_begin, int64_t plane_end, int step, float beta1,
                     float beta2, float lr, float eps, int adam_mode, void* stream);

/* ---- ub360_utils_cuda (FourierGrid/cuda/ub360_utils.cpp:20-22) -------------------------------- */
/* ub360_utils_cuda.cumdist_thres              ub360_utils.cpp:13-18 / ub360_utils_kernel.cu:13-47 */
int ubn_cumdist_thres(const float* dist, float thres, int64_t n_rays, int64_t n_pts, uint8_t* mask,
                      void* stream);

/* ---- rays and batches: the step either side of the march (SURVEY.md 8f rank 2) ---------------------
 * dvgo.get_rays_of_a_view                      FourierGrid/dvgo.py:492-555 (get_rays + ndc_rays + viewdirs)
 * One launch writes rays_o, rays_d, viewdirs [H*W,3] of one view.  K_host: 3x3 row-major intrinsics, c2w_host: camera-
 * to-world rows of length c2w_row_stride (4 for a 3x4 / 4x4 pose) -- both HOST pointers (21 scalars).  mode: 0 'lefttop',
 * 1 'center', 2 'random' with `jitter` = device [2,H,W] uniform(0,1) offsets (plane 0 for i, plane 1 for j; the caller
 * draws them, torch.rand_like in the reference).  ndc uses near = 1, focal = K[0][0] like dvgo.py:553-554. */
int ubn_get_rays_of_a_view(int H, int W, const float* K_host, const float* c2w_host, int c2w_row_stride, int ndc,
                           int inverse_y, int flip_x, int flip_y, int mode, const float* jitter, float* rays_o,
                           float* rays_d, float* viewdirs, void* stream);

/* Per-step batch assembly, run_train.py:204-212 (target / rays_o / rays_d / viewdirs = *_tr[sel_i]): gathers rows idx[k]
 * of up to four [n_src,3] fp32 arrays in ONE launch.  src / dst: HOST arrays of n_arrays device pointers.  Negative
 * indices wrap like Python; an out-of-range index sets *oob_flag (device int, caller-zeroed) instead of faulting. */
int ubn_gather_rays(const float* const* src, float* const* dst, int n_arrays, const int64_t* idx, int64_t n_sel,
                    int64_t n_src, int* oob_flag, void* stream);

/* ---- in-kernel training losses (SURVEY.md 8f rank 1) ------------------------------------------------
 * FourierGrid/run_train.py:253-279: loss = w_main * F.mse_loss(rgb_marched, target)
 *   + w_freq * FourierMSELoss(rgb_marched, target)            (FourierGrid_model.py:114-130; real part of the colour-axis FFT, :255-257)
 *   + w_entropy * entropy_last(alphainv_last.clamp(1e-6, 1-1e-6))                                                        (:258-261)
 *   + w_nearclip * sum_{t_m < near_thres} (density_m - density_m.detach())   (value 0, gradient w_nearclip on raw_density,  :262-268)
 *   + w_rgbper * sum_m weights_m |raw_rgb_m - target[ray_id_m]|^2 / n_rays                               (weights detached, :275-278)
 * and d loss / d {rgb_marched [n_rays,3], alphainv_last [n_rays], raw_rgb [n_pts,3], raw_density [n_pts]} in two launches.
 * out5 = {loss, mse, entropy_last, rgbper, freq} (device).  alphainv_last / raw_rgb / t_pts may be NULL (term off; their gradient
 * buffers are then not written).  t_pts: the per-sample ray parameter ret_dict['t'] [n_pts].  scratch: >= 2368 doubles of device
 * memory (per-block partials, summed in a fixed order: the loss value is deterministic). */
int ubn_render_loss(const float* rgb_marched, const float* alphainv_last, const float* raw_rgb, const float* weights,
                    const int64_t* ray_id, const float* target, const float* t_pts, int64_t n_rays, int64_t n_pts,
                    float w_main, float w_entropy, float w_rgbper, float w_freq, float w_nearclip, float near_thres,
                    float* out5, float* grad_rgb_marched, float* grad_alphainv_last, float* grad_raw_rgb,
                    float* grad_raw_density, double* scratch, int64_t scratch_len, void* stream);

/* Distortion loss, torch_efficient_distloss.flatten_eff_distloss(w, s, interval, ray_id) as called at run_train.py:268-274
 * (maths in-tree at dcvgo.py:387-409): out1[0] = (1/R) sum_rays [ sum_i interval/3 w_i^2 + 2 sum_i w_i (s_i W_<i - WS_<i) ]
 * with R = ray_id.max() + 1 like the library (read on the device from the last element of the sorted ray_id: no host sync) and
 * grad_w = d out / d w (NULL = value only).  n_rays: any upper bound of R (the batch size) -- it only sizes the per-ray arrays;
 * ray_id sorted, n_pts >= 1; i_start / i_end: int64[n_rays] scratch; scratch: >= n_rays doubles.  Deterministic. */
int ubn_distortion_loss(const float* w, const float* s, const int64_t* ray_id, int64_t n_pts, int64_t n_rays,
                        float interval, int64_t* i_start, int64_t* i_end, float* out1, float* grad_w, double* scratch,
                        int64_t scratch_len, void* stream);

/* ---- trilinear voxel-grid reads: DenseGrid.forward (grid.py:50-61) and FourierGrid.forward
 *      (FourierGrid_grid.py:60-78) == torch F.grid_sample(bilinear, align_corners=True, zero padding)
 *      + its adjoint (grid_sampler_3d_backward wrt the grid) -------------------------------------
 * grid: P slabs x C channels x [X,Y,Z]; element (p,c,x,y,z) lives at
 *       grid[p*stride_p + c*stride_c + ((x*Y + y)*Z + z)*stride_v].
 *       reference layout [P,C,X,Y,Z] contiguous: stride_p=C*X*Y*Z, stride_c=X*Y*Z, stride_v=1
 *       channels-last storage [P,X,Y,Z,C]      : stride_p=X*Y*Z*C, stride_c=1,     stride_v=C
 * num_freqs: 0 -> DenseGrid / FourierGrid(use_nerf_pos=False) (P must be 1);
 *            F>0 -> FourierGrid with P = 1+2F slabs sampled at gamma_n(ind_norm), averaged over slabs.
 * out / grad_out: [n_pts, C] row-major.  xyz_min/xyz_max: HOST float[3]. */
typedef struct UbnGridDesc {
  int32_t P, C, X, Y, Z;
  int32_t num_freqs;
  int64_t stride_p, stride_c, stride_v;
  float xyz_min[3];
  float xyz_max[3];
} UbnGridDesc;

int ubn_grid_sample_fwd(const float* grid, const UbnGridDesc* desc, const float* xyz, int64_t n_pts,
                        float* out, void* stream);
int ubn_grid_sample_bwd(const float* grad_out, const UbnGridDesc* desc, const float* xyz, int64_t n_pts,
                        float* grad_grid, void* stream);

/* ---- grid-native occupancy / progressive-growing utilities (SURVEY.md 8a row a13) ---------------------------------------------
 * The reference builds these from whole-grid torch ops (meshgrid + grid_sample + max_pool3d, F.interpolate, an autograd backward
 * per 10 000 rays); each is one or two kernels here, lattice / sample coordinates generated in registers. */

/* update_occupancy_cache, step 1 (FourierGrid_model.py:443-450, dcvgo.py:216-222): alpha[i,j,k] = Raw2Alpha(density(p_ijk)),
 * p = lattice of linspace(lattice_min[a], lattice_max[a], m_a) points (HOST float[3] arrays), density = C = 1 grid `desc`. */
int ubn_lattice_alpha(const float* grid, const UbnGridDesc* desc, const float* lattice_min, const float* lattice_max, int64_t mX,
                      int64_t mY, int64_t mZ, float act_shift, float interval, float* alpha, void* stream);
/* step 2 (:451-452): mask &= F.max_pool3d(alpha, kernel 3, stride 1, padding 1) > thres.  mask: torch.bool bytes [X,Y,Z]. */
int ubn_maxpool3_gt_and(const float* alpha, int64_t X, int64_t Y, int64_t Z, float thres, uint8_t* mask, void* stream);
/* scale_volume_grid (grid.py:63-68, FourierGrid_grid.py:80-85): out = F.interpolate(in, size = out dims, mode = 'trilinear',
 * align_corners = True) for every slab / channel; either layout on either side (strides from the descriptors). */
int ubn_resample_grid(const float* in, const UbnGridDesc* in_desc, float* out, const UbnGridDesc* out_desc, void* stream);
/* voxel_count_views inner loop (FourierGrid_model.py:405-417, dvgo.py:255-270): grad += adjoint of DenseGrid(1, dims)(pts).sum() for
 * pts = o + d * (t_min + step * i / |d|), i < n_samples, t_min from the AABB of `desc` clamped to [near, far]; grad: [X,Y,Z]. */
int ubn_view_scatter_ones(const float* rays_o, const float* rays_d, int64_t n_rays, int64_t n_samples, float near, float far,
                          float step, const UbnGridDesc* desc, float* grad, void* stream);
/* count += (grad > thres)      (:418-419 `count += (ones.grid.grad > 1)`) */
int ubn_count_gt(const float* grad, float thres, int64_t n, float* count, void* stream);
/* maskout_near_cam_vox (FourierGrid_model.py:375-388): slab[v] = fill where min_c |lattice(v) - cams[c]| <= near_clip, lattice =
 * linspace(-1, 1, size) per axis, cams [n_cams, 3] device array already in the slab's (embedded, flipped) coordinates. */
int ubn_maskout_near_cam(float* slab, int64_t voxel_stride, int64_t X, int64_t Y, int64_t Z, const float* cams, int64_t n_cams,
                         float near_clip, float fill, void* stream);
/* maskout_near_cam_vox of DirectVoxGO (dvgo.py:185-198): as above on the lattice linspace(lattice_min[a], lattice_max[a], size)
 * (HOST float[3] arrays; the world bbox there), cams [n_cams, 3] device array in world coordinates. */
int ubn_maskout_near_cam_lattice(float* slab, int64_t voxel_stride, int64_t X, int64_t Y, int64_t Z, const float* lattice_min,
                                 const float* lattice_max, const float* cams, int64_t n_cams, float near_clip, float fill,
                                 void* stream);

/* ---- fused ray march: sample_ray + density query + Raw2Alpha + Alphas2Weights + thresholds + k0 query
 *      for FourierGridModel.forward (FourierGrid_model.py:509-621) and DirectContractedVoxGO.forward
 *      (dcvgo.py:228-331) ------------------------------------------------------------------------ */
typedef struct UbnMarchCfg {
  /* scene normalisation (rays_o - center) / radius: FourierGrid_model.py:522, dcvgo.py:239 */
  float scene_center[3];
  float scene_radius[3];
  /* contraction p/|p| * (contract_B - contract_A/|p|) when |p| > 1: B = 1+bg_len, A = bg_len, both
   * narrowed to float by the host exactly as torch narrows the Python scalars
   * (dcvgo.py:260, FourierGrid_model.py:541-547) */
  float contract_B;
  float contract_A;
  int32_t contracted_norm;      /* 0 = inf-norm, 1 = l2-norm */
  int32_t n_samples;            /* S = len(t) (host builds the t table exactly as the reference does) */
  float act_shift;              /* Raw2Alpha shift */
  float interval;               /* stepsize * voxel_size_ratio */
  float fast_color_thres;       /* <= 0: no thresholding (dense output, M = N*S) */
  int32_t use_cumdist;          /* dcvgo.py:286-294: keep inner points + cumdist_thres survivors */
  float cumdist_thres;
  int32_t use_maskcache;        /* dcvgo.py:297-302 */
  int32_t mask_sz[3];
  float mask_scale[3];
  float mask_shift[3];
} UbnMarchCfg;

/* per-sample flag bits written by pass A */
#define UBN_FLAG_QUERIED   1   /* density was queried (survived cumdist / mask-cache) */
#define UBN_FLAG_LISTED    2   /* member of the Alphas2Weights list (alpha > thres) */
#define UBN_FLAG_SCANNED   4   /* consumed by the transmittance scan before its early stop (i < i_end) */
#define UBN_FLAG_KEEP      8   /* survives every mask: feature query + compacted output */
#define UBN_FLAG_INNER    16   /* |p| <= 1 before contraction (inner_mask) */

/* update_occupancy_cache_lt_nviews inner loop (dcvgo.py:195-213: per view, `ones = grid.DenseGrid(1, world_size, xyz_min,
 * xyz_max)`, then `ones(sample_ray(rays_o, rays_d)[0]).sum().backward()` per 8192 rays): grad [X,Y,Z] += the trilinear weights
 * (align_corners=True) of every contracted sample t_table[s], s < cfg->n_samples, of every ray -- the points pass A generates,
 * with no inner-mask, cumdist or mask-cache filter.  Only the scene normalisation, contraction and n_samples fields of `cfg`
 * are read; `desc` is the single-slab ones grid (P = C = 1, unit voxel stride).  Follow with ubn_count_gt(grad, 1). */
int ubn_view_scatter_ones_contracted(const float* rays_o, const float* rays_d, int64_t n_rays, const float* t_table,
                                     const UbnMarchCfg* cfg, const UbnGridDesc* desc, float* grad, void* stream);

/* Pass A: per nominal sample (r,s): contracted point, masks, density, alpha, exact sequential
 * transmittance scan (identical arithmetic to alpha2weight, early stop at T < 1e-3 included), weights,
 * both thresholds.  Dense per-sample outputs [n_rays*S]: density, alpha, weight, T, flags.
 * Per ray: alphainv_last[n_rays], n_keep[n_rays] (number of UBN_FLAG_KEEP samples). */
int ubn_march_density_fwd(const float* rays_o, const float* rays_d, const float* t_table,
                          const float* density_grid, const UbnGridDesc* density_desc,
                          const uint8_t* mask_world, const UbnMarchCfg* cfg, int64_t n_rays,
                          float* density, float* alpha, float* weight, float* T, uint8_t* flags,
                          float* alphainv_last, int32_t* n_keep, void* stream);

/* Exclusive scan of n_keep -> offsets[n_rays+1] (offsets[n_rays] = M). scratch >= n_rays/1024+2 int64. */
int ubn_exclusive_scan_i32(const int32_t* in, int64_t n, int64_t* offsets, int64_t* scratch, void* stream);

/* Which pass-B kernel family serves 12-channel channels-last feature grids: 0 = warp-cooperative (lane = corner x channel quad),
 * 1 = lane-per-sample for the forward, 2 = lane-per-sample for forward and backward, 3 / 4 / 5 (the default) = lane-per-sample
 * forward + slab-major cooperative scatter (FourierGrid k0 grids: one slab of the gradient live at a time), each slab swept in 1 / 2 / 4
 * x-ranges (a quarter slab of the benchmarked grid fits the H100's L2); 6 = as 3 with the gather that gives a sample three lanes (one per channel quad), 8 samples per instruction.  Same results to fp32 rounding (the
 * lane-per-sample forward is bit-identical to F.grid_sample(...).mean(0)); process-wide, not thread-safe against concurrent
 * launches.  Returns cudaErrorInvalidValue for other values. */
int ubn_set_feature_kernel(int variant);
int ubn_get_feature_kernel(void);
/* How ubn_march_density_bwd scatters into the density-grid gradient (contiguous single-channel grids): 1 (the default) = two
 * launches, the reverse scan writing per-sample gradients to gd_scratch, then a frequency-major scatter that walks runs of
 * consecutive samples per lane and merges the contributions of samples that stay in the same cell before they leave as pair
 * reductions; 0 = every sample scatters its own 8 corners from the scan kernel.  Same sums up to fp32 addition order.
 * Process-wide like ubn_set_feature_kernel. */
int ubn_set_density_scatter(int variant);
int ubn_get_density_scatter(void);

/* Pass B: for every survivor (flags bit1), in (ray, step) order at offsets[ray]+rank: recompute the
 * contracted point, query the feature grid (k0), and emit the compacted per-survivor records.
 * k0: channels-last with C in {4, 8, 12, 16} (16-byte aligned), or C in {3, 15} with an odd slab count P <= 11 and >= 2 voxels
 * per axis (4-byte aligned records; features bit-identical to F.grid_sample(...).mean(0)). */
int ubn_march_feature_fwd(const float* rays_o, const float* rays_d, const float* t_table,
                          const float* k0_grid, const UbnGridDesc* k0_desc, const UbnMarchCfg* cfg,
                          int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                          const float* density, const float* alpha, const float* weight,
                          float* k0_feat, float* out_density, float* out_alpha, float* out_weight,
                          int64_t* ray_id, int64_t* step_id, float* out_t, uint8_t* out_inner, void* stream);

/* Pass B forward for COHERENT rays (a frame's image-ordered 8192-ray chunks, run_render.py:43-63) on a single-slab 12-channel
 * channels-last feature grid (DenseGrid k0 of DirectContractedVoxGO / DirectVoxGO): same arguments and outputs as
 * ubn_march_feature_fwd, but warp = 32 consecutive rays and the voxel brick a warp's 32 rays x 4 steps touch is staged in shared
 * memory by ONE TMA tensor load (cp.async.bulk.tensor 4-D box [8,8,8,12], mbarrier-signalled); blocks whose cells span more than
 * 7 lattice steps on an axis fall back to direct loads.  Correct for any rays (incoherent rays simply take the fallback).
 * Features are accumulated in ATen's corner order (bit-identical to F.grid_sample / ubn_grid_sample_fwd).
 * stats2: optional device uint64[2], += {blocks served by TMA, blocks served by the fallback}. */
int ubn_march_feature_fwd_tma(const float* rays_o, const float* rays_d, const float* t_table, const float* k0_grid,
                              const UbnGridDesc* k0_desc, const UbnMarchCfg* cfg, int64_t n_rays, const uint8_t* flags,
                              const int64_t* offsets, const float* density, const float* alpha, const float* weight, float* feat,
                              float* o_density, float* o_alpha, float* o_weight, int64_t* o_ray_id, int64_t* o_step_id, float* o_t,
                              uint8_t* o_inner, unsigned long long* stats2, void* stream);

/* Backward of pass B: scatter grad_feat[M,C] into grad_k0 (adjoint of the trilinear read). */
int ubn_march_feature_bwd(const float* rays_o, const float* rays_d, const float* t_table,
                          const UbnGridDesc* k0_desc, const UbnMarchCfg* cfg, int64_t n_rays,
                          const uint8_t* flags, const int64_t* offsets, const float* grad_feat,
                          float* grad_k0, void* stream);

/* Backward of pass A: grads wrt compacted weights / alpha / density and alphainv_last -> exact reverse
 * scan (alpha2weight_backward arithmetic) -> raw2alpha_backward -> scatter into grad_density.
 * gd_scratch: device float[n_rays * S] (S = the records' stride) that the run scatter passes the per-sample gradients through
 * from its first launch to its second; its contents are overwritten.  May be NULL only under ubn_set_density_scatter(0). */
int ubn_march_density_bwd(const float* rays_o, const float* rays_d, const float* t_table,
                          const UbnGridDesc* density_desc, const UbnMarchCfg* cfg, int64_t n_rays,
                          const float* density, const float* alpha, const float* weight, const float* T,
                          const uint8_t* flags, const float* alphainv_last, const int64_t* offsets,
                          const float* g_weight, const float* g_alpha, const float* g_density,
                          const float* g_last, float* grad_density_grid, float* gd_scratch, void* stream);

/* ---- fused NDC ray march for the forward-facing model DirectMPIGO.forward (FourierGrid/dmpigo.py:224-340):
 *      sample_ndc_pts_on_rays + bbox drop + mask cache + (density + act_shift) + Raw2Alpha(shift 0) + Alphas2Weights + both
 *      thresholds + k0 query.  Same three-launch forward (pass A, ubn_exclusive_scan_i32, pass B) and two-launch backward as the
 *      contracted march above, the same per-sample records and flag bits (UBN_FLAG_INNER is never set). ------------------- */
typedef struct UbnNdcMarchCfg {
  /* sample i of S: p = o + d * (i / (S-1)) exactly as render_utils_kernel.cu:260-263; S = int((mpi_depth-1)/stepsize)+1
   * (dmpigo.py:239); samples with p outside [xyz_min, xyz_max] (strict comparisons) are dropped (dmpigo.py:242-243) */
  float xyz_min[3];
  float xyz_max[3];
  int32_t n_samples;
  float interval;               /* stepsize * voxel_size_ratio (dmpigo.py:265) */
  float fast_color_thres;       /* <= 0: no thresholding */
  int32_t use_maskcache;        /* dmpigo.py:268-272 */
  int32_t mask_sz[3];
  float mask_scale[3];
  float mask_shift[3];
} UbnNdcMarchCfg;

/* Pass A: density = density_grid(p) + act_shift_grid(p) (dmpigo.py:275; one fp32 add), alpha = Raw2Alpha(density, 0, interval)
 * (:276), the exact sequential transmittance scan and both thresholds (:277-292).  density_grid: single-slab C = 1 grid;
 * act_shift_grid: the [1,1,1,1,mpi_depth] DenseGrid of dmpigo.py:47-57 (any C = 1 single-slab grid).  Outputs as
 * ubn_march_density_fwd; `density` receives the biased density. */
int ubn_march_ndc_density_fwd(const float* rays_o, const float* rays_d, const float* density_grid,
                              const UbnGridDesc* density_desc, const float* act_shift_grid, const UbnGridDesc* act_shift_desc,
                              const uint8_t* mask_world, const UbnNdcMarchCfg* cfg, int64_t n_rays, float* density,
                              float* alpha, float* weight, float* T, uint8_t* flags, float* alphainv_last, int32_t* n_keep,
                              void* stream);

/* Pass B: for every survivor, in (ray, step) order at offsets[ray] + rank, the k0 read (dmpigo.py:295, F.grid_sample arithmetic,
 * bit-identical) and the compacted records alpha, weight, ray_id, step_id (:321-327).  k0: single-slab channels-last grid with
 * C = 3 (rgbnet_dim = 0) or C = 9 (LLFF, rgbnet_dim = 9); out_alpha / out_weight may be NULL. */
int ubn_march_ndc_feature_fwd(const float* rays_o, const float* rays_d, const float* k0_grid, const UbnGridDesc* k0_desc,
                              const UbnNdcMarchCfg* cfg, int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                              const float* alpha, const float* weight, float* k0_feat, float* out_alpha, float* out_weight,
                              int64_t* ray_id, int64_t* step_id, void* stream);

/* Backward of pass B: grad_k0 += adjoint of the k0 read applied to grad_feat[M,C] (grid_sampler_3d_backward wrt the grid). */
int ubn_march_ndc_feature_bwd(const float* rays_o, const float* rays_d, const UbnGridDesc* k0_desc, const UbnNdcMarchCfg* cfg,
                              int64_t n_rays, const uint8_t* flags, const int64_t* offsets, const float* grad_feat,
                              float* grad_k0, void* stream);

/* Backward of pass A: exact reverse scan (alpha2weight_backward) -> raw2alpha_backward -> scatter into the density-grid gradient.
 * act_shift gets no gradient (requires_grad = False, dmpigo.py:50).  gd_scratch as for ubn_march_density_bwd. */
int ubn_march_ndc_density_bwd(const float* rays_o, const float* rays_d, const UbnGridDesc* density_desc,
                              const UbnNdcMarchCfg* cfg, int64_t n_rays, const float* density, const float* alpha,
                              const float* weight, const float* T, const uint8_t* flags, const float* alphainv_last,
                              const int64_t* offsets, const float* g_weight, const float* g_alpha, const float* g_last,
                              float* grad_density_grid, float* gd_scratch, void* stream);

/* ---- fused box march for the bounded-scene model DirectVoxGO.forward (FourierGrid/dvgo.py:306-397): sample_pts_on_rays +
 *      in-box drop + mask cache + density + Raw2Alpha + Alphas2Weights + both thresholds + k0 query.  Same three-launch forward
 *      (pass A, ubn_exclusive_scan_i32, pass B) and two-launch backward as the contracted march, the same per-sample records and
 *      flag bits (UBN_FLAG_INNER is never set).  Records are [n_rays * s_max]; ray r fills its first n_steps(r) of them only. ---- */
typedef struct UbnBoxMarchCfg {
  /* scene bbox: the AABB of render_utils_kernel.cu:12-79 (t_min / t_max) and the inclusive in-box test of :191-192 */
  float xyz_min[3];
  float xyz_max[3];
  float near;                   /* t clamp (render_utils_kernel.cu:37-38); far is 1e9 as dvgo.py:321 sets it */
  float stepdist;               /* stepsize * voxel_size (dvgo.py:324); sample i = start + dir * (stepdist * i) (:185-190) */
  int32_t s_max;                /* record stride: a host bound on n_steps = max(ceil((t_max - t_min) * |d| / stepdist), 1) (:53).
                                   A ray with more steps sets *overflow in pass A, it is never truncated silently. <= 4096 */
  float act_shift;              /* Raw2Alpha shift (dvgo.py:60, 357) */
  float interval;               /* stepsize * voxel_size_ratio (dvgo.py:347) */
  float fast_color_thres;       /* <= 0: no thresholding (dvgo.py:358-375) */
  int32_t use_maskcache;        /* dvgo.py:350-354: the lookup comes before the density query */
  int32_t mask_sz[3];           /* MaskGrid geometry (grid.py:223-242): mask dims, xyz2ijk_scale, xyz2ijk_shift */
  float mask_scale[3];
  float mask_shift[3];
} UbnBoxMarchCfg;

/* Pass A: density = density_grid(p) (single-slab C = 1 grid), alpha = Raw2Alpha(density, act_shift, interval), the exact sequential
 * transmittance scan and both thresholds; outputs as ubn_march_density_fwd.  overflow: device int32 the caller zeroes; set to 1 when
 * some ray's n_steps exceeds s_max (that ray is clamped to s_max samples and the caller must treat the result as an error). */
int ubn_march_box_density_fwd(const float* rays_o, const float* rays_d, const float* density_grid, const UbnGridDesc* density_desc,
                              const uint8_t* mask_world, const UbnBoxMarchCfg* cfg, int64_t n_rays, float* density, float* alpha,
                              float* weight, float* T, uint8_t* flags, float* alphainv_last, int32_t* n_keep, int32_t* overflow,
                              void* stream);
/* Pass B: for every survivor, in (ray, step) order at offsets[ray] + rank, the k0 read (F.grid_sample arithmetic, bit-identical)
 * and the compacted records alpha, weight, ray_id, step_id (step_id = the ray's own step index).  k0: single-slab channels-last
 * grid with C = 12 (16-byte aligned) or C = 3; k0_feat 16-byte aligned; out_alpha / out_weight may be NULL. */
int ubn_march_box_feature_fwd(const float* rays_o, const float* rays_d, const float* k0_grid, const UbnGridDesc* k0_desc,
                              const UbnBoxMarchCfg* cfg, int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                              const float* alpha, const float* weight, float* k0_feat, float* out_alpha, float* out_weight,
                              int64_t* ray_id, int64_t* step_id, void* stream);
/* Backward of pass B: grad_k0 += adjoint of the k0 read applied to grad_feat[M,C]. */
int ubn_march_box_feature_bwd(const float* rays_o, const float* rays_d, const UbnGridDesc* k0_desc, const UbnBoxMarchCfg* cfg,
                              int64_t n_rays, const uint8_t* flags, const int64_t* offsets, const float* grad_feat,
                              float* grad_k0, void* stream);
/* Backward of pass A: exact reverse scan -> raw2alpha_backward -> scatter into the density-grid gradient.  gd_scratch as for
 * ubn_march_density_bwd, with S = cfg->s_max. */
int ubn_march_box_density_bwd(const float* rays_o, const float* rays_d, const UbnGridDesc* density_desc,
                              const UbnBoxMarchCfg* cfg, int64_t n_rays, const float* density, const float* alpha,
                              const float* weight, const float* T, const uint8_t* flags, const float* alphainv_last,
                              const int64_t* offsets, const float* g_weight, const float* g_alpha, const float* g_last,
                              float* grad_density_grid, float* gd_scratch, void* stream);

/* ---- rgbnet: rgb = sigmoid(rgbnet(cat[k0_feat, viewdirs_emb[ray_id]])) (FourierGrid_model.py:231-242,631-637;
 *      dcvgo.py:103-114,337-342) for the 3-layer, width-128, 12-feature configuration every shipped config uses.
 * The per-ray part of layer 1 is hoisted by the host: view_bias[n_rays,128] = emb(viewdirs) . W1[:,12:]^T + b1, so the
 * kernel sees W1k = W1[:, :12] ([128,12] row-major), W2 [128,128], b2 [128], W3 [3,128], b3 [3] (nn.Linear layout).
 * fp32 arithmetic; activations stay on chip.  h1_save / h2_save: NULL for inference, or [n_pts,128] buffers that
 * receive the post-ReLU hidden activations for ubn_rgbnet_bwd. */
int ubn_rgbnet_fwd(const float* feat, const float* view_bias, const int64_t* ray_id, const float* W1k, const float* W2,
                   const float* b2, const float* W3, const float* b3, int64_t n_pts, float* rgb, float* h1_save,
                   float* h2_save, void* stream);
/* Same contract on the tensor cores: the two 128-wide layers run as mma.sync m16n8k8 TF32 (16-sample units per warp,
 * accumulators and the layer-2 A operand in registers).  single_pass = 0: 3xTF32 split accumulation (fp32-grade,
 * meets the 1e-5 parity gate); single_pass bit 0: one TF32 pass (~1e-3 relative); bit 1: 4 warps per CTA instead of 8 (A/B);
 * bit 2: h1_save / h2_save are written in the PANEL layout [ceil(n_pts/128)][32 column quads][128 rows][4 floats] -- coalesced
 * for the tensor-core fragments on both sides -- and must hold ceil(n_pts/128)*128 rows; only ubn_rgbnet_bwd_tc_fused called
 * with the same bit reads that layout.  h1_mask (bit 2 only; may be NULL): ceil(n_pts/128)*512 uint32 that receive the ReLU masks
 * of H1, [tile][32-unit chunk][row], bit = unit -- ubn_rgbnet_bwd_tc_fused then gates dH1 with them instead of loading H1 rows
 * (pass the same h1_mask there). */
int ubn_rgbnet_fwd_tc(const float* feat, const float* view_bias, const int64_t* ray_id, const float* W1k, const float* W2,
                      const float* b2, const float* W3, const float* b3, int64_t n_pts, float* rgb, float* h1_save,
                      float* h2_save, uint32_t* h1_mask, int single_pass, void* stream);
/* Backward of the above wrt feat (grad_feat[n_pts,12], fully written) and, ACCUMULATED into zero-initialised buffers,
 * view_bias (grad_view_bias[n_rays,128]), W1k, W2, b2, W3, b3.  ray_id must be sorted. */
int ubn_rgbnet_bwd(const float* feat, const int64_t* ray_id, const float* W1k, const float* W2, const float* W3,
                   const float* rgb, const float* h1_save, const float* h2_save, const float* grad_rgb, int64_t n_pts,
                   float* grad_feat, float* grad_view_bias, float* grad_W1k, float* grad_W2, float* grad_b2,
                   float* grad_W3, float* grad_b3, void* stream);

/* Tensor-core backward, in two launches with the same net effect as ubn_rgbnet_bwd:
 *  ubn_rgbnet_bwd_tc_data : dZ2 -> dH1 = dZ2.W2 (tensor cores, A in registers) -> dZ1 -> dz1_out[n_pts,128]; and
 *                           grad_W2 += dZ2^T.H1 (split-K tensor-core GEMM over shared-memory chunks; 3xTF32 split).
 *  ubn_rgbnet_bwd_small   : from dz1: grad_feat, grad_view_bias (accumulated), grad_W1k, and grad_b2 / grad_W3 / grad_b3. */
int ubn_rgbnet_bwd_tc_data(const float* W2, const float* W3, const float* rgb, const float* h1_save, const float* h2_save,
                           const float* grad_rgb, int64_t n_pts, float* dz1_out, float* grad_W2, void* stream);
int ubn_rgbnet_bwd_small(const float* feat, const int64_t* ray_id, const float* W1k, const float* W3, const float* rgb,
                         const float* h2_save, const float* grad_rgb, const float* dz1, int64_t n_pts, float* grad_feat,
                         float* grad_view_bias, float* grad_W1k, float* grad_b2, float* grad_W3, float* grad_b3, void* stream);

/* Tensor-core backward in two launches without any intermediate in HBM (same arguments and net effect as ubn_rgbnet_bwd):
 *  launch 1: dZ2 -> dH1 = dZ2.W2 -> dZ1 -> dX = dZ1.W1k (three tensor-core GEMMs chained through registers) -> grad_feat, and every
 *            reduction over samples except dW2 (grad_view_bias per ray, grad_W1k, grad_b2, grad_W3, grad_b3) as tensor-core GEMMs
 *            over 16-sample tiles of H2 / dZ1 turned through shared memory;   launch 2: grad_W2 += dZ2^T.H1 (split-K tensor-core GEMM).
 * Replaces ubn_rgbnet_bwd_tc_data + ubn_rgbnet_bwd_small (which round-tripped dZ1 [n_pts,128] through HBM and re-read H2).
 * single_pass bit 0: one TF32 pass per product instead of the 3-pass split (the opt-in reduced-precision training mode);
 * bit 1: launch 1 with 4 warps per CTA instead of 8 (A/B);
 * bit 2: h1_save / h2_save are in the panel layout of ubn_rgbnet_fwd_tc.
 * h2_mask_scratch: NULL, or ceil(n_pts/128)*512 uint32 of scratch.  With bit 2 set and a scratch given, launch 1 leaves the ReLU
 * masks of H2 there ([tile][32-unit chunk][row], bit = unit) and launch 2 rebuilds dZ2 from them (dz3 . W3 gated by the mask)
 * instead of reading h2_save a second time.  h1_mask: NULL, or the masks ubn_rgbnet_fwd_tc wrote (bit 2 only): launch 1 then reads
 * 16 bytes per sample instead of the H1 row. */
int ubn_rgbnet_bwd_tc_fused(const float* feat, const int64_t* ray_id, const float* W1k, const float* W2, const float* W3,
                            const float* rgb, const float* h1_save, const float* h2_save, const float* grad_rgb, int64_t n_pts,
                            float* grad_feat, float* grad_view_bias, float* grad_W1k, float* grad_W2, float* grad_b2,
                            float* grad_W3, float* grad_b3, uint32_t* h2_mask_scratch, const uint32_t* h1_mask, int single_pass,
                            void* stream);
/* ubn_rgbnet_fwd_tc / ubn_rgbnet_bwd_tc_fused for n_feat in {3, 12, 15} feature columns (rgbnet_dim = 3: the Waymo / Mega-NeRF
 * FourierGrid configs; 15: Tanks&Temples Train): feat / grad_feat are [n_pts, n_feat], W1k = W1[:, :n_feat] ([128, n_feat]
 * row-major), grad_W1k [128, n_feat]; everything else as above.  n_feat = 12 runs the very kernels of the two functions above.
 * At n_feat = 15 launch 1 of the backward always runs with 4 warps per CTA (8 would not fit shared memory).  Any other n_feat:
 * cudaErrorInvalidValue. */
int ubn_rgbnet_fwd_tc_k(int n_feat, const float* feat, const float* view_bias, const int64_t* ray_id, const float* W1k,
                        const float* W2, const float* b2, const float* W3, const float* b3, int64_t n_pts, float* rgb, float* h1_save,
                        float* h2_save, uint32_t* h1_mask, int single_pass, void* stream);
int ubn_rgbnet_bwd_tc_fused_k(int n_feat, const float* feat, const int64_t* ray_id, const float* W1k, const float* W2,
                              const float* W3, const float* rgb, const float* h1_save, const float* h2_save, const float* grad_rgb,
                              int64_t n_pts, float* grad_feat, float* grad_view_bias, float* grad_W1k, float* grad_W2, float* grad_b2,
                              float* grad_W3, float* grad_b3, uint32_t* h2_mask_scratch, const uint32_t* h1_mask, int single_pass,
                              void* stream);
/* ubn_rgbnet_fwd_tc_k / ubn_rgbnet_bwd_tc_fused_k with the hidden width as an argument (rgbnet_width), for the forward-facing
 * DirectMPIGO of llff_default (rgbnet_dim = 9, rgbnet_width = 64, viewbase_pe = 0: a 12 -> 64 -> 64 -> 3 MLP; replaces
 * dmpigo.py:84-92, 297-306).  Every buffer that is 128 wide above is n_hidden wide here: view_bias / grad_view_bias
 * [n_rays, n_hidden], W1k / grad_W1k [n_hidden, n_feat], W2 / grad_W2 [n_hidden, n_hidden], b2 [n_hidden], W3 [3, n_hidden];
 * the panel saves hold ceil(n_pts/128)*128 rows of n_hidden floats ([tile][n_hidden/4 column quads][128 rows][4]) and the
 * ReLU masks ceil(n_pts/128)*128*n_hidden/32 uint32 ([tile][n_hidden/32 chunks][128 rows]).
 * (n_feat, n_hidden) = (3 | 12 | 15, 128) runs exactly the kernels of the _k pair.  (9, 64): the forward writes saves only in the
 * panel layout (bit 2 must be set when h1_save / h2_save are given), the backward needs bit 2, h1_mask and h2_mask_scratch, and
 * bit 1 (4 warps) is ignored: the width-64 kernels have one launch configuration each.  Any other pair, or a width-64 call
 * without what it needs: cudaErrorInvalidValue. */
int ubn_rgbnet_fwd_tc_kw(int n_feat, int n_hidden, const float* feat, const float* view_bias, const int64_t* ray_id,
                         const float* W1k, const float* W2, const float* b2, const float* W3, const float* b3, int64_t n_pts,
                         float* rgb, float* h1_save, float* h2_save, uint32_t* h1_mask, int single_pass, void* stream);
int ubn_rgbnet_bwd_tc_fused_kw(int n_feat, int n_hidden, const float* feat, const int64_t* ray_id, const float* W1k,
                               const float* W2, const float* W3, const float* rgb, const float* h1_save, const float* h2_save,
                               const float* grad_rgb, int64_t n_pts, float* grad_feat, float* grad_view_bias, float* grad_W1k,
                               float* grad_W2, float* grad_b2, float* grad_W3, float* grad_b3, uint32_t* h2_mask_scratch,
                               const uint32_t* h1_mask, int single_pass, void* stream);
/* Which kernel computes grad_W2 in the width-128 fused backward with panel saves (bit 2) and h2_mask_scratch: 1 (the default) =
 * warpgroup MMA (wgmma) with a producer warpgroup staging H1 in shared memory; 0 = the mma.sync kernel.  Same products and the
 * same per-chunk fp32 running sums, so the same results up to the tensor cores' accumulation order.  Process-wide like
 * ubn_set_feature_kernel.  Returns cudaErrorInvalidValue for other values. */
int ubn_set_dw2_engine(int engine);

/* ---- TensoRFGrid: the vector-matrix (VM) factorised grid (FourierGrid/grid.py:90-201) ------------------------------------------
 * Six factors, in this order everywhere: 0 xy_plane [1,Rxy,X,Y], 1 xz_plane [1,R,X,Z], 2 yz_plane [1,R,Y,Z], 3 x_vec [1,R,X,1],
 * 4 y_vec [1,R,Y,1], 5 z_vec [1,Rxy,Z,1], and, for C > 1, f_vec [R+R+Rxy, C] (row-major).  Factor f element (r, a, b) sits at
 * factor[r * stride_r[f] + a * stride_a[f] + b * stride_b[f]] (vectors: a = the node, b = 0), so the reference-contiguous layout and
 * the channels-last one (a corner's R components contiguous: stride_r == 1) are both described; the kernels take 128-bit loads and
 * reductions when every factor is channels-last with R, Rxy multiples of 4 and 16-byte aligned bases.  Gradient buffers have the
 * strides of their factors.  A point p reads the factors at ind = (p - xyz_min) / (xyz_max - xyz_min) * 2 - 1 (no axis flip) with
 * F.grid_sample(bilinear, align_corners=True, zero padding) arithmetic, corners in ATen's order nw, ne, sw, se; feat =
 * [xy.z, xz.y, yz.x] (3R products); out = sum(feat) for C = 1, feat . f_vec for C > 1.  C must be 1, 3 or 12; R + R + Rxy <= 96. */
typedef struct UbnTensorfDesc {
  int32_t X, Y, Z, R, Rxy, C;
  int64_t stride_r[6], stride_a[6], stride_b[6];
  float xyz_min[3], xyz_max[3];
} UbnTensorfDesc;

/* CTAs of the backward's persistent launch: the f_vec partial sums of the scratch below hold one [R+R+Rxy, C] block per CTA. */
#define UBN_TENSORF_BWD_MAX_CTAS 528

/* TensoRFGrid.forward: out[M, C] (fully written) for the points xyz[M, 3].  f_vec is ignored (may be NULL) when C == 1. */
int ubn_tensorf_fwd(const float* const* factors, const float* f_vec, const UbnTensorfDesc* desc, const float* xyz, int64_t M,
                    float* out, void* stream);
/* Adjoint of ubn_tensorf_fwd for grad_out[M, C]: ADDED into grads[6] (the factor gradients) and grad_f_vec (C > 1).  Plane
 * gradients are reduced straight into grads; the vector gradients go through vec_copies (1..64) replicated copies in scratch
 * (copy = blockIdx % vec_copies), summed in a fixed order by a closing launch.  grad_f_vec = feat^T . grad_out is summed as
 * per-128-sample partials added into one fp32 running sum per CTA, the CTAs' sums added in CTA order by the closing launch.
 * scratch: device floats, at least vec_copies * (X*R + Y*R + Z*Rxy) + UBN_TENSORF_BWD_MAX_CTAS * (R+R+Rxy) * C, 16-byte aligned. */
int ubn_tensorf_bwd(const float* const* factors, const float* f_vec, const UbnTensorfDesc* desc, const float* xyz, int64_t M,
                    const float* grad_out, float* const* grads, float* grad_f_vec, int vec_copies, float* scratch, void* stream);
/* TensoRFGrid.total_variation_add_grad: grads[f] += the gradient of the reference's smooth-L1 TV sum over the planes' two axes and
 * the vectors' length, weighted wx / wy / wz by the world axis each factor axis spans, divided by 6.  One launch for all six. */
int ubn_tensorf_tv_add_grad(const float* const* factors, float* const* grads, const UbnTensorfDesc* desc, float wx, float wy,
                            float wz, void* stream);
/* TensoRFGrid.get_dense_grid: out [1, C, X, Y, Z] (contiguous, fully written) = the node products (no interpolation), summed for
 * C == 1, projected by f_vec for C > 1. */
int ubn_tensorf_dense(const float* const* factors, const float* f_vec, const UbnTensorfDesc* desc, float* out, void* stream);

/* ---- the fused box march with TensoRF grids (DirectVoxGO.forward, dvgo.py:330-366, with density_type / k0_type 'TensoRFGrid';
 *      grid.py:111-129 / 174-201 for the read).  Same records, flags, scan and thresholds as ubn_march_box_density_fwd; the density
 *      is the TensoRF read of ubn_tensorf_fwd (C = 1) at the same box point, so every output is bit-identical to sample_pts_on_rays
 *      + mask cache + TensoRFGrid + Raw2Alpha + Alphas2Weights composed op by op. ---- */
/* Pass A with a TensoRF density: desc->C == 1, factors and desc as for ubn_tensorf_fwd; everything else as
 * ubn_march_box_density_fwd.  Samples outside the mask cache are not read. */
int ubn_march_box_tensorf_density_fwd(const float* rays_o, const float* rays_d, const float* const* factors, const UbnTensorfDesc* desc,
                                      const uint8_t* mask_world, const UbnBoxMarchCfg* cfg, int64_t n_rays, float* density,
                                      float* alpha, float* weight, float* T, uint8_t* flags, float* alphainv_last, int32_t* n_keep,
                                      int32_t* overflow, void* stream);
/* Backward of the above: the reverse scan of ubn_march_box_density_bwd leaves every sample's density gradient in gd_scratch
 * [n_rays * s_max]; a second launch walks each ray's own n_steps, recomputes the point of every record with a nonzero gradient and
 * ADDS the adjoint of the read into grads[6] as ubn_tensorf_bwd does (planes reduced directly, vectors through vec_copies (1..64)
 * replicated copies in vec_scratch -- at least vec_copies * (X*R + Y*R + Z*Rxy) floats, 16-byte aligned -- summed in copy order
 * by a closing launch). */
int ubn_march_box_tensorf_density_bwd(const float* rays_o, const float* rays_d, const float* const* factors, const UbnTensorfDesc* desc,
                                      const UbnBoxMarchCfg* cfg, int64_t n_rays, const float* density, const float* alpha,
                                      const float* weight, const float* T, const uint8_t* flags, const float* alphainv_last,
                                      const int64_t* offsets, const float* g_weight, const float* g_alpha, const float* g_last,
                                      float* const* grads, int vec_copies, float* gd_scratch, float* vec_scratch, void* stream);
/* Pass B for a k0 read elsewhere (the k0 of a TensoRF model, read by its own forward on these points): the compacted records of
 * ubn_march_box_feature_fwd (out_alpha / out_weight may be NULL) and, instead of the feature read, each survivor's point
 * xyz[M, 3] -- the point sample_pts_on_rays gives that step (render_utils_kernel.cu:185-190). */
int ubn_march_box_points_fwd(const float* rays_o, const float* rays_d, const UbnBoxMarchCfg* cfg, int64_t n_rays, const uint8_t* flags,
                             const int64_t* offsets, const float* alpha, const float* weight, float* xyz, float* out_alpha,
                             float* out_weight, int64_t* ray_id, int64_t* step_id, void* stream);

/* ---- scene bounds (FourierGrid/bbox_compute.py) ------------------------------------------------------------------------------
 * Each call widens bounds = device float[6] (xyz_min then xyz_max; pass +inf / -inf to start empty) IN PLACE: bounds[a] =
 * min(bounds[a], min of the points' axis a), bounds[3+a] likewise with max.  A NaN coordinate makes that bound NaN (torch.minimum
 * / amin propagate NaN).  Min and max are order independent: results are exact and deterministic. */

/* compute_bbox_by_cam_frustrm's ray branches (:10-45, :96-110) over n_views views of the 'center' rays of get_rays_of_a_view
 * (same bits as ubn_get_rays_of_a_view).  hw: device int32 [n_views, 2] (H, W); K: device [n_views, 9]; c2w: device
 * [n_views, 12] (c2w[:3, :4]); max_pixels: the largest H * W (host).  inward = 1: the points rays_o + rays_d * near
 * (unbounded-inward / nerfpp, near = near_clip); inward = 0: rays_o + dir * near and rays_o + dir * far with dir = rays_d when
 * ndc, viewdirs otherwise.  No ray is written. */
int ubn_frustum_bounds(const int* hw, const float* K, const float* c2w, int64_t n_views, int64_t max_pixels, int ndc, int inverse_y,
                       int flip_x, int flip_y, int inward, float near, float far, float* bounds, void* stream);
/* compute_bbox_by_coarse_geo's lattice (:144-149): xyz[X*Y*Z, 3] (k fastest) = lattice_min * (1 - t) + lattice_max * t with
 * t = torch.linspace(0, 1, n) per axis; lattice_min / lattice_max: HOST float[3]. */
int ubn_lattice_points(const float* lattice_min, const float* lattice_max, int64_t X, int64_t Y, int64_t Z, float* xyz,
                       void* stream);
/* compute_bbox_by_coarse_geo (:150-160) fused: the points of ubn_lattice_points whose alpha = Raw2Alpha(density(point), act_shift,
 * interval) exceeds thres widen bounds, and their number is ADDED to *count (device int64).  density = the C = 1 grid `desc`,
 * read as ubn_grid_sample_fwd reads it; Raw2Alpha as ubn_raw2alpha.  No point, density or alpha tensor is written. */
int ubn_lattice_bounds(const float* grid, const UbnGridDesc* desc, const float* lattice_min, const float* lattice_max, int64_t X,
                       int64_t Y, int64_t Z, float act_shift, float interval, float thres, float* bounds, int64_t* count,
                       void* stream);
/* The same reduction over a precomputed alpha[X*Y*Z] (device), for densities the fused read does not cover (TensoRFGrid). */
int ubn_lattice_bounds_alpha(const float* alpha, const float* lattice_min, const float* lattice_max, int64_t X, int64_t Y,
                             int64_t Z, float thres, float* bounds, int64_t* count, void* stream);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif  /* UBNERF_B200_H_ */
