// render_bounded.cu -- whole-frame render of DirectVoxGO (box march) and DirectMPIGO (NDC march) in one fused pass, sm_90a.
//
// The same per-warp loop as the contracted render (render.cu, render_warp.cuh): pass A's march on the model's sampling policy,
// the ray left at T < 1e-3, the k0 read of the kept samples, 16-row tiles on the tensor-core rgbnet (or sigmoid(k0)) and the
// composite in step order by the slot's own lane.  What differs per geometry:
//   * box (DirectVoxGO, dvgo.py:306-415): BoxSampler -- t_min / t_max from the AABB, the ray's own n_steps clamped to the cfg's
//     S_max (a longer ray sets *overflow, as pass A does), samples start + dir * (stepdist * s) inside the box; the density with the
//     cfg's scalar act_shift; depth term = step_id; always + alphainv_last * bg;
//   * NDC (DirectMPIGO, dmpigo.py:224-331): NdcSampler -- S = int((mpi_depth - 1) / stepsize) + 1 samples o + d * s / (S - 1) inside
//     the strict bbox; the density plus the act_shift grid (one fp32 add); depth term = (step_id + 0.5) / S in fp32; + alphainv_last
//     * bg (the render has no global_step, so never rand_bkgd).
// The k0 read (lane_features at one slab) is the arithmetic of pass B's k_march_ndc_feature: float4 records at C = 12, scalar
// loads at C = 9 / 3.
//
// Instances: box (C, pe, width) = (12, 4, 128) (the fine stage), (9, 4, 64) (the free-dataset lab config) and sigmoid(k0) at C = 3
// (the coarse stage); NDC (9, 0, 64) (llff_default) and sigmoid(k0) at C = 3.  Width 128 runs one CTA of 12 warps per SM, as the
// contracted kernel (168 registers).  At width 64 the W2 fragments are a quarter as large and layer 1 / 2 hold half the
// accumulators, so the kernel fits 128 registers and one CTA of 16 warps.
#include "render_warp.cuh"

namespace ubn {
namespace rnd {

// warps per CTA of an instance (one CTA per SM); kW is ignored without an rgbnet
__host__ __device__ constexpr int bounded_warps(bool net, int w) { return net && w == 64 ? 16 : 12; }

template <int kC, int kPe, bool kNet, int kW>
__global__ void __launch_bounds__(32 * bounded_warps(kNet, kW), 1) k_render_box(Args a) {
  render_warps<BoxSampler, kC, kPe, kNet, kW, bounded_warps(kNet, kW)>(a);
}

template <int kC, int kPe, bool kNet, int kW>
__global__ void __launch_bounds__(32 * bounded_warps(kNet, kW), 1) k_render_ndc(Args a) {
  render_warps<NdcSampler, kC, kPe, kNet, kW, bounded_warps(kNet, kW)>(a);
}

template <class Smp, int kC, int kPe, bool kNet, int kW>
static int launch_bounded(const Args& a, cudaStream_t st) {
  constexpr int kWarps = bounded_warps(kNet, kW);
  constexpr uint32_t smem = Layout<kC, kPe, kNet, kW, kWarps>::smem;
  if constexpr (std::is_same<Smp, BoxSampler>::value) return launch_render<kWarps>(k_render_box<kC, kPe, kNet, kW>, smem, a, st);
  else return launch_render<kWarps>(k_render_ndc<kC, kPe, kNet, kW>, smem, a, st);
}

}  // namespace rnd
}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_render_box(const float* rays_o, const float* rays_d, const float* viewdirs, const float* density_grid,
                   const UbnGridDesc* density_desc, const float* k0_grid, const UbnGridDesc* k0_desc, const uint8_t* mask_world,
                   const UbnBoxMarchCfg* cfg, int64_t n_rays, const float* W1, const float* b1, const float* W2, const float* b2,
                   const float* W3, const float* b3, int width, int viewbase_pe, float bg, float* rgb_marched, float* depth,
                   float* alphainv_last, int32_t* n_shaded, int32_t* n_marched, int32_t* overflow, void* stream) {
  if (n_rays <= 0) return 0;
  rnd::Args a = rnd::render_args(rays_o, rays_d, viewdirs, density_grid, density_desc, k0_grid, k0_desc, mask_world, n_rays, W1, b1,
                                 W2, b2, W3, b3, 1, bg, rgb_marched, depth, alphainv_last, n_shaded, n_marched);
  a.p = make_box_params(cfg, overflow);
  const int C = a.gk.C;
  const bool net = W1 != nullptr;
  if (!rnd::render_args_ok(a) || cfg->s_max < 1) return finish(cudaErrorInvalidValue);
  const cudaStream_t st = as_stream(stream);
  if (net && C == 12 && viewbase_pe == 4 && width == 128) return rnd::launch_bounded<BoxSampler, 12, 4, true, 128>(a, st);
  if (net && C == 9 && viewbase_pe == 4 && width == 64) return rnd::launch_bounded<BoxSampler, 9, 4, true, 64>(a, st);
  if (!net && C == 3) return rnd::launch_bounded<BoxSampler, 3, 0, false, 128>(a, st);
  return finish(cudaErrorInvalidValue);
}

int ubn_render_ndc(const float* rays_o, const float* rays_d, const float* viewdirs, const float* density_grid,
                   const UbnGridDesc* density_desc, const float* act_shift_grid, const UbnGridDesc* act_shift_desc,
                   const float* k0_grid, const UbnGridDesc* k0_desc, const uint8_t* mask_world, const UbnNdcMarchCfg* cfg,
                   int64_t n_rays, const float* W1, const float* b1, const float* W2, const float* b2, const float* W3,
                   const float* b3, int width, int viewbase_pe, float bg, float* rgb_marched, float* depth, float* alphainv_last,
                   int32_t* n_shaded, int32_t* n_marched, void* stream) {
  if (n_rays <= 0) return 0;
  rnd::Args a = rnd::render_args(rays_o, rays_d, viewdirs, density_grid, density_desc, k0_grid, k0_desc, mask_world, n_rays, W1, b1,
                                 W2, b2, W3, b3, 1, bg, rgb_marched, depth, alphainv_last, n_shaded, n_marched);
  if (!act_shift_grid || !act_shift_desc) return finish(cudaErrorInvalidValue);
  a.p = make_ndc_params(cfg, make_view(act_shift_grid, act_shift_desc));
  if (a.p.shift_grid.P != 1 || a.p.shift_grid.C != 1) return finish(cudaErrorInvalidValue);   // one single-channel slab
  const int C = a.gk.C;
  const bool net = W1 != nullptr;
  if (!rnd::render_args_ok(a) || cfg->n_samples < 2) return finish(cudaErrorInvalidValue);
  const cudaStream_t st = as_stream(stream);
  if (net && C == 9 && viewbase_pe == 0 && width == 64) return rnd::launch_bounded<NdcSampler, 9, 0, true, 64>(a, st);
  if (!net && C == 3) return rnd::launch_bounded<NdcSampler, 3, 0, false, 128>(a, st);
  return finish(cudaErrorInvalidValue);
}

}  // extern "C"
