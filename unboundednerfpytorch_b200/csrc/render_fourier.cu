// render_fourier.cu -- whole-frame render of FourierGridModel with Fourier slabs (P = 7, 9, 11 density and k0 slabs, 12-channel
// k0, the reference's (12, 4) width-128 rgbnet) in one fused pass, sm_90a.
//
// The kernel is render.cu's: render_warp.cuh's per-warp loop (march, early stop, k0 read of the kept samples, the rgbnet on the
// tensor cores in 16-row tiles that span rays, step-order composite by each ray's slot lane), one CTA of 12 warps per SM, here
// instantiated on the slab count.  The density is read as pass A reads it (grid_density_fast at 7 and 9 slabs, grid_density_at
// at 11), so alphainv_last and the kept samples are forward's bit for bit; the k0 read is lane_features' lean form (the slab loop
// rolled, four corner records in flight: the same arithmetic), which keeps the 168-register kernel free of spills.
//
// Why 12 warps that both march and shade, and not march warps feeding a tensor-core consumer warpgroup: such a kernel (8 march
// warps at 152 registers via setmaxnreg, one wgmma consumer warpgroup, sub-tiles handed over through mbarriers) was built and
// timed against this one in one process on the truck and 7-slab frames (DESIGN.md §7).  Its single consumer bounded it on dense
// frames (1176 ms against 919 ms for this kernel on the dense truck frame; 568 ms with the consumer's rgbnet stubbed out), and it
// was no faster on the opaque ones.
#include "render_warp.cuh"

namespace ubn {
namespace rfo {

constexpr int kC = 12, kPe = 4, kW = 128;
constexpr int kWarps = 12;             // as k_render_contracted: 168 registers, one CTA per SM

template <int kP>
__global__ void __launch_bounds__(32 * kWarps, 1) k_render_fourier(rnd::Args a) {
  rnd::render_warps<ContractedSampler, kC, kPe, true, kW, kWarps, kP>(a);
}

template <int kP>
static int launch(const rnd::Args& a, cudaStream_t st) {
  return rnd::launch_render<kWarps>(k_render_fourier<kP>, rnd::Layout<kC, kPe, true, kW, kWarps>::smem, a, st);
}

// density: contiguous single-channel grid of P slabs (8-byte aligned, 32-bit offsets inside a slab: pass A's fast read); k0: the
// same slab count, 12 channels channels-last, float4-aligned records in every slab (32-bit voxel offsets)
static bool grids_ok(const GridView& gd, const GridView& gk) {
  const bool dens_ok = gd.C == 1 && gd.sv == 1 && gd.X >= 2 && gd.Y >= 2 && gd.Z >= 2 &&
                       (int64_t)gd.X * gd.Y * gd.Z < (1ll << 31) && ((uintptr_t)gd.data & 7) == 0;
  const bool k0_ok = gk.P == gd.P && gk.C == kC && gk.sc == 1 && gk.sv == kC && gk.X >= 2 && gk.Y >= 2 && gk.Z >= 2 &&
                     (int64_t)gk.X * gk.Y * gk.Z * kC < (1ll << 31) && ((uintptr_t)gk.data & 15) == 0 && gk.sp % 4 == 0;
  return dens_ok && k0_ok;
}

}  // namespace rfo
}  // namespace ubn

using namespace ubn;

extern "C" int ubn_render_fourier(const float* rays_o, const float* rays_d, const float* viewdirs, const float* t_table,
                                  const float* density_grid, const UbnGridDesc* density_desc, const float* k0_grid,
                                  const UbnGridDesc* k0_desc, const uint8_t* mask_world, const UbnMarchCfg* cfg, int64_t n_rays,
                                  const float* W1, const float* b1, const float* W2, const float* b2, const float* W3,
                                  const float* b3, int width, int viewbase_pe, int use_bg, float bg, float* rgb_marched,
                                  float* depth, float* alphainv_last, int32_t* n_shaded, int32_t* n_marched, void* stream) {
  if (!density_desc || !k0_desc || !cfg) return finish(cudaErrorInvalidValue);
  if (n_rays <= 0) return 0;
  rnd::Args a = rnd::render_args(rays_o, rays_d, viewdirs, density_grid, density_desc, k0_grid, k0_desc, mask_world, n_rays, W1, b1,
                                 W2, b2, W3, b3, use_bg, bg, rgb_marched, depth, alphainv_last, n_shaded, n_marched);
  a.t_table = t_table;
  a.p = make_params(cfg);
  const bool args_ok = rays_o && rays_d && viewdirs && t_table && W1 && b1 && W2 && b2 && W3 && b3 && rgb_marched && depth &&
                       alphainv_last && (!a.p.use_mask || mask_world);
  if (!args_ok || width != rfo::kW || viewbase_pe != rfo::kPe || !rfo::grids_ok(a.gd, a.gk)) return finish(cudaErrorInvalidValue);
  const cudaStream_t st = as_stream(stream);
  switch (a.gd.P) {
    case 7: return rfo::launch<7>(a, st);
    case 9: return rfo::launch<9>(a, st);
    case 11: return rfo::launch<11>(a, st);
    default: return finish(cudaErrorInvalidValue);
  }
}
