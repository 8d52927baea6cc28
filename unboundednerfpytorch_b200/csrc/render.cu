// render.cu -- whole-frame render of the contracted models (FourierGridModel, DirectContractedVoxGO) in one fused pass, sm_90a.
//
// One-slab density and k0 grids only: DirectContractedVoxGO, and FourierGridModel at fourier_freq_num 0.  With Fourier slabs
// (the reference's FourierGridModel configs: 7 - 11 slabs) a 9-slab instance of this kernel rendered an opaque frame 8x faster than
// the chunk loop but a dense one 0.79x as fast (its slab reads are latency-bound at 12 warps per SM).  Those models render through
// render_fourier.cu's slab instances of this loop when the caller opts in (render_kwargs['fused_slabs']), else through the chunk loop.
//
// Rendering needs three numbers per ray: rgb_marched, depth and alphainv_last.  The training path (march.cu + march_feature.cu +
// shade_tc.cu + composite) writes dense per-sample records, compacts the survivors, reads their features, runs the rgbnet and
// composites, with every intermediate in HBM.  Here one warp walks its rays one after another and nothing per sample leaves the SM:
//   * march: march_common.cuh's march_chunk_point / march_alpha / transmittance_scan, the arithmetic of pass A, chunk by chunk; the
//     warp leaves the ray when T < 1e-3 (after the stop no sample gets a weight, so alphainv_last is final there and the stop is exact);
//   * kept samples (listed, scanned, and weight > fast_color_thres when the threshold is on) read their k0 features with
//     lane_features, pass B's lane-per-sample read, so the features are bit-identical to what pass B hands the rgbnet;
//   * a kept sample becomes one row of the warp's 16-row staging tile in shared memory (feature, weight, s and the slot of its
//     ray).  A tile spans as many rays as it takes to fill; when it is full (or the warp has no rays left) one 16-sample unit runs:
//     the 3-layer rgbnet on the tensor cores with rgbnet_tc.cuh's 3xTF32 warp GEMM and epilogues, or sigmoid(k0) without an rgbnet;
//   * the view embedding cat[v, sin(v 2^i), cos(v 2^i)] is computed once per ray into a per-warp ring of 16 slots (a tile
//     references at most 16 rays) and enters layer 1 as further k columns of the row, next to its features: layer 1 runs
//     ceil((C + E) / 8) k-steps (5 at C = 12 / pe 4, 7 at C = 3 / pe 8) instead of ceil(C / 8) plus a per-ray [W]-wide view bias.
//     That costs about 14 % more layer-1+2 MMA work than a per-ray bias, and saves the bias ring (8 KB per warp) and the W1 view
//     half (26 KB per CTA) of shared memory; with layer 2 evaluated in four groups of 4 column tiles (16 live accumulators instead
//     of 64) the kernel fits 168 registers, so one CTA of 12 warps runs per SM instead of 8 (§7 of DESIGN.md: the dense garden frame
//     went from parity with the chunk loop to 1.15x faster);
//   * composite: every slot's w . rgb and w . s (s = 1 - 1 / (1 + t), as torch evaluates it) are added in step order by the slot's
//     own lane, so a ray's sums do not depend on which tiles its rows fell into; DirectContractedVoxGO adds alphainv_last . bg.
// Every output element is written once by one lane: no atomics, run-to-run deterministic, and independent of how the rays are
// batched (mma rows are independent).
//
// The loop itself is render_warp.cuh's render_warps, which the box and NDC kernels (render_bounded.cu) share.
#include "render_warp.cuh"

namespace ubn {
namespace rnd {

constexpr int kWarps = 12;             // one CTA of 12 warps per SM (168 registers; 16 warps at 128 spill and measured the same speedup)
constexpr int kW = 128;                // rgbnet width

// kPe: viewbase_pe of the rgbnet.  One-slab density and k0 grids (DirectContractedVoxGO; FourierGridModel at fourier_freq_num 0).
template <int kC, int kPe, bool kNet>
__global__ void __launch_bounds__(32 * kWarps, 1) k_render_contracted(Args a) {
  render_warps<ContractedSampler, kC, kPe, kNet, kW, kWarps>(a);
}

template <int kC, int kPe, bool kNet>
static int launch(const Args& a, cudaStream_t st) {
  return launch_render<kWarps>(k_render_contracted<kC, kPe, kNet>, Layout<kC, kPe, kNet, kW, kWarps>::smem, a, st);
}

}  // namespace rnd
}  // namespace ubn

using namespace ubn;

extern "C" int ubn_render_contracted(const float* rays_o, const float* rays_d, const float* viewdirs, const float* t_table,
                                     const float* density_grid, const UbnGridDesc* density_desc, const float* k0_grid,
                                     const UbnGridDesc* k0_desc, const uint8_t* mask_world, const UbnMarchCfg* cfg, int64_t n_rays,
                                     const float* W1, const float* b1, const float* W2, const float* b2, const float* W3,
                                     const float* b3, int width, int viewbase_pe, int use_bg, float bg, float* rgb_marched,
                                     float* depth, float* alphainv_last, int32_t* n_shaded, int32_t* n_marched, void* stream) {
  if (n_rays <= 0) return 0;
  rnd::Args a = rnd::render_args(rays_o, rays_d, viewdirs, density_grid, density_desc, k0_grid, k0_desc, mask_world, n_rays, W1, b1,
                                 W2, b2, W3, b3, use_bg, bg, rgb_marched, depth, alphainv_last, n_shaded, n_marched);
  a.t_table = t_table;
  a.p = make_params(cfg);
  const int C = a.gk.C;
  const bool net = W1 != nullptr;
  if (!rnd::render_args_ok(a) || (net && width != rnd::kW) || !t_table) return finish(cudaErrorInvalidValue);
  const cudaStream_t st = as_stream(stream);
  if (net && C == 12 && viewbase_pe == 4) return rnd::launch<12, 4, true>(a, st);
  if (net && C == 3 && viewbase_pe == 8) return rnd::launch<3, 8, true>(a, st);
  if (!net && C == 3) return rnd::launch<3, 0, false>(a, st);
  return finish(cudaErrorInvalidValue);
}
