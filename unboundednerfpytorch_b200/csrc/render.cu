// render.cu -- whole-frame render of the contracted models (FourierGridModel, DirectContractedVoxGO) in one fused pass, sm_90a.
//
// One-slab density and k0 grids only: DirectContractedVoxGO, and FourierGridModel at fourier_freq_num 0.  With Fourier slabs
// (the reference's FourierGridModel configs: 7 - 11 slabs) a 9-slab instance of this kernel rendered an opaque frame 8x faster than
// the chunk loop but a dense one 0.79x as fast (its slab reads are latency-bound at 12 warps per SM), and nothing observable before
// the render tells the two apart, so those models keep the chunk loop.
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
#include <algorithm>

#include "march_common.cuh"
#include "rgbnet_tc.cuh"

namespace ubn {
namespace rnd {

constexpr int kWarps = 12;             // one CTA of 12 warps per SM (168 registers; 16 warps at 128 spill and measured the same speedup)
constexpr int kRows = tc::kUnit;       // rows of a staging tile = samples of one mma unit
constexpr int kW = 128;                // rgbnet width
constexpr int kNT = tc::n_tiles(kW);

struct Args {
  const float *rays_o, *rays_d, *viewdirs, *t_table;
  GridView gd, gk;                     // density, k0
  const uint8_t* mask_world;
  MarchParams p;
  int64_t n_rays;
  const float *W1, *b1, *W2, *b2, *W3, *b3;   // nn.Linear weights: W1 [kW][C + E], W2 [kW][kW], W3 [3][kW]
  int use_bg;
  float bg;
  float *rgb, *depth, *last;
  int32_t *n_shaded, *n_marched;
};

// Shared memory of one instance.  With an rgbnet: W2 and W1 as fp32 B fragments, b1, b2, W3; then one block per warp (floats):
// slot rays [16] (int64), feature tile [16][C], rgb [16][4], w [16], s [16], row slot [16], slot sums [16][4], slot
// alphainv_last [16], slot embeddings [16][kEs] (with an rgbnet: the k columns of layer 1 past C, zero past C + E)
template <int kC, int kPe, bool kNet>
struct Layout {
  static constexpr int kE = kNet ? 3 + 6 * kPe : 0;
  static constexpr int kKS = kNet ? (kC + kE + 7) / 8 : 0;         // layer-1 k-steps
  static constexpr int kEs = kNet ? 8 * kKS - kC : 0;
  static constexpr uint32_t oW1 = kNet ? kNT * kNT * 32 * 8 : 0;
  static constexpr uint32_t oB1 = oW1 + kNT * kKS * 32 * 8;
  static constexpr uint32_t oB2 = oB1 + (kNet ? kW * 4 : 0);
  static constexpr uint32_t oW3 = oB2 + (kNet ? kW * 4 : 0);
  static constexpr uint32_t oWarp = oW3 + (kNet ? 3 * kW * 4 : 0);
  static constexpr int kRayF = 0, kTileF = kRayF + 2 * kRows, kRgbF = kTileF + kRows * kC, kWF = kRgbF + kRows * 4,
                       kSF = kWF + kRows, kSlotF = kSF + kRows, kAccF = kSlotF + kRows, kLastF = kAccF + kRows * 4,
                       kEmbF = kLastF + kRows, kWarpF = (kEmbF + kRows * kEs + 3) / 4 * 4;
  static constexpr uint32_t smem = oWarp + kWarps * kWarpF * 4;
};

// kPe: viewbase_pe of the rgbnet.  One-slab density and k0 grids (DirectContractedVoxGO; FourierGridModel at fourier_freq_num 0).
template <int kC, int kPe, bool kNet>
__global__ void __launch_bounds__(32 * kWarps, 1) k_render_contracted(Args a) {
  using L = Layout<kC, kPe, kNet>;
  constexpr int kKS = L::kKS, kEs = L::kEs;
  extern __shared__ __align__(16) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const MarchParams& p = a.p;
  const uint2* fW2 = reinterpret_cast<const uint2*>(smem);
  const uint2* fW1 = reinterpret_cast<const uint2*>(smem + L::oW1);
  float* sB1 = reinterpret_cast<float*>(smem + L::oB1);
  float* sB2 = reinterpret_cast<float*>(smem + L::oB2);
  float* sW3 = reinterpret_cast<float*>(smem + L::oW3);
  float* wb = reinterpret_cast<float*>(smem + L::oWarp) + warp * L::kWarpF;
  int64_t* sRay = reinterpret_cast<int64_t*>(wb + L::kRayF);
  float* tF = wb + L::kTileF;
  float* tRgb = wb + L::kRgbF;
  float* tW = wb + L::kWF;
  float* tS = wb + L::kSF;
  int* tSlot = reinterpret_cast<int*>(wb + L::kSlotF);
  float* sAcc = wb + L::kAccF;
  float* sLast = wb + L::kLastF;
  float* sEmb = wb + L::kEmbF;
  if constexpr (kNet) {
    constexpr int ld = kC + L::kE;
    tc::stage_frags_f32(a.W2, kW, kW, kW, kNT, kNT, reinterpret_cast<uint2*>(smem), tid, 32 * kWarps, true);
    tc::stage_frags_f32(a.W1, ld, ld, kW, kKS, kNT, reinterpret_cast<uint2*>(smem + L::oW1), tid, 32 * kWarps, true);
    for (int i = tid; i < kW; i += 32 * kWarps) { sB1[i] = a.b1[i]; sB2[i] = a.b2[i]; }
    for (int i = tid; i < 3 * kW; i += 32 * kWarps) sW3[i] = a.W3[i];
  }
  for (int i = lane; i < L::kWarpF - L::kTileF; i += 32) wb[L::kTileF + i] = 0.f;   // no stale NaN reaches a live row
  __syncthreads();
  float b3v[3] = {0.f, 0.f, 0.f};
  if constexpr (kNet) b3v[0] = __ldg(a.b3), b3v[1] = __ldg(a.b3 + 1), b3v[2] = __ldg(a.b3 + 2);

  // ---- one 16-row unit: rgb of rows [0, fill) into tRgb ----
  auto shade_tile = [&](int fill) {
    if constexpr (kNet) {
      const int g = lane >> 2, t = lane & 3;
      const int slot[2] = {g < fill ? tSlot[g] : 0, g + 8 < fill ? tSlot[g + 8] : 0};
      // layer 1's A operand: column k of row r is feature k (k < C), else embedding column k - C of the row's ray
      float x[kKS][4];
#pragma unroll
      for (int s = 0; s < kKS; ++s)
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int row = g + 8 * r, col = 8 * s + 2 * t + e;
            x[s][2 * r + e] = col < kC ? tF[row * kC + col] : sEmb[slot[r] * kEs + col - kC];
          }
      float h[kNT][4];
#pragma unroll
      for (int j = 0; j < kNT; ++j) h[j][0] = h[j][1] = h[j][2] = h[j][3] = 0.f;
      tc::warp_gemm_f<kKS, kNT, true>(h, x, fW1, lane);
      tc::epi_bias_relu<kNT>(
          h, t, [&](int, int c) { return *reinterpret_cast<const float2*>(sB1 + c); }, [](int, int, float, float) {});
      // layer 2 in kParts groups of column tiles (fW2 is n-tile major), each followed by its part of epilogue 2 and layer 3
      constexpr int kParts = 4, kNTp = kNT / kParts;
      float q[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll 1
      for (int part = 0; part < kParts; ++part) {               // rolled: the split h is not kept across the parts
        float z[kNTp][4];
#pragma unroll
        for (int j = 0; j < kNTp; ++j) z[j][0] = z[j][1] = z[j][2] = z[j][3] = 0.f;
        tc::warp_gemm_f<kNT, kNTp, true>(z, h, fW2 + part * kNTp * kNT * 32, lane);
        tc::epi_hidden_layer3<kW, kNTp>(z, part * kNTp, t, sB2, sW3, q, [](int, int, float, float) {});
      }
      tc::epi_rgb(q, b3v, t, [&](int r, const float (&v)[3]) {
        if (g + 8 * r < fill) {
#pragma unroll
          for (int i = 0; i < 3; ++i) tRgb[(g + 8 * r) * 4 + i] = v[i];
        }
      });
    } else {
      for (int i = lane; i < fill * 3; i += 32) {
        const int row = i / 3, c = i - 3 * row;
        tRgb[row * 4 + c] = 1.f / (1.f + expf(-tF[row * kC + c]));
      }
    }
    __syncwarp();
  };

  // ---- a finished ray's outputs from its slot (lane = slot) ----
  auto emit = [&](int j) {
    const int64_t ray = sRay[j];
    const float T = sLast[j];
    float c[3] = {sAcc[4 * j], sAcc[4 * j + 1], sAcc[4 * j + 2]};
    if (a.use_bg) {
#pragma unroll
      for (int i = 0; i < 3; ++i) c[i] = __fadd_rn(c[i], __fmul_rn(T, a.bg));
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) a.rgb[3 * ray + i] = c[i];
    a.depth[ray] = sAcc[4 * j + 3];
    a.last[ray] = T;
  };

  int fill = 0;          // rows in the tile (warp-uniform)
  int nslot = 0;         // slots [0, nslot) are referenced by rows of the tile
  int cur = 0;           // slot of the ray being marched
  bool cur_rows = false; // that ray has rows in the tile

  // shade the tile, add every row into its slot in step order, emit the slots of finished rays; `marching`: the ray in slot cur
  // goes on, so its slot moves to 0 and stays open
  auto flush = [&](bool marching) {
    shade_tile(fill);
    if (lane < nslot) {
      float acc[4] = {sAcc[4 * lane], sAcc[4 * lane + 1], sAcc[4 * lane + 2], sAcc[4 * lane + 3]};
      for (int i = 0; i < fill; ++i) {
        if (tSlot[i] != lane) continue;
        const float w = tW[i];
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(w, tRgb[i * 4 + c]));
        acc[3] = __fadd_rn(acc[3], __fmul_rn(w, tS[i]));
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) sAcc[4 * lane + c] = acc[c];
      if (!(marching && lane == cur)) emit(lane);
    }
    __syncwarp();
    if (marching && cur != 0) {
      if constexpr (kNet)
        for (int i = lane; i < kEs; i += 32) sEmb[i] = sEmb[cur * kEs + i];
      if (lane < 4) sAcc[lane] = sAcc[4 * cur + lane];
      if (lane == 0) sRay[0] = sRay[cur];
      __syncwarp();
    }
    fill = 0;
    nslot = 0;
    cur = 0;
    cur_rows = false;
  };

  const int64_t n_warps = (int64_t)gridDim.x * kWarps;
  for (int64_t ray = (int64_t)blockIdx.x * kWarps + warp; ray < a.n_rays; ray += n_warps) {
    cur = nslot;
    cur_rows = false;
    if constexpr (kNet) {
      // _view_embed's column order: v, sin(v_d 2^i) at 3 + d pe + i, cos(v_d 2^i) at 3 + 3 pe + d pe + i; zero past E
      const float* vd = a.viewdirs + 3 * ray;
      for (int e = lane; e < kEs; e += 32) {
        float v = 0.f;
        if (e < 3) {
          v = vd[e];
        } else if (e < L::kE) {
          const int k = (e - 3) % (3 * kPe), d = k / kPe, i = k - d * kPe;
          const float arg = __fmul_rn(vd[d], (float)(1 << i));
          v = (e - 3 < 3 * kPe) ? sinf(arg) : cosf(arg);
        }
        sEmb[cur * kEs + e] = v;
      }
    }
    if (lane < 4) sAcc[4 * cur + lane] = 0.f;
    if (lane == 0) sRay[cur] = ray;
    __syncwarp();

    const Ray r = load_ray(a.rays_o + 3 * ray, a.rays_d + 3 * ray, p);
    float T_cum = 1.f, cum = 0.f;
    bool done = false, carry_over = false;
    int n_kept = 0, n_marched = 0;
    for (int base = 0; base < r.n && !done; base += 32) {
      n_marched = min(base + 32, r.n);
      const MarchSample ms = march_chunk_point<ContractedSampler>(r, a.t_table, a.mask_world, p, base, lane, cum, carry_over);
      float alpha = 0.f;
      if (ms.queried) {
        alpha = march_alpha(grid_density_fast<1>(a.gd, ms.x, ms.y, ms.z), p);
      }
      const bool listed = march_listed(ms.queried, alpha, p);
      float myT, myW;
      bool scanned;
      transmittance_scan(listed, alpha, lane, T_cum, done, myT, myW, scanned);
      // pass A's keep, without the zero-weight samples a threshold of 0 lists after the stop
      const bool keep = listed && scanned && (p.thres > 0.f ? (myW > p.thres) : true);
      const unsigned km = __ballot_sync(0xffffffffu, keep);
      if (km == 0) continue;
      const int nk = __popc(km), rank = __popc(km & ((1u << lane) - 1));
      n_kept += nk;
      float f[kC];
      float sv = 0.f;
      if (keep) {
        lane_features<kC, 1>(a.gk, norm_coord(ms.x, a.gk.mn[0], a.gk.len[0]), norm_coord(ms.y, a.gk.mn[1], a.gk.len[1]),
                               norm_coord(ms.z, a.gk.mn[2], a.gk.len[2]), f);
        sv = __fsub_rn(1.f, __frcp_rn(__fadd_rn(1.f, a.t_table[base + lane])));   // torch: 1 - 1 / (1 + t)
      }
      for (int put = 0; put < nk;) {
        const int take = min(kRows - fill, nk - put);
        if (!cur_rows) {
          cur_rows = true;
          nslot = cur + 1;
        }
        if (keep && rank >= put && rank < put + take) {
          const int row = fill + rank - put;
#pragma unroll
          for (int c = 0; c < kC; ++c) tF[row * kC + c] = f[c];
          tW[row] = myW;
          tS[row] = sv;
          tSlot[row] = cur;
        }
        __syncwarp();
        fill += take;
        put += take;
        if (fill == kRows) flush(true);
      }
    }
    if (lane == 0) {
      sLast[cur] = T_cum;
      if (a.n_shaded) a.n_shaded[ray] = n_kept;
      if (a.n_marched) a.n_marched[ray] = n_marched;
    }
    __syncwarp();
    if (!cur_rows) {                       // nothing of this ray waits in the tile: its sums are final
      if (lane == cur) emit(cur);
      __syncwarp();
    }
  }
  if (fill > 0 || nslot > 0) flush(false);
}

template <int kC, int kPe, bool kNet>
static int launch(const Args& a, cudaStream_t st) {
  const auto kernel = k_render_contracted<kC, kPe, kNet>;
  const int smem = (int)Layout<kC, kPe, kNet>::smem;
  // the attribute, the occupancy and the SM count are those of the current device, queried on every call
  int dev = 0, sms = 0, per_sm = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 32 * kWarps, smem);
  if (e != cudaSuccess) return finish(e);
  const int64_t want = (a.n_rays + kWarps - 1) / kWarps;
  const unsigned blocks = (unsigned)std::min<int64_t>(want, (int64_t)std::max(per_sm, 1) * sms);
  kernel<<<blocks, 32 * kWarps, smem, st>>>(a);
  UBN_LAUNCH_CHECK();
  return 0;
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
  rnd::Args a{};
  a.rays_o = rays_o; a.rays_d = rays_d; a.viewdirs = viewdirs; a.t_table = t_table;
  a.gd = make_view(density_grid, density_desc);
  a.gk = make_view(k0_grid, k0_desc);
  a.mask_world = mask_world;
  a.p = make_params(cfg);
  a.n_rays = n_rays;
  a.W1 = W1; a.b1 = b1; a.W2 = W2; a.b2 = b2; a.W3 = W3; a.b3 = b3;
  a.use_bg = use_bg; a.bg = bg;
  a.rgb = rgb_marched; a.depth = depth; a.last = alphainv_last; a.n_shaded = n_shaded; a.n_marched = n_marched;
  const GridView& gd = a.gd;
  const GridView& gk = a.gk;
  const int C = gk.C;
  const bool net = W1 != nullptr;
  // one-slab grids: a contiguous density (pass A's fast read: 8-byte aligned, 32-bit offsets) and a channels-last k0 (32-bit offsets,
  // float4-aligned records at C = 12)
  const bool dens_ok = gd.C == 1 && gd.P == 1 && gd.sv == 1 && gd.X >= 2 && gd.Y >= 2 && gd.Z >= 2 &&
                       (int64_t)gd.X * gd.Y * gd.Z < (1ll << 31) && ((uintptr_t)gd.data & 7) == 0;
  const bool k0_ok = gk.P == 1 && gk.sc == 1 && gk.sv == C && gk.X >= 2 && gk.Y >= 2 && gk.Z >= 2 &&
                     (int64_t)gk.X * gk.Y * gk.Z * C < (1ll << 31) && ((uintptr_t)gk.data & 3) == 0 &&
                     (C != 12 || ((uintptr_t)gk.data & 15) == 0);
  const bool net_ok = !net || (width == rnd::kW && b1 && W2 && b2 && W3 && b3 && viewdirs);
  if (!dens_ok || !k0_ok || !net_ok || !rays_o || !rays_d || !t_table || !rgb_marched || !depth || !alphainv_last ||
      (a.p.use_mask && !mask_world))
    return finish(cudaErrorInvalidValue);
  const cudaStream_t st = as_stream(stream);
  if (net && C == 12 && viewbase_pe == 4) return rnd::launch<12, 4, true>(a, st);
  if (net && C == 3 && viewbase_pe == 8) return rnd::launch<3, 8, true>(a, st);
  if (!net && C == 3) return rnd::launch<3, 0, false>(a, st);
  return finish(cudaErrorInvalidValue);
}
