// render_warp.cuh -- the per-warp loop of the fused whole-frame render, shared by the contracted (render.cu), box and NDC
// (render_bounded.cu) kernels.  What differs per geometry is the sampling policy Smp (march_common.cuh: ray set-up, sample point,
// the raw density) and the depth term of a sample (render_depth_term); the rgbnet width is a template parameter.  See render.cu
// for the structure of the loop.
#pragma once
#include <algorithm>
#include <type_traits>

#include "march_common.cuh"
#include "rgbnet_tc.cuh"

namespace ubn {
namespace rnd {

constexpr int kRows = tc::kUnit;       // rows of a staging tile = samples of one mma unit

struct Args {
  const float *rays_o, *rays_d, *viewdirs, *t_table;   // t_table: contracted models only
  GridView gd, gk;                     // density, k0
  const uint8_t* mask_world;
  MarchParams p;
  int64_t n_rays;
  const float *W1, *b1, *W2, *b2, *W3, *b3;   // nn.Linear weights: W1 [W][C + E], W2 [W][W], W3 [3][W]
  int use_bg;
  float bg;
  float *rgb, *depth, *last;
  int32_t *n_shaded, *n_marched;
};

// The term a sample adds to depth with its weight: s = 1 - 1 / (1 + t) as torch evaluates it (dcvgo.py:366), the step index
// (dvgo.py:415: weights * step_id), or (step_id + 0.5) / N_samples in fp32 (dmpigo.py:331)
template <class Smp>
__device__ __forceinline__ float render_depth_term(const Args& a, int s) {
  if constexpr (std::is_same<Smp, BoxSampler>::value) return (float)s;
  else if constexpr (std::is_same<Smp, NdcSampler>::value) return __fdiv_rn(__fadd_rn((float)s, 0.5f), (float)a.p.S);
  else return __fsub_rn(1.f, __frcp_rn(__fadd_rn(1.f, a.t_table[s])));
}

// The raw density Raw2Alpha activates, given the density grid's value d: Smp::density, with NdcSampler's act_shift grid read as
// grid_density_at reads it at its one slab (ubn_render_ndc requires P = 1), so no run-time slab loop (and no sinf / cosf frame)
template <class Smp>
__device__ __forceinline__ float render_density(const MarchParams& p, float d, float x, float y, float z) {
  if constexpr (std::is_same<Smp, NdcSampler>::value) {
    const GridView& g = p.shift_grid;
    SlabMean acc;
    acc.add(0, trilerp1(g.data, g.sv, g.X, g.Y, g.Z, src_index(norm_coord(x, g.mn[0], g.len[0]), g.X),
                        src_index(norm_coord(y, g.mn[1], g.len[1]), g.Y), src_index(norm_coord(z, g.mn[2], g.len[2]), g.Z)));
    return __fadd_rn(d, acc.mean(1));
  } else {
    return Smp::density(p, d, x, y, z);
  }
}

// The density grid's value at (x, y, z) as pass A reads it: grid_density_fast at the slab counts its fast path takes (1 - 9),
// grid_density_at at 11 (pass A's generic read of FourierGridModel at fourier_freq_num 5)
template <int kP>
__device__ __forceinline__ float render_grid_density(const GridView& g, float x, float y, float z) {
  if constexpr (kP <= 9) return grid_density_fast<kP>(g, x, y, z);
  else return grid_density_at(g, x, y, z);
}

// Shared memory of one instance.  With an rgbnet: W2 and W1 as fp32 B fragments, b1, b2, W3; then one block per warp (floats):
// slot rays [16] (int64), feature tile [16][C], rgb [16][4], w [16], s [16], row slot [16], slot sums [16][4], slot
// alphainv_last [16], slot embeddings [16][kEs] (with an rgbnet: the k columns of layer 1 past C, zero past C + E)
template <int kC, int kPe, bool kNet, int kW, int kWarps>
struct Layout {
  static constexpr int kNT = tc::n_tiles(kW);
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

// The body of a render kernel of kWarps warps: kC-channel k0, rgbnet of width kW at viewbase_pe kPe (kNet) or sigmoid(k0).
// kP-slab density and k0 grids (kP > 1: FourierGridModel's Fourier slabs, render_fourier.cu; the k0 read in lane_features' lean
// form, which keeps the kernel at 168 registers without spills).
template <class Smp, int kC, int kPe, bool kNet, int kW, int kWarps, int kP = 1>
__device__ __forceinline__ void render_warps(const Args& a) {
  using L = Layout<kC, kPe, kNet, kW, kWarps>;
  constexpr int kKS = L::kKS, kEs = L::kEs, kNT = L::kNT;
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
      // layer 2 in kParts groups of 4 column tiles (fW2 is n-tile major), each followed by its part of epilogue 2 and layer 3
      constexpr int kNTp = 4, kParts = kNT / kNTp;
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
        } else if constexpr (kPe > 0) {          // at pe 0 the embedding is viewdirs alone
          if (e < L::kE) {
            const int k = (e - 3) % (3 * kPe), d = k / kPe, i = k - d * kPe;
            const float arg = __fmul_rn(vd[d], (float)(1 << i));
            v = (e - 3 < 3 * kPe) ? sinf(arg) : cosf(arg);
          }
        }
        sEmb[cur * kEs + e] = v;
      }
    }
    if (lane < 4) sAcc[4 * cur + lane] = 0.f;
    if (lane == 0) sRay[cur] = ray;
    __syncwarp();

    const Ray r = Smp::load(a.rays_o + 3 * ray, a.rays_d + 3 * ray, p);
    float T_cum = 1.f, cum = 0.f;
    bool done = false, carry_over = false;
    int n_kept = 0, n_marched = 0;
    for (int base = 0; base < r.n && !done; base += 32) {
      n_marched = min(base + 32, r.n);
      const MarchSample ms = march_chunk_point<Smp>(r, a.t_table, a.mask_world, p, base, lane, cum, carry_over);
      float alpha = 0.f;
      if (ms.queried) {
        alpha = march_alpha(render_density<Smp>(p, render_grid_density<kP>(a.gd, ms.x, ms.y, ms.z), ms.x, ms.y, ms.z), p);
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
        lane_features<kC, kP, (kP > 1)>(a.gk, norm_coord(ms.x, a.gk.mn[0], a.gk.len[0]), norm_coord(ms.y, a.gk.mn[1], a.gk.len[1]),
                               norm_coord(ms.z, a.gk.mn[2], a.gk.len[2]), f);
        sv = render_depth_term<Smp>(a, base + lane);
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

// One launch of a render kernel: the dynamic shared memory attribute, and as many CTAs as fit on the device (persistent warps).
// The attribute, the occupancy and the SM count are those of the current device, queried on every call.
template <int kWarps, class K>
static int launch_render(K kernel, uint32_t smem_bytes, const Args& a, cudaStream_t st) {
  const int smem = (int)smem_bytes;
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

// The one-slab grids every render kernel reads: a contiguous density (pass A's fast read: 8-byte aligned, 32-bit offsets) and a
// channels-last k0 (32-bit offsets, float4-aligned records at C = 12)
inline bool render_grids_ok(const GridView& gd, const GridView& gk) {
  const int C = gk.C;
  const bool dens_ok = gd.C == 1 && gd.P == 1 && gd.sv == 1 && gd.X >= 2 && gd.Y >= 2 && gd.Z >= 2 &&
                       (int64_t)gd.X * gd.Y * gd.Z < (1ll << 31) && ((uintptr_t)gd.data & 7) == 0;
  const bool k0_ok = gk.P == 1 && gk.sc == 1 && gk.sv == C && gk.X >= 2 && gk.Y >= 2 && gk.Z >= 2 &&
                     (int64_t)gk.X * gk.Y * gk.Z * C < (1ll << 31) && ((uintptr_t)gk.data & 3) == 0 &&
                     (C != 12 || ((uintptr_t)gk.data & 15) == 0);
  return dens_ok && k0_ok;
}

// The arguments every render entry takes, bar the geometry (p, t_table)
inline Args render_args(const float* rays_o, const float* rays_d, const float* viewdirs, const float* density_grid,
                        const UbnGridDesc* density_desc, const float* k0_grid, const UbnGridDesc* k0_desc, const uint8_t* mask_world,
                        int64_t n_rays, const float* W1, const float* b1, const float* W2, const float* b2, const float* W3,
                        const float* b3, int use_bg, float bg, float* rgb_marched, float* depth, float* alphainv_last,
                        int32_t* n_shaded, int32_t* n_marched) {
  Args a{};
  a.rays_o = rays_o; a.rays_d = rays_d; a.viewdirs = viewdirs;
  a.gd = make_view(density_grid, density_desc);
  a.gk = make_view(k0_grid, k0_desc);
  a.mask_world = mask_world;
  a.n_rays = n_rays;
  a.W1 = W1; a.b1 = b1; a.W2 = W2; a.b2 = b2; a.W3 = W3; a.b3 = b3;
  a.use_bg = use_bg; a.bg = bg;
  a.rgb = rgb_marched; a.depth = depth; a.last = alphainv_last; a.n_shaded = n_shaded; a.n_marched = n_marched;
  return a;
}

// What every render entry requires of its arguments (the widths and (C, pe) pairs are the dispatch's): supported grids, the
// rgbnet complete with its view directions, and the outputs
inline bool render_args_ok(const Args& a) {
  const bool net_ok = !a.W1 || (a.b1 && a.W2 && a.b2 && a.W3 && a.b3 && a.viewdirs);
  return render_grids_ok(a.gd, a.gk) && net_ok && a.rays_o && a.rays_d && a.rgb && a.depth && a.last &&
         (!a.p.use_mask || a.mask_world);
}

}  // namespace rnd
}  // namespace ubn
