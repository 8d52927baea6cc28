// render_tma.cu -- pass B (feature-grid read) of the fused march for COHERENT rays on a single-slab (DenseGrid) feature grid:
// the render path of DirectContractedVoxGO / DirectVoxGO-style models (run_render.py:43-63 renders a frame as 8192-ray chunks of
// image-ordered rays), with the voxel bricks staged in shared memory by TMA.
//
// Why a second kernel: for random training rays a sample needs eight 48-byte records at unrelated addresses and no tile is
// reused (march_feature.cu: warp-cooperative 128-bit gathers).  32 ADJACENT pixels are different: at any step their samples sit
// within a few voxels of each other (pixel footprint t / focal in world units, which the contraction keeps at ~0.1 voxel per
// pixel at every depth), so the 32 rays x 4 steps of a warp's block touch one small brick of the grid.  Here
//   warp = 32 consecutive rays of the chunk (lane = ray), block = 4 consecutive steps;
//   the warp reduces the bounding box of the block's cell bases (min / max over lanes and steps);
//   if the box spans <= 7 cells per axis, ONE cp.async.bulk.tensor (TMA, 4-D box [8 x][8 y][8 z][12 ch] = 24 KB, zero fill
//   outside the grid) brings the brick into the warp's shared-memory buffer, signalled on an mbarrier, and all 128 samples
//   interpolate from shared memory (8 corners x 3 LDS.128);  otherwise (row wrap of the image, grazing geometry) the lanes
//   fall back to direct global loads for that block.
// Parallelism: a chunk of 8192 rays is only 256 ray groups, so the step axis is split too: a warp owns (32 rays) x (a segment of
// 64 steps = 16 blocks); its output cursor starts after the survivors of the earlier segments, counted from the flag bytes
// (16-byte loads, 4 bytes of flags per step block).  First version (one warp per ray group, all 128 blocks): 3x slower than the
// gather kernel on the garden frame, because 64 CTAs per chunk left more than half of the SMs idle.
// The trilinear sum runs in ATen's corner order (tnw .. bse, FMA chain), so the features are bit-identical to the stand-alone
// grid op (trilinear.cu) and to torch F.grid_sample, which the reference calls, at every sample whose unnormalised coordinates
// ((c + 1) / 2) * (size - 1) lie in [0, size - 1] -- every sample of the contracted models, whose points stay inside the k0
// grid's bounds.  A coordinate beyond a face (a k0 grid with narrower bounds than the points) keeps its clamped cell (cell_of,
// as march_feature.cu::make_cell) and extrapolates linearly, where F.grid_sample zero-pads the corners past the face.
// Outputs = those of ubn_march_feature_fwd.
#include <cuda.h>

#include <algorithm>
#include <cstring>

#include "march_common.cuh"

namespace ubn {

namespace rt {
constexpr int kBox = 8;                                  // lattice points per axis in a staged brick
constexpr int kChan = 12;
constexpr int kSteps = 4;                                // steps per block
constexpr int kSegSteps = 64;                            // steps per warp (16 blocks)
constexpr uint32_t kBoxBytes = kBox * kBox * kBox * kChan * 4;   // 24 576
constexpr int kWarps = 4;
constexpr uint32_t kSmemBytes = kWarps * kBoxBytes + kWarps * 8 + 128;   // + mbarriers (+ slack for 128-byte alignment)

__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// 4-D tiled TMA load: coordinates in tensor-map order (innermost first) = {channel, z, y, x}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

struct Cell3 {
  int x0, y0, z0;
  float fx, fy, fz;
};

// same clamping as march_feature.cu::make_cell: base in [0, size - 2], fraction in [0, 1]
__device__ __forceinline__ Cell3 cell_of(float cx, float cy, float cz, int X, int Y, int Z) {
  Cell3 c;
  const float x0 = fminf(fmaxf(floorf(cx), 0.f), (float)(X - 2));
  const float y0 = fminf(fmaxf(floorf(cy), 0.f), (float)(Y - 2));
  const float z0 = fminf(fmaxf(floorf(cz), 0.f), (float)(Z - 2));
  c.fx = cx - x0; c.fy = cy - y0; c.fz = cz - z0;
  c.x0 = (int)x0; c.y0 = (int)y0; c.z0 = (int)z0;
  return c;
}

// corner weight in ATen's product order (wz * wy) * wx with w0 = (f0 + 1) - c  == 1 - frac, w1 = frac
__device__ __forceinline__ float cweight(const Cell3& c, int bx, int by, int bz) {
  return ((bz ? c.fz : 1.f - c.fz) * (by ? c.fy : 1.f - c.fy)) * (bx ? c.fx : 1.f - c.fx);
}

}  // namespace rt

__global__ void __launch_bounds__(32 * rt::kWarps, 2) k_march_feature_tma(
    const __grid_constant__ CUtensorMap tmap, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
    const float* __restrict__ t_table, GridView g, MarchParams p, int64_t n_rays, const uint8_t* __restrict__ flags,
    const int64_t* __restrict__ offsets, const float* __restrict__ density, const float* __restrict__ alpha,
    const float* __restrict__ weight, float* __restrict__ feat, float* __restrict__ o_density, float* __restrict__ o_alpha,
    float* __restrict__ o_weight, int64_t* __restrict__ o_ray_id, int64_t* __restrict__ o_step_id, float* __restrict__ o_t,
    uint8_t* __restrict__ o_inner, unsigned long long* __restrict__ stats) {
  using namespace rt;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float* box = reinterpret_cast<float*>(smem + w * kBoxBytes);
  const uint32_t box_addr = smem_u32(box);
  const uint32_t bar = smem_u32(smem + kWarps * kBoxBytes + w * 8);
  if (lane == 0) mbar_init(bar, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();

  const int S = p.S;
  const int n_seg = (S + kSegSteps - 1) / kSegSteps;
  const int64_t unit = (int64_t)blockIdx.x * kWarps + w;                 // (ray group, step segment)
  const int64_t group = unit / n_seg;
  const int seg = (int)(unit - group * n_seg);
  const int64_t ray = group * 32 + lane;
  const bool ray_ok = ray < n_rays;
  Ray r = {0, 0, 0, 0, 0, 1};
  int64_t cursor = 0;
  const int seg_begin = seg * kSegSteps, seg_end = min(seg_begin + kSegSteps, S);
  if (ray_ok) {
    r = load_ray(rays_o + 3 * ray, rays_d + 3 * ray, p);
    // survivors of this ray in the earlier segments: KEEP is bit 3 of every flag byte
    const uint8_t* fr = flags + ray * S;
    int before = 0;
    if ((S & 15) == 0) {
      for (int i = 0; i < seg_begin; i += 16) {
        const uint4 v = *reinterpret_cast<const uint4*>(fr + i);
        before += __popc(v.x & 0x08080808u) + __popc(v.y & 0x08080808u) + __popc(v.z & 0x08080808u) + __popc(v.w & 0x08080808u);
      }
    } else {
      for (int i = 0; i < seg_begin; ++i) before += (fr[i] & UBN_FLAG_KEEP) ? 1 : 0;
    }
    cursor = offsets[ray] + before;
  }
  uint32_t phase = 0;
  unsigned long long n_tma = 0, n_fallback = 0;

  for (int s0 = seg_begin; s0 < seg_end; s0 += kSteps) {
    // ---- this lane's up-to-4 samples of the block ----
    Cell3 cell[kSteps];
    float tt[kSteps];
    bool keep[kSteps];
    uint8_t fl[kSteps];
    int lo_x = INT_MAX, lo_y = INT_MAX, lo_z = INT_MAX, hi_x = INT_MIN, hi_y = INT_MIN, hi_z = INT_MIN;
#pragma unroll
    for (int j = 0; j < kSteps; ++j) {
      const int s = s0 + j;
      fl[j] = (ray_ok && s < seg_end) ? flags[ray * S + s] : 0;
      keep[j] = (fl[j] & UBN_FLAG_KEEP) != 0;
      tt[j] = 0.f;
      cell[j] = Cell3{0, 0, 0, 0.f, 0.f, 0.f};
      if (keep[j]) {
        float x, y, z;
        tt[j] = t_table[s];
        sample_point(r, tt[j], p, x, y, z);
        cell[j] = cell_of(src_index(norm_coord(x, g.mn[0], g.len[0]), g.X), src_index(norm_coord(y, g.mn[1], g.len[1]), g.Y),
                          src_index(norm_coord(z, g.mn[2], g.len[2]), g.Z), g.X, g.Y, g.Z);
        lo_x = min(lo_x, cell[j].x0); hi_x = max(hi_x, cell[j].x0);
        lo_y = min(lo_y, cell[j].y0); hi_y = max(hi_y, cell[j].y0);
        lo_z = min(lo_z, cell[j].z0); hi_z = max(hi_z, cell[j].z0);
      }
    }
    const bool any_here = keep[0] | keep[1] | keep[2] | keep[3];
    if (!__any_sync(0xffffffffu, any_here)) continue;                   // warp-uniform
    lo_x = __reduce_min_sync(0xffffffffu, lo_x); hi_x = __reduce_max_sync(0xffffffffu, hi_x);
    lo_y = __reduce_min_sync(0xffffffffu, lo_y); hi_y = __reduce_max_sync(0xffffffffu, hi_y);
    lo_z = __reduce_min_sync(0xffffffffu, lo_z); hi_z = __reduce_max_sync(0xffffffffu, hi_z);
    const bool fits = (hi_x - lo_x <= kBox - 2) && (hi_y - lo_y <= kBox - 2) && (hi_z - lo_z <= kBox - 2);   // corner x0 + 1 <= lo + 7
    if (fits) {
      if (lane == 0) {
        mbar_expect_tx(bar, kBoxBytes);
        tma_load_4d(box_addr, &tmap, bar, 0, lo_z, lo_y, lo_x);
        ++n_tma;
      }
      mbar_wait(bar, phase);
      phase ^= 1;
    } else if (lane == 0) {
      ++n_fallback;
    }
#pragma unroll
    for (int j = 0; j < kSteps; ++j) {
      if (!keep[j]) continue;
      const Cell3 c = cell[j];
      float4 a0 = make_float4(0, 0, 0, 0), a1 = a0, a2 = a0;
#pragma unroll
      for (int corner = 0; corner < 8; ++corner) {                       // tnw, tne, tsw, tse, bnw, bne, bsw, bse: z fastest
        const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
        const float wgt = cweight(c, bx, by, bz);
        float4 v0, v1, v2;
        if (fits) {
          const float4* rec = reinterpret_cast<const float4*>(
              box + ((((c.x0 - lo_x + bx) * kBox) + (c.y0 - lo_y + by)) * kBox + (c.z0 - lo_z + bz)) * kChan);
          v0 = rec[0]; v1 = rec[1]; v2 = rec[2];
        } else {
          const float4* rec = reinterpret_cast<const float4*>(
              g.data + ((int64_t)((c.x0 + bx) * g.Y + (c.y0 + by)) * g.Z + (c.z0 + bz)) * kChan);
          v0 = __ldg(rec); v1 = __ldg(rec + 1); v2 = __ldg(rec + 2);
        }
        a0.x = fmaf(v0.x, wgt, a0.x); a0.y = fmaf(v0.y, wgt, a0.y); a0.z = fmaf(v0.z, wgt, a0.z); a0.w = fmaf(v0.w, wgt, a0.w);
        a1.x = fmaf(v1.x, wgt, a1.x); a1.y = fmaf(v1.y, wgt, a1.y); a1.z = fmaf(v1.z, wgt, a1.z); a1.w = fmaf(v1.w, wgt, a1.w);
        a2.x = fmaf(v2.x, wgt, a2.x); a2.y = fmaf(v2.y, wgt, a2.y); a2.z = fmaf(v2.z, wgt, a2.z); a2.w = fmaf(v2.w, wgt, a2.w);
      }
      const int64_t o = cursor++;
      const int64_t i = ray * S + s0 + j;
      float4* fo = reinterpret_cast<float4*>(feat + o * kChan);
      fo[0] = a0; fo[1] = a1; fo[2] = a2;
      o_density[o] = density[i];
      o_alpha[o] = alpha[i];
      o_weight[o] = weight[i];
      o_ray_id[o] = ray;
      o_step_id[o] = s0 + j;
      o_t[o] = tt[j];
      o_inner[o] = (fl[j] & UBN_FLAG_INNER) ? 1 : 0;
    }
    __syncwarp();          // every lane has consumed the brick before the next TMA overwrites it
  }
  if (stats && lane == 0 && (n_tma | n_fallback)) {
    atomicAdd(stats, n_tma);
    atomicAdd(stats + 1, n_fallback);
  }
}

}  // namespace ubn

using namespace ubn;

namespace {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}
}  // namespace

extern "C" int ubn_march_feature_fwd_tma(const float* rays_o, const float* rays_d, const float* t_table, const float* k0_grid,
                                         const UbnGridDesc* k0_desc, const UbnMarchCfg* cfg, int64_t n_rays, const uint8_t* flags,
                                         const int64_t* offsets, const float* density, const float* alpha, const float* weight,
                                         float* feat, float* o_density, float* o_alpha, float* o_weight, int64_t* o_ray_id,
                                         int64_t* o_step_id, float* o_t, uint8_t* o_inner, unsigned long long* stats2, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(k0_grid, k0_desc);
  // single slab, 12 channels, channels-last, 16-byte aligned, at least 2 lattice points per axis
  if (g.P != 1 || g.C != rt::kChan || g.sc != 1 || g.sv != g.C || ((uintptr_t)k0_grid & 15) || g.X < 2 || g.Y < 2 || g.Z < 2)
    return finish(cudaErrorInvalidValue);
  EncodeTiledFn enc = encode_tiled();
  if (!enc) return finish(cudaErrorNotSupported);
  CUtensorMap tmap;
  const cuuint64_t dims[4] = {(cuuint64_t)g.C, (cuuint64_t)g.Z, (cuuint64_t)g.Y, (cuuint64_t)g.X};          // innermost first
  const cuuint64_t strides[3] = {(cuuint64_t)g.C * 4, (cuuint64_t)g.Z * g.C * 4, (cuuint64_t)g.Y * g.Z * g.C * 4};
  const cuuint32_t box[4] = {(cuuint32_t)rt::kChan, rt::kBox, rt::kBox, rt::kBox};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult cr = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(k0_grid), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_params(cfg);
  cudaError_t e = cudaFuncSetAttribute(k_march_feature_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rt::kSmemBytes);
  if (e != cudaSuccess) return finish(e);
  const int64_t n_seg = (p.S + rt::kSegSteps - 1) / rt::kSegSteps;
  const int64_t units = ((n_rays + 31) / 32) * n_seg;                    // (ray group, step segment) pairs, one warp each
  k_march_feature_tma<<<blocks_for(units, rt::kWarps), 32 * rt::kWarps, rt::kSmemBytes, as_stream(stream)>>>(
      tmap, rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat, o_density, o_alpha, o_weight,
      o_ray_id, o_step_id, o_t, o_inner, stats2);
  UBN_LAUNCH_CHECK();
  return 0;
}
