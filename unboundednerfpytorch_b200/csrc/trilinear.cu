// trilinear.cu -- stand-alone voxel-grid read (DenseGrid.forward / FourierGrid.forward) and its adjoint.
//
// Replaces the torch F.grid_sample call of grid.py:57 and FourierGrid_grid.py:71,74 (ATen
// grid_sampler_3d forward / backward wrt the grid) with kernels that understand a channels-last voxel
// layout: a warp fetches the 8 corner records of one point with ONE 128-bit load instruction
// (lane = corner x channel-quad), instead of 8*C scattered 4-byte loads on C separate planes.
#include <algorithm>

#include "trilinear.cuh"

namespace ubn {

// ------------------------------------------------------------------------------------------------
// path 1: C == 1 (density grids), one lane per point, any layout
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_grid_fwd_c1(GridView g, const float* __restrict__ xyz, int64_t n_pts,
                                                     float* __restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pts) return;
  const float nx = norm_coord(xyz[3 * p], g.mn[0], g.len[0]);
  const float ny = norm_coord(xyz[3 * p + 1], g.mn[1], g.len[1]);
  const float nz = norm_coord(xyz[3 * p + 2], g.mn[2], g.len[2]);
  SlabMean acc;
  for (int s = 0; s < g.P; ++s) {
    const float cx = src_index_guarded(fourier_gamma(s, nx), g.X);
    const float cy = src_index_guarded(fourier_gamma(s, ny), g.Y);
    const float cz = src_index_guarded(fourier_gamma(s, nz), g.Z);
    acc.add(s, trilerp1(g.data + s * g.sp, g.sv, g.X, g.Y, g.Z, cx, cy, cz));
  }
  out[p] = acc.mean(g.P);
}

__global__ void __launch_bounds__(256) k_grid_bwd_c1(GridView g, const float* __restrict__ xyz, int64_t n_pts,
                                                     const float* __restrict__ grad_out, float* __restrict__ grad_grid) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pts) return;
  float go = grad_out[p];
  if (go == 0.f) return;
  go = slab_mean_scale(go, g.P);   // d mean / d slab
  const float nx = norm_coord(xyz[3 * p], g.mn[0], g.len[0]);
  const float ny = norm_coord(xyz[3 * p + 1], g.mn[1], g.len[1]);
  const float nz = norm_coord(xyz[3 * p + 2], g.mn[2], g.len[2]);
  for (int s = 0; s < g.P; ++s) {
    const float cx = src_index_guarded(fourier_gamma(s, nx), g.X);
    const float cy = src_index_guarded(fourier_gamma(s, ny), g.Y);
    const float cz = src_index_guarded(fourier_gamma(s, nz), g.Z);
    trilerp1_scatter(grad_grid + s * g.sp, g.sv, g.X, g.Y, g.Z, cx, cy, cz, go);
  }
}

// ------------------------------------------------------------------------------------------------
// path 2: generic C, any layout, one lane per point (coarse-stage C=3 grids, reference-layout tensors)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_grid_fwd_generic(GridView g, const float* __restrict__ xyz, int64_t n_pts,
                                                          float* __restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pts) return;
  const float nx = norm_coord(xyz[3 * p], g.mn[0], g.len[0]);
  const float ny = norm_coord(xyz[3 * p + 1], g.mn[1], g.len[1]);
  const float nz = norm_coord(xyz[3 * p + 2], g.mn[2], g.len[2]);
  for (int c = 0; c < g.C; ++c) {
    SlabMean acc;
    for (int s = 0; s < g.P; ++s) {
      const float cx = src_index_guarded(fourier_gamma(s, nx), g.X);
      const float cy = src_index_guarded(fourier_gamma(s, ny), g.Y);
      const float cz = src_index_guarded(fourier_gamma(s, nz), g.Z);
      acc.add(s, trilerp1(g.data + s * g.sp + c * g.sc, g.sv, g.X, g.Y, g.Z, cx, cy, cz));
    }
    out[p * g.C + c] = acc.mean(g.P);
  }
}

__global__ void __launch_bounds__(256) k_grid_bwd_generic(GridView g, const float* __restrict__ xyz, int64_t n_pts,
                                                          const float* __restrict__ grad_out,
                                                          float* __restrict__ grad_grid) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pts) return;
  const float nx = norm_coord(xyz[3 * p], g.mn[0], g.len[0]);
  const float ny = norm_coord(xyz[3 * p + 1], g.mn[1], g.len[1]);
  const float nz = norm_coord(xyz[3 * p + 2], g.mn[2], g.len[2]);
  for (int s = 0; s < g.P; ++s) {
    const float cx = src_index_guarded(fourier_gamma(s, nx), g.X);
    const float cy = src_index_guarded(fourier_gamma(s, ny), g.Y);
    const float cz = src_index_guarded(fourier_gamma(s, nz), g.Z);
    for (int c = 0; c < g.C; ++c) {
      float go = grad_out[p * g.C + c];
      go = slab_mean_scale(go, g.P);
      trilerp1_scatter(grad_grid + s * g.sp + c * g.sc, g.sv, g.X, g.Y, g.Z, cx, cy, cz, go);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// path 3: channels-last, C in {4,8,12,16}: warp-cooperative record fetch.
//   phase 1 (lane = point)  : normalised coords -> per-slab continuous indices -> shared memory
//   phase 2 (warp per point): lane = (corner = lane>>2, quad = lane&3); one LDG.128 per slab fetches the
//                             8 x C corner record; per-lane FMA; xor-shuffle reduction over corners.
// ------------------------------------------------------------------------------------------------
constexpr int kCoopWarps = 4;
constexpr int kMaxSlabs = 16;

template <bool kBackward>
__global__ void __launch_bounds__(32 * kCoopWarps) k_grid_coop(GridView g, const float* __restrict__ xyz,
                                                               int64_t n_pts, float* __restrict__ out_or_gin,
                                                               float* __restrict__ grad_grid) {
  extern __shared__ float4 s_idx[];   // [kCoopWarps][32][P]  continuous indices (cx,cy,cz,-)
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float4* my_idx = s_idx + (size_t)w * 32 * g.P;
  const int corner = lane >> 2, quad = lane & 3;
  const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
  const int nq = g.C >> 2;
  const bool quad_on = quad < nq;
  const float inv_p_is_needed = (g.P > 1) ? 1.f : 0.f;

  const int64_t n_groups = ceil_div<int64_t>(n_pts, 32);
  for (int64_t grp = (int64_t)blockIdx.x * kCoopWarps + w; grp < n_groups; grp += (int64_t)gridDim.x * kCoopWarps) {
    const int64_t p = grp * 32 + lane;
    if (p < n_pts) {
      const float nx = norm_coord(xyz[3 * p], g.mn[0], g.len[0]);
      const float ny = norm_coord(xyz[3 * p + 1], g.mn[1], g.len[1]);
      const float nz = norm_coord(xyz[3 * p + 2], g.mn[2], g.len[2]);
      for (int s = 0; s < g.P; ++s)
        my_idx[lane * g.P + s] = make_float4(src_index_guarded(fourier_gamma(s, nx), g.X), src_index_guarded(fourier_gamma(s, ny), g.Y),
                                             src_index_guarded(fourier_gamma(s, nz), g.Z), 0.f);
    }
    __syncwarp();
    const int n_here = (int)min((int64_t)32, n_pts - grp * 32);
    for (int i = 0; i < n_here; ++i) {
      const int64_t pt = grp * 32 + i;
      float4 acc = make_float4(0, 0, 0, 0);
      float4 gin = make_float4(0, 0, 0, 0);
      if (kBackward) {
        if (quad_on) gin = *reinterpret_cast<const float4*>(out_or_gin + pt * g.C + quad * 4);
        if (inv_p_is_needed != 0.f) {
          gin.x = slab_mean_scale(gin.x, g.P); gin.y = slab_mean_scale(gin.y, g.P); gin.z = slab_mean_scale(gin.z, g.P); gin.w = slab_mean_scale(gin.w, g.P);
        }
      }
      for (int s = 0; s < g.P; ++s) {
        const float4 ci = my_idx[i * g.P + s];   // broadcast read
        const Cell c = locate(ci.x, ci.y, ci.z);
        const bool in = corner_inside(c, bx, by, bz, g.X, g.Y, g.Z) && quad_on;
        const float wgt = corner_weight(c, bx, by, bz);
        const int64_t v = ((int64_t)(c.x0 + bx) * g.Y + (c.y0 + by)) * g.Z + (c.z0 + bz);
        if (!kBackward) {
          if (in) {
            const float4 val = __ldg(reinterpret_cast<const float4*>(g.data + s * g.sp + v * g.sv + quad * 4));
            acc.x += val.x * wgt; acc.y += val.y * wgt; acc.z += val.z * wgt; acc.w += val.w * wgt;
          }
        } else {
          if (in) red_add_v4(grad_grid + s * g.sp + v * g.sv + quad * 4,
                             make_float4(wgt * gin.x, wgt * gin.y, wgt * gin.z, wgt * gin.w));
        }
      }
      if (!kBackward) {
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o);
          acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
          acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o);
          acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
        }
        if (corner == 0 && quad_on) {
          acc.x = slab_mean_scale(acc.x, g.P); acc.y = slab_mean_scale(acc.y, g.P); acc.z = slab_mean_scale(acc.z, g.P); acc.w = slab_mean_scale(acc.w, g.P);
          *reinterpret_cast<float4*>(out_or_gin + pt * g.C + quad * 4) = acc;
        }
      }
    }
    __syncwarp();
  }
}

static bool coop_ok(const GridView& g, const void* io) {
  return g.sc == 1 && g.sv == g.C && (g.C == 4 || g.C == 8 || g.C == 12 || g.C == 16) && g.P <= kMaxSlabs &&
         ((uintptr_t)g.data & 15) == 0 && ((uintptr_t)io & 15) == 0 && (g.sp % 4) == 0;
}

}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_grid_sample_fwd(const float* grid, const UbnGridDesc* desc, const float* xyz, int64_t n_pts, float* out,
                        void* stream) {
  if (n_pts <= 0) return 0;
  const GridView g = make_view(grid, desc);
  if ((g.num_freqs > 0 && g.P != 1 + 2 * g.num_freqs) || (g.num_freqs <= 0 && g.P != 1)) return finish(cudaErrorInvalidValue);
  cudaStream_t st = as_stream(stream);
  if (g.C == 1) {
    k_grid_fwd_c1<<<blocks_for(n_pts, 256), 256, 0, st>>>(g, xyz, n_pts, out);
  } else if (coop_ok(g, out)) {
    const int64_t groups = ceil_div<int64_t>(n_pts, 32);
    const unsigned nb = (unsigned)std::min<int64_t>(ceil_div<int64_t>(groups, kCoopWarps), (int64_t)kNumSMs * 8);
    const size_t smem = sizeof(float4) * kCoopWarps * 32 * g.P;
    k_grid_coop<false><<<nb, 32 * kCoopWarps, smem, st>>>(g, xyz, n_pts, out, nullptr);
  } else {
    k_grid_fwd_generic<<<blocks_for(n_pts, 256), 256, 0, st>>>(g, xyz, n_pts, out);
  }
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_grid_sample_bwd(const float* grad_out, const UbnGridDesc* desc, const float* xyz, int64_t n_pts,
                        float* grad_grid, void* stream) {
  if (n_pts <= 0) return 0;
  GridView g = make_view(grad_grid, desc);
  if ((g.num_freqs > 0 && g.P != 1 + 2 * g.num_freqs) || (g.num_freqs <= 0 && g.P != 1)) return finish(cudaErrorInvalidValue);
  cudaStream_t st = as_stream(stream);
  if (g.C == 1) {
    k_grid_bwd_c1<<<blocks_for(n_pts, 256), 256, 0, st>>>(g, xyz, n_pts, grad_out, grad_grid);
  } else if (coop_ok(g, grad_out)) {
    const int64_t groups = ceil_div<int64_t>(n_pts, 32);
    const unsigned nb = (unsigned)std::min<int64_t>(ceil_div<int64_t>(groups, kCoopWarps), (int64_t)kNumSMs * 8);
    const size_t smem = sizeof(float4) * kCoopWarps * 32 * g.P;
    k_grid_coop<true><<<nb, 32 * kCoopWarps, smem, st>>>(g, xyz, n_pts, const_cast<float*>(grad_out), grad_grid);
  } else {
    k_grid_bwd_generic<<<blocks_for(n_pts, 256), 256, 0, st>>>(g, xyz, n_pts, grad_out, grad_grid);
  }
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
