// march_feature.cu -- pass B of the fused march (feature-grid read for the surviving samples and its adjoint),
// second generation.  Same outputs as k_march_feature in march.cu (kept as the generic fallback); restructured after
// profiling the first version, which ran far below the algorithmic roofline with almost no L1
// hits (its per-warp staging buffers forced a 200 KB shared-memory carve-out and every sample touched all P
// slabs before the next sample re-touched the same voxels) and one load in flight per warp.  Here:
//   * no shared memory at all: the per-(sample, slab) cell (base voxel + 3 fractions) lives in the registers of the
//     lane that owns the sample and is broadcast with warp shuffles -> the whole 228 KB stays L1;
//   * samples are processed in groups (2 forward, 4 backward) with the slab loop OUTSIDE the sample loop, so the corner records of
//     consecutive samples (which share 4-8 corners at half-voxel steps) are re-read while still in L1;
//   * the 8 loads of a group are issued back to back (independent) before their FMAs: 8x the memory-level parallelism;
//   * cells are pre-clamped (base in [0, size-2], fraction in [0,1]) by the owning lane, so no per-corner bounds
//     predicate is needed: contracted / Fourier-warped coordinates never leave [-1,1] (asserted by the host side).
// Lane roles in the cooperative phase: corner = lane >> 2 (bit2 = x, bit1 = y, bit0 = z), quad = lane & 3 (channels
// 4*quad .. 4*quad+3 of the C-channel voxel record); C in {4, 8, 12, 16}, channels-last grid.
#include "march_common.cuh"

namespace ubn {

template <int kP, bool kBackward, int kGroup>
__global__ void __launch_bounds__(32 * kMarchWarps, (kGroup <= 1 ? 8 : (kGroup <= 2 ? 6 : (kGroup <= 4 ? 4 : 5)))) k_march_feature_v2(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ t_table,
    GridView g, MarchParams p, int64_t n_rays, const uint8_t* __restrict__ flags,
    const int64_t* __restrict__ offsets, const float* __restrict__ density, const float* __restrict__ alpha,
    const float* __restrict__ weight, float* __restrict__ feat /* out (fwd) or grad in (bwd) */,
    float* __restrict__ grad_grid, float* __restrict__ o_density, float* __restrict__ o_alpha,
    float* __restrict__ o_weight, int64_t* __restrict__ o_ray_id, int64_t* __restrict__ o_step_id,
    float* __restrict__ o_t, uint8_t* __restrict__ o_inner) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  int64_t out_base = offsets[ray];
  const int64_t out_end = offsets[ray + 1];
  if (out_base == out_end) return;
  const int corner = lane >> 2, quad = lane & 3;
  const bool bx = corner & 4, by = corner & 2, bz = corner & 1;
  const bool quad_on = quad < (g.C >> 2);
  // this lane's constant offset inside a cell: corner displacement + channel quad
  const int lane_off = (((bx ? 1 : 0) * g.Y + (by ? 1 : 0)) * g.Z + (bz ? 1 : 0)) * g.C + quad * 4;
  const Ray r = load_ray(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int S = p.S;
  const float inv_p = 1.f;   // the slab mean is applied as a division below (matches torch mean(0))

  for (int base = 0; base < S && out_base < out_end; base += 32) {
    const int s = base + lane;
    const uint8_t f = (s < S) ? flags[ray * S + s] : 0;
    const bool keep = (f & UBN_FLAG_KEEP) != 0;
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (km == 0) continue;
    const int n_here = __popc(km);
    const int rank = __popc(km & ((1u << lane) - 1));

    // ---- lane = sample: the P cells of my sample (registers) + compacted per-survivor records ----
    CellR cell[kP];
    {
      float x = 0, y = 0, z = 0, t = 0;
      if (keep) {
        t = t_table[s];
        sample_point(r, t, p, x, y, z);
      }
      const float nx = norm_coord(x, g.mn[0], g.len[0]);
      const float ny = norm_coord(y, g.mn[1], g.len[1]);
      const float nz = norm_coord(z, g.mn[2], g.len[2]);
#pragma unroll
      for (int sl = 0; sl < kP; ++sl)
        cell[sl] = make_cell(src_index(fourier_gamma(sl, nx), g.X), src_index(fourier_gamma(sl, ny), g.Y),
                             src_index(fourier_gamma(sl, nz), g.Z), g.X, g.Y, g.Z);
      if (!kBackward && keep) {
        const int64_t o = out_base + rank;
        const int64_t i = ray * S + s;
        o_density[o] = density[i];
        o_alpha[o] = alpha[i];
        o_weight[o] = weight[i];
        o_ray_id[o] = ray;
        o_step_id[o] = s;
        o_t[o] = t;
        o_inner[o] = (f & UBN_FLAG_INNER) ? 1 : 0;
      }
    }
    // compact: slot i (i-th survivor of the chunk) must be readable from lane i
    if (km != 0xffffffffu) {
      const int src = __fns(km, 0, lane + 1) & 31;   // lane holding the (lane+1)-th set bit (garbage when lane >= n_here)
#pragma unroll
      for (int sl = 0; sl < kP; ++sl) {
        cell[sl].v = __shfl_sync(0xffffffffu, cell[sl].v, src);
        cell[sl].fx = __shfl_sync(0xffffffffu, cell[sl].fx, src);
        cell[sl].fy = __shfl_sync(0xffffffffu, cell[sl].fy, src);
        cell[sl].fz = __shfl_sync(0xffffffffu, cell[sl].fz, src);
      }
    }

    // ---- cooperative phase: groups of kGroup survivors, slab loop outside the sample loop ----
    for (int g0 = 0; g0 < n_here; g0 += kGroup) {
      float4 acc[kGroup];
      float4 gin[kGroup];
#pragma unroll
      for (int j = 0; j < kGroup; ++j) {
        acc[j] = make_float4(0, 0, 0, 0);
        gin[j] = make_float4(0, 0, 0, 0);
        if (kBackward) {
          if (quad_on && g0 + j < n_here) gin[j] = *reinterpret_cast<const float4*>(feat + (out_base + g0 + j) * g.C + quad * 4);
          gin[j].x = slab_mean_scale(gin[j].x, kP); gin[j].y = slab_mean_scale(gin[j].y, kP); gin[j].z = slab_mean_scale(gin[j].z, kP); gin[j].w = slab_mean_scale(gin[j].w, kP);
        }
      }
#pragma unroll
      for (int sl = 0; sl < kP; ++sl) {
        const float* slab = g.data + sl * g.sp + lane_off;
        float wgt[kGroup];
        int64_t off[kGroup];
#pragma unroll
        for (int j = 0; j < kGroup; ++j) {
          const int src = (g0 + j) & 31;
          const int v = __shfl_sync(0xffffffffu, cell[sl].v, src);
          const float fx = __shfl_sync(0xffffffffu, cell[sl].fx, src);
          const float fy = __shfl_sync(0xffffffffu, cell[sl].fy, src);
          const float fz = __shfl_sync(0xffffffffu, cell[sl].fz, src);
          // (wz * wy) * wx, the product order of ATen's tnw..bse corner weights
          wgt[j] = ((bz ? fz : 1.f - fz) * (by ? fy : 1.f - fy)) * (bx ? fx : 1.f - fx);
          off[j] = (int64_t)v * g.C;
        }
        if (!kBackward) {
          float4 val[kGroup];
#pragma unroll
          for (int j = 0; j < kGroup; ++j) {
            val[j] = make_float4(0, 0, 0, 0);
            if (quad_on && g0 + j < n_here) val[j] = __ldg(reinterpret_cast<const float4*>(slab + off[j]));
          }
#pragma unroll
          for (int j = 0; j < kGroup; ++j) {
            acc[j].x = fmaf(val[j].x, wgt[j], acc[j].x); acc[j].y = fmaf(val[j].y, wgt[j], acc[j].y);
            acc[j].z = fmaf(val[j].z, wgt[j], acc[j].z); acc[j].w = fmaf(val[j].w, wgt[j], acc[j].w);
          }
        } else {
#pragma unroll
          for (int j = 0; j < kGroup; ++j)
            if (quad_on && g0 + j < n_here)
              red_add_v4(grad_grid + sl * g.sp + lane_off + off[j],
                         make_float4(wgt[j] * gin[j].x, wgt[j] * gin[j].y, wgt[j] * gin[j].z, wgt[j] * gin[j].w));
        }
      }
      if (!kBackward) {
#pragma unroll
        for (int j = 0; j < kGroup; ++j) {
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            acc[j].x += __shfl_xor_sync(0xffffffffu, acc[j].x, o);
            acc[j].y += __shfl_xor_sync(0xffffffffu, acc[j].y, o);
            acc[j].z += __shfl_xor_sync(0xffffffffu, acc[j].z, o);
            acc[j].w += __shfl_xor_sync(0xffffffffu, acc[j].w, o);
          }
        }
        // lane (corner j, quad) writes sample j's channel quad: 8 samples x 48 B = one contiguous 384-byte run
#pragma unroll
        for (int j = 0; j < kGroup; ++j) {
          if (corner == j && quad_on && g0 + j < n_here) {
            float4 v = acc[j];
            v.x = slab_mean_scale(v.x, kP); v.y = slab_mean_scale(v.y, kP); v.z = slab_mean_scale(v.z, kP); v.w = slab_mean_scale(v.w, kP);
            *reinterpret_cast<float4*>(feat + (out_base + g0 + j) * g.C + quad * 4) = v;
          }
        }
      }
    }
    out_base += n_here;
  }
  (void)inv_p;
}

template <int kP, int kGroup>
static int launch_v2(bool backward, const float* rays_o, const float* rays_d, const float* t_table, const GridView& g,
                     const MarchParams& p, int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                     const float* density, const float* alpha, const float* weight, float* feat, float* grad_grid,
                     float* o_density, float* o_alpha, float* o_weight, int64_t* o_ray_id, int64_t* o_step_id, float* o_t,
                     uint8_t* o_inner, cudaStream_t st) {
  const unsigned nb = blocks_for(n_rays, kMarchWarps);
  if (backward)
    k_march_feature_v2<kP, true, kGroup><<<nb, 32 * kMarchWarps, 0, st>>>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets,
                                                                 density, alpha, weight, feat, grad_grid, o_density, o_alpha,
                                                                 o_weight, o_ray_id, o_step_id, o_t, o_inner);
  else
    k_march_feature_v2<kP, false, kGroup><<<nb, 32 * kMarchWarps, 0, st>>>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets,
                                                                  density, alpha, weight, feat, grad_grid, o_density, o_alpha,
                                                                  o_weight, o_ray_id, o_step_id, o_t, o_inner);
  UBN_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================================
// Third generation: LANE = SAMPLE.  The cooperative kernels above spend one warp instruction per (sample, slab) -- 24 of 32
// lanes fetch the 8 x 48-byte corner records of ONE sample, then 12 shuffles reduce the corners: ~17 issue slots and 4 broadcast
// shuffles per sample-slab, few independent loads in flight per warp (profiled: few warps resident, long-scoreboard bound).  Here every lane owns one surviving sample of the chunk and walks its own 8 corners:
//   * 24 independent 128-bit loads per lane and slab (8 corners x 3 channel quads), no shuffles, no cross-lane reduction:
//     ~4.7 issue slots per sample-slab, and 8-24 loads in flight per LANE instead of per warp;
//   * adjacent lanes are adjacent samples of a ray (half a voxel apart), so the same-corner loads of a warp instruction
//     fall into a handful of neighbouring records and coalesce in the LSU;
//   * per slab the 8 products are accumulated in ATen's corner order (FMA chain tnw .. bse) and the slabs are combined in
//     torch-CUDA's mean order (four interleaved accumulators, trilinear.cuh::SlabMean): the features are bit-identical to
//     F.grid_sample(...).mean(0), i.e. to the reference's GPU path;
//   * survivors of a 32-sample chunk are compacted to the low lanes (3 shuffles per chunk) so output rows are written
//     coalesced in (ray, step) order.
// C = 12 channels-last grids (every shipped config); other channel counts keep the cooperative kernels.
// =====================================================================================================================
template <int kP>
__device__ __forceinline__ void slab_cell(const GridView& g, int sl, float nx, float ny, float nz, CellR& c) {
  c = make_cell(src_index(fourier_gamma(sl, nx), g.X), src_index(fourier_gamma(sl, ny), g.Y), src_index(fourier_gamma(sl, nz), g.Z),
                g.X, g.Y, g.Z);
}

template <int kP, bool kBackward>
__global__ void __launch_bounds__(32 * kMarchWarps, 4) k_march_feature_v3(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ t_table,
    GridView g, MarchParams p, int64_t n_rays, const uint8_t* __restrict__ flags,
    const int64_t* __restrict__ offsets, const float* __restrict__ density, const float* __restrict__ alpha,
    const float* __restrict__ weight, float* __restrict__ feat /* out (fwd) or grad in (bwd) */,
    float* __restrict__ grad_grid, float* __restrict__ o_density, float* __restrict__ o_alpha,
    float* __restrict__ o_weight, int64_t* __restrict__ o_ray_id, int64_t* __restrict__ o_step_id,
    float* __restrict__ o_t, uint8_t* __restrict__ o_inner) {
  constexpr int kC = 12;
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  int64_t out_base = offsets[ray];
  const int64_t out_end = offsets[ray + 1];
  if (out_base == out_end) return;
  const Ray r = load_ray(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int S = p.S;
  const int dY = g.Z * kC, dX = g.Y * g.Z * kC;        // record strides (floats) of +1 in y / x; +1 in z is kC

  for (int base = 0; base < S && out_base < out_end; base += 32) {
    const int s = base + lane;
    const uint8_t f = (s < S) ? flags[ray * S + s] : 0;
    const bool keep = (f & UBN_FLAG_KEEP) != 0;
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (km == 0) continue;
    const int n_here = __popc(km);
    const int rank = __popc(km & ((1u << lane) - 1));
    float nx = 0.f, ny = 0.f, nz = 0.f;
    if (keep) {
      float x, y, z;
      const float t = t_table[s];
      sample_point(r, t, p, x, y, z);
      nx = norm_coord(x, g.mn[0], g.len[0]);
      ny = norm_coord(y, g.mn[1], g.len[1]);
      nz = norm_coord(z, g.mn[2], g.len[2]);
      if (!kBackward) {
        const int64_t o = out_base + rank;
        const int64_t i = ray * S + s;
        o_density[o] = density[i];
        o_alpha[o] = alpha[i];
        o_weight[o] = weight[i];
        o_ray_id[o] = ray;
        o_step_id[o] = s;
        o_t[o] = t;
        o_inner[o] = (f & UBN_FLAG_INNER) ? 1 : 0;
      }
    }
    if (km != 0xffffffffu) {            // compact: lane i takes the i-th survivor of the chunk
      const int src = __fns(km, 0, lane + 1) & 31;
      nx = __shfl_sync(0xffffffffu, nx, src);
      ny = __shfl_sync(0xffffffffu, ny, src);
      nz = __shfl_sync(0xffffffffu, nz, src);
    }
    const bool act = lane < n_here;
    const int64_t row = out_base + lane;
    if (!kBackward) {
      // slabs visited in torch's mean order: accumulator a = slab & 3, i.e. 0,4,8 | 1,5,9 | 2,6 | 3,7 ...; `tot` = ((a0 + a1) + a2) + a3
      float tot[kC], grp[kC];
#pragma unroll
      for (int a = 0; a < 4 && a < kP; ++a) {
#pragma unroll
        for (int sl = a; sl < kP; sl += 4) {
          float val[kC];
#pragma unroll
          for (int c = 0; c < kC; ++c) val[c] = 0.f;
          if (act) {
            CellR cell;
            slab_cell<kP>(g, sl, nx, ny, nz, cell);
            const float* rec = g.data + sl * g.sp + (int64_t)cell.v * kC;
#pragma unroll
            for (int corner = 0; corner < 8; ++corner) {          // tnw, tne, tsw, tse, bnw, bne, bsw, bse (z fastest)
              const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
              const float wgt = ((bz ? cell.fz : 1.f - cell.fz) * (by ? cell.fy : 1.f - cell.fy)) * (bx ? cell.fx : 1.f - cell.fx);
              const float4* q = reinterpret_cast<const float4*>(rec + bx * dX + by * dY + bz * kC);
              const float4 v0 = __ldg(q), v1 = __ldg(q + 1), v2 = __ldg(q + 2);
              val[0] = fmaf(v0.x, wgt, val[0]); val[1] = fmaf(v0.y, wgt, val[1]); val[2] = fmaf(v0.z, wgt, val[2]); val[3] = fmaf(v0.w, wgt, val[3]);
              val[4] = fmaf(v1.x, wgt, val[4]); val[5] = fmaf(v1.y, wgt, val[5]); val[6] = fmaf(v1.z, wgt, val[6]); val[7] = fmaf(v1.w, wgt, val[7]);
              val[8] = fmaf(v2.x, wgt, val[8]); val[9] = fmaf(v2.y, wgt, val[9]); val[10] = fmaf(v2.z, wgt, val[10]); val[11] = fmaf(v2.w, wgt, val[11]);
            }
          }
#pragma unroll
          for (int c = 0; c < kC; ++c) grp[c] = (sl == a) ? __fadd_rn(0.f, val[c]) : __fadd_rn(grp[c], val[c]);
        }
#pragma unroll
        for (int c = 0; c < kC; ++c) tot[c] = (a == 0) ? grp[c] : __fadd_rn(tot[c], grp[c]);
      }
      if (act) {
        float4* o = reinterpret_cast<float4*>(feat + row * kC);
        o[0] = make_float4(slab_mean_scale(tot[0], kP), slab_mean_scale(tot[1], kP), slab_mean_scale(tot[2], kP), slab_mean_scale(tot[3], kP));
        o[1] = make_float4(slab_mean_scale(tot[4], kP), slab_mean_scale(tot[5], kP), slab_mean_scale(tot[6], kP), slab_mean_scale(tot[7], kP));
        o[2] = make_float4(slab_mean_scale(tot[8], kP), slab_mean_scale(tot[9], kP), slab_mean_scale(tot[10], kP), slab_mean_scale(tot[11], kP));
      }
    } else if (act) {
      const float4* gi = reinterpret_cast<const float4*>(feat + row * kC);
      float4 g0 = gi[0], g1 = gi[1], g2 = gi[2];
      g0.x = slab_mean_scale(g0.x, kP); g0.y = slab_mean_scale(g0.y, kP); g0.z = slab_mean_scale(g0.z, kP); g0.w = slab_mean_scale(g0.w, kP);
      g1.x = slab_mean_scale(g1.x, kP); g1.y = slab_mean_scale(g1.y, kP); g1.z = slab_mean_scale(g1.z, kP); g1.w = slab_mean_scale(g1.w, kP);
      g2.x = slab_mean_scale(g2.x, kP); g2.y = slab_mean_scale(g2.y, kP); g2.z = slab_mean_scale(g2.z, kP); g2.w = slab_mean_scale(g2.w, kP);
#pragma unroll
      for (int sl = 0; sl < kP; ++sl) {
        CellR cell;
        slab_cell<kP>(g, sl, nx, ny, nz, cell);
        float* rec = grad_grid + sl * g.sp + (int64_t)cell.v * kC;
#pragma unroll
        for (int corner = 0; corner < 8; ++corner) {
          const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
          const float wgt = ((bz ? cell.fz : 1.f - cell.fz) * (by ? cell.fy : 1.f - cell.fy)) * (bx ? cell.fx : 1.f - cell.fx);
          float* q = rec + bx * dX + by * dY + bz * kC;
          red_add_v4(q, make_float4(wgt * g0.x, wgt * g0.y, wgt * g0.z, wgt * g0.w));
          red_add_v4(q + 4, make_float4(wgt * g1.x, wgt * g1.y, wgt * g1.z, wgt * g1.w));
          red_add_v4(q + 8, make_float4(wgt * g2.x, wgt * g2.y, wgt * g2.z, wgt * g2.w));
        }
      }
    }
    out_base += n_here;
  }
}

// =====================================================================================================================
// Fourth generation of the gather: EIGHT samples per instruction, three lanes per sample (lane = sample j of 8, channel quad q).
// The lane-per-sample kernel above is bound by L1 wavefronts: one LDG.128 of its 24 per slab sends
// 32 lanes to up to 32 different 128-byte lines.  Here the three quad lanes of a sample read the 48 contiguous bytes of ONE
// corner record, so an instruction touches 8 records instead of 32 and a slab costs 8 load instructions per 8 samples.  The
// accumulation stays inside the lane (4 channels of its quad over the 8 corners in ATen's order, slabs in torch-CUDA's mean
// order), so there is still no cross-lane reduction and the features keep their bits.  The cells are computed once per sample
// (lane = sample, as before) and handed to the (j, q) lanes by 4 shuffles per (pass, slab).
// =====================================================================================================================
template <int kP>
__global__ void __launch_bounds__(32 * kMarchWarps, 4) k_march_feature_v4(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ t_table,
    GridView g, MarchParams p, int64_t n_rays, const uint8_t* __restrict__ flags,
    const int64_t* __restrict__ offsets, const float* __restrict__ density, const float* __restrict__ alpha,
    const float* __restrict__ weight, float* __restrict__ feat, float* __restrict__ o_density, float* __restrict__ o_alpha,
    float* __restrict__ o_weight, int64_t* __restrict__ o_ray_id, int64_t* __restrict__ o_step_id,
    float* __restrict__ o_t, uint8_t* __restrict__ o_inner) {
  constexpr int kC = 12;
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  int64_t out_base = offsets[ray];
  const int64_t out_end = offsets[ray + 1];
  if (out_base == out_end) return;
  const Ray r = load_ray(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int S = p.S;
  const int dY = g.Z * kC, dX = g.Y * g.Z * kC;
  const int jq = lane >> 2, q = lane & 3;                 // sample of the pass, channel quad (q == 3: idle lane)

  for (int base = 0; base < S && out_base < out_end; base += 32) {
    const int s = base + lane;
    const uint8_t f = (s < S) ? flags[ray * S + s] : 0;
    const bool keep = (f & UBN_FLAG_KEEP) != 0;
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (km == 0) continue;
    const int n_here = __popc(km);
    const int rank = __popc(km & ((1u << lane) - 1));
    float nx = 0.f, ny = 0.f, nz = 0.f;
    if (keep) {
      float x, y, z;
      const float t = t_table[s];
      sample_point(r, t, p, x, y, z);
      nx = norm_coord(x, g.mn[0], g.len[0]);
      ny = norm_coord(y, g.mn[1], g.len[1]);
      nz = norm_coord(z, g.mn[2], g.len[2]);
      const int64_t o = out_base + rank;
      const int64_t i = ray * S + s;
      o_density[o] = density[i];
      o_alpha[o] = alpha[i];
      o_weight[o] = weight[i];
      o_ray_id[o] = ray;
      o_step_id[o] = s;
      o_t[o] = t;
      o_inner[o] = (f & UBN_FLAG_INNER) ? 1 : 0;
    }
    if (km != 0xffffffffu) {            // compact: lane i takes the i-th survivor of the chunk
      const int src = __fns(km, 0, lane + 1) & 31;
      nx = __shfl_sync(0xffffffffu, nx, src);
      ny = __shfl_sync(0xffffffffu, ny, src);
      nz = __shfl_sync(0xffffffffu, nz, src);
    }
    // the kP cells of MY sample (lane = i-th survivor), one sincosf per axis and frequency
    CellR cell[kP];
    for_each_slab<kP>(g, nx, ny, nz, [&](int sl, float cx, float cy, float cz) { cell[sl] = make_cell(cx, cy, cz, g.X, g.Y, g.Z); });
#pragma unroll 1
    for (int pass = 0; pass < 4; ++pass) {
      if (pass * 8 >= n_here) break;                      // warp-uniform
      const int j = pass * 8 + jq;
      const bool act = q < 3 && j < n_here;
      float4 tot = make_float4(0, 0, 0, 0), grp = make_float4(0, 0, 0, 0);
#pragma unroll
      for (int a = 0; a < 4 && a < kP; ++a) {
#pragma unroll
        for (int sl = a; sl < kP; sl += 4) {
          const int v = __shfl_sync(0xffffffffu, cell[sl].v, j);
          const float fx = __shfl_sync(0xffffffffu, cell[sl].fx, j);
          const float fy = __shfl_sync(0xffffffffu, cell[sl].fy, j);
          const float fz = __shfl_sync(0xffffffffu, cell[sl].fz, j);
          float4 val = make_float4(0, 0, 0, 0);
          if (act) {
            const float* rec = g.data + sl * g.sp + (int64_t)v * kC + q * 4;
#pragma unroll
            for (int corner = 0; corner < 8; ++corner) {          // tnw, tne, tsw, tse, bnw, bne, bsw, bse (z fastest)
              const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
              const float wgt = ((bz ? fz : 1.f - fz) * (by ? fy : 1.f - fy)) * (bx ? fx : 1.f - fx);
              const float4 c4 = __ldg(reinterpret_cast<const float4*>(rec + bx * dX + by * dY + bz * kC));
              val.x = fmaf(c4.x, wgt, val.x); val.y = fmaf(c4.y, wgt, val.y); val.z = fmaf(c4.z, wgt, val.z); val.w = fmaf(c4.w, wgt, val.w);
            }
          }
          if (sl == a) { grp.x = __fadd_rn(0.f, val.x); grp.y = __fadd_rn(0.f, val.y); grp.z = __fadd_rn(0.f, val.z); grp.w = __fadd_rn(0.f, val.w); }
          else { grp.x = __fadd_rn(grp.x, val.x); grp.y = __fadd_rn(grp.y, val.y); grp.z = __fadd_rn(grp.z, val.z); grp.w = __fadd_rn(grp.w, val.w); }
        }
        if (a == 0) tot = grp;
        else { tot.x = __fadd_rn(tot.x, grp.x); tot.y = __fadd_rn(tot.y, grp.y); tot.z = __fadd_rn(tot.z, grp.z); tot.w = __fadd_rn(tot.w, grp.w); }
      }
      if (act)
        *reinterpret_cast<float4*>(feat + (out_base + j) * kC + q * 4) =
            make_float4(slab_mean_scale(tot.x, kP), slab_mean_scale(tot.y, kP), slab_mean_scale(tot.z, kP), slab_mean_scale(tot.w, kP));
    }
    out_base += n_here;
  }
}

template <int kP>
static int launch_v4(const float* rays_o, const float* rays_d, const float* t_table, const GridView& g, const MarchParams& p,
                     int64_t n_rays, const uint8_t* flags, const int64_t* offsets, const float* density, const float* alpha,
                     const float* weight, float* feat, float* o_density, float* o_alpha, float* o_weight, int64_t* o_ray_id,
                     int64_t* o_step_id, float* o_t, uint8_t* o_inner, cudaStream_t st) {
  k_march_feature_v4<kP><<<blocks_for(n_rays, kMarchWarps), 32 * kMarchWarps, 0, st>>>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets,
                                                                                        density, alpha, weight, feat, o_density, o_alpha,
                                                                                        o_weight, o_ray_id, o_step_id, o_t, o_inner);
  UBN_LAUNCH_CHECK();
  return 0;
}

template <int kP>
static int launch_v3(bool backward, const float* rays_o, const float* rays_d, const float* t_table, const GridView& g,
                     const MarchParams& p, int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                     const float* density, const float* alpha, const float* weight, float* feat, float* grad_grid,
                     float* o_density, float* o_alpha, float* o_weight, int64_t* o_ray_id, int64_t* o_step_id, float* o_t,
                     uint8_t* o_inner, cudaStream_t st) {
  const unsigned nb = blocks_for(n_rays, kMarchWarps);
  if (backward)
    k_march_feature_v3<kP, true><<<nb, 32 * kMarchWarps, 0, st>>>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha,
                                                                  weight, feat, grad_grid, o_density, o_alpha, o_weight, o_ray_id,
                                                                  o_step_id, o_t, o_inner);
  else
    k_march_feature_v3<kP, false><<<nb, 32 * kMarchWarps, 0, st>>>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha,
                                                                   weight, feat, grad_grid, o_density, o_alpha, o_weight, o_ray_id,
                                                                   o_step_id, o_t, o_inner);
  UBN_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================================
// Slab-major scatter (variant 3).  The k0 gradient of the truck workload is 9 slabs x 172 MB: with the slab loop inside the
// kernel every resident warp spreads its reductions over all 1.55 GB, far more than the L2 holds, and nearly every vector
// reduction costs a DRAM sector fetch + write-back at random addresses.  Here the SLAB is the slow grid dimension
// (blockIdx.y): the CTAs of slab s are scheduled before the CTAs of slab s + 1, the live gradient footprint at any moment is
// ONE slab (172 MB; split in x-ranges by variants 4 / 5 to fit the H100's 50 MB L2), and every sector of a
// slab goes to DRAM about once.  Cost: the chunk preamble (flags, sample point, compaction) runs once per slab instead of
// once, and the 48-byte gradient rows are re-read 9 times (coalesced, L2 hits after the first slab).  Same lane roles and
// the same addends as k_march_feature_v2<.., true, ..>: the gradients differ only by the atomics' summation order.
// =====================================================================================================================
template <int kP, int kGroup, int kMinBlocks, bool kPreScale>
__global__ void __launch_bounds__(32 * kMarchWarps, kMinBlocks) k_march_feature_bwd_slab(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ t_table,
    GridView g, MarchParams p, int64_t n_rays, const uint8_t* __restrict__ flags,
    const int64_t* __restrict__ offsets, const float* __restrict__ gfeat, float* __restrict__ grad_grid, int n_split) {
  // n_split > 1: every slab is swept n_split times, pass `part` scattering only the samples whose cell starts in the part-th
  // x-range of the slab, so the live gradient footprint is 1 / n_split of a slab (86 / 43 MB for two / four parts of a
  // 153^3 x 12 slab; the H100's L2 is 50 MB) at the price of repeating the chunk preamble
  const int lane = threadIdx.x & 31;
  const int sl = blockIdx.y / n_split, part = blockIdx.y - sl * n_split;
  const int v_lo = (int)(((int64_t)(g.X - 1) * part) / n_split) * g.Y * g.Z;
  const int v_hi = (part + 1 == n_split) ? 0x7fffffff : (int)(((int64_t)(g.X - 1) * (part + 1)) / n_split) * g.Y * g.Z;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  int64_t out_base = offsets[ray];
  const int64_t out_end = offsets[ray + 1];
  if (out_base == out_end) return;
  const int corner = lane >> 2, quad = lane & 3;
  const bool bx = corner & 4, by = corner & 2, bz = corner & 1;
  const bool quad_on = quad < (g.C >> 2);
  const int lane_off = (((bx ? 1 : 0) * g.Y + (by ? 1 : 0)) * g.Z + (bz ? 1 : 0)) * g.C + quad * 4;
  float* slab = grad_grid + sl * g.sp + lane_off;
  const Ray r = load_ray(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int S = p.S;

  for (int base = 0; base < S && out_base < out_end; base += 32) {
    const int s = base + lane;
    const uint8_t f = (s < S) ? flags[ray * S + s] : 0;
    const bool keep = (f & UBN_FLAG_KEEP) != 0;
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (km == 0) continue;
    CellR cell;
    {
      float x = 0, y = 0, z = 0;
      if (keep) sample_point(r, t_table[s], p, x, y, z);
      const float nx = norm_coord(x, g.mn[0], g.len[0]);
      const float ny = norm_coord(y, g.mn[1], g.len[1]);
      const float nz = norm_coord(z, g.mn[2], g.len[2]);
      cell = make_cell(src_index(fourier_gamma(sl, nx), g.X), src_index(fourier_gamma(sl, ny), g.Y),
                       src_index(fourier_gamma(sl, nz), g.Z), g.X, g.Y, g.Z);
    }
    // survivors of the chunk that this pass serves; `row` = their position in the compacted gradient rows
    const unsigned sm = __ballot_sync(0xffffffffu, keep && cell.v >= v_lo && cell.v < v_hi);
    const int n_here = __popc(sm);
    int row = __popc(km & ((1u << lane) - 1));
    if (sm != 0xffffffffu) {
      const int src = __fns(sm, 0, lane + 1) & 31;
      cell.v = __shfl_sync(0xffffffffu, cell.v, src);
      cell.fx = __shfl_sync(0xffffffffu, cell.fx, src);
      cell.fy = __shfl_sync(0xffffffffu, cell.fy, src);
      cell.fz = __shfl_sync(0xffffffffu, cell.fz, src);
      row = __shfl_sync(0xffffffffu, row, src);
    }
    for (int g0 = 0; g0 < n_here; g0 += kGroup) {
      float4 gin[kGroup];
#pragma unroll
      for (int j = 0; j < kGroup; ++j) {
        gin[j] = make_float4(0, 0, 0, 0);
        const int rj = __shfl_sync(0xffffffffu, row, (g0 + j) & 31);
        if (quad_on && g0 + j < n_here) gin[j] = __ldg(reinterpret_cast<const float4*>(gfeat + (out_base + rj) * g.C + quad * 4));
      }
      // Consecutive samples of a ray are half a voxel apart in slab 0 and at most that in the sin / cos slabs of the lowest
      // frequency, so neighbours of a group often fall into the SAME cell: their contributions are added in registers and leave as
      // one vector reduction (the scatter is bound by the number of L2 reduction sectors).  The cell index is warp-uniform after the shuffle, so the test costs no divergence.
      // (Handing the shared FACE of two neighbouring cells over the same way -- four of eight corners, one xor-shuffle per float --
      // was measured slower: half-populated reduction instructions do not halve the cost of an instruction.  So was a run-length
      // merge carried across groups and chunks -- the open run serialises the group's reductions; and so was pairing neighbours
      // 16 positions apart with alternating issue -- fewer merges, and nothing gained from spacing.)
      int vj[kGroup];
      float4 val[kGroup];
#pragma unroll
      for (int j = 0; j < kGroup; ++j) {
        const int src = (g0 + j) & 31;
        vj[j] = __shfl_sync(0xffffffffu, cell.v, src);
        const float fx = __shfl_sync(0xffffffffu, cell.fx, src);
        const float fy = __shfl_sync(0xffffffffu, cell.fy, src);
        const float fz = __shfl_sync(0xffffffffu, cell.fz, src);
        float wgt = ((bz ? fz : 1.f - fz) * (by ? fy : 1.f - fy)) * (bx ? fx : 1.f - fx);
        const float4 q = gin[j];
        if (kPreScale) {                                   // 1 / P folded into the corner weight: one multiply instead of four
          wgt = slab_mean_scale(wgt, kP);
          val[j] = make_float4(wgt * q.x, wgt * q.y, wgt * q.z, wgt * q.w);
        } else {
          val[j] = make_float4(wgt * slab_mean_scale(q.x, kP), wgt * slab_mean_scale(q.y, kP), wgt * slab_mean_scale(q.z, kP),
                               wgt * slab_mean_scale(q.w, kP));
        }
        if (g0 + j >= n_here) vj[j] = -1 - j;              // past the end: never equal to a neighbour, never written
      }
#pragma unroll
      for (int j = 0; j < kGroup; ++j) {
        if (j + 1 < kGroup && vj[j] == vj[j + 1]) {        // warp-uniform: same cell as the next sample -> carry the sum forward
          val[j + 1].x += val[j].x; val[j + 1].y += val[j].y; val[j + 1].z += val[j].z; val[j + 1].w += val[j].w;
        } else if (quad_on && vj[j] >= 0) {
          red_add_v4(slab + (int64_t)vj[j] * g.C, val[j]);
        }
      }
    }
    out_base += __popc(km);
  }
}

template <int kP>
static int launch_bwd_slab(const float* rays_o, const float* rays_d, const float* t_table, const GridView& g, const MarchParams& p,
                           int64_t n_rays, const uint8_t* flags, const int64_t* offsets, const float* gfeat, float* grad_grid,
                           int n_split, cudaStream_t st) {
  const dim3 grid(blocks_for(n_rays, kMarchWarps), kP * n_split);
  // 8 resident blocks (64 registers) and 1 / P folded into the corner weight: measured faster than fewer blocks and than groups of 8
  k_march_feature_bwd_slab<kP, 4, 8, true><<<grid, 32 * kMarchWarps, 0, st>>>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, gfeat, grad_grid,
                                                                              n_split);
  UBN_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================================
// C = 3 and C = 15 (FourierGridModel with rgbnet_dim = 3 -- the Waymo / Mega-NeRF configs -- or 15, and every colour-grid stage
// with rgbnet_dim <= 0).  A 12- or 60-byte record is only 4-byte aligned, so neither the float4 quads of the kernels above nor
// their lane roles apply.
//   Gather: lane = sample, as k_march_feature_v3: scalar loads, every channel accumulated in ATen's corner order (fma chain
//   tnw .. bse) and the slabs combined in torch-CUDA's mean order, so the features are bit-identical to
//   F.grid_sample(...).mean(0).
//   Scatter: slab-major with the x-range split, as k_march_feature_bwd_slab.  Lane (corner = lane >> 2, run = lane & 3): the
//   survivors of a chunk that this pass serves are cut into 4 contiguous runs, and the 8 corner lanes of a run walk its samples in
//   order, adding the contributions of consecutive samples that share a cell in registers.  A cell leaves as one record of
//   red_add_record (red.v4 / red.v2 / scalar, whatever each address allows) when the run moves on or ends.
// =====================================================================================================================
template <int kC, int kP>
__global__ void __launch_bounds__(32 * kMarchWarps, 4) k_march_feature_narrow(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ t_table,
    GridView g, MarchParams p, int64_t n_rays, const uint8_t* __restrict__ flags,
    const int64_t* __restrict__ offsets, const float* __restrict__ density, const float* __restrict__ alpha,
    const float* __restrict__ weight, float* __restrict__ feat, float* __restrict__ o_density, float* __restrict__ o_alpha,
    float* __restrict__ o_weight, int64_t* __restrict__ o_ray_id, int64_t* __restrict__ o_step_id,
    float* __restrict__ o_t, uint8_t* __restrict__ o_inner) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  int64_t out_base = offsets[ray];
  const int64_t out_end = offsets[ray + 1];
  if (out_base == out_end) return;
  const Ray r = load_ray(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int S = p.S;
  const int dY = g.Z * kC, dX = g.Y * g.Z * kC;

  for (int base = 0; base < S && out_base < out_end; base += 32) {
    const int s = base + lane;
    const uint8_t f = (s < S) ? flags[ray * S + s] : 0;
    const bool keep = (f & UBN_FLAG_KEEP) != 0;
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (km == 0) continue;
    const int n_here = __popc(km);
    const int rank = __popc(km & ((1u << lane) - 1));
    float nx = 0.f, ny = 0.f, nz = 0.f;
    if (keep) {
      float x, y, z;
      const float t = t_table[s];
      sample_point(r, t, p, x, y, z);
      nx = norm_coord(x, g.mn[0], g.len[0]);
      ny = norm_coord(y, g.mn[1], g.len[1]);
      nz = norm_coord(z, g.mn[2], g.len[2]);
      const int64_t o = out_base + rank;
      const int64_t i = ray * S + s;
      o_density[o] = density[i];
      o_alpha[o] = alpha[i];
      o_weight[o] = weight[i];
      o_ray_id[o] = ray;
      o_step_id[o] = s;
      o_t[o] = t;
      o_inner[o] = (f & UBN_FLAG_INNER) ? 1 : 0;
    }
    if (km != 0xffffffffu) {            // compact: lane i takes the i-th survivor of the chunk
      const int src = __fns(km, 0, lane + 1) & 31;
      nx = __shfl_sync(0xffffffffu, nx, src);
      ny = __shfl_sync(0xffffffffu, ny, src);
      nz = __shfl_sync(0xffffffffu, nz, src);
    }
    if (lane < n_here) {
      // slabs visited in torch's mean order: accumulator a = slab & 3; `tot` = ((a0 + a1) + a2) + a3
      float tot[kC], grp[kC];
#pragma unroll
      for (int a = 0; a < 4 && a < kP; ++a) {
#pragma unroll
        for (int sl = a; sl < kP; sl += 4) {
          CellR cell;
          slab_cell<kP>(g, sl, nx, ny, nz, cell);
          const float* rec = g.data + sl * g.sp + (int64_t)cell.v * kC;
          float val[kC];
#pragma unroll
          for (int c = 0; c < kC; ++c) val[c] = 0.f;
#pragma unroll
          for (int corner = 0; corner < 8; ++corner) {        // tnw, tne, tsw, tse, bnw, bne, bsw, bse (z fastest)
            const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
            const float wgt = ((bz ? cell.fz : 1.f - cell.fz) * (by ? cell.fy : 1.f - cell.fy)) * (bx ? cell.fx : 1.f - cell.fx);
            const float* q = rec + bx * dX + by * dY + bz * kC;
#pragma unroll
            for (int c = 0; c < kC; ++c) val[c] = fmaf(__ldg(q + c), wgt, val[c]);
          }
#pragma unroll
          for (int c = 0; c < kC; ++c) grp[c] = (sl == a) ? __fadd_rn(0.f, val[c]) : __fadd_rn(grp[c], val[c]);
        }
#pragma unroll
        for (int c = 0; c < kC; ++c) tot[c] = (a == 0) ? grp[c] : __fadd_rn(tot[c], grp[c]);
      }
      float* o = feat + (out_base + lane) * kC;
#pragma unroll
      for (int c = 0; c < kC; ++c) o[c] = slab_mean_scale(tot[c], kP);
    }
    out_base += n_here;
  }
}

template <int kC, int kP>
__global__ void __launch_bounds__(32 * kMarchWarps, 8) k_march_feature_bwd_narrow(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ t_table,
    GridView g, MarchParams p, int64_t n_rays, const uint8_t* __restrict__ flags,
    const int64_t* __restrict__ offsets, const float* __restrict__ gfeat, float* __restrict__ grad_grid, int n_split) {
  const int lane = threadIdx.x & 31;
  const int sl = blockIdx.y / n_split, part = blockIdx.y - sl * n_split;
  const int v_lo = (int)(((int64_t)(g.X - 1) * part) / n_split) * g.Y * g.Z;
  const int v_hi = (part + 1 == n_split) ? 0x7fffffff : (int)(((int64_t)(g.X - 1) * (part + 1)) / n_split) * g.Y * g.Z;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  int64_t out_base = offsets[ray];
  const int64_t out_end = offsets[ray + 1];
  if (out_base == out_end) return;
  const int corner = lane >> 2, run = lane & 3;
  const bool bx = corner & 4, by = corner & 2, bz = corner & 1;
  float* slab = grad_grid + sl * g.sp + (((bx ? 1 : 0) * g.Y + (by ? 1 : 0)) * g.Z + (bz ? 1 : 0)) * kC;
  const Ray r = load_ray(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int S = p.S;

  for (int base = 0; base < S && out_base < out_end; base += 32) {
    const int s = base + lane;
    const uint8_t f = (s < S) ? flags[ray * S + s] : 0;
    const bool keep = (f & UBN_FLAG_KEEP) != 0;
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (km == 0) continue;
    CellR cell;
    {
      float x = 0, y = 0, z = 0;
      if (keep) sample_point(r, t_table[s], p, x, y, z);
      const float nx = norm_coord(x, g.mn[0], g.len[0]);
      const float ny = norm_coord(y, g.mn[1], g.len[1]);
      const float nz = norm_coord(z, g.mn[2], g.len[2]);
      if (kP == 1) cell = make_cell(src_index(nx, g.X), src_index(ny, g.Y), src_index(nz, g.Z), g.X, g.Y, g.Z);
      else cell = make_cell(src_index(fourier_gamma(sl, nx), g.X), src_index(fourier_gamma(sl, ny), g.Y),
                            src_index(fourier_gamma(sl, nz), g.Z), g.X, g.Y, g.Z);
    }
    // survivors of the chunk that this pass serves; `row` = their position in the compacted gradient rows
    const unsigned sm = __ballot_sync(0xffffffffu, keep && cell.v >= v_lo && cell.v < v_hi);
    const int n_here = __popc(sm);
    int row = __popc(km & ((1u << lane) - 1));
    if (sm != 0xffffffffu) {
      const int src = __fns(sm, 0, lane + 1) & 31;
      cell.v = __shfl_sync(0xffffffffu, cell.v, src);
      cell.fx = __shfl_sync(0xffffffffu, cell.fx, src);
      cell.fy = __shfl_sync(0xffffffffu, cell.fy, src);
      cell.fz = __shfl_sync(0xffffffffu, cell.fz, src);
      row = __shfl_sync(0xffffffffu, row, src);
    }
    const int len = (n_here + 3) >> 2;                     // samples per run (warp-uniform)
    const int i0 = min(run * len, n_here), i1 = min(i0 + len, n_here);
    int open = -1;                                         // cell of the open sum (-1: none)
    float acc[kC];
#pragma unroll
    for (int c = 0; c < kC; ++c) acc[c] = 0.f;
    for (int i = 0; i < len; ++i) {
      const int src = (i0 + i) & 31;
      const int v = __shfl_sync(0xffffffffu, cell.v, src);
      const float fx = __shfl_sync(0xffffffffu, cell.fx, src);
      const float fy = __shfl_sync(0xffffffffu, cell.fy, src);
      const float fz = __shfl_sync(0xffffffffu, cell.fz, src);
      const int rj = __shfl_sync(0xffffffffu, row, src);
      if (i0 + i >= i1) continue;                          // the last run may be shorter; every lane keeps shuffling
      // 1 / P folded into the corner weight
      const float wgt = slab_mean_scale(((bz ? fz : 1.f - fz) * (by ? fy : 1.f - fy)) * (bx ? fx : 1.f - fx), kP);
      const float* gi = gfeat + (out_base + rj) * kC;
      if (v != open) {
        if (open >= 0) red_add_record<kC>(slab + (int64_t)open * kC, acc);
        open = v;
#pragma unroll
        for (int c = 0; c < kC; ++c) acc[c] = wgt * __ldg(gi + c);
      } else {
#pragma unroll
        for (int c = 0; c < kC; ++c) acc[c] += wgt * __ldg(gi + c);
      }
    }
    if (open >= 0) red_add_record<kC>(slab + (int64_t)open * kC, acc);
    out_base += __popc(km);
  }
}

template <int kC, int kP>
static int launch_narrow(bool backward, const float* rays_o, const float* rays_d, const float* t_table, const GridView& g,
                         const MarchParams& p, int64_t n_rays, const uint8_t* flags, const int64_t* offsets, const float* density,
                         const float* alpha, const float* weight, float* feat, float* grad_grid, float* o_density, float* o_alpha,
                         float* o_weight, int64_t* o_ray_id, int64_t* o_step_id, float* o_t, uint8_t* o_inner, int n_split,
                         cudaStream_t st) {
  if (backward)
    k_march_feature_bwd_narrow<kC, kP><<<dim3(blocks_for(n_rays, kMarchWarps), kP * n_split), 32 * kMarchWarps, 0, st>>>(
        rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, feat, grad_grid, n_split);
  else
    k_march_feature_narrow<kC, kP><<<blocks_for(n_rays, kMarchWarps), 32 * kMarchWarps, 0, st>>>(
        rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat, o_density, o_alpha, o_weight, o_ray_id,
        o_step_id, o_t, o_inner);
  UBN_LAUNCH_CHECK();
  return 0;
}

template <int kC>
static int march_feature_narrow(bool backward, const float* rays_o, const float* rays_d, const float* t_table, const GridView& g,
                                const MarchParams& p, int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                                const float* density, const float* alpha, const float* weight, float* feat, float* grad_grid,
                                float* o_density, float* o_alpha, float* o_weight, int64_t* o_ray_id, int64_t* o_step_id, float* o_t,
                                uint8_t* o_inner, int n_split, cudaStream_t st) {
#define UBN_NARROW(P)                                                                                                            \
  case P:                                                                                                                        \
    return launch_narrow<kC, P>(backward, rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat,    \
                                grad_grid, o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, n_split, st)
  switch (g.P) {
    UBN_NARROW(1);
    UBN_NARROW(3);
    UBN_NARROW(5);
    UBN_NARROW(7);
    UBN_NARROW(9);
    UBN_NARROW(11);
    default: return -1;
  }
#undef UBN_NARROW
}

// Pass-B kernel family, set through ubn_set_feature_kernel (the GPU tests exercise every value):
//   0  warp-cooperative gather and scatter (k_march_feature_v2)
//   1  lane-per-sample gather (k_march_feature_v3) + cooperative scatter
//   2  lane-per-sample gather and scatter
//   3  lane-per-sample gather -- the 8-samples-per-instruction k_march_feature_v4 for single-slab grids -- + SLAB-MAJOR
//      cooperative scatter with the equal-cell merge (k_march_feature_bwd_slab)
//   4 / 5  as 3 with every slab swept in 2 / 4 x-ranges (5 = default)
//   6  as 3 with k_march_feature_v4 for every slab count
// The scatter stays cooperative: one warp instruction issues the 24 vector reductions of a sample into 8 x 48 contiguous bytes,
// whereas lane-per-sample reductions hit 32 unrelated records per instruction.
// Scatter of the truck workload (8192 x 512, 9 slabs of 172 MB) on one H100 80GB HBM3 at a 400 W power limit, two alternating
// runs of bench.py --only-timed --feature-kernel V: 6.61 / 6.61 ms (3), 6.19 / 6.17 ms (4), 5.98 / 5.98 ms (5).  A quarter slab
// (43 MB) fits the 50 MB L2, and that saves more than the repeated chunk preamble costs, so 5 is the default.
static int g_feature_kernel = 5;
void set_feature_kernel(int v) { g_feature_kernel = v; }
int get_feature_kernel() { return g_feature_kernel; }

// returns -1 when this configuration is not covered (caller falls back to the generic kernel)
int march_feature_v2(bool backward, const float* rays_o, const float* rays_d, const float* t_table, const GridView& g,
                     const MarchParams& p, int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                     const float* density, const float* alpha, const float* weight, float* feat, float* grad_grid,
                     float* o_density, float* o_alpha, float* o_weight, int64_t* o_ray_id, int64_t* o_step_id, float* o_t,
                     uint8_t* o_inner, cudaStream_t st) {
  if (g.X < 2 || g.Y < 2 || g.Z < 2) return -1;
  if ((int64_t)g.X * g.Y * g.Z * g.C >= (1ll << 31)) return -1;   // 32-bit voxel offsets inside a slab
  if (g.C == 3 || g.C == 15) {                            // every variant: the lane-per-sample gather, the slab-major run scatter
    const int n_split = g_feature_kernel == 4 ? 2 : g_feature_kernel == 5 ? 4 : 1;
    if (g.C == 3)
      return march_feature_narrow<3>(backward, rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat,
                                     grad_grid, o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, n_split, st);
    return march_feature_narrow<15>(backward, rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat,
                                    grad_grid, o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, n_split, st);
  }
  if (backward && g_feature_kernel >= 3 && g.P > 1) {     // 3 / 4 / 5: slab-major scatter, each slab swept in 1 / 2 / 4 x-ranges; 6: as 3
    const int n_split = g_feature_kernel == 6 ? 1 : 1 << (g_feature_kernel - 3);
    switch (g.P) {
      case 3: return launch_bwd_slab<3>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, feat, grad_grid, n_split, st);
      case 5: return launch_bwd_slab<5>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, feat, grad_grid, n_split, st);
      case 7: return launch_bwd_slab<7>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, feat, grad_grid, n_split, st);
      case 9: return launch_bwd_slab<9>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, feat, grad_grid, n_split, st);
      default: break;
    }
  }
  // 8 samples x 3 channel quads per instruction: explicitly (6), and with 3 / 4 / 5 (5 = default) for single-slab grids, where it
  // measured faster than the lane-per-sample gather; on the 9-slab FourierGrid the shuffled cells cost more than the wavefronts save
  if (g.C == 12 && !backward && (g_feature_kernel == 6 || (g_feature_kernel >= 3 && g_feature_kernel <= 5 && g.P == 1))) {
    switch (g.P) {
      case 1: return launch_v4<1>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat, o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, st);
      case 3: return launch_v4<3>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat, o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, st);
      case 5: return launch_v4<5>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat, o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, st);
      case 7: return launch_v4<7>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat, o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, st);
      case 9: return launch_v4<9>(rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat, o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, st);
      default: break;
    }
  }
  if (g.C == 12 && (g_feature_kernel == 2 || ((g_feature_kernel == 1 || g_feature_kernel >= 3) && !backward))) {
#define UBN_V3(P)                                                                                                               \
  case P:                                                                                                                       \
    return launch_v3<P>(backward, rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, feat, grad_grid, \
                        o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, st)
    switch (g.P) {
      UBN_V3(1);
      UBN_V3(3);
      UBN_V3(5);
      UBN_V3(7);
      UBN_V3(9);
      default: break;
    }
#undef UBN_V3
  }
  // forward: groups of 2 samples (80 registers, 6 CTAs/SM won the occupancy sweep); backward: groups of 4 (the vector reductions
  // need no result, deeper batching costs nothing).  Round 1's other variants (groups of 1 / 8, the env switch) are gone.
#define UBN_V2(P)                                                                                                       \
  case P:                                                                                                               \
    return backward ? launch_v2<P, 4>(backward, rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, \
                                      feat, grad_grid, o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, st)    \
                    : launch_v2<P, 2>(backward, rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, \
                                      feat, grad_grid, o_density, o_alpha, o_weight, o_ray_id, o_step_id, o_t, o_inner, st)
  switch (g.P) {
    UBN_V2(1);
    UBN_V2(3);
    UBN_V2(5);
    UBN_V2(7);
    UBN_V2(9);
    default: return -1;
  }
#undef UBN_V2
}

}  // namespace ubn
