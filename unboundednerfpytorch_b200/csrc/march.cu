// march.cu -- fused per-ray march kernels of libubnerf_b200.so (the hot path).
//
// One warp owns one ray and walks its S nominal samples in chunks of 32 (lane = sample), fusing what the
// reference does with ~40 separate torch / extension launches per model.forward:
//   FourierGridModel.sample_ray (FourierGrid_model.py:509-552) / DirectContractedVoxGO.sample_ray
//   (dcvgo.py:228-262)  -> cumdist_thres (dcvgo.py:286-294, ub360_utils_kernel.cu:13-32)
//   -> mask_cache lookup (dcvgo.py:297-302, render_utils_kernel.cu:374-392)
//   -> density grid read (grid.py:50-61 / FourierGrid_grid.py:60-78)
//   -> Raw2Alpha (dvgo.py:430-443, render_utils_kernel.cu:431-443)
//   -> fast_color_thres mask -> Alphas2Weights (dvgo.py:472-479, render_utils_kernel.cu:577-605)
//   -> fast_color_thres mask -> feature grid read (k0) for the survivors, compacted in (ray, step) order.
// Pass A = everything up to the weights (dense per-sample records + per-ray survivor counts); a tiny scan
// turns the counts into offsets; pass B = warp-cooperative k0 read for the survivors (lane = corner x
// channel-quad, one 128-bit load per sample-slab) and the compacted outputs the model returns.
// The backward kernels mirror them: exact reverse transmittance scan + raw2alpha' + atomic scatter into
// the density grid gradient, and vector-red scatter of the feature gradient into the k0 grid gradient.
//
// Order-sensitive float recurrences (transmittance product with early stop, cumdist accumulate-reset)
// are evaluated in the reference's sequential order (a warp-uniform loop over the lanes) so that the
// index-like outputs (which samples are listed / scanned / kept) stay bit-exact.
#include <algorithm>
#include <type_traits>

#include "march_common.cuh"
#include "tensorf.cuh"

namespace ubn {

__device__ __forceinline__ float grid_density(const GridView& g, float x, float y, float z) { return grid_density_at(g, x, y, z); }

// ------------------------------------------------------------------------------------------------
// pass A forward
// ------------------------------------------------------------------------------------------------
// kP > 0: compile-time slab count + contiguous single-channel grid -> grid_density_fast (march_common.cuh); kP = 0: generic layout;
// kP < 0: the TensoRF density tf (C = 1) instead of g, read as ubn_tensorf_fwd reads it (tensorf.cuh's tf_read) with W = -kP
// components per load (4: 128-bit records, tf_records4).  Smp: the sampling policy (ContractedSampler / NdcSampler / BoxSampler,
// march_common.cuh).
template <class Smp, int kP>
__global__ void __launch_bounds__(32 * kMarchWarps) k_march_density_fwd(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ t_table,
    GridView g, const uint8_t* __restrict__ mask_world, MarchParams p, int64_t n_rays,
    float* __restrict__ o_density, float* __restrict__ o_alpha, float* __restrict__ o_weight,
    float* __restrict__ o_T, uint8_t* __restrict__ o_flags, float* __restrict__ o_last,
    int32_t* __restrict__ o_nkeep, TfView tf) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const Ray r = Smp::load(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int S = p.S;      // record stride
  const int n = r.n;      // samples of this ray (warp-uniform): S, or the box march's n_steps

  float T_cum = 1.f;      // warp-uniform
  bool done = false;      // warp-uniform: early stop reached
  float cum = 0.f;        // cumdist accumulator (warp-uniform)
  bool carry_over = false;   // cumdist flag for the first sample of the next chunk
  int n_keep = 0;

  for (int base = 0; base < n; base += 32) {
    const int s = base + lane;
    const MarchSample ms = march_chunk_point<Smp>(r, t_table, mask_world, p, base, lane, cum, carry_over);
    const bool valid = ms.valid, inner = ms.inner, queried = ms.queried;
    const float x = ms.x, y = ms.y, z = ms.z;

    float dens = 0.f, alpha = 0.f;
    if (queried) {
      if constexpr (kP < 0) {
        const float c[3] = {tf_coord(tf, 0, x), tf_coord(tf, 1, y), tf_coord(tf, 2, z)};
        tf_read<1, -kP>(tf, c, nullptr, &dens);
      } else {
        dens = kP > 0 ? grid_density_fast<(kP > 0 ? kP : 1)>(g, x, y, z) : grid_density(g, x, y, z);
      }
      dens = Smp::density(p, dens, x, y, z);
      alpha = march_alpha(dens, p);
    }
    const bool listed = march_listed(queried, alpha, p);

    float myT, myW;
    bool scanned;
    transmittance_scan(listed, alpha, lane, T_cum, done, myT, myW, scanned);
    const bool keep = listed && (p.thres > 0.f ? (myW > p.thres) : true);
    n_keep += __popc(__ballot_sync(0xffffffffu, keep));

    if (valid) {
      const int64_t o = ray * S + s;
      o_density[o] = dens;
      o_alpha[o] = alpha;
      o_weight[o] = myW;
      o_T[o] = myT;
      o_flags[o] = (uint8_t)((queried ? UBN_FLAG_QUERIED : 0) | (listed ? UBN_FLAG_LISTED : 0) |
                             (scanned ? UBN_FLAG_SCANNED : 0) | (keep ? UBN_FLAG_KEEP : 0) |
                             (inner ? UBN_FLAG_INNER : 0));
    }
  }
  if (lane == 0) {
    o_last[ray] = T_cum;
    o_nkeep[ray] = n_keep;
  }
}

// ------------------------------------------------------------------------------------------------
// pass B forward / backward (feature grid, warp-cooperative)
// ------------------------------------------------------------------------------------------------
template <bool kBackward>
__global__ void __launch_bounds__(32 * kMarchWarps) k_march_feature(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ t_table,
    GridView g, MarchParams p, int64_t n_rays, const uint8_t* __restrict__ flags,
    const int64_t* __restrict__ offsets, const float* __restrict__ density, const float* __restrict__ alpha,
    const float* __restrict__ weight, float* __restrict__ feat /* out (fwd) or grad in (bwd) */,
    float* __restrict__ grad_grid, float* __restrict__ o_density, float* __restrict__ o_alpha,
    float* __restrict__ o_weight, int64_t* __restrict__ o_ray_id, int64_t* __restrict__ o_step_id,
    float* __restrict__ o_t, uint8_t* __restrict__ o_inner) {
  extern __shared__ float4 s_idx[];   // [kMarchWarps][32][P]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + w;
  if (ray >= n_rays) return;
  float4* my_idx = s_idx + (size_t)w * 32 * g.P;
  const int corner = lane >> 2, quad = lane & 3;
  const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
  const bool quad_on = quad < (g.C >> 2);
  const Ray r = load_ray(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int S = p.S;
  int64_t out_base = offsets[ray];
  const int64_t out_end = offsets[ray + 1];
  if (out_base == out_end) return;

  for (int base = 0; base < S && out_base < out_end; base += 32) {
    const int s = base + lane;
    const uint8_t f = (s < S) ? flags[ray * S + s] : 0;
    const bool keep = (f & UBN_FLAG_KEEP) != 0;
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (km == 0) continue;
    const int rank = __popc(km & ((1u << lane) - 1));
    if (keep) {
      float x, y, z;
      const float t = t_table[s];
      sample_point(r, t, p, x, y, z);
      const float nx = norm_coord(x, g.mn[0], g.len[0]);
      const float ny = norm_coord(y, g.mn[1], g.len[1]);
      const float nz = norm_coord(z, g.mn[2], g.len[2]);
      for (int sl = 0; sl < g.P; ++sl)
        my_idx[rank * g.P + sl] = make_float4(src_index(fourier_gamma(sl, nx), g.X), src_index(fourier_gamma(sl, ny), g.Y),
                                              src_index(fourier_gamma(sl, nz), g.Z), 0.f);
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
    __syncwarp();
    const int n_here = __popc(km);
    for (int i = 0; i < n_here; ++i) {
      const int64_t pt = out_base + i;
      float4 acc = make_float4(0, 0, 0, 0);
      float4 gin = make_float4(0, 0, 0, 0);
      if (kBackward) {
        if (quad_on) gin = *reinterpret_cast<const float4*>(feat + pt * g.C + quad * 4);
        gin.x = slab_mean_scale(gin.x, g.P); gin.y = slab_mean_scale(gin.y, g.P); gin.z = slab_mean_scale(gin.z, g.P); gin.w = slab_mean_scale(gin.w, g.P);
      }
      for (int sl = 0; sl < g.P; ++sl) {
        const float4 ci = my_idx[i * g.P + sl];
        const Cell c = locate(ci.x, ci.y, ci.z);
        const bool in = corner_inside(c, bx, by, bz, g.X, g.Y, g.Z) && quad_on;
        const float wgt = corner_weight(c, bx, by, bz);
        const int64_t v = ((int64_t)(c.x0 + bx) * g.Y + (c.y0 + by)) * g.Z + (c.z0 + bz);
        if (!kBackward) {
          if (in) {
            const float4 val = __ldg(reinterpret_cast<const float4*>(g.data + sl * g.sp + v * g.sv + quad * 4));
            acc.x += val.x * wgt; acc.y += val.y * wgt; acc.z += val.z * wgt; acc.w += val.w * wgt;
          }
        } else {
          if (in) red_add_v4(grad_grid + sl * g.sp + v * g.sv + quad * 4,
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
          *reinterpret_cast<float4*>(feat + pt * g.C + quad * 4) = acc;
        }
      }
    }
    __syncwarp();
    out_base += n_here;
  }
}

// ------------------------------------------------------------------------------------------------
// pass A backward
// ------------------------------------------------------------------------------------------------
constexpr int kMaxChunks = 128;   // S <= 4096

// kRuns (kP > 0 only): launch 1 of the run scatter.  The reverse scan (lane = sample of a 32-sample chunk) writes every sample's
// density gradient, already divided by the slab count, to gd_out[ray * S + s] and scatters nothing; k_march_density_scatter
// (launch 2) adds them into the grid.  Otherwise every sample scatters its own 8 corners in every slab right here.
template <class Smp, int kP, bool kRuns>
__global__ void __launch_bounds__(32 * kMarchWarps) k_march_density_bwd(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ t_table,
    GridView g /* data = grad grid */, MarchParams p, int64_t n_rays, const float* __restrict__ density,
    const float* __restrict__ alpha, const float* __restrict__ weight, const float* __restrict__ T,
    const uint8_t* __restrict__ flags, const float* __restrict__ last, const int64_t* __restrict__ offsets,
    const float* __restrict__ g_weight, const float* __restrict__ g_alpha, const float* __restrict__ g_density,
    const float* __restrict__ g_last, float* __restrict__ grad_grid, float* __restrict__ gd_out) {
  __shared__ int s_cnt[kMarchWarps][kMaxChunks];
  __shared__ __align__(16) float2 s_pair[kMarchWarps][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + w;
  if (ray >= n_rays) return;
  const Ray r = Smp::load(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int S = p.S;                                       // record stride
  const int n = r.n;                                       // samples of this ray (S, or the box march's n_steps)
  const int n_chunks = (n + 31) / 32;

  // exclusive prefix of KEEP counts per chunk -> compact index of every kept sample
  int run = 0;
  for (int c = 0; c < n_chunks; ++c) {
    const int s = c * 32 + lane;
    const bool keep = (s < n) && (flags[ray * S + s] & UBN_FLAG_KEEP);
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_cnt[w][c] = run;
    run += __popc(km);
  }
  __syncwarp();
  const int64_t off = offsets[ray];

  float back_cum = (g_last ? g_last[ray] : 0.f) * last[ray];   // warp-uniform
  for (int c = n_chunks - 1; c >= 0; --c) {
    const int s = c * 32 + lane;
    const bool valid = s < n;
    const int64_t i = ray * S + s;
    const uint8_t f = valid ? flags[i] : 0;
    const bool keep = f & UBN_FLAG_KEEP;
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    const int64_t ci = off + s_cnt[w][c] + __popc(km & ((1u << lane) - 1));
    const float gw = (keep && g_weight) ? g_weight[ci] : 0.f;
    const float wt = valid ? weight[i] : 0.f;
    // reverse sequential accumulation over the scanned samples (alpha2weight_backward order).  The chain is inherently serial
    // (one fp32 fma per scanned sample, in the reference's order), so every lane runs it redundantly on warp-uniform operands.
    // They used to be fetched with two shuffles per sample from a data-dependent lane (profiled: mio_throttle + short
    // scoreboard stalls dominated); now the chunk's 32 (grad, weight) pairs go through 256 bytes of shared
    // memory and come back as 16 broadcast LDS.128 in a fully unrolled loop.
    const unsigned m = __ballot_sync(0xffffffffu, (f & UBN_FLAG_SCANNED) != 0);
    float my_back = 0.f;
    if (m) {
      s_pair[w][lane] = make_float2(gw, wt);
      __syncwarp();
#pragma unroll
      for (int jj = 15; jj >= 0; --jj) {
        const float4 v = *reinterpret_cast<const float4*>(&s_pair[w][2 * jj]);      // pairs 2jj (x, y) and 2jj + 1 (z, w)
        if (m & (2u << (2 * jj))) {
          if (lane == 2 * jj + 1) my_back = back_cum;
          back_cum = fmaf(v.z, v.w, back_cum);            // float fma (render_utils_kernel.cu:674)
        }
        if (m & (1u << (2 * jj))) {
          if (lane == 2 * jj) my_back = back_cum;
          back_cum = fmaf(v.x, v.y, back_cum);
        }
      }
      __syncwarp();
    }
    float gd = 0.f;
    if (f & UBN_FLAG_QUERIED) {
      const float a = alpha[i];
      float ga = (keep && g_alpha) ? g_alpha[ci] : 0.f;
      if (f & UBN_FLAG_SCANNED) ga += (float)(gw * T[i] - my_back / (1 - a + 1e-10));
      const float d = density[i];
      gd = (keep && g_density) ? g_density[ci] : 0.f;
      if (ga != 0.f) {
        const float e = expf(d + p.shift);
        gd += (float)(fmin((double)e, 1e10) * powf(1 + e, -p.interval - 1) * p.interval * ga);
      }
    }
    if (kRuns) {
      if (valid) gd_out[i] = slab_mean_scale(gd, g.P);
      continue;
    }
    if (gd == 0.f) continue;
    // scatter into the density grid gradient (adjoint of grid_density)
    float x, y, z;
    bool inner;
    Smp::point(r, t_table, s, p, x, y, z, inner);
    const float nx = norm_coord(x, g.mn[0], g.len[0]);
    const float ny = norm_coord(y, g.mn[1], g.len[1]);
    const float nz = norm_coord(z, g.mn[2], g.len[2]);
    gd = slab_mean_scale(gd, g.P);
    if (kP > 0) {
      grid_density_scatter_fast<(kP > 0 ? kP : 1)>(grad_grid, g, nx, ny, nz, gd);
      continue;
    }
    for (int sl = 0; sl < g.P; ++sl) {
      const float cx = src_index(fourier_gamma(sl, nx), g.X);
      const float cy = src_index(fourier_gamma(sl, ny), g.Y);
      const float cz = src_index(fourier_gamma(sl, nz), g.Z);
      if (g.sv == 1) trilerp1_scatter_pairs(grad_grid + sl * g.sp, g.X, g.Y, g.Z, cx, cy, cz, gd);
      else trilerp1_scatter(grad_grid + sl * g.sp, g.sv, g.X, g.Y, g.Z, cx, cy, cz, gd);
    }
  }
}

// Launch 2 of the run scatter: adds launch 1's per-sample gradients gd[ray * S + s] into the density-grid gradient.
// Warp = ray, lane = a run of L = ceil(n / 32) consecutive samples.  The lane keeps the cell it is in open in registers (cell
// index + its 8 corner sums): samples that stay in the cell -- a large share of the steps in slab 0 and the lowest sin / cos slabs
// at half-voxel spacing -- are added in registers, and a cell leaves as four pair reductions only when the ray moves on.  The
// scatter is bound by L2 reduction requests, so it needs both few requests and requests that hit in L2.
// Frequency-major: blockIdx.y = k * n_split + part.  Pass k = 0 scatters slab 0, pass k > 0 the sin / cos slab pair 2k - 1 / 2k
// (one sincosf per axis serves both).  The CTAs of one blockIdx.y are scheduled before those of the next, so the live part of the
// gradient is one slab or one pair instead of all P slabs (129 MB for the 153^3 x 9 truck grid, against the H100's 50 MB L2).
// n_split > 1 cuts it further into x-ranges, as k_march_feature_bwd_slab does: part `part` adds only the cells whose base voxel
// lies in its range of x planes.
template <class Smp, int kP>
__global__ void __launch_bounds__(32 * kMarchWarps) k_march_density_scatter(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ t_table, GridView g,
    MarchParams p, int64_t n_rays, const float* __restrict__ gd_in, float* __restrict__ grad_grid, int n_split) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const int k = blockIdx.y / n_split, part = blockIdx.y - k * n_split;
  const int v_lo = (int)(((int64_t)(g.X - 1) * part) / n_split) * g.Y * g.Z;
  const int v_hi = (part + 1 == n_split) ? 0x7fffffff : (int)(((int64_t)(g.X - 1) * (part + 1)) / n_split) * g.Y * g.Z;
  const Ray r = Smp::load(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int n = r.n;
  const int L = (n + 31) / 32;
  const float* gd_ray = gd_in + ray * p.S;
  const int dY = g.Z, dX = g.Y * g.Z;
  struct Run { int v; float c[8]; };
  auto flush = [&](const Run& run, float* slab) {          // the four (x, y) edges of the open cell as pair reductions
    float* rec = slab + run.v;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float* a = rec + (e >> 1) * dX + (e & 1) * dY;
      const float w0 = run.c[2 * e], w1 = run.c[2 * e + 1];
      const bool odd = (reinterpret_cast<uintptr_t>(a) & 4) != 0;
      red_add_v2(a - (odd ? 1 : 0), odd ? 0.f : w0, odd ? w0 : w1);
      if (odd) atomicAdd(a + 1, w1);
    }
  };
  auto visit = [&](Run& run, float* slab, float cx, float cy, float cz, float gd) {
    const CellR c = make_cell(cx, cy, cz, g.X, g.Y, g.Z);
    if (c.v < v_lo || c.v >= v_hi) return;                 // another part's cell
    float wgt[8];
#pragma unroll
    for (int e = 0; e < 4; ++e) {                          // same products as grid_density_scatter_fast: ((wz * wy) * wx) * gd
      const int bx = e >> 1, by = e & 1;
      const float wy = by ? c.fy : 1.f - c.fy, wx = bx ? c.fx : 1.f - c.fx;
      wgt[2 * e] = (((1.f - c.fz) * wy) * wx) * gd;
      wgt[2 * e + 1] = ((c.fz * wy) * wx) * gd;
    }
    if (c.v == run.v) {
#pragma unroll
      for (int q = 0; q < 8; ++q) run.c[q] += wgt[q];
    } else {
      if (run.v >= 0) flush(run, slab);
      run.v = c.v;
#pragma unroll
      for (int q = 0; q < 8; ++q) run.c[q] = wgt[q];
    }
  };
  Run ra, rb;
  ra.v = -1; rb.v = -1;
  float* slab_a = grad_grid + (int64_t)(k == 0 ? 0 : 2 * k - 1) * g.sp;
  float* slab_b = grad_grid + (int64_t)(2 * k) * g.sp;
  const float m = (float)(1 << (k > 0 ? k - 1 : 0));
  for (int i = 0; i < L; ++i) {
    const int s = lane * L + i;
    if (s >= n) break;
    const float gd = gd_ray[s];
    if (gd == 0.f) continue;
    float x, y, z;
    bool inner;
    Smp::point(r, t_table, s, p, x, y, z, inner);
    const float nx = norm_coord(x, g.mn[0], g.len[0]);
    const float ny = norm_coord(y, g.mn[1], g.len[1]);
    const float nz = norm_coord(z, g.mn[2], g.len[2]);
    if (kP == 1 || k == 0) {
      visit(ra, slab_a, src_index(nx, g.X), src_index(ny, g.Y), src_index(nz, g.Z), gd);
    } else {
      float sx, cx, sy, cy, sz, cz;
      sincosf(__fmul_rn(m, nx), &sx, &cx);
      sincosf(__fmul_rn(m, ny), &sy, &cy);
      sincosf(__fmul_rn(m, nz), &sz, &cz);
      visit(ra, slab_a, src_index(sx, g.X), src_index(sy, g.Y), src_index(sz, g.Z), gd);
      visit(rb, slab_b, src_index(cx, g.X), src_index(cy, g.Y), src_index(cz, g.Z), gd);
    }
  }
  if (ra.v >= 0) flush(ra, slab_a);
  if (rb.v >= 0) flush(rb, slab_b);
}

// Launch 2 of the TensoRF density's backward.  Launch 1 (k_march_density_bwd<BoxSampler, 1, true>, the dense grid's launch 1) left
// every sample's density gradient in gd_in[ray * S + s].  Warp = ray, lane = every 32nd step of the ray's own n_steps: a record
// with a nonzero gradient recomputes its point from (ray, step) and runs the per-sample adjoint of ubn_tensorf_bwd (tensorf.cuh's
// tf_sample_bwd): plane gradients reduced straight into grads, vector gradients into copy blockIdx % vec_copies.
template <int W>
__global__ void __launch_bounds__(32 * kMarchWarps) k_march_box_tensorf_scatter(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, TfView t, MarchParams p, int64_t n_rays,
    const float* __restrict__ gd_in, TfGrads gr, float* __restrict__ vcopies, int64_t copy_len, int vec_copies) {
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const Ray r = BoxSampler::load(rays_o + 3 * ray, rays_d + 3 * ray, p);
  float* vc = vcopies + (int64_t)(blockIdx.x % vec_copies) * copy_len;
  for (int s = threadIdx.x & 31; s < r.n; s += 32) {
    const float gd = gd_in[ray * p.S + s];
    if (gd == 0.f) continue;
    float x, y, z;
    bool inner;
    BoxSampler::point(r, nullptr, s, p, x, y, z, inner);
    const float c[3] = {tf_coord(t, 0, x), tf_coord(t, 1, y), tf_coord(t, 2, z)};
    tf_sample_bwd<1, W>(t, c, &gd, nullptr, nullptr, 0, gr, vc);
  }
}

// the fast density paths need: contiguous single channel, >= 2 voxels per axis, 32-bit offsets inside a slab, and an 8-byte aligned
// buffer (the pair reductions align on the ADDRESS, so odd-sized slabs -- 153^3 -- are fine: the +0 half of a pair may fall on the
// last voxel of the previous slab, never before the buffer)
static int density_fast_slabs(const GridView& g) {
  const bool ok = g.sv == 1 && g.X >= 2 && g.Y >= 2 && g.Z >= 2 && (int64_t)g.X * g.Y * g.Z < (1ll << 31) &&
                  ((uintptr_t)g.data & 7) == 0;
  if (!ok) return 0;
  return (g.P == 1 || g.P == 3 || g.P == 5 || g.P == 7 || g.P == 9) ? g.P : 0;
}

// second-generation feature kernels (march_feature.cu); -1 = configuration not covered, use the generic kernel
int march_feature_v2(bool backward, const float* rays_o, const float* rays_d, const float* t_table, const GridView& g,
                     const MarchParams& p, int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                     const float* density, const float* alpha, const float* weight, float* feat, float* grad_grid,
                     float* o_density, float* o_alpha, float* o_weight, int64_t* o_ray_id, int64_t* o_step_id, float* o_t,
                     uint8_t* o_inner, cudaStream_t st);

void set_feature_kernel(int v);
int get_feature_kernel();
static int g_density_scatter = 1;      // 1 = run-merging two-launch scatter (default), 0 = per-sample scatter
static int get_density_scatter() { return g_density_scatter; }

static bool feature_grid_ok(const GridView& g) {
  if (g.C == 3 || g.C == 9 || g.C == 15)   // march_feature.cu's scalar-channel kernels: 4-byte aligned records, odd P <= 11, >= 2 voxels per axis
    return g.sc == 1 && g.sv == g.C && g.P >= 1 && g.P <= 11 && (g.P & 1) && g.X >= 2 && g.Y >= 2 && g.Z >= 2 &&
           ((uintptr_t)g.data & 3) == 0;
  return g.sc == 1 && g.sv == g.C && (g.C == 4 || g.C == 8 || g.C == 12 || g.C == 16) && g.P <= 16 &&
         ((uintptr_t)g.data & 15) == 0 && (g.sp % 4) == 0;
}

template <class Smp>
static int launch_density_fwd(const float* rays_o, const float* rays_d, const float* t_table, const GridView& g,
                              const uint8_t* mask_world, const MarchParams& p, int64_t n_rays, float* density, float* alpha,
                              float* weight, float* T, uint8_t* flags, float* alphainv_last, int32_t* n_keep, cudaStream_t st) {
#define UBN_DFWD(P)                                                                                              \
  k_march_density_fwd<Smp, P><<<blocks_for(n_rays, kMarchWarps), 32 * kMarchWarps, 0, st>>>(                   \
      rays_o, rays_d, t_table, g, mask_world, p, n_rays, density, alpha, weight, T, flags, alphainv_last, n_keep, TfView{})
  if constexpr (std::is_same<Smp, BoxSampler>::value) {      // DVGO's density: one contiguous slab, the fast path only
    if (density_fast_slabs(g) != 1) return finish(cudaErrorInvalidValue);
    UBN_DFWD(1);
  } else {
    switch (density_fast_slabs(g)) {
      case 1: UBN_DFWD(1); break;
      case 3: UBN_DFWD(3); break;
      case 5: UBN_DFWD(5); break;
      case 7: UBN_DFWD(7); break;
      case 9: UBN_DFWD(9); break;
      default: UBN_DFWD(0); break;
    }
  }
#undef UBN_DFWD
  UBN_LAUNCH_CHECK();
  return 0;
}

// x-ranges per frequency pass of k_march_density_scatter.  A pass reduces into its live part of the gradient (one slab, or a
// sin / cos pair) while the per-sample gradients stream through the same L2; n_split = ceil((live part + per-sample gradients) /
// (3/4 of the L2)).  A rule fit to measurements on an H100 (50 MB L2, launch 2's time by split count): truck, 153^3 x 9 slabs,
// 8192 x 512 samples -> 2 (1 / 2 / 4: 1.66 / 1.57 / 1.88 ms for both launches); bicycle, one 320^3 slab -> 4 (1 / 2 / 4 / 8: 0.33 /
// 0.28 / 0.29 / 0.40 ms).  Fewer parts leave the reductions missing in L2, more repeat the per-sample work of the pass.
static int density_scatter_split(const GridView& g, int kP, int64_t n_samples, int& n_split) {
  int dev = 0, l2 = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev);
  if (e != cudaSuccess) return finish(e);
  const int64_t live = (int64_t)(kP > 1 ? 2 : 1) * g.X * g.Y * g.Z * (int64_t)sizeof(float);
  const int64_t need = live + n_samples * (int64_t)sizeof(float);
  const int64_t budget = std::max<int64_t>((int64_t)l2 * 3 / 4, 1);
  n_split = (int)std::min<int64_t>((need + budget - 1) / budget, g.X - 1);
  return 0;
}

template <class Smp, int kP>
static int launch_density_bwd_p(const float* rays_o, const float* rays_d, const float* t_table, const GridView& g,
                                const MarchParams& p, int64_t n_rays, const float* density, const float* alpha,
                                const float* weight, const float* T, const uint8_t* flags, const float* alphainv_last,
                                const int64_t* offsets, const float* g_weight, const float* g_alpha, const float* g_density,
                                const float* g_last, float* grad_density_grid, float* gd_scratch, cudaStream_t st) {
  const unsigned blocks = blocks_for(n_rays, kMarchWarps);
  // run-merging scatter (two launches) by default; ubn_set_density_scatter(0) selects the per-sample scatter (A/B, tests)
  if constexpr (kP > 0) {
    if (get_density_scatter() == 1) {
      if (!gd_scratch) return finish(cudaErrorInvalidValue);
      int n_split = 1;
      if (const int e = density_scatter_split(g, kP, n_rays * p.S, n_split)) return e;
      k_march_density_bwd<Smp, kP, true><<<blocks, 32 * kMarchWarps, 0, st>>>(
          rays_o, rays_d, t_table, g, p, n_rays, density, alpha, weight, T, flags, alphainv_last, offsets, g_weight, g_alpha,
          g_density, g_last, grad_density_grid, gd_scratch);
      UBN_LAUNCH_CHECK();
      k_march_density_scatter<Smp, kP><<<dim3(blocks, (kP + 1) / 2 * n_split), 32 * kMarchWarps, 0, st>>>(
          rays_o, rays_d, t_table, g, p, n_rays, gd_scratch, grad_density_grid, n_split);
      UBN_LAUNCH_CHECK();
      return 0;
    }
  }
  k_march_density_bwd<Smp, kP, false><<<blocks, 32 * kMarchWarps, 0, st>>>(
      rays_o, rays_d, t_table, g, p, n_rays, density, alpha, weight, T, flags, alphainv_last, offsets, g_weight, g_alpha,
      g_density, g_last, grad_density_grid, nullptr);
  UBN_LAUNCH_CHECK();
  return 0;
}

template <class Smp>
static int launch_density_bwd(const float* rays_o, const float* rays_d, const float* t_table, const GridView& g,
                              const MarchParams& p, int64_t n_rays, const float* density, const float* alpha, const float* weight,
                              const float* T, const uint8_t* flags, const float* alphainv_last, const int64_t* offsets,
                              const float* g_weight, const float* g_alpha, const float* g_density, const float* g_last,
                              float* grad_density_grid, float* gd_scratch, cudaStream_t st) {
#define UBN_DBWD(P)                                                                                                      \
  return launch_density_bwd_p<Smp, P>(rays_o, rays_d, t_table, g, p, n_rays, density, alpha, weight, T, flags,          \
                                      alphainv_last, offsets, g_weight, g_alpha, g_density, g_last, grad_density_grid,  \
                                      gd_scratch, st)
  if constexpr (std::is_same<Smp, BoxSampler>::value) {
    if (density_fast_slabs(g) != 1) return finish(cudaErrorInvalidValue);
    UBN_DBWD(1);
  } else {
    switch (density_fast_slabs(g)) {
      case 1: UBN_DBWD(1);
      case 3: UBN_DBWD(3);
      case 5: UBN_DBWD(5);
      case 7: UBN_DBWD(7);
      case 9: UBN_DBWD(9);
      default: UBN_DBWD(0);
    }
  }
#undef UBN_DBWD
}

}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_set_feature_kernel(int variant) {
  if (variant < 0 || variant > 6) return finish(cudaErrorInvalidValue);
  set_feature_kernel(variant);
  return 0;
}
int ubn_get_feature_kernel(void) { return get_feature_kernel(); }

int ubn_set_density_scatter(int variant) {
  if (variant < 0 || variant > 1) return finish(cudaErrorInvalidValue);
  g_density_scatter = variant;
  return 0;
}
int ubn_get_density_scatter(void) { return g_density_scatter; }

int ubn_march_density_fwd(const float* rays_o, const float* rays_d, const float* t_table, const float* density_grid,
                          const UbnGridDesc* density_desc, const uint8_t* mask_world, const UbnMarchCfg* cfg,
                          int64_t n_rays, float* density, float* alpha, float* weight, float* T, uint8_t* flags,
                          float* alphainv_last, int32_t* n_keep, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(density_grid, density_desc);
  if (g.C != 1) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_params(cfg);
  if (p.use_mask && !mask_world) return finish(cudaErrorInvalidValue);
  return launch_density_fwd<ContractedSampler>(rays_o, rays_d, t_table, g, mask_world, p, n_rays, density, alpha, weight, T,
                                               flags, alphainv_last, n_keep, as_stream(stream));
}

int ubn_march_feature_fwd(const float* rays_o, const float* rays_d, const float* t_table, const float* k0_grid,
                          const UbnGridDesc* k0_desc, const UbnMarchCfg* cfg, int64_t n_rays, const uint8_t* flags,
                          const int64_t* offsets, const float* density, const float* alpha, const float* weight,
                          float* k0_feat, float* out_density, float* out_alpha, float* out_weight, int64_t* ray_id,
                          int64_t* step_id, float* out_t, uint8_t* out_inner, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(k0_grid, k0_desc);
  if (!feature_grid_ok(g) || ((uintptr_t)k0_feat & 15)) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_params(cfg);
  {
    const int e = march_feature_v2(false, rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight,
                                   k0_feat, nullptr, out_density, out_alpha, out_weight, ray_id, step_id, out_t, out_inner,
                                   as_stream(stream));
    if (e >= 0) return e;
  }
  if (g.C % 4) return finish(cudaErrorInvalidValue);     // C = 3 / 9 / 15 beyond 32-bit slab offsets: no kernel
  const size_t smem = sizeof(float4) * kMarchWarps * 32 * g.P;
  k_march_feature<false><<<blocks_for(n_rays, kMarchWarps), 32 * kMarchWarps, smem, as_stream(stream)>>>(
      rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, density, alpha, weight, k0_feat, nullptr, out_density,
      out_alpha, out_weight, ray_id, step_id, out_t, out_inner);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_march_feature_bwd(const float* rays_o, const float* rays_d, const float* t_table, const UbnGridDesc* k0_desc,
                          const UbnMarchCfg* cfg, int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                          const float* grad_feat, float* grad_k0, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(grad_k0, k0_desc);
  if (!feature_grid_ok(g) || ((uintptr_t)grad_feat & 15)) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_params(cfg);
  {
    const int e = march_feature_v2(true, rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, nullptr, nullptr, nullptr,
                                   const_cast<float*>(grad_feat), grad_k0, nullptr, nullptr, nullptr, nullptr, nullptr,
                                   nullptr, nullptr, as_stream(stream));
    if (e >= 0) return e;
  }
  if (g.C % 4) return finish(cudaErrorInvalidValue);     // C = 3 / 9 / 15 beyond 32-bit slab offsets: no kernel
  const size_t smem = sizeof(float4) * kMarchWarps * 32 * g.P;
  k_march_feature<true><<<blocks_for(n_rays, kMarchWarps), 32 * kMarchWarps, smem, as_stream(stream)>>>(
      rays_o, rays_d, t_table, g, p, n_rays, flags, offsets, nullptr, nullptr, nullptr, const_cast<float*>(grad_feat),
      grad_k0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_march_density_bwd(const float* rays_o, const float* rays_d, const float* t_table,
                          const UbnGridDesc* density_desc, const UbnMarchCfg* cfg, int64_t n_rays, const float* density,
                          const float* alpha, const float* weight, const float* T, const uint8_t* flags,
                          const float* alphainv_last, const int64_t* offsets, const float* g_weight,
                          const float* g_alpha, const float* g_density, const float* g_last, float* grad_density_grid,
                          float* gd_scratch, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(grad_density_grid, density_desc);
  if (g.C != 1) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_params(cfg);
  if (p.S > 32 * kMaxChunks) return finish(cudaErrorInvalidValue);
  return launch_density_bwd<ContractedSampler>(rays_o, rays_d, t_table, g, p, n_rays, density, alpha, weight, T, flags,
                                               alphainv_last, offsets, g_weight, g_alpha, g_density, g_last, grad_density_grid,
                                               gd_scratch, as_stream(stream));
}

int ubn_march_ndc_density_fwd(const float* rays_o, const float* rays_d, const float* density_grid,
                              const UbnGridDesc* density_desc, const float* act_shift_grid, const UbnGridDesc* act_shift_desc,
                              const uint8_t* mask_world, const UbnNdcMarchCfg* cfg, int64_t n_rays, float* density,
                              float* alpha, float* weight, float* T, uint8_t* flags, float* alphainv_last, int32_t* n_keep,
                              void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(density_grid, density_desc);
  const GridView sg = make_view(act_shift_grid, act_shift_desc);
  if (g.C != 1 || g.P != 1 || sg.C != 1 || sg.P != 1 || cfg->n_samples < 2) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_ndc_params(cfg, sg);
  if (p.use_mask && !mask_world) return finish(cudaErrorInvalidValue);
  return launch_density_fwd<NdcSampler>(rays_o, rays_d, nullptr, g, mask_world, p, n_rays, density, alpha, weight, T, flags,
                                         alphainv_last, n_keep, as_stream(stream));
}

int ubn_march_ndc_density_bwd(const float* rays_o, const float* rays_d, const UbnGridDesc* density_desc,
                              const UbnNdcMarchCfg* cfg, int64_t n_rays, const float* density, const float* alpha,
                              const float* weight, const float* T, const uint8_t* flags, const float* alphainv_last,
                              const int64_t* offsets, const float* g_weight, const float* g_alpha, const float* g_last,
                              float* grad_density_grid, float* gd_scratch, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(grad_density_grid, density_desc);
  if (g.C != 1 || g.P != 1 || cfg->n_samples < 2) return finish(cudaErrorInvalidValue);
  GridView none{};
  const MarchParams p = make_ndc_params(cfg, none);
  if (p.S > 32 * kMaxChunks) return finish(cudaErrorInvalidValue);
  return launch_density_bwd<NdcSampler>(rays_o, rays_d, nullptr, g, p, n_rays, density, alpha, weight, T, flags, alphainv_last,
                                         offsets, g_weight, g_alpha, nullptr, g_last, grad_density_grid, gd_scratch,
                                         as_stream(stream));
}

// S_max (cfg->s_max) is the record stride of pass A; the backward's chunk table holds 32 * kMaxChunks samples of a ray
static bool box_cfg_ok(const UbnBoxMarchCfg* c) { return c->s_max >= 1 && c->s_max <= 32 * kMaxChunks && c->stepdist > 0.f; }

int ubn_march_box_density_fwd(const float* rays_o, const float* rays_d, const float* density_grid, const UbnGridDesc* density_desc,
                              const uint8_t* mask_world, const UbnBoxMarchCfg* cfg, int64_t n_rays, float* density, float* alpha,
                              float* weight, float* T, uint8_t* flags, float* alphainv_last, int32_t* n_keep, int32_t* overflow,
                              void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(density_grid, density_desc);
  if (g.C != 1 || g.P != 1 || !box_cfg_ok(cfg) || !overflow) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_box_params(cfg, overflow);
  if (p.use_mask && !mask_world) return finish(cudaErrorInvalidValue);
  return launch_density_fwd<BoxSampler>(rays_o, rays_d, nullptr, g, mask_world, p, n_rays, density, alpha, weight, T, flags,
                                        alphainv_last, n_keep, as_stream(stream));
}

int ubn_march_box_density_bwd(const float* rays_o, const float* rays_d, const UbnGridDesc* density_desc,
                              const UbnBoxMarchCfg* cfg, int64_t n_rays, const float* density, const float* alpha,
                              const float* weight, const float* T, const uint8_t* flags, const float* alphainv_last,
                              const int64_t* offsets, const float* g_weight, const float* g_alpha, const float* g_last,
                              float* grad_density_grid, float* gd_scratch, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(grad_density_grid, density_desc);
  if (g.C != 1 || g.P != 1 || !box_cfg_ok(cfg)) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_box_params(cfg, nullptr);
  return launch_density_bwd<BoxSampler>(rays_o, rays_d, nullptr, g, p, n_rays, density, alpha, weight, T, flags, alphainv_last,
                                        offsets, g_weight, g_alpha, nullptr, g_last, grad_density_grid, gd_scratch,
                                        as_stream(stream));
}

int ubn_march_box_tensorf_density_fwd(const float* rays_o, const float* rays_d, const float* const* factors, const UbnTensorfDesc* desc,
                                      const uint8_t* mask_world, const UbnBoxMarchCfg* cfg, int64_t n_rays, float* density,
                                      float* alpha, float* weight, float* T, uint8_t* flags, float* alphainv_last, int32_t* n_keep,
                                      int32_t* overflow, void* stream) {
  if (n_rays <= 0) return 0;
  TfView t;
  if (!make_tf_view(factors, desc, t) || t.C != 1 || !box_cfg_ok(cfg) || !overflow) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_box_params(cfg, overflow);
  if (p.use_mask && !mask_world) return finish(cudaErrorInvalidValue);
  const unsigned blocks = blocks_for(n_rays, kMarchWarps);
  const cudaStream_t st = as_stream(stream);
  const GridView none{};
  if (tf_records4(t, nullptr))
    k_march_density_fwd<BoxSampler, -4><<<blocks, 32 * kMarchWarps, 0, st>>>(rays_o, rays_d, nullptr, none, mask_world, p, n_rays,
                                                                            density, alpha, weight, T, flags, alphainv_last, n_keep, t);
  else
    k_march_density_fwd<BoxSampler, -1><<<blocks, 32 * kMarchWarps, 0, st>>>(rays_o, rays_d, nullptr, none, mask_world, p, n_rays,
                                                                            density, alpha, weight, T, flags, alphainv_last, n_keep, t);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_march_box_tensorf_density_bwd(const float* rays_o, const float* rays_d, const float* const* factors, const UbnTensorfDesc* desc,
                                      const UbnBoxMarchCfg* cfg, int64_t n_rays, const float* density, const float* alpha,
                                      const float* weight, const float* T, const uint8_t* flags, const float* alphainv_last,
                                      const int64_t* offsets, const float* g_weight, const float* g_alpha, const float* g_last,
                                      float* const* grads, int vec_copies, float* gd_scratch, float* vec_scratch, void* stream) {
  if (n_rays <= 0) return 0;
  TfView t;
  TfGrads gr;
  if (!make_tf_view(factors, desc, t) || t.C != 1 || !make_tf_grads(grads, gr) || !box_cfg_ok(cfg) || !gd_scratch || !vec_scratch ||
      !aligned16(vec_scratch) || vec_copies < 1 || vec_copies > 64)
    return finish(cudaErrorInvalidValue);
  const MarchParams p = make_box_params(cfg, nullptr);
  const cudaStream_t st = as_stream(stream);
  const unsigned blocks = blocks_for(n_rays, kMarchWarps);
  const int64_t copy_len = tf_copy_len(t);
  const cudaError_t e = cudaMemsetAsync(vec_scratch, 0, (size_t)vec_copies * copy_len * sizeof(float), st);
  if (e != cudaSuccess) return finish(e);
  GridView g{};     // launch 1 reads only the slab count
  g.P = 1;
  k_march_density_bwd<BoxSampler, 1, true><<<blocks, 32 * kMarchWarps, 0, st>>>(
      rays_o, rays_d, nullptr, g, p, n_rays, density, alpha, weight, T, flags, alphainv_last, offsets, g_weight, g_alpha, nullptr,
      g_last, nullptr, gd_scratch);
  UBN_LAUNCH_CHECK();
  if (tf_records4(t, grads))
    k_march_box_tensorf_scatter<4><<<blocks, 32 * kMarchWarps, 0, st>>>(rays_o, rays_d, t, p, n_rays, gd_scratch, gr, vec_scratch,
                                                                        copy_len, vec_copies);
  else
    k_march_box_tensorf_scatter<1><<<blocks, 32 * kMarchWarps, 0, st>>>(rays_o, rays_d, t, p, n_rays, gd_scratch, gr, vec_scratch,
                                                                        copy_len, vec_copies);
  UBN_LAUNCH_CHECK();
  k_tensorf_bwd_finish<<<blocks_for(copy_len, 256), 256, 0, st>>>(t, gr, vec_scratch, copy_len, vec_copies, nullptr, 0, 0, nullptr);
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
