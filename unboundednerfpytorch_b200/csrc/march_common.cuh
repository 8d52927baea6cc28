// march_common.cuh -- ray set-up and contracted sampling shared by the fused march kernels.
#pragma once
#include "trilinear.cuh"

namespace ubn {

struct MarchParams {
  float cx, cy, cz, rx, ry, rz;   // scene center / radius
  float B, A;                     // contraction constants
  int l2norm;
  int S;
  float shift, interval, thres;
  int use_cumdist;
  float cumdist_thres;
  int use_mask;
  int msz[3];
  float mscale[3], mshift[3];
  float bmin[3], bmax[3];         // NDC march: samples outside this box (strict comparisons) are dropped
  GridView shift_grid;            // NDC march: the act_shift DenseGrid, added to the raw density
  float near, stepdist;           // box march: t_min clamp and the step length of a sample
  int* overflow;                  // box march, pass A: set to 1 when a ray needs more than S steps (else NULL)
};

inline MarchParams make_params(const UbnMarchCfg* c) {
  MarchParams p{};
  p.cx = c->scene_center[0]; p.cy = c->scene_center[1]; p.cz = c->scene_center[2];
  p.rx = c->scene_radius[0]; p.ry = c->scene_radius[1]; p.rz = c->scene_radius[2];
  p.B = c->contract_B; p.A = c->contract_A;
  p.l2norm = c->contracted_norm;
  p.S = c->n_samples;
  p.shift = c->act_shift; p.interval = c->interval; p.thres = c->fast_color_thres;
  p.use_cumdist = c->use_cumdist; p.cumdist_thres = c->cumdist_thres;
  p.use_mask = c->use_maskcache;
  for (int a = 0; a < 3; ++a) { p.msz[a] = c->mask_sz[a]; p.mscale[a] = c->mask_scale[a]; p.mshift[a] = c->mask_shift[a]; }
  return p;
}

// DirectMPIGO (dmpigo.py:224-340): no contraction, no cumdist, Raw2Alpha with shift 0 (the per-plane bias is in the density)
inline MarchParams make_ndc_params(const UbnNdcMarchCfg* c, const GridView& shift_grid) {
  MarchParams p{};
  p.S = c->n_samples;
  p.shift = 0.f; p.interval = c->interval; p.thres = c->fast_color_thres;
  p.use_cumdist = 0;
  p.use_mask = c->use_maskcache;
  for (int a = 0; a < 3; ++a) {
    p.msz[a] = c->mask_sz[a]; p.mscale[a] = c->mask_scale[a]; p.mshift[a] = c->mask_shift[a];
    p.bmin[a] = c->xyz_min[a]; p.bmax[a] = c->xyz_max[a];
  }
  p.shift_grid = shift_grid;
  return p;
}

struct Ray {
  float ox, oy, oz, dx, dy, dz;   // normalised origin, unit direction (box march: rays_start, rays_dir)
  int n;                          // samples of this ray: S, or the box march's own n_steps (<= S)
};

// ||v|| exactly as torch's CUDA reduction evaluates x.norm(dim=-1) on 3-vectors: the lanes of the reduced
// dimension are combined by a shuffle tree, i.e. sqrt((x*x + z*z) + y*y) with every product and sum rounded
// separately (scripts/probe_mean_order.py-style probe against torch: the "natural" orders do not match).
// The reference runs these norms as torch ops (dcvgo.py:240,253,288; FourierGrid_model.py:523,537), so matching
// them bit-for-bit keeps the threshold decisions downstream (inner mask, cumdist, mask-cache rounding) identical.
__device__ __forceinline__ float norm3_torch(float x, float y, float z) {
  return sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z)), __fmul_rn(y, y)));
}

// rays_o = (o - center) / radius ; rays_d = d / ||d||     (torch elementwise: no fma contraction)
__device__ __forceinline__ Ray load_ray(const float* __restrict__ o, const float* __restrict__ d, const MarchParams& p) {
  Ray r;
  r.ox = __fdiv_rn(__fsub_rn(o[0], p.cx), p.rx);
  r.oy = __fdiv_rn(__fsub_rn(o[1], p.cy), p.ry);
  r.oz = __fdiv_rn(__fsub_rn(o[2], p.cz), p.rz);
  const float n = norm3_torch(d[0], d[1], d[2]);
  r.dx = __fdiv_rn(d[0], n);
  r.dy = __fdiv_rn(d[1], n);
  r.dz = __fdiv_rn(d[2], n);
  r.n = p.S;
  return r;
}

// contracted sample position at parameter t; returns inner flag (norm <= 1)
__device__ __forceinline__ bool sample_point(const Ray& r, float t, const MarchParams& p, float& x, float& y, float& z) {
  x = __fadd_rn(r.ox, __fmul_rn(r.dx, t));
  y = __fadd_rn(r.oy, __fmul_rn(r.dy, t));
  z = __fadd_rn(r.oz, __fmul_rn(r.dz, t));
  float n;
  if (p.l2norm) n = norm3_torch(x, y, z);
  else          n = fmaxf(fmaxf(fabsf(x), fabsf(y)), fabsf(z));
  const bool inner = (n <= 1.f);
  if (!inner) {
    // torch evaluates `bg_len / norm` (Python scalar / tensor) as norm.reciprocal() * bg_len -- Tensor.__rtruediv__ --
    // i.e. two roundings; reproduced here so contracted points match the reference's torch ops bit-for-bit
    const float f = __fsub_rn(p.B, __fmul_rn(__frcp_rn(n), p.A));
    x = __fmul_rn(__fdiv_rn(x, n), f);
    y = __fmul_rn(__fdiv_rn(y, n), f);
    z = __fmul_rn(__fdiv_rn(z, n), f);
  }
  return inner;
}

// Sampling policies of the fused march kernels (march.cu, march_ndc.cu).  A policy says where sample s of a ray lies, whether the
// model samples there at all, and what is added to the density-grid value before Raw2Alpha.  The scan, flags, compaction and
// backward scan code is written once against this interface.
//   point(r, t_table, s, p, x, y, z, inner) -> false when the sample is outside the model's domain; `inner` -> UBN_FLAG_INNER
//   density(p, d, x, y, z)                  -> the raw density that Raw2Alpha(shift = p.shift) activates
struct ContractedSampler {      // FourierGrid_model.py:509-552, dcvgo.py:228-262: contracted point at t_table[s]
  __device__ static Ray load(const float* o, const float* d, const MarchParams& p) { return load_ray(o, d, p); }
  __device__ static bool point(const Ray& r, const float* t_table, int s, const MarchParams& p, float& x, float& y, float& z,
                               bool& inner) {
    inner = sample_point(r, t_table[s], p, x, y, z);
    return true;
  }
  __device__ static float density(const MarchParams&, float d, float, float, float) { return d; }
};

struct NdcSampler {             // dmpigo.py:224-249, 275: NDC point inside the strict bbox; density + act_shift(p)
  __device__ static Ray load(const float* o, const float* d, const MarchParams& p) {
    Ray r;
    r.ox = o[0]; r.oy = o[1]; r.oz = o[2];
    r.dx = d[0]; r.dy = d[1]; r.dz = d[2];
    r.n = p.S;
    return r;
  }
  __device__ static bool point(const Ray& r, const float*, int s, const MarchParams& p, float& x, float& y, float& z,
                               bool& inner) {
    ndc_point(r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, s, p.S, x, y, z);
    inner = false;
    return !((p.bmin[0] > x) | (p.bmin[1] > y) | (p.bmin[2] > z) | (p.bmax[0] < x) | (p.bmax[1] < y) | (p.bmax[2] < z));
  }
  // act_shift is a [1,1,1,1,D] grid: X = Y = 1, so the pre-clamped cell does not apply; the general trilinear read is
  // F.grid_sample's arithmetic for any shape.  One fp32 add, as torch's `density(p) + act_shift(p)`.
  __device__ static float density(const MarchParams& p, float d, float x, float y, float z) {
    return __fadd_rn(d, grid_density_at(p.shift_grid, x, y, z));
  }
};

struct BoxSampler {             // dvgo.py:306-328, render_utils_kernel.cu:12-79,167-194: start + dir * (stepdist * s), s < n_steps
  // t_min / t_max from the AABB (near clamp, far = 1e9 as sample_ray sets it), n_steps, start and dir with the very functions
  // ubn_sample_pts_* use (common.cuh).  n_steps > S (the host's S_max) raises p.overflow and is clamped so no record is out of range.
  __device__ static Ray load(const float* o, const float* d, const MarchParams& p) {
    const RayBox b = ray_aabb(o, d, p.bmin, p.bmax, p.near, 1e9f);
    const int64_t n = ray_n_samples(d, b.t_min, b.t_max, p.stepdist);
    float start[3], dir[3];
    ray_start_dir(o, d, b.t_min, start, dir);
    Ray r;
    r.ox = start[0]; r.oy = start[1]; r.oz = start[2];
    r.dx = dir[0]; r.dy = dir[1]; r.dz = dir[2];
    r.n = (int)min(n, (int64_t)p.S);
    if (n > p.S && p.overflow) *p.overflow = 1;
    return r;
  }
  __device__ static bool point(const Ray& r, const float*, int s, const MarchParams& p, float& x, float& y, float& z,
                               bool& inner) {
    const float start[3] = {r.ox, r.oy, r.oz}, dir[3] = {r.dx, r.dy, r.dz};
    box_point(start, dir, p.stepdist, s, x, y, z);
    inner = false;
    return !outside_box(p.bmin, p.bmax, x, y, z);
  }
  __device__ static float density(const MarchParams&, float d, float, float, float) { return d; }
};

// DirectVoxGO (dvgo.py:330-397): no contraction, no cumdist; Raw2Alpha with the scalar act_shift; mask cache before the density
inline MarchParams make_box_params(const UbnBoxMarchCfg* c, int* overflow) {
  MarchParams p{};
  p.S = c->s_max;
  p.shift = c->act_shift; p.interval = c->interval; p.thres = c->fast_color_thres;
  p.use_cumdist = 0;
  p.use_mask = c->use_maskcache;
  for (int a = 0; a < 3; ++a) {
    p.msz[a] = c->mask_sz[a]; p.mscale[a] = c->mask_scale[a]; p.mshift[a] = c->mask_shift[a];
    p.bmin[a] = c->xyz_min[a]; p.bmax[a] = c->xyz_max[a];
  }
  p.near = c->near;
  p.stepdist = c->stepdist;
  p.overflow = overflow;
  return p;
}

struct CellR {
  int v;            // base voxel index  (x0*Y + y0)*Z + z0, pre-clamped
  float fx, fy, fz; // fractions in [0,1]
};

__device__ __forceinline__ CellR make_cell(float cx, float cy, float cz, int X, int Y, int Z) {
  CellR c;
  const float x0 = fminf(fmaxf(floorf(cx), 0.f), (float)(X - 2));
  const float y0 = fminf(fmaxf(floorf(cy), 0.f), (float)(Y - 2));
  const float z0 = fminf(fmaxf(floorf(cz), 0.f), (float)(Z - 2));
  c.fx = cx - x0; c.fy = cy - y0; c.fz = cz - z0;
  c.v = ((int)x0 * Y + (int)y0) * Z + (int)z0;
  return c;
}

// Visit the kP slabs of a FourierGrid in natural order with their continuous source indices.  Slabs 2k+1 / 2k+2 are sin / cos
// of the SAME argument 2^k x, so one sincosf per (axis, frequency) serves both: half the range reductions of separate sinf / cosf
// calls.  sincosf is bit-identical to the pair on this toolchain for every float |a| <= 8 (scripts/probe_sincos.cu checks all
// 2.18e9 arguments), so every coordinate -- and with it raw_density -- keeps its bits; the at-size parity tests pin it.
template <int kP, typename F>
__device__ __forceinline__ void for_each_slab(const GridView& g, float nx, float ny, float nz, F&& f) {
  f(0, src_index(nx, g.X), src_index(ny, g.Y), src_index(nz, g.Z));
#pragma unroll
  for (int k = 0; k < (kP - 1) / 2; ++k) {
    const float m = (float)(1 << k);
    float sx, cx, sy, cy, sz, cz;
    sincosf(__fmul_rn(m, nx), &sx, &cx);
    sincosf(__fmul_rn(m, ny), &sy, &cy);
    sincosf(__fmul_rn(m, nz), &sz, &cz);
    f(2 * k + 1, src_index(sx, g.X), src_index(sy, g.Y), src_index(sz, g.Z));
    f(2 * k + 2, src_index(cx, g.X), src_index(cy, g.Y), src_index(cz, g.Z));
  }
}

// grid_density_at for a contiguous single-channel grid (sv == 1) with kP slabs known at compile time, 32-bit voxel offsets and
// pre-clamped cells: no per-corner bounds predicates, no 64-bit index arithmetic, no runtime slab loop.  Contracted / Fourier-warped
// coordinates never leave [-1, 1], where the clamped cell gives the same eight (value, weight) pairs in the same order as
// trilerp1 (a corner that trilerp1 skips as out of range has weight exactly 0 here), so the result is bit-identical.
template <int kP>
__device__ __forceinline__ float grid_density_fast(const GridView& g, float x, float y, float z) {
  const float nx = norm_coord(x, g.mn[0], g.len[0]);
  const float ny = norm_coord(y, g.mn[1], g.len[1]);
  const float nz = norm_coord(z, g.mn[2], g.len[2]);
  const int dY = g.Z, dX = g.Y * g.Z;
  SlabMean acc;
  for_each_slab<kP>(g, nx, ny, nz, [&](int s, float cx, float cy, float cz) {
    const CellR c = make_cell(cx, cy, cz, g.X, g.Y, g.Z);
    const float* rec = g.data + (int64_t)s * g.sp + c.v;
    float a = 0.f;
#pragma unroll
    for (int corner = 0; corner < 8; ++corner) {          // tnw .. bse, z fastest (ATen's order)
      const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
      const float w = ((bz ? c.fz : 1.f - c.fz) * (by ? c.fy : 1.f - c.fy)) * (bx ? c.fx : 1.f - c.fx);
      a = fmaf(__ldg(rec + bx * dX + by * dY + bz), w, a);
    }
    acc.add(s, a);
  });
  return acc.mean(kP);
}

// adjoint of grid_density_fast: the four (x, y) edges of the cell, two z-adjacent floats each.  An edge whose lower corner is
// 8-byte aligned goes out as one red.v2 {w0, w1}; otherwise as red.v2 {0, w0} at the aligned pair below it (adding +0 to the
// neighbouring voxel: a no-op on the value) plus one scalar red for the upper corner -- the same instruction stream for every
// lane, no divergent alignment branch, 4 + (0..4) reduction instructions per slab instead of 4..12.
template <int kP>
__device__ __forceinline__ void grid_density_scatter_fast(float* __restrict__ grad, const GridView& g, float nx, float ny, float nz,
                                                          float gd) {
  const int dY = g.Z, dX = g.Y * g.Z;
  for_each_slab<kP>(g, nx, ny, nz, [&](int s, float cx, float cy, float cz) {
    const CellR c = make_cell(cx, cy, cz, g.X, g.Y, g.Z);
    float* rec = grad + (int64_t)s * g.sp + c.v;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int bx = e >> 1, by = e & 1;
      const float wxy_lo = (1.f - c.fz) * (by ? c.fy : 1.f - c.fy), wxy_hi = c.fz * (by ? c.fy : 1.f - c.fy);
      const float wx = bx ? c.fx : 1.f - c.fx;
      const float w0 = (wxy_lo * wx) * gd, w1 = (wxy_hi * wx) * gd;
      float* a = rec + bx * dX + by * dY;
      const bool odd = (reinterpret_cast<uintptr_t>(a) & 4) != 0;
      red_add_v2(a - (odd ? 1 : 0), odd ? 0.f : w0, odd ? w0 : w1);
      if (odd) atomicAdd(a + 1, w1);
    }
  });
}

// v[kCh ..] added into q[kCh ..] when q + kCh sits at 4-byte phase kPh of a 16-byte line: the widest reduction the address
// allows at every step (red.v4 at phase 0, red.v2 at even phases, scalar otherwise), all channel indices known at compile time
template <int kC, int kCh, int kPh>
__device__ __forceinline__ void red_add_from(float* q, const float* v) {
  if constexpr (kCh < kC) {
    if constexpr (kPh == 0 && kCh + 4 <= kC) {
      red_add_v4(q + kCh, make_float4(v[kCh], v[kCh + 1], v[kCh + 2], v[kCh + 3]));
      red_add_from<kC, kCh + 4, 0>(q, v);
    } else if constexpr ((kPh & 1) == 0 && kCh + 2 <= kC) {
      red_add_v2(q + kCh, v[kCh], v[kCh + 1]);
      red_add_from<kC, kCh + 2, (kPh + 2) & 3>(q, v);
    } else {
      atomicAdd(q + kCh, v[kCh]);
      red_add_from<kC, kCh + 1, (kPh + 1) & 3>(q, v);
    }
  }
}

// q[0 .. kC) += v for a record that starts at any of the four 4-byte phases of a 16-byte line: one unrolled reduction sequence
// per phase, so every channel index is a compile-time constant and v stays in registers
template <int kC>
__device__ __forceinline__ void red_add_record_phased(float* q, const float* v) {
  switch ((reinterpret_cast<uintptr_t>(q) >> 2) & 3) {
    case 0: red_add_from<kC, 0, 0>(q, v); break;
    case 1: red_add_from<kC, 0, 1>(q, v); break;
    case 2: red_add_from<kC, 0, 2>(q, v); break;
    default: red_add_from<kC, 0, 3>(q, v); break;
  }
}

// q[0 .. kC) += v with the widest reductions each address allows (red.v4 at 16-byte, red.v2 at 8-byte alignment, scalar
// otherwise): the k0 scatters of the NDC / box march (C = 3, 9, 12) and of the contracted march at C = 3 and 15
template <int kC>
__device__ __forceinline__ void red_add_record(float* q, const float* v) {
  if constexpr (kC % 4 == 0) {                // 16-byte aligned records (C = 12): all red.v4
#pragma unroll
    for (int c4 = 0; c4 < kC; c4 += 4) red_add_v4(q + c4, make_float4(v[c4], v[c4 + 1], v[c4 + 2], v[c4 + 3]));
    return;
  }
  if constexpr (kC == 3) {                    // the same reductions as the loop below, without its run-time channel index
    if ((reinterpret_cast<uintptr_t>(q) & 7) == 0) {
      red_add_v2(q, v[0], v[1]);
      atomicAdd(q + 2, v[2]);
    } else {
      atomicAdd(q, v[0]);
      red_add_v2(q + 1, v[1], v[2]);
    }
    return;
  }
  if constexpr (kC == 15) {                   // a 60-byte record starts at any of the four phases of a 16-byte line
    red_add_record_phased<kC>(q, v);
    return;
  }
  int ch = 0;
#pragma unroll
  for (int step = 0; step < kC; ++step) {     // at most kC iterations; each consumes 1, 2 or 4 channels
    if (ch >= kC) break;
    const uintptr_t a = reinterpret_cast<uintptr_t>(q + ch);
    if (ch + 4 <= kC && (a & 15) == 0) {
      red_add_v4(q + ch, make_float4(v[ch], v[ch + 1], v[ch + 2], v[ch + 3]));
      ch += 4;
    } else if (ch + 2 <= kC && (a & 7) == 0) {
      red_add_v2(q + ch, v[ch], v[ch + 1]);
      ch += 2;
    } else {
      atomicAdd(q + ch, v[ch]);
      ch += 1;
    }
  }
}

constexpr int kMarchWarps = 4;

// ------------------------------------------------------------------------------------------------
// One 32-sample chunk of the forward march (lane = sample base + lane), shared by pass A (march.cu) and the fused render
// (render.cu).  march_chunk_point: sample point, cumdist filter and mask cache -> whether the density is queried; the caller
// reads the density, then march_alpha (Raw2Alpha) and march_listed (the `alpha > thres` listing).  cum / carry_over are the
// warp-uniform cumdist state carried from chunk to chunk.
// ------------------------------------------------------------------------------------------------
struct MarchSample {
  float x, y, z;
  bool valid, inner, queried;
};

template <class Smp>
__device__ __forceinline__ MarchSample march_chunk_point(const Ray& r, const float* __restrict__ t_table,
                                                         const uint8_t* __restrict__ mask_world, const MarchParams& p, int base,
                                                         int lane, float& cum, bool& carry_over) {
  const int S = p.S;
  const int s = base + lane;
  MarchSample m;
  m.valid = s < r.n;
  m.x = 0; m.y = 0; m.z = 0;
  m.inner = false;
  bool in_domain = false;
  if (m.valid) in_domain = Smp::point(r, t_table, s, p, m.x, m.y, m.z, m.inner);

  bool queried = m.valid && in_domain;
  if (p.use_cumdist) {
    // dist[s] = || pts[s+1] - pts[s] || (torch .norm), s <= S-2; mask[s+1] |= cumdist(dist)[s]
    float dist = 0.f;
    if (s + 1 < S) {
      float x1, y1, z1;
      bool inner1;
      Smp::point(r, t_table, s + 1, p, x1, y1, z1, inner1);
      const float ex = __fsub_rn(x1, m.x), ey = __fsub_rn(y1, m.y), ez = __fsub_rn(z1, m.z);
      dist = norm3_torch(ex, ey, ez);
    }
    bool over_here = false;   // result for dist index s (applies to sample s+1)
    const int n_d = min(32, S - 1 - base);
    for (int j = 0; j < n_d; ++j) {
      const float dj = __shfl_sync(0xffffffffu, dist, j);
      cum += dj;
      const bool over = (cum > p.cumdist_thres);
      cum *= float(!over);
      if (lane == j) over_here = over;
    }
    // shift by one sample: sample s gets the flag of dist index s-1
    const int prev = __shfl_up_sync(0xffffffffu, (int)over_here, 1);
    const bool flag_for_me = (lane == 0) ? carry_over : (prev != 0);
    carry_over = __shfl_sync(0xffffffffu, (int)over_here, 31) != 0;
    queried = m.valid && (m.inner || (s > 0 && flag_for_me));
  }
  if (p.use_mask && queried) {
    const int i = roundf(m.x * p.mscale[0] + p.mshift[0]);
    const int j = roundf(m.y * p.mscale[1] + p.mshift[1]);
    const int k = roundf(m.z * p.mscale[2] + p.mshift[2]);
    bool hit = false;
    if (0 <= i && i < p.msz[0] && 0 <= j && j < p.msz[1] && 0 <= k && k < p.msz[2])
      hit = mask_world[((int64_t)i * p.msz[1] + j) * p.msz[2] + k] != 0;
    queried = hit;
  }

  m.queried = queried;
  return m;
}

// Raw2Alpha (render_utils_kernel.cu:431-443) of a queried sample's raw density
__device__ __forceinline__ float march_alpha(float dens, const MarchParams& p) {
  const float e = expf(dens + p.shift);
  return 1 - powf(1 + e, -p.interval);
}

__device__ __forceinline__ bool march_listed(bool queried, float alpha, const MarchParams& p) {
  return queried && (p.thres > 0.f ? (alpha > p.thres) : true);
}

// exact sequential transmittance scan over the listed samples of this chunk (alpha2weight order): myT / myW of the lanes it reaches,
// T_cum and `done` (T < 1e-3, render_utils_kernel.cu:591-603) carried warp-uniform from chunk to chunk
__device__ __forceinline__ void transmittance_scan(bool listed, float alpha, int lane, float& T_cum, bool& done, float& myT, float& myW,
                                                   bool& scanned) {
  myT = 1.f;
  myW = 0.f;
  scanned = false;
  unsigned m = __ballot_sync(0xffffffffu, listed);
  if (!done) {
    while (m) {
      const int j = __ffs(m) - 1;
      m &= m - 1;
      const float a = __shfl_sync(0xffffffffu, alpha, j);
      if (lane == j) { myT = T_cum; myW = T_cum * alpha; scanned = true; }
      T_cum *= (1. - a);            // double intermediate (render_utils_kernel.cu:596)
      if (T_cum < 1e-3) { done = true; break; }
    }
  }
}

// The k0 features of one sample at normalised coordinates (nx, ny, nz), lane = sample: every channel accumulated in ATen's corner
// order (fma chain tnw .. bse) and the slabs combined in torch-CUDA's mean order (accumulator a = slab & 3, ((a0 + a1) + a2) + a3),
// so the features are bit-identical to F.grid_sample(...).mean(0).  Records of C % 4 == 0 channels are read as float4.
// kLean: the slab loop rolled and four corner records in flight instead of eight, for callers with a smaller register budget
// (render_fourier.cu's march warps); the same arithmetic in the same order
template <int kC, int kP, bool kLean = false>
__device__ __forceinline__ void lane_features(const GridView& g, float nx, float ny, float nz, float (&out)[kC]) {
  const int dY = g.Z * kC, dX = g.Y * g.Z * kC;
  float tot[kC], grp[kC];
  auto corner_add = [&](const float* rec, const CellR& cell, int corner, float (&val)[kC]) {   // tnw .. bse (z fastest)
    const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
    const float wgt = ((bz ? cell.fz : 1.f - cell.fz) * (by ? cell.fy : 1.f - cell.fy)) * (bx ? cell.fx : 1.f - cell.fx);
    const float* q = rec + bx * dX + by * dY + bz * kC;
    if constexpr (kC % 4 == 0) {
#pragma unroll
      for (int c4 = 0; c4 < kC; c4 += 4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(q + c4));
        val[c4] = fmaf(v.x, wgt, val[c4]); val[c4 + 1] = fmaf(v.y, wgt, val[c4 + 1]);
        val[c4 + 2] = fmaf(v.z, wgt, val[c4 + 2]); val[c4 + 3] = fmaf(v.w, wgt, val[c4 + 3]);
      }
    } else {
#pragma unroll
      for (int c = 0; c < kC; ++c) val[c] = fmaf(__ldg(q + c), wgt, val[c]);
    }
  };
  auto slab_add = [&](int a, int sl) {
    const CellR cell = make_cell(src_index(fourier_gamma(sl, nx), g.X), src_index(fourier_gamma(sl, ny), g.Y),
                                 src_index(fourier_gamma(sl, nz), g.Z), g.X, g.Y, g.Z);
    const float* rec = g.data + sl * g.sp + (int64_t)cell.v * kC;
    float val[kC];
#pragma unroll
    for (int c = 0; c < kC; ++c) val[c] = 0.f;
    if constexpr (kLean) {
#pragma unroll 4
      for (int corner = 0; corner < 8; ++corner) corner_add(rec, cell, corner, val);
    } else {
#pragma unroll
      for (int corner = 0; corner < 8; ++corner) corner_add(rec, cell, corner, val);
    }
#pragma unroll
    for (int c = 0; c < kC; ++c) grp[c] = (sl == a) ? __fadd_rn(0.f, val[c]) : __fadd_rn(grp[c], val[c]);
  };
#pragma unroll
  for (int a = 0; a < 4 && a < kP; ++a) {
    if constexpr (kLean) {
#pragma unroll 1
      for (int sl = a; sl < kP; sl += 4) slab_add(a, sl);
    } else {
#pragma unroll
      for (int sl = a; sl < kP; sl += 4) slab_add(a, sl);
    }
#pragma unroll
    for (int c = 0; c < kC; ++c) tot[c] = (a == 0) ? grp[c] : __fadd_rn(tot[c], grp[c]);
  }
#pragma unroll
  for (int c = 0; c < kC; ++c) out[c] = slab_mean_scale(tot[c], kP);
}

}  // namespace ubn
