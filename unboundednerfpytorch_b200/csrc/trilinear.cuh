// trilinear.cuh -- device-side trilinear voxel-grid read / scatter primitives shared by the stand-alone
// grid ops (trilinear.cu) and the fused ray-march kernels (march.cu).
//
// Semantics = torch F.grid_sample(mode='bilinear', padding_mode='zeros', align_corners=True) on a
// [P,C,X,Y,Z] volume as the reference calls it (grid.py:55-57, FourierGrid_grid.py:66-72):
//   ind_norm = ((xyz - xyz_min) / (xyz_max - xyz_min)).flip(-1) * 2 - 1      (elementwise float ops)
//   slab n is sampled at gamma_n(ind_norm), gamma = [x, sin(2^k x), cos(2^k x)]_k   (FourierGrid only)
//   source index c = ((coord + 1) / 2) * (size - 1); corners floor(c), floor(c)+1; out-of-range corners
//   contribute zero; corner weights are products of the distances to the opposite corner.
// World axis x indexes grid dim X (slowest), z indexes Z (fastest) -- the .flip(-1) in the reference
// exists only because grid_sample's coordinate order is (W,H,D).
#pragma once
#include "common.cuh"

namespace ubn {

struct GridView {
  const float* data;
  int P, C, X, Y, Z;
  int num_freqs;
  int64_t sp, sc, sv;   // strides (elements) of slab, channel, voxel
  float mn[3];          // xyz_min
  float len[3];         // xyz_max - xyz_min  (float subtraction, as torch computes it)
};

inline GridView make_view(const float* data, const UbnGridDesc* d) {
  GridView g;
  g.data = data;
  g.P = d->P; g.C = d->C; g.X = d->X; g.Y = d->Y; g.Z = d->Z;
  g.num_freqs = d->num_freqs;
  g.sp = d->stride_p; g.sc = d->stride_c; g.sv = d->stride_v;
  for (int a = 0; a < 3; ++a) { g.mn[a] = d->xyz_min[a]; g.len[a] = d->xyz_max[a] - d->xyz_min[a]; }
  return g;
}

// normalised coordinate in [-1,1] of one world axis: ((p - min) / len) * 2 - 1   (no contraction issue:
// the *2 is exact, so fma(t,2,-1) == (t*2)-1)
__device__ __forceinline__ float norm_coord(float p, float mn, float len) {
  return __fdiv_rn(__fsub_rn(p, mn), len) * 2.f - 1.f;
}

// gamma_n of FourierGrid_grid.py:32-36: slab 0 identity, slab 2k+1 = sin(2^k x), slab 2k+2 = cos(2^k x)
__device__ __forceinline__ float fourier_gamma(int slab, float x) {
  if (slab == 0) return x;
  const int k = (slab - 1) >> 1;
  const float a = __fmul_rn((float)(1 << k), x);
  return ((slab - 1) & 1) ? cosf(a) : sinf(a);
}

// continuous source index along one axis: ((coord + 1) / 2) * (size - 1)
__device__ __forceinline__ float src_index(float coord, int size) {
  return __fmul_rn(__fmul_rn(__fadd_rn(coord, 1.f), 0.5f), (float)(size - 1));
}

// src_index followed by ATen's guard (GridSampler.cuh: safe_downgrade_to_int_range): an index that is NaN, infinite or outside the
// int range becomes -100, so every corner of it lies outside the grid.  A point with a NaN or inf coordinate -- or the sin / cos
// of one -- then reads 0 and scatters nothing, as F.grid_sample does, instead of carrying NaN weights into in-range corners.
// The stand-alone grid ops and the view count use it; the fused march's points are finite by construction.
__device__ __forceinline__ float src_index_guarded(float coord, int size) {
  const float c = src_index(coord, size);
  return (c > (float)(INT_MAX - 1) || c < (float)INT_MIN || !isfinite(c)) ? -100.f : c;
}

// Mean over the P slabs exactly as torch-CUDA evaluates `out.mean(0)` on the grid_sample output (FourierGrid_grid.py:72), as
// probed with scripts/probe_mean_order.py (the sequential and the pairwise-tree orders do not match): ATen's reduction keeps four interleaved accumulators a[i & 3] += x_i, combines them ((a0 + a1) + a2) + a3
// and multiplies by the fp32 reciprocal of P.  Matching it makes raw_density -- and with it alpha, the weights and every
// threshold decision downstream -- bit-identical to the reference's GPU path (alpha = 1 - (1+e)^-interval is ill-conditioned:
// one ulp of density can move a dense-mode alpha by 1e-3 of its value).
struct SlabMean {
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  __device__ __forceinline__ void add(int slab, float v) {
    switch (slab & 3) {
      case 0: a0 = __fadd_rn(a0, v); break;
      case 1: a1 = __fadd_rn(a1, v); break;
      case 2: a2 = __fadd_rn(a2, v); break;
      default: a3 = __fadd_rn(a3, v); break;
    }
  }
  __device__ __forceinline__ float mean(int P) const {
    const float sum = __fadd_rn(__fadd_rn(__fadd_rn(a0, a1), a2), a3);
    return (P > 1) ? __fmul_rn(sum, __frcp_rn((float)P)) : sum;
  }
};

// d mean / d slab as torch's autograd evaluates it: grad / P is a multiplication by the fp32 reciprocal on CUDA
__device__ __forceinline__ float slab_mean_scale(float g, int P) { return (P > 1) ? __fmul_rn(g, __frcp_rn((float)P)) : g; }

struct Cell {
  int x0, y0, z0;
  float wx0, wx1, wy0, wy1, wz0, wz1;   // weight of corner 0 / corner 1 along each axis
};

__device__ __forceinline__ Cell locate(float cx, float cy, float cz) {
  Cell c;
  const float fx = floorf(cx), fy = floorf(cy), fz = floorf(cz);
  c.x0 = (int)fx; c.y0 = (int)fy; c.z0 = (int)fz;
  c.wx1 = cx - fx; c.wx0 = (fx + 1.f) - cx;
  c.wy1 = cy - fy; c.wy0 = (fy + 1.f) - cy;
  c.wz1 = cz - fz; c.wz0 = (fz + 1.f) - cz;
  return c;
}

// weight of corner (bx,by,bz): (wz * wy) * wx, the product order of ATen's tnw..bse
__device__ __forceinline__ float corner_weight(const Cell& c, int bx, int by, int bz) {
  return ((bz ? c.wz1 : c.wz0) * (by ? c.wy1 : c.wy0)) * (bx ? c.wx1 : c.wx0);
}

__device__ __forceinline__ bool corner_inside(const Cell& c, int bx, int by, int bz, int X, int Y, int Z) {
  const int x = c.x0 + bx, y = c.y0 + by, z = c.z0 + bz;
  return (unsigned)x < (unsigned)X && (unsigned)y < (unsigned)Y && (unsigned)z < (unsigned)Z;
}

// Single-channel read of one slab at continuous index (cx,cy,cz); `slab` points at channel 0 of the slab,
// `sv` is the voxel stride.  Accumulation order tnw,tne,tsw,tse,bnw,bne,bsw,bse = binary count, z fastest.
__device__ __forceinline__ float trilerp1(const float* __restrict__ slab, int64_t sv, int X, int Y, int Z,
                                          float cx, float cy, float cz) {
  const Cell c = locate(cx, cy, cz);
  float acc = 0.f;
#pragma unroll
  for (int corner = 0; corner < 8; ++corner) {
    const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
    if (corner_inside(c, bx, by, bz, X, Y, Z)) {
      const int64_t v = ((int64_t)(c.x0 + bx) * Y + (c.y0 + by)) * Z + (c.z0 + bz);
      acc += __ldg(slab + v * sv) * corner_weight(c, bx, by, bz);
    }
  }
  return acc;
}

// single-channel grid value at world position (x, y, z): mean over the P slabs of the trilinear reads at gamma_s(normalised coords)
// -- DenseGrid.forward (grid.py:50-61) for P = 1, FourierGrid.forward (FourierGrid_grid.py:60-78) otherwise
__device__ __forceinline__ float grid_density_at(const GridView& g, float x, float y, float z) {
  const float nx = norm_coord(x, g.mn[0], g.len[0]);
  const float ny = norm_coord(y, g.mn[1], g.len[1]);
  const float nz = norm_coord(z, g.mn[2], g.len[2]);
  SlabMean acc;
  for (int s = 0; s < g.P; ++s) {
    const float cx = src_index(fourier_gamma(s, nx), g.X);
    const float cy = src_index(fourier_gamma(s, ny), g.Y);
    const float cz = src_index(fourier_gamma(s, nz), g.Z);
    acc.add(s, trilerp1(g.data + s * g.sp, g.sv, g.X, g.Y, g.Z, cx, cy, cz));
  }
  return acc.mean(g.P);
}

// adjoint of trilerp1: grad_slab[corner] += w_corner * g
__device__ __forceinline__ void trilerp1_scatter(float* __restrict__ slab, int64_t sv, int X, int Y, int Z,
                                                 float cx, float cy, float cz, float g) {
  const Cell c = locate(cx, cy, cz);
#pragma unroll
  for (int corner = 0; corner < 8; ++corner) {
    const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
    if (corner_inside(c, bx, by, bz, X, Y, Z)) {
      const int64_t v = ((int64_t)(c.x0 + bx) * Y + (c.y0 + by)) * Z + (c.z0 + bz);
      atomicAdd(slab + v * sv, corner_weight(c, bx, by, bz) * g);
    }
  }
}

// 64-bit vector reduction (sm_90+): two consecutive floats at an 8-byte aligned address in one L2 atomic operation
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// trilerp1_scatter for unit voxel stride: the two z corners of an (x, y) edge are adjacent floats, so when both are
// inside and the lower one is 8-byte aligned they go out as ONE vector reduction (the scatter is bound by the number of
// L2 atomic operations, not by bytes).  Same addends as the scalar form.
__device__ __forceinline__ void trilerp1_scatter_pairs(float* __restrict__ slab, int X, int Y, int Z, float cx, float cy,
                                                       float cz, float g) {
  const Cell c = locate(cx, cy, cz);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int bx = e >> 1, by = e & 1;
    const bool in0 = corner_inside(c, bx, by, 0, X, Y, Z), in1 = corner_inside(c, bx, by, 1, X, Y, Z);
    if (!(in0 || in1)) continue;
    float* a = slab + ((int64_t)(c.x0 + bx) * Y + (c.y0 + by)) * Z + c.z0;
    const float w0 = corner_weight(c, bx, by, 0) * g, w1 = corner_weight(c, bx, by, 1) * g;
    if (in0 && in1 && ((reinterpret_cast<uintptr_t>(a) & 7) == 0)) {
      red_add_v2(a, w0, w1);
    } else {
      if (in0) atomicAdd(a, w0);
      if (in1) atomicAdd(a + 1, w1);
    }
  }
}

// 128-bit vector reduction (sm_90+): one instruction adds 4 consecutive floats at a 16-byte aligned address
__device__ __forceinline__ void red_add_v4(float* addr, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

}  // namespace ubn
