// tensorf.cuh -- the per-sample TensoRF read and its adjoint (FourierGrid/grid.py:111-129, 174-201), shared by the stand-alone
// TensoRFGrid kernels (tensorf.cu) and the fused box march's TensoRF density (march.cu), so that both give the same bits.
//
// Everything here sits in an unnamed namespace: each translation unit gets its own internal copy, and the kernels of tensorf.cu
// keep the names they had when these helpers were local to it.  Their SASS is unchanged too, except that ptxas orders the
// instructions of k_tensorf_bwd differently now that its per-sample body is tf_sample_bwd (same instructions, same arithmetic,
// same time: DESIGN.md section 7).
#pragma once
#include "trilinear.cuh"

namespace ubn {
namespace {

constexpr int kTfMaxFeat = 96;    // R + R + Rxy: one grad_f_vec row per thread of tensorf.cu's 128-thread CTA

struct TfView {
  const float* f[6];             // xy_plane, xz_plane, yz_plane, x_vec, y_vec, z_vec
  int64_t sr[6], sa[6], sb[6];   // component / first / second spatial stride of each factor (elements)
  int S[3];                      // X, Y, Z
  int R, Rxy, C;
  float mn[3], len[3];
};

struct TfGrads {
  float* g[6];
};

// Product group g = plane g times vector 5 - g:  0: xy_plane . z_vec (Rxy),  1: xz_plane . y_vec (R),  2: yz_plane . x_vec (R).
__device__ __forceinline__ int grp_axis_a(int g) { return g == 2 ? 1 : 0; }
__device__ __forceinline__ int grp_axis_b(int g) { return g == 0 ? 1 : 2; }
__device__ __forceinline__ int grp_axis_l(int g) { return 2 - g; }
__device__ __forceinline__ int grp_comps(const TfView& t, int g) { return g == 0 ? t.Rxy : t.R; }
__device__ __forceinline__ int grp_feat0(const TfView& t, int g) { return g == 0 ? 0 : (g == 1 ? t.Rxy : t.Rxy + t.R); }

// Bilinear corners of a plane read at continuous index (ca, cb) as ATen's 2-D grid_sample forms them: the grid's x (W) coordinate
// is the plane's second axis b, y (H) the first axis a; corners nw (a0,b0), ne (a0,b1), sw (a1,b0), se (a1,b1);
// weights nw = (ix_se - ix) * (iy_se - iy) and so on.
struct Corners4 {
  int64_t off[4];
  float w[4];
  bool in[4];
};

__device__ __forceinline__ Corners4 plane_corners(float ca, int A, float cb, int B, int64_t sa, int64_t sb) {
  Corners4 q;
  const float fa = floorf(ca), fb = floorf(cb);
  const int a0 = (int)fa, b0 = (int)fb;
  const float wa1 = ca - fa, wa0 = (fa + 1.f) - ca, wb1 = cb - fb, wb0 = (fb + 1.f) - cb;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int da = c >> 1, db = c & 1;
    const int a = a0 + da, b = b0 + db;
    q.in[c] = (unsigned)a < (unsigned)A && (unsigned)b < (unsigned)B;
    q.off[c] = (int64_t)a * sa + (int64_t)b * sb;
    q.w[c] = (db ? wb1 : wb0) * (da ? wa1 : wa0);
  }
  return q;
}

// A vector [1,R,L,1] read at grid (0, ind): the width-1 axis puts the x coordinate at 0, so ne / se fall outside and the read is
// the linear interpolation nw = 1 * (iy_se - iy), sw = 1 * (iy - iy_nw) along the length.
struct Corners2 {
  int node[2];
  float w[2];
  bool in[2];
};

__device__ __forceinline__ Corners2 line_nodes(float cl, int L) {
  Corners2 q;
  const float fl = floorf(cl);
  const int l0 = (int)fl;
  q.node[0] = l0;
  q.node[1] = l0 + 1;
  q.w[0] = (fl + 1.f) - cl;
  q.w[1] = cl - fl;
  q.in[0] = (unsigned)l0 < (unsigned)L;
  q.in[1] = (unsigned)(l0 + 1) < (unsigned)L;
  return q;
}

template <int W>
__device__ __forceinline__ void load_w(const float* p, float* v) {
  if constexpr (W == 4) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
    v[0] = __ldg(p);
  }
}

template <int W>
__device__ __forceinline__ void red_w(float* p, const float* v, float s) {
  if constexpr (W == 4) {
    red_add_v4(p, make_float4(v[0] * s, v[1] * s, v[2] * s, v[3] * s));
  } else {
    atomicAdd(p, v[0] * s);
  }
}

// W consecutive components (from component offset roff) of the plane read and of the vector read
template <int W>
__device__ __forceinline__ void plane_val(const float* base, const Corners4& q, int64_t roff, float* v) {
#pragma unroll
  for (int j = 0; j < W; ++j) v[j] = 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (q.in[c]) {
      float t[W];
      load_w<W>(base + q.off[c] + roff, t);
#pragma unroll
      for (int j = 0; j < W; ++j) v[j] += t[j] * q.w[c];
    }
  }
}

template <int W>
__device__ __forceinline__ void line_val(const float* base, const Corners2& q, int64_t sl, int64_t roff, float* v) {
#pragma unroll
  for (int j = 0; j < W; ++j) v[j] = 0.f;
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    if (q.in[c]) {
      float t[W];
      load_w<W>(base + (int64_t)q.node[c] * sl + roff, t);
#pragma unroll
      for (int j = 0; j < W; ++j) v[j] += t[j] * q.w[c];
    }
  }
}

// continuous factor index of world coordinate p on axis a: ((p - min) / len * 2 - 1 + 1) / 2 * (size - 1)
__device__ __forceinline__ float tf_coord(const TfView& t, int a, float p) { return src_index(norm_coord(p, t.mn[a], t.len[a]), t.S[a]); }

// The read at continuous index c[3]: the 3R products folded into acc[kC] in group, component order -- summed for kC = 1 (the
// density), projected by f_vec (staged in shared memory as sf[nfeat][kC]) otherwise.
template <int kC, int W>
__device__ __forceinline__ void tf_read(const TfView& t, const float* c, const float* sf, float* acc) {
#pragma unroll
  for (int ch = 0; ch < kC; ++ch) acc[ch] = 0.f;
#pragma unroll
  for (int g = 0; g < 3; ++g) {
    const int ia = grp_axis_a(g), ib = grp_axis_b(g), il = grp_axis_l(g), v = 5 - g;
    const Corners4 pq = plane_corners(c[ia], t.S[ia], c[ib], t.S[ib], t.sa[g], t.sb[g]);
    const Corners2 lq = line_nodes(c[il], t.S[il]);
    const int n = grp_comps(t, g), k0 = grp_feat0(t, g);
#pragma unroll 2
    for (int r = 0; r < n; r += W) {
      float pv[W], lv[W];
      plane_val<W>(t.f[g], pq, r * t.sr[g], pv);
      line_val<W>(t.f[v], lq, t.sa[v], r * t.sr[v], lv);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        const float p = pv[j] * lv[j];
        if constexpr (kC == 1) {
          acc[0] += p;
        } else {
#pragma unroll
          for (int ch = 0; ch < kC; ++ch) acc[ch] = fmaf(p, sf[(k0 + r + j) * kC + ch], acc[ch]);
        }
      }
    }
  }
}

// vector copy layout in scratch: [x_vec X*R | y_vec Y*R | z_vec Z*Rxy], each [node][component]
__device__ __host__ __forceinline__ int64_t vcopy_base(int f, int X, int Y, int R) {
  return f == 3 ? 0 : (f == 4 ? (int64_t)X * R : (int64_t)X * R + (int64_t)Y * R);
}

// Adjoint of tf_read for one sample with output gradient go[kC]: plane gradients reduced straight into gr, vector gradients into
// the copy vc; for kC > 1 the sample's products are also left in feat[row ..] (its row of the grad_f_vec tile).
template <int kC, int W>
__device__ __forceinline__ void tf_sample_bwd(const TfView& t, const float* c, const float* go, const float* sf, float* feat, int row,
                                              const TfGrads& gr, float* vc) {
#pragma unroll
  for (int g = 0; g < 3; ++g) {
    const int ia = grp_axis_a(g), ib = grp_axis_b(g), il = grp_axis_l(g), v = 5 - g;
    const Corners4 pq = plane_corners(c[ia], t.S[ia], c[ib], t.S[ib], t.sa[g], t.sb[g]);
    const Corners2 lq = line_nodes(c[il], t.S[il]);
    const int n = grp_comps(t, g), k0 = grp_feat0(t, g);
    float* vq = vc + vcopy_base(v, t.S[0], t.S[1], t.R);
#pragma unroll 1
    for (int r = 0; r < n; r += W) {
      float pv[W], lv[W], gp[W], gl[W];
      plane_val<W>(t.f[g], pq, r * t.sr[g], pv);
      line_val<W>(t.f[v], lq, t.sa[v], r * t.sr[v], lv);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        float gf;
        if constexpr (kC == 1) {
          gf = go[0];
        } else {
          gf = 0.f;
#pragma unroll
          for (int ch = 0; ch < kC; ++ch) gf = fmaf(go[ch], sf[(k0 + r + j) * kC + ch], gf);
          feat[row + k0 + r + j] = pv[j] * lv[j];
        }
        gp[j] = gf * lv[j];      // d out / d plane component = g_feat . line value
        gl[j] = gf * pv[j];      // d out / d vector component = g_feat . plane value
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (pq.in[q]) red_w<W>(gr.g[g] + pq.off[q] + r * t.sr[g], gp, pq.w[q]);
#pragma unroll
      for (int q = 0; q < 2; ++q)
        if (lq.in[q]) red_w<W>(vq + (int64_t)lq.node[q] * n + r, gl, lq.w[q]);
    }
  }
}

// closing launch: vector gradients += the vec_copies copies summed in copy order; grad_f_vec += the CTAs' sums in CTA order
__global__ void __launch_bounds__(256) k_tensorf_bwd_finish(TfView t, TfGrads gr, const float* __restrict__ vcopies, int64_t copy_len,
                                                            int vec_copies, const float* __restrict__ fpart, int nblk, int nfc,
                                                            float* __restrict__ grad_fvec) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < copy_len) {
    float s = 0.f;
    for (int q = 0; q < vec_copies; ++q) s += vcopies[(int64_t)q * copy_len + idx];
    const int64_t xr = (int64_t)t.S[0] * t.R, yr = (int64_t)t.S[1] * t.R;
    int f, n;
    int64_t e;
    if (idx < xr) { f = 3; n = t.R; e = idx; }
    else if (idx < xr + yr) { f = 4; n = t.R; e = idx - xr; }
    else { f = 5; n = t.Rxy; e = idx - xr - yr; }
    const int64_t node = e / n, r = e - node * n;
    float* p = gr.g[f] + r * t.sr[f] + node * t.sa[f];
    *p += s;
  } else if (idx < copy_len + nfc) {
    const int64_t j = idx - copy_len;
    float s = 0.f;
    for (int b = 0; b < nblk; ++b) s += fpart[(int64_t)b * nfc + j];
    grad_fvec[j] += s;
  }
}

// ---- host side ----------------------------------------------------------------------------------------------------------------
bool make_tf_view(const float* const* factors, const UbnTensorfDesc* d, TfView& t) {
  if (!factors || !d) return false;
  if (d->X < 1 || d->Y < 1 || d->Z < 1 || d->R < 1 || d->Rxy < 1) return false;
  if (d->C != 1 && d->C != 3 && d->C != 12) return false;
  if (2 * d->R + d->Rxy > kTfMaxFeat) return false;
  for (int f = 0; f < 6; ++f) {
    if (!factors[f]) return false;
    t.f[f] = factors[f];
    t.sr[f] = d->stride_r[f]; t.sa[f] = d->stride_a[f]; t.sb[f] = d->stride_b[f];
  }
  t.S[0] = d->X; t.S[1] = d->Y; t.S[2] = d->Z;
  t.R = d->R; t.Rxy = d->Rxy; t.C = d->C;
  for (int a = 0; a < 3; ++a) { t.mn[a] = d->xyz_min[a]; t.len[a] = d->xyz_max[a] - d->xyz_min[a]; }
  return true;
}

bool make_tf_grads(float* const* grads, TfGrads& gr) {
  if (!grads) return false;
  for (int f = 0; f < 6; ++f) {
    if (!grads[f]) return false;
    gr.g[f] = grads[f];
  }
  return true;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// 128-bit component records: every factor channels-last (component stride 1) with R, Rxy multiples of 4 and 16-byte aligned
// records; `also` (the gradients in the backward) must be aligned too
bool tf_records4(const TfView& t, float* const* also) {
  if (t.R % 4 || t.Rxy % 4) return false;
  for (int f = 0; f < 6; ++f) {
    if (t.sr[f] != 1 || t.sa[f] % 4 || (f < 3 && t.sb[f] % 4) || !aligned16(t.f[f])) return false;
    if (also && !aligned16(also[f])) return false;
  }
  return true;
}

// floats of the vector-gradient copies: vec_copies * (X*R + Y*R + Z*Rxy); copies start 16-byte aligned when R and Rxy are
// multiples of 4 (the only case that takes 128-bit reductions)
int64_t tf_copy_len(const TfView& t) { return (int64_t)t.S[0] * t.R + (int64_t)t.S[1] * t.R + (int64_t)t.S[2] * t.Rxy; }

}  // namespace
}  // namespace ubn
