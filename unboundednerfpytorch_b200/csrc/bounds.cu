// bounds.cu -- the scene bounding boxes a training run starts from (FourierGrid/bbox_compute.py), as reductions:
//   compute_bbox_by_cam_frustrm, bounded / unbounded-inward / nerfpp branches (:10-45, :96-110) -> ubn_frustum_bounds
//   compute_bbox_by_coarse_geo (:136-165)                                                   -> ubn_lattice_bounds[_alpha]
// The reference materialises every ray of every training view (~20 torch ops per view) or a [X,Y,Z,3] lattice, a density and an
// alpha tensor, only to keep a min and a max per axis.  Here each thread generates its ray or lattice point in registers with the
// arithmetic of the kernels that write them (pixel_ray of ray_gen.cuh, linspace_at / raw2alpha_one of common.cuh, the dense-grid
// read of trilinear.cuh), and the bounds are reduced warp -> block -> one atomicMin / atomicMax per block and axis on an
// order-preserving integer encoding of the float.  Min and max are order independent, so the result is exact and deterministic.
#include "ray_gen.cuh"
#include "trilinear.cuh"

namespace ubn {

constexpr int kBoundsThreads = 256;

// Order-preserving map float -> uint32 (a < b  <=>  enc(a) < enc(b) for non-NaN floats; -0 sorts below +0).  NaN maps to the
// bottom of the min order and to the top of the max order, so a NaN anywhere wins both reductions, as torch.minimum / amin
// propagate it; both extreme codes decode to a NaN.
__device__ __forceinline__ uint32_t enc_ordered(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ uint32_t enc_for_min(float f) { return f != f ? 0u : enc_ordered(f); }
__device__ __forceinline__ uint32_t enc_for_max(float f) { return f != f ? 0xffffffffu : enc_ordered(f); }
__device__ __forceinline__ float dec_ordered(uint32_t e) {
  return __uint_as_float((e & 0x80000000u) ? (e & 0x7fffffffu) : ~e);
}

// The running bounds of one thread: mn[] in min order, mx[] in max order; starts empty (the identities of the two reductions).
struct BoundsAcc {
  uint32_t mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu};
  uint32_t mx[3] = {0u, 0u, 0u};
  __device__ __forceinline__ void add(float x, float y, float z) {
    mn[0] = min(mn[0], enc_for_min(x)); mn[1] = min(mn[1], enc_for_min(y)); mn[2] = min(mn[2], enc_for_min(z));
    mx[0] = max(mx[0], enc_for_max(x)); mx[1] = max(mx[1], enc_for_max(y)); mx[2] = max(mx[2], enc_for_max(z));
  }
};

// Block reduction of every thread's BoundsAcc (and count) into acc[6] (encoded: min xyz, max xyz) and *count.  Every thread of the
// block calls it.
__device__ __forceinline__ void commit_bounds(const BoundsAcc& a, uint32_t cnt, uint32_t* __restrict__ acc,
                                              unsigned long long* __restrict__ count) {
  __shared__ uint32_t s[kBoundsThreads / 32][7];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t v[7];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    v[k] = __reduce_min_sync(0xffffffffu, a.mn[k]);
    v[3 + k] = __reduce_max_sync(0xffffffffu, a.mx[k]);
  }
  v[6] = __reduce_add_sync(0xffffffffu, cnt);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 7; ++k) s[warp][k] = v[k];
  }
  __syncthreads();
  if (threadIdx.x < 7) {
    const int k = threadIdx.x;
    uint32_t r = s[0][k];
    for (int w = 1; w < kBoundsThreads / 32; ++w) r = k < 3 ? min(r, s[w][k]) : (k < 6 ? max(r, s[w][k]) : r + s[w][k]);
    if (k < 3) {
      if (r != 0xffffffffu) atomicMin(acc + k, r);
    } else if (k < 6) {
      if (r != 0u) atomicMax(acc + k, r);
    } else if (count && r) {
      atomicAdd(count, (unsigned long long)r);
    }
  }
}

// bounds[6] floats <-> the encoded accumulator, in place (one thread per slot)
__global__ void k_bounds_encode(uint32_t* __restrict__ acc) {
  const int k = threadIdx.x;
  if (k < 6) acc[k] = k < 3 ? enc_for_min(__uint_as_float(acc[k])) : enc_for_max(__uint_as_float(acc[k]));
}
__global__ void k_bounds_decode(uint32_t* __restrict__ acc) {
  const int k = threadIdx.x;
  if (k < 6) acc[k] = __float_as_uint(dec_ordered(acc[k]));
}

struct FrustumArgs {
  const int* hw;          // [n_views, 2] (H, W), device
  const float* K;         // [n_views, 9], device
  const float* c2w;       // [n_views, 12] = c2w[:3, :4], device
  int ndc, inverse_y, flip_x, flip_y;
  int inward;             // 1: rays_o + rays_d * near (unbounded-inward / nerfpp); 0: the bounded near and far points
  float near, far;
};

// one view per blockIdx.y (view0 + blockIdx.y), its pixels strided over blockIdx.x; pixel ray as k_rays_of_a_view (mode 'center')
__global__ void __launch_bounds__(kBoundsThreads) k_frustum_bounds(FrustumArgs a, int64_t view0, uint32_t* __restrict__ acc) {
  const int64_t view = view0 + blockIdx.y;
  ViewParams v;
  v.H = a.hw[2 * view]; v.W = a.hw[2 * view + 1];
  const float* K = a.K + 9 * view;
  const float* c = a.c2w + 12 * view;
  v.fx = K[0]; v.cx = K[2]; v.fy = K[4]; v.cy = K[5];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int q = 0; q < 3; ++q) v.r[r][q] = c[4 * r + q];
    v.t[r] = c[4 * r + 3];
  }
  v.ndc = a.ndc; v.inverse_y = a.inverse_y; v.flip_x = a.flip_x; v.flip_y = a.flip_y;
  v.pix = 0.5f;
  v.sw = v.sh = 0.f;
  if (v.ndc) ndc_scales(v.H, v.W, v.fx, v.sw, v.sh);
  const int64_t n = (int64_t)v.H * v.W;
  BoundsAcc b;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const int row = (int)(p / v.W), col = (int)(p - (int64_t)row * v.W);
    float ro[3], rd[3], vd[3];
    pixel_ray(v, row, col, nullptr, ro, rd, vd);
    if (a.inward) {   // pts = rays_o + rays_d * near_clip  (bbox_compute.py:19, :38)
      b.add(__fadd_rn(ro[0], __fmul_rn(rd[0], a.near)), __fadd_rn(ro[1], __fmul_rn(rd[1], a.near)),
            __fadd_rn(ro[2], __fmul_rn(rd[2], a.near)));
    } else {          // rays_o + dir * near / far, dir = rays_d under NDC, viewdirs otherwise  (:104-107)
      const float* d = v.ndc ? rd : vd;
      b.add(__fadd_rn(ro[0], __fmul_rn(d[0], a.near)), __fadd_rn(ro[1], __fmul_rn(d[1], a.near)),
            __fadd_rn(ro[2], __fmul_rn(d[2], a.near)));
      b.add(__fadd_rn(ro[0], __fmul_rn(d[0], a.far)), __fadd_rn(ro[1], __fmul_rn(d[1], a.far)),
            __fadd_rn(ro[2], __fmul_rn(d[2], a.far)));
    }
  }
  commit_bounds(b, 0u, acc, nullptr);
}

struct Lattice {
  float lo[3], hi[3];
  int X, Y, Z;
};

// dense_xyz[i,j,k] = xyz_min * (1 - t) + xyz_max * t with t = linspace(0, 1, n) per axis (bbox_compute.py:144-149): torch's
// four elementwise kernels, each rounded (no fma contraction across them)
__device__ __forceinline__ void lattice_point(const Lattice& L, int64_t idx, float& x, float& y, float& z) {
  const int k = (int)(idx % L.Z), j = (int)((idx / L.Z) % L.Y), i = (int)(idx / ((int64_t)L.Z * L.Y));
  const float tx = linspace_at(0.f, 1.f, L.X, i), ty = linspace_at(0.f, 1.f, L.Y, j), tz = linspace_at(0.f, 1.f, L.Z, k);
  x = __fadd_rn(__fmul_rn(L.lo[0], __fsub_rn(1.f, tx)), __fmul_rn(L.hi[0], tx));
  y = __fadd_rn(__fmul_rn(L.lo[1], __fsub_rn(1.f, ty)), __fmul_rn(L.hi[1], ty));
  z = __fadd_rn(__fmul_rn(L.lo[2], __fsub_rn(1.f, tz)), __fmul_rn(L.hi[2], tz));
}

__global__ void __launch_bounds__(256) k_lattice_points(Lattice L, float* __restrict__ xyz) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)L.X * L.Y * L.Z) return;
  float x, y, z;
  lattice_point(L, idx, x, y, z);
  xyz[3 * idx] = x; xyz[3 * idx + 1] = y; xyz[3 * idx + 2] = z;
}

// bounds and count of the lattice points whose alpha > thres; alpha = Raw2Alpha(density(point)) read from the grid (kFused), or
// alpha[idx] precomputed by the caller
template <bool kFused>
__global__ void __launch_bounds__(kBoundsThreads) k_lattice_bounds(GridView g, const float* __restrict__ alpha_in, Lattice L,
                                                                   float shift, float interval, float thres,
                                                                   uint32_t* __restrict__ acc, unsigned long long* __restrict__ count) {
  const int64_t n = (int64_t)L.X * L.Y * L.Z;
  BoundsAcc b;
  uint32_t cnt = 0;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * blockDim.x) {
    float x, y, z;
    lattice_point(L, idx, x, y, z);
    float alpha;
    if (kFused) {
      float e;
      raw2alpha_one(grid_density_at(g, x, y, z), shift, interval, &e, &alpha);
    } else {
      alpha = alpha_in[idx];
    }
    if (alpha > thres) {
      b.add(x, y, z);
      ++cnt;
    }
  }
  commit_bounds(b, cnt, acc, count);
}

inline Lattice make_lattice(const float* lo, const float* hi, int64_t X, int64_t Y, int64_t Z) {
  Lattice L;
  for (int a = 0; a < 3; ++a) { L.lo[a] = lo[a]; L.hi[a] = hi[a]; }
  L.X = (int)X; L.Y = (int)Y; L.Z = (int)Z;
  return L;
}

// enough blocks to fill the H100 several times over; each block then strides over its share and commits once
inline unsigned reduce_blocks(int64_t n) {
  const int64_t cap = (int64_t)kNumSMs * 16;
  const int64_t need = (n + kBoundsThreads - 1) / kBoundsThreads;
  return (unsigned)(need < cap ? (need > 0 ? need : 1) : cap);
}

}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_frustum_bounds(const int* hw, const float* K, const float* c2w, int64_t n_views, int64_t max_pixels, int ndc, int inverse_y,
                       int flip_x, int flip_y, int inward, float near, float far, float* bounds, void* stream) {
  if (n_views < 0 || max_pixels < 0) return finish(cudaErrorInvalidValue);
  uint32_t* acc = reinterpret_cast<uint32_t*>(bounds);
  const cudaStream_t s = as_stream(stream);
  k_bounds_encode<<<1, 32, 0, s>>>(acc);
  UBN_LAUNCH_CHECK();
  if (n_views > 0 && max_pixels > 0) {
    FrustumArgs a;
    a.hw = hw; a.K = K; a.c2w = c2w;
    a.ndc = ndc; a.inverse_y = inverse_y; a.flip_x = flip_x; a.flip_y = flip_y;
    a.inward = inward; a.near = near; a.far = far;
    // about kNumSMs * 16 blocks over all views, at most one block per 256 pixels of the largest view
    const int64_t per_view = ((int64_t)kNumSMs * 16 + n_views - 1) / n_views;
    const int64_t most = (max_pixels + kBoundsThreads - 1) / kBoundsThreads;
    const unsigned bx = (unsigned)(per_view < most ? per_view : most);
    for (int64_t v0 = 0; v0 < n_views; v0 += 65535) {
      const unsigned by = (unsigned)(n_views - v0 < 65535 ? n_views - v0 : 65535);
      k_frustum_bounds<<<dim3(bx, by), kBoundsThreads, 0, s>>>(a, v0, acc);
      UBN_LAUNCH_CHECK();
    }
  }
  k_bounds_decode<<<1, 32, 0, s>>>(acc);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_lattice_points(const float* lattice_min, const float* lattice_max, int64_t X, int64_t Y, int64_t Z, float* xyz,
                       void* stream) {
  const int64_t n = X * Y * Z;
  if (X < 0 || Y < 0 || Z < 0 || X > INT32_MAX || Y > INT32_MAX || Z > INT32_MAX) return finish(cudaErrorInvalidValue);
  if (n <= 0) return 0;
  k_lattice_points<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(make_lattice(lattice_min, lattice_max, X, Y, Z), xyz);
  UBN_LAUNCH_CHECK();
  return 0;
}

static int lattice_bounds(const float* grid, const UbnGridDesc* desc, const float* alpha, const float* lattice_min,
                          const float* lattice_max, int64_t X, int64_t Y, int64_t Z, float act_shift, float interval, float thres,
                          float* bounds, int64_t* count, void* stream) {
  if (X < 0 || Y < 0 || Z < 0 || X > INT32_MAX || Y > INT32_MAX || Z > INT32_MAX) return finish(cudaErrorInvalidValue);
  const int64_t n = X * Y * Z;
  uint32_t* acc = reinterpret_cast<uint32_t*>(bounds);
  unsigned long long* cnt = reinterpret_cast<unsigned long long*>(count);
  const cudaStream_t s = as_stream(stream);
  const Lattice L = make_lattice(lattice_min, lattice_max, X, Y, Z);
  k_bounds_encode<<<1, 32, 0, s>>>(acc);
  UBN_LAUNCH_CHECK();
  if (n > 0) {
    if (grid) {
      k_lattice_bounds<true><<<reduce_blocks(n), kBoundsThreads, 0, s>>>(make_view(grid, desc), nullptr, L, act_shift, interval,
                                                                         thres, acc, cnt);
    } else {
      GridView none{};
      k_lattice_bounds<false><<<reduce_blocks(n), kBoundsThreads, 0, s>>>(none, alpha, L, 0.f, 0.f, thres, acc, cnt);
    }
    UBN_LAUNCH_CHECK();
  }
  k_bounds_decode<<<1, 32, 0, s>>>(acc);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_lattice_bounds(const float* grid, const UbnGridDesc* desc, const float* lattice_min, const float* lattice_max, int64_t X,
                       int64_t Y, int64_t Z, float act_shift, float interval, float thres, float* bounds, int64_t* count,
                       void* stream) {
  if (!grid || !desc || desc->C != 1) return finish(cudaErrorInvalidValue);
  return lattice_bounds(grid, desc, nullptr, lattice_min, lattice_max, X, Y, Z, act_shift, interval, thres, bounds, count, stream);
}

int ubn_lattice_bounds_alpha(const float* alpha, const float* lattice_min, const float* lattice_max, int64_t X, int64_t Y,
                             int64_t Z, float thres, float* bounds, int64_t* count, void* stream) {
  if (!alpha && X * Y * Z > 0) return finish(cudaErrorInvalidValue);
  return lattice_bounds(nullptr, nullptr, alpha, lattice_min, lattice_max, X, Y, Z, 0.f, 0.f, thres, bounds, count, stream);
}

}  // extern "C"
