// color.cu -- the colour transfer of the ARF stylizer: arf.py:60-89 (ARF.match_colors_for_image_set) -> ubn_color_moments and
// ubn_color_affine.
//
// The reference uploads the rendered set, centres it twice, forms the 3 x 3 covariance with one fp32 cuBLAS matmul whose inner
// dimension is the pixel count, and applies the transform with a second matmul, an add and a clamp: about ten set-sized passes
// and three set-sized buffers alive at once.  Here the work is one read for the moments and one read + one write for the
// transform; the 3 x 3 algebra in between runs on the host in fp64.
//
// Moments.  Each pixel x contributes d = x - k, with k the set's first pixel, to nine fp64 sums: d0, d1, d2 and the six distinct
// products d_i d_j.  The shift keeps the covariance from cancelling catastrophically (sum(x x^T) - n mu mu^T loses everything
// where the variance is small against mu^2).  Every thread walks the set with a grid stride and 64-bit indices; where the pixel
// run is 16-byte aligned it reads four pixels as three float4, with at most three scalar pixels before and after.  The sums are
// reduced in a fixed order -- xor shuffles, the block's warps in index order, per-block fp64 partials, then one closing block that
// adds the partials in block order -- and the grid size depends on n_px only, so two calls on the same input give the same bits.
//
// Affine.  y = clamp(T x + b, 0, 1) per pixel, each channel evaluated as fma(T[c][2], x2, fma(T[c][1], x1, fma(T[c][0], x0, b[c])))
// and clamped as ATen's CUDA clamp does (NaN passes through, then fminf(fmaxf(y, 0), 1)).  In place (in == out) is allowed.
#include "common.cuh"

namespace ubn {

constexpr int kColorThreads = 256;
constexpr int kColorWarps = kColorThreads / 32;

struct ColorAffine {
  float t[9];  // row-major T
  float b[3];
};

// The number of leading pixels before the first pixel whose address is 16-byte aligned.  A pixel is 12 bytes, so pixel j of a
// 4-byte aligned pointer p sits at p + 12 j = p - 4 j (mod 16): pixel (p mod 16) / 4 is aligned.
__host__ __device__ __forceinline__ int64_t color_head(const float* p, int64_t n_px) {
  const int64_t head = (int64_t)((reinterpret_cast<uintptr_t>(p) & 15u) >> 2);
  return head < n_px ? head : n_px;
}

struct Moments {
  double s[9];  // d0, d1, d2, d0d0, d0d1, d0d2, d1d1, d1d2, d2d2

  __device__ __forceinline__ void add(float x0, float x1, float x2, double k0, double k1, double k2) {
    const double d0 = (double)x0 - k0, d1 = (double)x1 - k1, d2 = (double)x2 - k2;
    s[0] += d0;
    s[1] += d1;
    s[2] += d2;
    s[3] = fma(d0, d0, s[3]);
    s[4] = fma(d0, d1, s[4]);
    s[5] = fma(d0, d2, s[5]);
    s[6] = fma(d1, d1, s[6]);
    s[7] = fma(d1, d2, s[7]);
    s[8] = fma(d2, d2, s[8]);
  }
};

// The nine sums of the block, in a fixed order (xor tree within each warp, then the warps in index order), valid in thread 0.
__device__ __forceinline__ void block_sum9(double* v) {
  __shared__ double warp_sums[kColorWarps][9];
#pragma unroll
  for (int i = 0; i < 9; ++i) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int i = 0; i < 9; ++i) warp_sums[threadIdx.x >> 5][i] = v[i];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      double s = 0.0;
      for (int w = 0; w < kColorWarps; ++w) s += warp_sums[w][i];
      v[i] = s;
    }
  }
}

__global__ void __launch_bounds__(kColorThreads) k_color_moments(const float* __restrict__ px, int64_t n_px, int64_t head,
                                                                 double* __restrict__ partial) {
  const double k0 = px[0], k1 = px[1], k2 = px[2];
  Moments m;
#pragma unroll
  for (int i = 0; i < 9; ++i) m.s[i] = 0.0;
  const int64_t tid = (int64_t)blockIdx.x * kColorThreads + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * kColorThreads;
  const int64_t n_groups = (n_px - head) / 4;
  const int64_t tail0 = head + 4 * n_groups;
  if (tid < head) m.add(px[3 * tid], px[3 * tid + 1], px[3 * tid + 2], k0, k1, k2);
  const float4* v = reinterpret_cast<const float4*>(px + 3 * head);
  for (int64_t g = tid; g < n_groups; g += stride) {
    const float4 a = __ldg(v + 3 * g), b = __ldg(v + 3 * g + 1), c = __ldg(v + 3 * g + 2);
    m.add(a.x, a.y, a.z, k0, k1, k2);
    m.add(a.w, b.x, b.y, k0, k1, k2);
    m.add(b.z, b.w, c.x, k0, k1, k2);
    m.add(c.y, c.z, c.w, k0, k1, k2);
  }
  if (tid < n_px - tail0) {
    const int64_t p = tail0 + tid;
    m.add(px[3 * p], px[3 * p + 1], px[3 * p + 2], k0, k1, k2);
  }
  block_sum9(m.s);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < 9; ++i) partial[(int64_t)blockIdx.x * 9 + i] = m.s[i];
  }
}

// out = [mu0, mu1, mu2, c00, c01, c02, c11, c12, c22]: the partials of n_blocks blocks added in block order (each thread a fixed
// stride, then the fixed tree); m = S / n, mu = k + m, c_ij = S_ij / n - m_i m_j (population covariance, as arf.py:68-69).
__global__ void __launch_bounds__(kColorThreads) k_color_moments_close(const float* __restrict__ px, int64_t n_px,
                                                                       const double* __restrict__ partial, int n_blocks,
                                                                       double* __restrict__ out) {
  double v[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) v[i] = 0.0;
  for (int b = threadIdx.x; b < n_blocks; b += kColorThreads) {
#pragma unroll
    for (int i = 0; i < 9; ++i) v[i] += partial[(int64_t)b * 9 + i];
  }
  block_sum9(v);
  if (threadIdx.x == 0) {
    const double n = (double)n_px;
    const double m0 = v[0] / n, m1 = v[1] / n, m2 = v[2] / n;
    out[0] = (double)px[0] + m0;
    out[1] = (double)px[1] + m1;
    out[2] = (double)px[2] + m2;
    out[3] = __dsub_rn(v[3] / n, __dmul_rn(m0, m0));
    out[4] = __dsub_rn(v[4] / n, __dmul_rn(m0, m1));
    out[5] = __dsub_rn(v[5] / n, __dmul_rn(m0, m2));
    out[6] = __dsub_rn(v[6] / n, __dmul_rn(m1, m1));
    out[7] = __dsub_rn(v[7] / n, __dmul_rn(m1, m2));
    out[8] = __dsub_rn(v[8] / n, __dmul_rn(m2, m2));
  }
}

__device__ __forceinline__ float clamp01(float y) { return (y != y) ? y : fminf(fmaxf(y, 0.f), 1.f); }

__device__ __forceinline__ void affine_px(const ColorAffine& a, float x0, float x1, float x2, float& y0, float& y1, float& y2) {
  y0 = clamp01(fmaf(a.t[2], x2, fmaf(a.t[1], x1, fmaf(a.t[0], x0, a.b[0]))));
  y1 = clamp01(fmaf(a.t[5], x2, fmaf(a.t[4], x1, fmaf(a.t[3], x0, a.b[1]))));
  y2 = clamp01(fmaf(a.t[8], x2, fmaf(a.t[7], x1, fmaf(a.t[6], x0, a.b[2]))));
}

// No __restrict__: in == out is allowed (each element is read before it is written, by the same thread).
__global__ void __launch_bounds__(kColorThreads) k_color_affine(const float* in, float* out, int64_t n_px, int64_t head,
                                                                ColorAffine a) {
  const int64_t tid = (int64_t)blockIdx.x * kColorThreads + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * kColorThreads;
  const int64_t n_groups = (n_px - head) / 4;
  const int64_t tail0 = head + 4 * n_groups;
  float y0, y1, y2;
  if (tid < head) {
    affine_px(a, in[3 * tid], in[3 * tid + 1], in[3 * tid + 2], y0, y1, y2);
    out[3 * tid] = y0; out[3 * tid + 1] = y1; out[3 * tid + 2] = y2;
  }
  const float4* vi = reinterpret_cast<const float4*>(in + 3 * head);
  float4* vo = reinterpret_cast<float4*>(out + 3 * head);
  for (int64_t g = tid; g < n_groups; g += stride) {
    const float4 p = vi[3 * g], q = vi[3 * g + 1], r = vi[3 * g + 2];
    float4 P, Q, R;
    affine_px(a, p.x, p.y, p.z, P.x, P.y, P.z);
    affine_px(a, p.w, q.x, q.y, P.w, Q.x, Q.y);
    affine_px(a, q.z, q.w, r.x, Q.z, Q.w, R.x);
    affine_px(a, r.y, r.z, r.w, R.y, R.z, R.w);
    vo[3 * g] = P; vo[3 * g + 1] = Q; vo[3 * g + 2] = R;
  }
  if (tid < n_px - tail0) {
    const int64_t p = tail0 + tid;
    affine_px(a, in[3 * p], in[3 * p + 1], in[3 * p + 2], y0, y1, y2);
    out[3 * p] = y0; out[3 * p + 1] = y1; out[3 * p + 2] = y2;
  }
}

// Where in and out are aligned differently no pixel is 16-byte aligned in both: one pixel per thread, scalar loads and stores.
__global__ void __launch_bounds__(kColorThreads) k_color_affine_scalar(const float* in, float* out, int64_t n_px, ColorAffine a) {
  const int64_t stride = (int64_t)gridDim.x * kColorThreads;
  for (int64_t p = (int64_t)blockIdx.x * kColorThreads + threadIdx.x; p < n_px; p += stride) {
    float y0, y1, y2;
    affine_px(a, in[3 * p], in[3 * p + 1], in[3 * p + 2], y0, y1, y2);
    out[3 * p] = y0; out[3 * p + 1] = y1; out[3 * p + 2] = y2;
  }
}

inline int color_blocks(int64_t work) {
  const int64_t b = ceil_div<int64_t>(work, kColorThreads);
  return (int)(b < 1 ? 1 : (b < UBN_COLOR_MAX_CTAS ? b : UBN_COLOR_MAX_CTAS));
}

}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_color_moments(const float* px, int64_t n_px, double* scratch, double* out, void* stream) {
  if (!px || !scratch || !out || n_px < 1 || (reinterpret_cast<uintptr_t>(px) & 3u)) return finish(cudaErrorInvalidValue);
  const int64_t head = color_head(px, n_px);
  const int blocks = color_blocks((n_px - head) / 4 > 4 ? (n_px - head) / 4 : 4);
  const cudaStream_t s = as_stream(stream);
  k_color_moments<<<blocks, kColorThreads, 0, s>>>(px, n_px, head, scratch);
  UBN_LAUNCH_CHECK();
  k_color_moments_close<<<1, kColorThreads, 0, s>>>(px, n_px, scratch, blocks, out);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_color_affine(const float* in, float* out, int64_t n_px, const float* T, const float* b, void* stream) {
  if (!in || !out || !T || !b || n_px < 0 || ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 3u))
    return finish(cudaErrorInvalidValue);
  if (n_px == 0) return 0;
  ColorAffine a;
  for (int i = 0; i < 9; ++i) a.t[i] = T[i];
  for (int i = 0; i < 3; ++i) a.b[i] = b[i];
  const cudaStream_t s = as_stream(stream);
  const int64_t head = color_head(in, n_px);
  if (head == color_head(out, n_px)) {
    k_color_affine<<<color_blocks((n_px - head) / 4 > 4 ? (n_px - head) / 4 : 4), kColorThreads, 0, s>>>(in, out, n_px, head, a);
  } else {
    k_color_affine_scalar<<<color_blocks(n_px), kColorThreads, 0, s>>>(in, out, n_px, a);
  }
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
