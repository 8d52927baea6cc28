// metrics.cu -- the image-quality score of the evaluation step: utils.rgb_ssim (FourierGrid/utils.py:79-125) -> ubn_rgb_ssim.
//
// The reference runs it as scipy convolve2d on the CPU.  Its precision is what this kernel reproduces: img**2 and img0*img1 are
// numpy float32 products (rounded to fp32), while the convolutions and everything after them run in fp64 (scipy promotes the
// float32 image against the float64 taps).  So the three products are formed in fp32 and every moment is accumulated in fp64;
// fp32 moments move the map by up to ~1e-4 on smooth images.
//
// One block stages an output tile plus its f - 1 halo of one channel of both images in shared memory, once.  A horizontal pass
// writes the five filtered moments (mu0, mu1, E[x^2], E[y^2], E[xy]) of every staged row, a vertical pass finishes them and the
// epilogue forms the SSIM map in numpy's order of operations.  Blocks walk the tiles in a fixed order and each writes one fp64
// partial sum of its map values; a one-block closing launch adds the partials in index order.  No floating-point atomics: two
// calls give the same bits.
#include "common.cuh"

namespace ubn {

constexpr int kSsimTW = 32;                                    // output tile width: one warp across
constexpr int kSsimTH = 32;                                    // output tile height
constexpr int kSsimThreads = 256;                              // 32 columns x 8 row groups
constexpr int kSsimRows = kSsimTH / (kSsimThreads / kSsimTW);  // output rows per thread in the vertical pass (4)

struct SsimTaps {
  double w[UBN_SSIM_MAX_TAPS];
};

struct SsimArgs {
  const float* img0;
  const float* img1;
  double* map;                  // [Ho, Wo, 3] or NULL
  int H, W, f, Ho, Wo, tiles_x;
  int64_t n_tiles;              // 3 channels x tiles_y x tiles_x
  double c1, c2;
};

inline size_t ssim_smem_bytes(int f) {
  const size_t RH = kSsimTH + f - 1, RW = kSsimTW + f - 1;
  return 5 * RH * kSsimTW * sizeof(double) + 2 * RH * RW * sizeof(float) + UBN_SSIM_MAX_TAPS * sizeof(double);
}

// numpy's NaN-propagating element functions (CUDA's fmax / fmin drop a NaN operand):
// np.maximum(0., s) = (0 >= s) ? 0 : s;  np.minimum(a, b) = (a <= b || isnan(a)) ? a : b;  np.sign(NaN) = NaN.
__device__ __forceinline__ double np_maximum0(double s) { return (0.0 >= s) ? 0.0 : s; }
__device__ __forceinline__ double np_minimum(double a, double b) { return (a <= b || a != a) ? a : b; }
__device__ __forceinline__ double np_sign(double s) { return s > 0.0 ? 1.0 : (s < 0.0 ? -1.0 : (s == 0.0 ? 0.0 : s)); }

// utils.py:106-123 for one element, every operation rounded on its own in numpy's order: a contracted fma(mu0, mu0, mu1 * mu1)
// differs from 2 * (mu0 * mu1), and identical frames would no longer score exactly 1.
__device__ __forceinline__ double ssim_of(double mu0, double mu1, double e00, double e11, double e01, double c1, double c2) {
  const double mu00 = __dmul_rn(mu0, mu0), mu11 = __dmul_rn(mu1, mu1), mu01 = __dmul_rn(mu0, mu1);
  const double s00 = np_maximum0(__dsub_rn(e00, mu00));
  const double s11 = np_maximum0(__dsub_rn(e11, mu11));
  double s01 = __dsub_rn(e01, mu01);
  s01 = __dmul_rn(np_sign(s01), np_minimum(__dsqrt_rn(__dmul_rn(s00, s11)), fabs(s01)));
  const double numer = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mu01), c1), __dadd_rn(__dmul_rn(2.0, s01), c2));
  const double denom = __dmul_rn(__dadd_rn(__dadd_rn(mu00, mu11), c1), __dadd_rn(__dadd_rn(s00, s11), c2));
  return __ddiv_rn(numer, denom);
}

// Sum of v over the block, in a fixed order (xor-shuffle tree, then the warps in index order); the result is valid in thread 0.
__device__ __forceinline__ double block_sum_fixed(double v) {
  __shared__ double warp_sums[kSsimThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();                                   // warp_sums may still be read by a previous call
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kSsimThreads / 32; ++w) s += warp_sums[w];
  return s;
}

__global__ void __launch_bounds__(kSsimThreads) k_rgb_ssim(SsimArgs a, SsimTaps taps, double* __restrict__ partial) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int f = a.f, RH = kSsimTH + f - 1, RW = kSsimTW + f - 1;
  double* hm = reinterpret_cast<double*>(smem);            // [5][RH][kSsimTW] horizontally filtered moments
  double* w = hm + 5 * RH * kSsimTW;                       // [f] taps
  float* sx = reinterpret_cast<float*>(w + UBN_SSIM_MAX_TAPS);  // [RH][RW] staged img0 channel
  float* sy = sx + RH * RW;                                // [RH][RW] staged img1 channel
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  if (threadIdx.x < f) w[threadIdx.x] = taps.w[threadIdx.x];
  double acc = 0.0;
  for (int64_t tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    const int c = (int)(tile % 3);                         // the three channels of a tile are neighbours: they share lines in L2
    const int64_t rest = tile / 3;
    const int x0 = (int)(rest % a.tiles_x) * kSsimTW, y0 = (int)(rest / a.tiles_x) * kSsimTH;
    __syncthreads();                                       // the previous tile's readers are done (and the taps are written)
    for (int i = threadIdx.x; i < RH * RW; i += kSsimThreads) {
      const int r = i / RW, q = i - r * RW;
      const int gy = y0 + r, gx = x0 + q;
      float x = 0.f, y = 0.f;                              // beyond the image only outputs beyond the map read these
      if (gy < a.H && gx < a.W) {
        const int64_t o = ((int64_t)gy * a.W + gx) * 3 + c;
        x = __ldg(a.img0 + o);
        y = __ldg(a.img1 + o);
      }
      sx[i] = x;
      sy[i] = y;
    }
    __syncthreads();
    // horizontal pass ('valid' convolution along W): h[r][j] = sum_k w[k] * z[r][j + f - 1 - k]
    for (int i = threadIdx.x; i < RH * kSsimTW; i += kSsimThreads) {
      const int r = i / kSsimTW, j = i - r * kSsimTW;
      const float* px = sx + r * RW + j + f - 1;
      const float* py = sy + r * RW + j + f - 1;
      double m0 = 0.0, m1 = 0.0, m00 = 0.0, m11 = 0.0, m01 = 0.0;
      for (int k = 0; k < f; ++k) {
        const float x = px[-k], y = py[-k];
        const double wk = w[k];
        m0 = fma(wk, (double)x, m0);
        m1 = fma(wk, (double)y, m1);
        m00 = fma(wk, (double)__fmul_rn(x, x), m00);     // the fp32 products of img0**2, img1**2, img0*img1
        m11 = fma(wk, (double)__fmul_rn(y, y), m11);
        m01 = fma(wk, (double)__fmul_rn(x, y), m01);
      }
      hm[(0 * RH + r) * kSsimTW + j] = m0;
      hm[(1 * RH + r) * kSsimTW + j] = m1;
      hm[(2 * RH + r) * kSsimTW + j] = m00;
      hm[(3 * RH + r) * kSsimTW + j] = m11;
      hm[(4 * RH + r) * kSsimTW + j] = m01;
    }
    __syncthreads();
    // vertical pass: thread (tx, ty) finishes rows i0 .. i0 + kSsimRows - 1 of column tx; each staged row is read once and added
    // into every output whose window holds it (out[i0 + s] takes row i0 + q with tap k = s + f - 1 - q)
    const int i0 = ty * kSsimRows;
    double m[kSsimRows][5];
#pragma unroll
    for (int s = 0; s < kSsimRows; ++s)
#pragma unroll
      for (int v = 0; v < 5; ++v) m[s][v] = 0.0;
    for (int q = 0; q < f + kSsimRows - 1; ++q) {
      double h[5];
#pragma unroll
      for (int v = 0; v < 5; ++v) h[v] = hm[(v * RH + i0 + q) * kSsimTW + tx];
#pragma unroll
      for (int s = 0; s < kSsimRows; ++s) {
        const int k = s + f - 1 - q;
        if (k >= 0 && k < f) {
          const double wk = w[k];
#pragma unroll
          for (int v = 0; v < 5; ++v) m[s][v] = fma(wk, h[v], m[s][v]);
        }
      }
    }
    const int gx = x0 + tx;
#pragma unroll
    for (int s = 0; s < kSsimRows; ++s) {
      const int gy = y0 + i0 + s;
      if (gy < a.Ho && gx < a.Wo) {
        const double v = ssim_of(m[s][0], m[s][1], m[s][2], m[s][3], m[s][4], a.c1, a.c2);
        if (a.map) a.map[((int64_t)gy * a.Wo + gx) * 3 + c] = v;
        acc += v;
      }
    }
  }
  const double s = block_sum_fixed(acc);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// mean = (partial[0] + ... + partial[n - 1]) / count, every thread's stride and the tree in a fixed order
__global__ void __launch_bounds__(kSsimThreads) k_ssim_mean(const double* __restrict__ partial, int n, double count,
                                                            double* __restrict__ mean) {
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += kSsimThreads) v += partial[i];
  const double s = block_sum_fixed(v);
  if (threadIdx.x == 0) *mean = __ddiv_rn(s, count);
}

}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_rgb_ssim(const float* img0, const float* img1, int64_t H, int64_t W, int filter_size, const double* taps, double c1,
                 double c2, double* map, double* scratch, double* mean, void* stream) {
  if (!img0 || !img1 || !taps || !scratch || !mean || filter_size < 1 || filter_size > UBN_SSIM_MAX_TAPS || H < filter_size ||
      W < filter_size || H > INT32_MAX || W > INT32_MAX)
    return finish(cudaErrorInvalidValue);
  SsimArgs a;
  a.img0 = img0; a.img1 = img1; a.map = map;
  a.H = (int)H; a.W = (int)W; a.f = filter_size;
  a.Ho = (int)(H - filter_size + 1); a.Wo = (int)(W - filter_size + 1);
  a.tiles_x = ceil_div(a.Wo, kSsimTW);
  a.n_tiles = 3 * (int64_t)ceil_div(a.Ho, kSsimTH) * a.tiles_x;
  a.c1 = c1; a.c2 = c2;
  SsimTaps t = {};
  for (int k = 0; k < filter_size; ++k) t.w[k] = taps[k];
  const size_t smem = ssim_smem_bytes(filter_size);
  cudaError_t e = cudaFuncSetAttribute(k_rgb_ssim, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return finish(e);
  const int blocks = (int)(a.n_tiles < UBN_SSIM_MAX_CTAS ? a.n_tiles : UBN_SSIM_MAX_CTAS);
  const cudaStream_t s = as_stream(stream);
  k_rgb_ssim<<<blocks, kSsimThreads, smem, s>>>(a, t, scratch);
  UBN_LAUNCH_CHECK();
  k_ssim_mean<<<1, kSsimThreads, 0, s>>>(scratch, blocks, (double)a.Ho * (double)a.Wo * 3.0, mean);
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
