// rgbnet_tc.cuh -- the tensor-core (mma.sync m16n8k8, kind TF32, 3xTF32) building blocks of the rgbnet: B-fragment staging,
// the hi / lo split and the warp GEMM over 16-sample units.  Shared by shade_tc.cu (the rgbnet kernels) and render.cu (the fused
// render), so both evaluate every product in the same order.
#pragma once
#include "common.cuh"

namespace ubn {
namespace tc {

// Hidden width kW is a template parameter of every kernel: 128 (every 12-channel config, the FourierGrid K = 3 / 15 configs)
// or 64 (DirectMPIGO's llff_default, K = 9).  Everything below that sizes a layer derives from it.
constexpr int kHidden = 128;            // the width of the kernels that keep their own names (k_shade_fwd_tc, k_shade_bwd_tc, ...)
constexpr int kFeat = 12;               // feature columns of every shipped 12-channel config; kernels take kF in {3, 9, 12, 15}
constexpr int kUnit = 16;               // samples per warp unit (the M of one mma)
constexpr int kPanelRows = 128;         // row block of the panel save layout
__host__ __device__ constexpr int n_tiles(int w) { return w / 8; }      // 8-column tiles of a w-wide layer
__host__ __device__ constexpr int stride(int w) { return w + 8; }       // floats per row of a shared-memory operand tile
                                                                        // (conflict-free both ways)

// B-fragment tables (uint4 per lane): [n-tile][k-step][32 lanes]
__host__ __device__ constexpr uint32_t frag_w2(int w) { return n_tiles(w) * n_tiles(w) * 32 * 16; }  // 128 KB at w = 128
__host__ __device__ constexpr uint32_t frag_w1(int w) { return n_tiles(w) * 2 * 32 * 16; }  // layer 1: K <= 16 (2 k-steps)

__device__ __forceinline__ uint32_t tf32_hi_bits(float x) { return __float_as_uint(x) & 0xFFFFE000u; }

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void split4(const float (&v)[4], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    hi[i] = tf32_hi_bits(v[i]);
    lo[i] = __float_as_uint(v[i] - __uint_as_float(hi[i]));
  }
}

// d += a . b with (a, b) given as hi / lo halves; kThree adds the two cross terms
template <bool kThree>
__device__ __forceinline__ void mma3(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], uint4 b) {
  if (kThree) {
    mma_tf32(d, al, b.x, b.y);
    mma_tf32(d, ah, b.z, b.w);
  }
  mma_tf32(d, ah, b.x, b.y);
}

// Stage B[k][n] (k < K, n < N; zero outside) as B fragments for k-steps reading units 8 s + 2 t / 8 s + 2 t + 1:
// lane (g, t) of (n-tile j, k-step s) gets {hi(B[8s+2t][8j+g]), hi(B[8s+2t+1][8j+g]), lo(..), lo(..)}.
// B[k][n] = trans ? W[n * ld + k] : W[k * ld + n].
inline __device__ void stage_frags(const float* __restrict__ W, int ld, bool trans, int K, int N, int n_ksteps, int n_ntiles,
                            uint4* dst, int tid, int nthreads) {
  for (int i = tid; i < n_ntiles * n_ksteps * 32; i += nthreads) {
    const int lane = i & 31, s = (i >> 5) % n_ksteps, j = (i >> 5) / n_ksteps;
    const int n = 8 * j + (lane >> 2), k0 = 8 * s + 2 * (lane & 3);
    float w[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int k = k0 + e;
      w[e] = (k < K && n < N) ? (trans ? W[n * ld + k] : W[k * ld + n]) : 0.f;
    }
    const uint32_t h0 = tf32_hi_bits(w[0]), h1 = tf32_hi_bits(w[1]);
    dst[i] = make_uint4(h0, h1, __float_as_uint(w[0] - __uint_as_float(h0)), __float_as_uint(w[1] - __uint_as_float(h1)));
  }
}

// acc[NT] += X . B, X given in accumulator layout (x[s] = column tile s of the previous layer), B from stage_frags
template <int KS, int NT, bool kThree>
__device__ __forceinline__ void warp_gemm(float (&acc)[NT][4], const float (&x)[KS][4], const uint4* __restrict__ frag, int lane) {
#pragma unroll
  for (int s = 0; s < KS; ++s) {
    const float av[4] = {x[s][0], x[s][2], x[s][1], x[s][3]};
    uint32_t ah[4], al[4];
    split4(av, ah, al);
#pragma unroll
    for (int j = 0; j < NT; ++j) mma3<kThree>(acc[j], ah, al, frag[(j * KS + s) * 32 + lane]);
  }
}

// lane (g, t) of (n-tile j, k-step s) gets the fp32 pair {B[8s+2t][8j+g], B[8s+2t+1][8j+g]}, B[k][n] = W[k * ld + n]
// trans: B[k][n] = W[n * ld + k] (the forward layers, as stage_frags)
inline __device__ void stage_frags_f32(const float* __restrict__ W, int ld, int K, int N, int n_ksteps, int n_ntiles, uint2* dst, int tid,
                                       int nthreads, bool trans = false) {
  for (int i = tid; i < n_ntiles * n_ksteps * 32; i += nthreads) {
    const int lane = i & 31, s = (i >> 5) % n_ksteps, j = (i >> 5) / n_ksteps;
    const int n = 8 * j + (lane >> 2), k = 8 * s + 2 * (lane & 3);
    const float w0 = (k < K && n < N) ? (trans ? W[n * ld + k] : W[k * ld + n]) : 0.f;
    const float w1 = (k + 1 < K && n < N) ? (trans ? W[n * ld + k + 1] : W[(k + 1) * ld + n]) : 0.f;
    dst[i] = make_uint2(__float_as_uint(w0), __float_as_uint(w1));
  }
}

// mma3 with the B fragment given as fp32: the same hi / lo split (and the same three products in the same order) as stage_frags
template <bool kThree>
__device__ __forceinline__ void mma3f(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], uint2 b) {
  const uint32_t h0 = b.x & 0xFFFFE000u, h1 = b.y & 0xFFFFE000u;
  if (kThree) {
    mma_tf32(d, al, h0, h1);
    mma_tf32(d, ah, __float_as_uint(__uint_as_float(b.x) - __uint_as_float(h0)),
             __float_as_uint(__uint_as_float(b.y) - __uint_as_float(h1)));
  }
  mma_tf32(d, ah, h0, h1);
}

template <int KS, int NT, bool kThree>
__device__ __forceinline__ void warp_gemm_f(float (&acc)[NT][4], const float (&x)[KS][4], const uint2* __restrict__ frag, int lane) {
#pragma unroll
  for (int s = 0; s < KS; ++s) {
    const float av[4] = {x[s][0], x[s][2], x[s][1], x[s][3]};
    uint32_t ah[4], al[4];
    split4(av, ah, al);
#pragma unroll
    for (int j = 0; j < NT; ++j) mma3f<kThree>(acc[j], ah, al, frag[(j * KS + s) * 32 + lane]);
  }
}

// ---- the forward's epilogues (lane (g, t) holds rows g, g + 8 and columns 8 j + 2 t, + 1 of every column tile j) ----
// epilogue 1: h += bias(r, c) (a float2 for columns c, c + 1 of the lane's row r), ReLU; sink(r, c, h_c, h_c+1) sees the result
template <int kNT, class Bias, class Sink>
__device__ __forceinline__ void epi_bias_relu(float (&h)[kNT][4], int t, Bias&& bias, Sink&& sink) {
#pragma unroll
  for (int j = 0; j < kNT; ++j)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float2 b = bias(r, 8 * j + 2 * t);
      h[j][2 * r] = fmaxf(h[j][2 * r] + b.x, 0.f);
      h[j][2 * r + 1] = fmaxf(h[j][2 * r + 1] + b.y, 0.f);
      sink(r, 8 * j + 2 * t, h[j][2 * r], h[j][2 * r + 1]);
    }
}

// epilogue 2 over the column tiles j0 .. j0 + kNT - 1 of the hidden layer: + b2, ReLU (sink(r, c, a_c, a_c+1) sees it), then the
// layer-3 partial products p[r][i] += a . W3[i] (N = 3: CUDA cores), in column order
template <int kW, int kNT, class Sink>
__device__ __forceinline__ void epi_hidden_layer3(const float (&z)[kNT][4], int j0, int t, const float* sB2, const float* sW3,
                                                  float (&p)[2][3], Sink&& sink) {
#pragma unroll
  for (int jj = 0; jj < kNT; ++jj) {
    const int c = 8 * (j0 + jj) + 2 * t;
    const float2 bb = *reinterpret_cast<const float2*>(sB2 + c);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float a0 = fmaxf(z[jj][2 * r] + bb.x, 0.f), a1 = fmaxf(z[jj][2 * r + 1] + bb.y, 0.f);
      sink(r, c, a0, a1);
#pragma unroll
      for (int i = 0; i < 3; ++i) p[r][i] = fmaf(a1, sW3[i * kW + c + 1], fmaf(a0, sW3[i * kW + c], p[r][i]));
    }
  }
}

// the layer-3 sums of the four t lanes of a row, + b3, sigmoid: sink(r, rgb[3]) on the t == 0 lanes
template <class Sink>
__device__ __forceinline__ void epi_rgb(float (&p)[2][3], const float (&b3)[3], int t, Sink&& sink) {
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      p[r][i] += __shfl_xor_sync(0xffffffffu, p[r][i], 1);
      p[r][i] += __shfl_xor_sync(0xffffffffu, p[r][i], 2);
    }
  if (t == 0) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float v[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) v[i] = 1.f / (1.f + expf(-(p[r][i] + b3[i])));
      sink(r, v);
    }
  }
}

}  // namespace tc
}  // namespace ubn
