// shade_tc.cu -- rgbnet forward and backward on the Hopper tensor cores (mma.sync m16n8k8, kind TF32), sm_90a.
//
// Same contract as k_shade_fwd / k_shade_bwd (shade.cu): rgb = sigmoid(W3 relu(W2 relu(W1k x + vb[ray]) + b2) + b3).
// Every warp owns 16-sample units and keeps the whole activation chain in registers: the accumulator fragment of one
// layer IS the A fragment of the next.  mma.m16n8k8 gives thread (g = lane / 4, t = lane % 4) the accumulator elements
// (row g, columns 2t, 2t + 1) and (row g + 8, same columns) of each 8-column tile, and wants A elements (row g, k = t) and
// (row g, k = t + 4).  The contraction order is free, so k-step s reads hidden units 8 s + 2 t as "k = t" and 8 s + 2 t + 1
// as "k = t + 4": the layer-1 accumulators of column tile s are the layer-2 A operand of k-step s without a shuffle.
// The weights are staged once per CTA in shared memory as ready-made B fragments in that same k order (one 16-byte
// {hi0, hi1, lo0, lo1} load per thread, tile and k-step, conflict-free).
//
// Precision: a single TF32 pass has ~1e-3 relative error, two orders of magnitude above the 1e-5 parity gate.  Every
// operand is therefore split into hi = tf32(x) and lo = x - hi (exact in fp32) and each product is the 3-term sum
// hi*hi + lo*hi + hi*lo accumulated in fp32 ("3xTF32", error ~2^-21).  single_pass (UBN_RGBNET_MODE=tc1) runs hi*hi only.
//
// Sample reductions of the backward (dW1k, dW3, db2, grad_view_bias) run on the tensor cores too: their contraction
// index is the sample, which the accumulator layout spreads over g, so the warp turns the 16 x 128 operand through a
// private shared-memory tile and reads it back as B fragments (sample = k).  Their per-unit results go into running sums
// that each warp owns, so the backward has no shared-memory atomics (sm_90 has no native shared fp32 add: those would be
// compare-and-swap loops).
#include <algorithm>

#include "rgbnet_tc.cuh"

namespace ubn {
namespace tc {

// element offset of (row, col) in a save buffer: row-major [n][kW], or the panel layout [n/128][kW/4 quads][128 rows][4]
template <bool kPanel, int kW>
__device__ __forceinline__ int64_t save_idx(int64_t row, int col) {
  if (kPanel) return (row >> 7) * (kPanelRows * kW) + (int64_t)(col >> 2) * (kPanelRows * 4) + (row & 127) * 4 + (col & 3);
  return row * kW + col;
}

// ReLU mask words: [n/128][kW/32 chunks of 32 units][128 rows], bit e = unit 32 c + e
template <int kW>
__device__ __forceinline__ int64_t mask_idx(int64_t row, int chunk) {
  return (row >> 7) * (kW / 32 * kPanelRows) + chunk * kPanelRows + (row & 127);
}

// OR of this thread's bits of chunk c (units 8 j + 2 t, + 1 for j = 4 c .. 4 c + 3) over the four t lanes of a row
template <int kNT>
__device__ __forceinline__ uint32_t mask_chunk(const float (&h)[kNT][4], int c, int e0, int t) {
  uint32_t w = 0;
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = 4 * c + jj;
    w |= (h[j][e0] > 0.f ? 1u : 0u) << (8 * jj + 2 * t);
    w |= (h[j][e0 + 1] > 0.f ? 1u : 0u) << (8 * jj + 2 * t + 1);
  }
  w |= __shfl_xor_sync(0xffffffffu, w, 1);
  w |= __shfl_xor_sync(0xffffffffu, w, 2);
  return w;
}

// ---- forward ---------------------------------------------------------------------------------------------------------
// shared memory: W2 fragments, W1k fragments, W3 [3][kW], b2 [kW]
namespace fw {
__host__ __device__ constexpr uint32_t oW1(int w) { return frag_w2(w); }
__host__ __device__ constexpr uint32_t oW3(int w) { return oW1(w) + frag_w1(w); }
__host__ __device__ constexpr uint32_t oB2(int w) { return oW3(w) + 3 * w * 4; }
__host__ __device__ constexpr uint32_t smem(int w) { return oB2(w) + w * 4; }
}  // namespace fw

#define UBN_SHADE_FWD_PARAMS                                                                                                 \
  const float* __restrict__ feat, const float* __restrict__ vb, const int64_t* __restrict__ ray_id,                          \
      const float* __restrict__ W1k, const float* __restrict__ W2, const float* __restrict__ b2, const float* __restrict__ W3, \
      const float* __restrict__ b3, int64_t n_pts, float* __restrict__ rgb, float* __restrict__ h1_out,                      \
      float* __restrict__ h2_out, uint32_t* __restrict__ h1_mask
#define UBN_SHADE_FWD_ARGS feat, vb, ray_id, W1k, W2, b2, W3, b3, n_pts, rgb, h1_out, h2_out, h1_mask

// kF feature columns: ceil(kF / 8) k-steps of layer 1 (1 for kF = 3, 2 for 9, 12 and 15); odd kF rows are 4-byte aligned
template <int kF, int kW, bool kSave, bool kThree, int kWarps, bool kPanel>
__device__ __forceinline__ void shade_fwd_tc(UBN_SHADE_FWD_PARAMS) {
  constexpr int kNT = n_tiles(kW);
  extern __shared__ __align__(16) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const uint4* fW2 = reinterpret_cast<const uint4*>(smem);
  const uint4* fW1 = reinterpret_cast<const uint4*>(smem + fw::oW1(kW));
  float* sW3 = reinterpret_cast<float*>(smem + fw::oW3(kW));
  float* sB2 = reinterpret_cast<float*>(smem + fw::oB2(kW));
  stage_frags(W2, kW, true, kW, kW, kNT, kNT, reinterpret_cast<uint4*>(smem), tid, 32 * kWarps);
  constexpr int kKS = (kF + 7) / 8;
  stage_frags(W1k, kF, true, kF, kW, kKS, kNT, reinterpret_cast<uint4*>(smem + fw::oW1(kW)), tid, 32 * kWarps);
  for (int i = tid; i < 3 * kW; i += 32 * kWarps) sW3[i] = W3[i];
  for (int i = tid; i < kW; i += 32 * kWarps) sB2[i] = b2[i];
  __syncthreads();
  const float b3v[3] = {b3[0], b3[1], b3[2]};

  const int64_t n_units = (n_pts + kUnit - 1) / kUnit;
  for (int64_t u = (int64_t)blockIdx.x * kWarps + (tid >> 5); u < n_units; u += (int64_t)gridDim.x * kWarps) {
    const int64_t row[2] = {u * kUnit + g, u * kUnit + g + 8};
    const bool live[2] = {row[0] < n_pts, row[1] < n_pts};
    // layer 1: X in accumulator layout, column tile s = features 8 s .. 8 s + 7 (kF .. 8 kKS - 1 are zero)
    float x[kKS][4];
#pragma unroll
    for (int s = 0; s < kKS; ++s)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float2 v = make_float2(0.f, 0.f);
        if constexpr (kF % 2 == 0) {
          if (live[r] && 8 * s + 2 * t < kF) v = *reinterpret_cast<const float2*>(feat + row[r] * kF + 8 * s + 2 * t);
        } else if (live[r]) {
          const int c = 8 * s + 2 * t;
          if (c < kF) v.x = feat[row[r] * kF + c];
          if (c + 1 < kF) v.y = feat[row[r] * kF + c + 1];
        }
        x[s][2 * r] = v.x;
        x[s][2 * r + 1] = v.y;
      }
    const int64_t ray[2] = {live[0] ? ray_id[row[0]] : 0, live[1] ? ray_id[row[1]] : 0};
    float h[kNT][4];
#pragma unroll
    for (int j = 0; j < kNT; ++j) h[j][0] = h[j][1] = h[j][2] = h[j][3] = 0.f;
    warp_gemm<kKS, kNT, kThree>(h, x, fW1, lane);
    // epilogue 1: + vb[ray], ReLU
    epi_bias_relu<kNT>(
        h, t, [&](int r, int c) { return __ldg(reinterpret_cast<const float2*>(vb + ray[r] * kW + c)); },
        [&](int r, int c, float v0, float v1) {
          if (kSave && live[r]) *reinterpret_cast<float2*>(h1_out + save_idx<kPanel, kW>(row[r], c)) = make_float2(v0, v1);
        });
    if (kSave && kPanel && h1_mask) {
#pragma unroll
      for (int c = 0; c < kW / 32; ++c)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const uint32_t w = mask_chunk(h, c, 2 * r, t);
          if (t == 0 && live[r]) h1_mask[mask_idx<kW>(row[r], c)] = w;
        }
    }
    // layer 2
    float z[kNT][4];
#pragma unroll
    for (int j = 0; j < kNT; ++j) z[j][0] = z[j][1] = z[j][2] = z[j][3] = 0.f;
    warp_gemm<kNT, kNT, kThree>(z, h, fW2, lane);
    // epilogue 2: + b2, ReLU, layer 3 (N = 3: CUDA cores), sigmoid
    float p[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    epi_hidden_layer3<kW, kNT>(z, 0, t, sB2, sW3, p, [&](int r, int c, float a0, float a1) {
      if (kSave && live[r]) *reinterpret_cast<float2*>(h2_out + save_idx<kPanel, kW>(row[r], c)) = make_float2(a0, a1);
    });
    epi_rgb(p, b3v, t, [&](int r, const float (&v)[3]) {
      if (live[r]) {
        float* o = rgb + row[r] * 3;
#pragma unroll
        for (int i = 0; i < 3; ++i) o[i] = v[i];
      }
    });
  }
}

template <int kF, bool kSave, bool kThree, int kWarps, bool kPanel>
__global__ void __launch_bounds__(32 * kWarps, 1) k_shade_fwd_tc(UBN_SHADE_FWD_PARAMS) {
  shade_fwd_tc<kF, kHidden, kSave, kThree, kWarps, kPanel>(UBN_SHADE_FWD_ARGS);
}

// other widths: kCtas resident CTAs per SM
template <int kF, int kW, bool kSave, bool kThree, int kWarps, int kCtas, bool kPanel>
__global__ void __launch_bounds__(32 * kWarps, kCtas) k_shade_fwd_tc_w(UBN_SHADE_FWD_PARAMS) {
  shade_fwd_tc<kF, kW, kSave, kThree, kWarps, kPanel>(UBN_SHADE_FWD_ARGS);
}
#undef UBN_SHADE_FWD_ARGS

// ---- backward, launch 1 --------------------------------------------------------------------------------------------------
//   dz3 = g_rgb * rgb (1 - rgb);  dZ2 = (dz3 . W3) * [H2 > 0];  dH1 = dZ2 . W2;  dZ1 = dH1 * [H1 > 0]
//   kDz1Out: write dZ1 [n,128] row-major and stop (ubn_rgbnet_bwd_small finishes on the CUDA cores); otherwise also
//   dX = dZ1 . W1k and every sample reduction except dW2:  dW1k^T = X^T . dZ1,  grad_view_bias[ray] += sum dZ1 of the
//   ray (segment indicators as extra A rows),  dW3 = dz3^T . H2,  E = dz3^T . [H2 > 0] (db2 = sum_i W3[i] * E[i]),  db3 = sum dz3.
//
// Each warp walks one contiguous, balanced range of 16-sample units.  The sample reductions restart their MMA accumulator every
// unit and add it with plain fp32 adds into running sums that the warp owns (its private slice of shared memory, db3 in a
// register), so no two warps ever touch the same word until the one cross-warp sum at the end of the CTA.  Because the range is
// contiguous and ray_id is sorted, the dZ1 sum of the ray that is still open at the end of a unit is carried (one more row of
// the warp's slice) into the next unit and written to grad_view_bias once, when its ray ends.
namespace bk {
// W2 fragments at offset 0 (dH1 = dZ2 . W2: B[k][n] = W2[k][n]), fp32 and split into hi / lo at the MMA: 64 KB at w = 128
__host__ __device__ constexpr uint32_t frag_w2f(int w) { return n_tiles(w) * n_tiles(w) * 32 * 8; }
__host__ __device__ constexpr uint32_t oW1T(int w) { return frag_w2f(w); }              // dX = dZ1 . W1k: B[k][n] = W1k[k][n]
__host__ __device__ constexpr uint32_t oW3(int w) { return oW1T(w) + 2 * n_tiles(w) * 32 * 8; }
__host__ __device__ constexpr uint32_t oWarp(int w) { return oW3(w) + 3 * w * 4; }
// per warp: operand tile [16][stride], the running sums dW1k^T [kF][stride], dW3 [3][stride], E [3][stride], and the
// open ray's dZ1 sum [stride]
__host__ __device__ constexpr uint32_t tile_bytes(int w) { return kUnit * stride(w) * 4; }
__host__ __device__ constexpr int sum_rows(int f) { return f + 3 + 3; }
__host__ __device__ constexpr uint32_t warp_bytes(int f, int w) { return tile_bytes(w) + (sum_rows(f) + 1) * stride(w) * 4; }
__host__ __device__ constexpr uint32_t smem_bytes(int warps, int f, int w) { return oWarp(w) + warps * warp_bytes(f, w); }
}  // namespace bk

// B fragment of the warp tile S[16][kStride] (sample = k): k-step s, column tile j -> S[8 s + t][8 j + g], S[8 s + t + 4][..]
template <int kStride>
__device__ __forceinline__ void tile_frag(const float* S, int s, int j, int g, int t, uint32_t (&hi)[2], uint32_t (&lo)[2]) {
  const float v[2] = {S[(8 * s + t) * kStride + 8 * j + g], S[(8 * s + t + 4) * kStride + 8 * j + g]};
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    hi[e] = tf32_hi_bits(v[e]);
    lo[e] = __float_as_uint(v[e] - __uint_as_float(hi[e]));
  }
}

// store a [16][8 kNT] accumulator-layout block into the warp tile
template <int kStride, int kNT>
__device__ __forceinline__ void tile_store(float* S, const float (&v)[kNT][4], int g, int t) {
#pragma unroll
  for (int j = 0; j < kNT; ++j) {
    *reinterpret_cast<float2*>(S + g * kStride + 8 * j + 2 * t) = make_float2(v[j][0], v[j][1]);
    *reinterpret_cast<float2*>(S + (g + 8) * kStride + 8 * j + 2 * t) = make_float2(v[j][2], v[j][3]);
  }
}

__device__ __forceinline__ void sum_add2(float* p, float a, float b) {
  float2 v = *reinterpret_cast<float2*>(p);
  v.x += a;
  v.y += b;
  *reinterpret_cast<float2*>(p) = v;
}

__device__ __forceinline__ void red_add2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// grad_view_bias[ray] += V for the columns 8 j + 2 t, + 1 (j < kW / 8) of a g-row of lanes
template <int kW>
__device__ __forceinline__ void emit_ray(float* grad_view_bias, int64_t ray, const float* V, int t) {
#pragma unroll
  for (int j = 0; j < n_tiles(kW); ++j) {
    const float2 v = *reinterpret_cast<const float2*>(V + 8 * j + 2 * t);
    red_add2(grad_view_bias + ray * kW + 8 * j + 2 * t, v.x, v.y);
  }
}

// kF feature columns: dX has ceil(kF / 8) n-tiles.  The dW1k^T sums and the ray-segment indicators share one 16-row A tile
// while kF <= 12 (features in rows 0 .. kF - 1, indicators in rows 12 .. 15); at kF = 15 the indicators get an m-tile of their own.
template <int kF, int kW, bool kThree, int kWarps, bool kPanel, bool kMask1, bool kDz1Out>
__device__ __forceinline__ void shade_bwd_tc(
    const float* __restrict__ feat, const int64_t* __restrict__ ray_id, const float* __restrict__ W1k,
    const float* __restrict__ W2, const float* __restrict__ W3, const float* __restrict__ rgb,
    const float* __restrict__ h1_save, const float* __restrict__ h2_save, const float* __restrict__ grad_rgb, int64_t n_pts,
    float* __restrict__ grad_feat, float* __restrict__ grad_view_bias, float* __restrict__ grad_W1k, float* __restrict__ grad_b2,
    float* __restrict__ grad_W3, float* __restrict__ grad_b3, uint32_t* __restrict__ h2_mask, const uint32_t* __restrict__ h1_mask,
    float* __restrict__ dz1_out) {
  extern __shared__ __align__(16) uint8_t smem[];
  constexpr int kThreads = 32 * kWarps;
  constexpr int kNTX = (kF + 7) / 8;                      // n-tiles of dX
  constexpr bool kSegTile = kF > 12;                      // indicators in a second m-tile
  constexpr int kNT = n_tiles(kW), kStride = stride(kW), kChunks = kW / 32;
  constexpr uint32_t kWarpBytes = bk::warp_bytes(kF, kW);
  const int tid = threadIdx.x, lane = tid & 31, g = lane >> 2, t = lane & 3, warp = tid >> 5;
  const uint2* fW2 = reinterpret_cast<const uint2*>(smem);
  const uint2* fW1T = reinterpret_cast<const uint2*>(smem + bk::oW1T(kW));
  float* sW3 = reinterpret_cast<float*>(smem + bk::oW3(kW));
  float* S = reinterpret_cast<float*>(smem + bk::oWarp(kW) + warp * kWarpBytes);
  float* sumW1 = S + kUnit * kStride;                     // dW1k^T [feature][unit]
  float* sumW3 = sumW1 + kF * kStride;
  float* sumE = sumW3 + 3 * kStride;
  float* vbc = sumE + 3 * kStride;                        // lanes g == 4: the open ray's sum of dZ1 so far
  stage_frags_f32(W2, kW, kW, kW, kNT, kNT, reinterpret_cast<uint2*>(smem), tid, kThreads);
  if (!kDz1Out) stage_frags_f32(W1k, kF, kW, kF, kNT, kNTX, reinterpret_cast<uint2*>(smem + bk::oW1T(kW)), tid, kThreads);
  for (int i = tid; i < 3 * kW; i += kThreads) sW3[i] = W3[i];
  if (!kDz1Out)
    for (int i = lane; i < bk::sum_rows(kF) * kStride; i += 32) sumW1[i] = 0.f;
  __syncthreads();

  float db3 = 0.f;                                        // lane i < 3: this warp's sum of dz3_i
  int64_t open_ray = -1;                                  // warp-uniform: the ray whose dZ1 sum vbc carries (-1: none)

  const int64_t n_units = (n_pts + kUnit - 1) / kUnit;
  const int64_t n_warps = (int64_t)gridDim.x * kWarps, wid = (int64_t)blockIdx.x * kWarps + warp;
  const int64_t u_end = n_units * (wid + 1) / n_warps;
  for (int64_t u = n_units * wid / n_warps; u < u_end; ++u) {
    const int64_t r0 = u * kUnit;
    const int64_t row[2] = {r0 + g, r0 + g + 8};
    const bool live[2] = {row[0] < n_pts, row[1] < n_pts};
    float dz3[2][3];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const float y = live[r] ? rgb[row[r] * 3 + i] : 0.f;
        dz3[r][i] = live[r] ? grad_rgb[row[r] * 3 + i] * y * (1.f - y) : 0.f;
      }
    // dZ2 in accumulator layout; H2 values kept for dW3 below (through the warp tile)
    float d2[kNT][4];
    uint32_t m2[2][kChunks] = {};
#pragma unroll
    for (int j = 0; j < kNT; ++j) {
      const int c = 8 * j + 2 * t;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float2 hv = live[r] ? *reinterpret_cast<const float2*>(h2_save + save_idx<kPanel, kW>(row[r], c)) : make_float2(0.f, 0.f);
        const float hv2[2] = {hv.x, hv.y};
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float dh = dz3[r][0] * sW3[c + e] + dz3[r][1] * sW3[kW + c + e] + dz3[r][2] * sW3[2 * kW + c + e];
          d2[j][2 * r + e] = hv2[e] > 0.f ? dh : 0.f;
          if (hv2[e] > 0.f) m2[r][j >> 2] |= 1u << (8 * (j & 3) + 2 * t + e);
        }
        if (!kDz1Out) *reinterpret_cast<float2*>(S + (g + 8 * r) * kStride + c) = hv;   // H2 tile for dW3 / db2
      }
    }
    if (h2_mask) {
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          uint32_t w = m2[r][c];
          w |= __shfl_xor_sync(0xffffffffu, w, 1);
          w |= __shfl_xor_sync(0xffffffffu, w, 2);
          if (t == 0 && live[r]) h2_mask[mask_idx<kW>(row[r], c)] = w;
        }
    }
    if (!kDz1Out) {
      __syncwarp();
      // dW3 = dz3^T . H2 and E = dz3^T . [H2 > 0]: A rows 0..2 = dz3^T, sample = k
      {
        // a0 = A[g][t], a1 = A[g + 8][t], a2 = A[g][t + 4], a3 = A[g + 8][t + 4]; A[i][k] = dz3 of sample k (rows >= 3: 0)
        // dz3 of sample k lives in lane (g = k % 8, any t) as dz3[k / 8][.]
        float av[2][4];
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          float a[4];
#pragma unroll
          for (int q = 0; q < 2; ++q) {                      // k = t (q = 0) or t + 4 (q = 1), sample 8 s + k
            const int src = 4 * (t + 4 * q);                 // lane holding sample row (t + 4 q) of this half
            float v0 = __shfl_sync(0xffffffffu, dz3[s][0], src), v1 = __shfl_sync(0xffffffffu, dz3[s][1], src),
                  v2 = __shfl_sync(0xffffffffu, dz3[s][2], src);
            a[2 * q] = g == 0 ? v0 : g == 1 ? v1 : g == 2 ? v2 : 0.f;
            a[2 * q + 1] = 0.f;                              // rows g + 8 >= 8: unused
          }
          av[s][0] = a[0]; av[s][1] = a[1]; av[s][2] = a[2]; av[s][3] = a[3];
        }
        uint32_t ah[2][4], al[2][4];
#pragma unroll
        for (int s = 0; s < 2; ++s) split4(av[s], ah[s], al[s]);
#pragma unroll
        for (int jh = 0; jh < kNT / 8; ++jh) {               // groups of 8 column tiles: at most 64 accumulators live
          constexpr int kH = 8;
          float dW3a[kH][4], Ea[kH][4];
#pragma unroll
          for (int jj = 0; jj < kH; ++jj) dW3a[jj][0] = dW3a[jj][1] = dW3a[jj][2] = dW3a[jj][3] = Ea[jj][0] = Ea[jj][1] = Ea[jj][2] = Ea[jj][3] = 0.f;
#pragma unroll
          for (int s = 0; s < 2; ++s) {
#pragma unroll
            for (int jj = 0; jj < kH; ++jj) {
              uint32_t bh[2], bl[2];
              tile_frag<kStride>(S, s, kH * jh + jj, g, t, bh, bl);
              mma3<kThree>(dW3a[jj], ah[s], al[s], make_uint4(bh[0], bh[1], bl[0], bl[1]));
              const uint32_t one = 0x3f800000u;
              const uint32_t mb0 = __uint_as_float(bh[0]) + __uint_as_float(bl[0]) > 0.f ? one : 0u;
              const uint32_t mb1 = __uint_as_float(bh[1]) + __uint_as_float(bl[1]) > 0.f ? one : 0u;
              if (kThree) mma_tf32(Ea[jj], al[s], mb0, mb1);
              mma_tf32(Ea[jj], ah[s], mb0, mb1);
            }
          }
          if (g < 3) {
#pragma unroll
            for (int jj = 0; jj < kH; ++jj) {
              const int c = 8 * (kH * jh + jj) + 2 * t;
              sum_add2(sumW3 + g * kStride + c, dW3a[jj][0], dW3a[jj][1]);
              sum_add2(sumE + g * kStride + c, Ea[jj][0], Ea[jj][1]);
            }
          }
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {                        // db3: the four t-lanes of a row hold the same dz3
          float s3 = dz3[0][i] + dz3[1][i];
          s3 += __shfl_xor_sync(0xffffffffu, s3, 4);
          s3 += __shfl_xor_sync(0xffffffffu, s3, 8);
          s3 += __shfl_xor_sync(0xffffffffu, s3, 16);
          if (lane == i) db3 += s3;
        }
      }
      __syncwarp();
    }
    // dH1 = dZ2 . W2
    float d1[kNT][4];
#pragma unroll
    for (int j = 0; j < kNT; ++j) d1[j][0] = d1[j][1] = d1[j][2] = d1[j][3] = 0.f;
    warp_gemm_f<kNT, kNT, kThree>(d1, d2, fW2, lane);
    // dZ1 = dH1 * [H1 > 0]
    if (kMask1) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        uint32_t w[kChunks] = {};
        if (live[r]) {
#pragma unroll
          for (int c = 0; c < kChunks; ++c) w[c] = h1_mask[mask_idx<kW>(row[r], c)];
        }
#pragma unroll
        for (int j = 0; j < kNT; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (!((w[j >> 2] >> (8 * (j & 3) + 2 * t + e)) & 1u)) d1[j][2 * r + e] = 0.f;
      }
    } else {
#pragma unroll
      for (int j = 0; j < kNT; ++j)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float2 hv = live[r] ? *reinterpret_cast<const float2*>(h1_save + save_idx<kPanel, kW>(row[r], 8 * j + 2 * t))
                                    : make_float2(0.f, 0.f);
          if (!(hv.x > 0.f)) d1[j][2 * r] = 0.f;
          if (!(hv.y > 0.f)) d1[j][2 * r + 1] = 0.f;
        }
    }
    if (kDz1Out) {
#pragma unroll
      for (int j = 0; j < kNT; ++j)
#pragma unroll
        for (int r = 0; r < 2; ++r)
          if (live[r]) *reinterpret_cast<float2*>(dz1_out + row[r] * kW + 8 * j + 2 * t) = make_float2(d1[j][2 * r], d1[j][2 * r + 1]);
      continue;
    }
    // dX = dZ1 . W1k
    {
      float dx[kNTX][4] = {};
      warp_gemm_f<kNT, kNTX, kThree>(dx, d1, fW1T, lane);
#pragma unroll
      for (int j = 0; j < kNTX; ++j)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int c = 8 * j + 2 * t;
          if constexpr (kF % 2 == 0) {
            if (live[r] && c < kF) *reinterpret_cast<float2*>(grad_feat + row[r] * kF + c) = make_float2(dx[j][2 * r], dx[j][2 * r + 1]);
          } else if (live[r]) {
            if (c < kF) grad_feat[row[r] * kF + c] = dx[j][2 * r];
            if (c + 1 < kF) grad_feat[row[r] * kF + c + 1] = dx[j][2 * r + 1];
          }
        }
    }
    // dW1k^T = X^T . dZ1 (A rows 0 .. kF - 1) and per-ray sums of dZ1 (A rows 12..15 = indicators of up to 4 ray segments; at
    // kF > 12 those rows of a second m-tile)
    tile_store<kStride>(S, d1, g, t);
    __syncwarp();                                             // the tile is read back across lanes as B fragments below
    const int64_t my_ray = (lane < kUnit && r0 + lane < n_pts) ? ray_id[r0 + lane] : -1;
    const int64_t prev_ray = __shfl_up_sync(0xffffffffu, my_ray, 1);
    const uint32_t starts = __ballot_sync(0xffffffffu, lane < kUnit && my_ray >= 0 && (lane == 0 || prev_ray != my_ray));
    const int nseg = __popc(starts);                          // >= 1: sample r0 is live
    const bool segs_fit = nseg <= 4;
    {
      float acc[kNT][4];
      // kF <= 12: one m-tile -- row g feature g, row g + 8 feature g + 8 (g < 4) or the indicator of segment g - 4 (g >= 4).
      // kF > 12: the features fill rows 0 .. kF - 1 and the indicators get rows 12..15 of a second m-tile.
      if constexpr (!kSegTile) {
#pragma unroll
        for (int j = 0; j < kNT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          float av[4];
#pragma unroll
          for (int q = 0; q < 2; ++q) {                       // sample k = 8 s + t + 4 q
            const int64_t rr = r0 + 8 * s + t + 4 * q;
            const int ks = 8 * s + t + 4 * q;
            const bool ok = rr < n_pts;
            av[2 * q] = (ok && (kF >= 8 || g < kF)) ? feat[rr * kF + g] : 0.f;   // A row g: feature g
            float lo = 0.f;                                                     // A row g + 8: feature g + 8 or segment g - 4
            if (ok) {
              if (g < 4) { if (kF >= 12 || g + 8 < kF) lo = feat[rr * kF + g + 8]; }
              else if (segs_fit) lo = (__popc(starts & ((2u << ks) - 1u)) - 1 == g - 4) ? 1.f : 0.f;
            }
            av[2 * q + 1] = lo;
          }
          const float a[4] = {av[0], av[1], av[2], av[3]};
          uint32_t ah[4], al[4];
          split4(a, ah, al);
#pragma unroll
          for (int j = 0; j < kNT; ++j) {
            uint32_t bh[2], bl[2];
            tile_frag<kStride>(S, s, j, g, t, bh, bl);
            mma3<kThree>(acc[j], ah, al, make_uint4(bh[0], bh[1], bl[0], bl[1]));
          }
        }
#pragma unroll
        for (int j = 0; j < kNT; ++j) {
          const int c = 8 * j + 2 * t;
          if (kF >= 8 || g < kF) sum_add2(sumW1 + g * kStride + c, acc[j][0], acc[j][1]);
          if (g < 4 && (kF >= 12 || g + 8 < kF)) sum_add2(sumW1 + (g + 8) * kStride + c, acc[j][2], acc[j][3]);
        }
      } else {
        // A[row][sample k] from row_lo (rows g) and row_hi (rows g + 8) of sample rr = r0 + k, zero past the last sample
        auto tile_gemm = [&](auto row_lo, auto row_hi) {
#pragma unroll
          for (int j = 0; j < kNT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
          for (int s = 0; s < 2; ++s) {
            float av[4];
#pragma unroll
            for (int q = 0; q < 2; ++q) {                     // sample k = 8 s + t + 4 q
              const int ks = 8 * s + t + 4 * q;
              const bool ok = r0 + ks < n_pts;
              av[2 * q] = ok ? row_lo(r0 + ks) : 0.f;
              av[2 * q + 1] = ok ? row_hi(r0 + ks, ks) : 0.f;
            }
            uint32_t ah[4], al[4];
            split4(av, ah, al);
#pragma unroll
            for (int j = 0; j < kNT; ++j) {
              uint32_t bh[2], bl[2];
              tile_frag<kStride>(S, s, j, g, t, bh, bl);
              mma3<kThree>(acc[j], ah, al, make_uint4(bh[0], bh[1], bl[0], bl[1]));
            }
          }
        };
        tile_gemm([&](int64_t rr) { return feat[rr * kF + g]; },                               // features 0 .. kF - 1
                  [&](int64_t rr, int) { return g + 8 < kF ? feat[rr * kF + g + 8] : 0.f; });
#pragma unroll
        for (int j = 0; j < kNT; ++j) {
          const int c = 8 * j + 2 * t;
          sum_add2(sumW1 + g * kStride + c, acc[j][0], acc[j][1]);
          if (g + 8 < kF) sum_add2(sumW1 + (g + 8) * kStride + c, acc[j][2], acc[j][3]);
        }
        tile_gemm([&](int64_t) { return 0.f; },                                                  // rows 12..15: segments g - 4
                  [&](int64_t, int ks) {
                    return (g >= 4 && segs_fit && __popc(starts & ((2u << ks) - 1u)) - 1 == g - 4) ? 1.f : 0.f;
                  });
      }
      // rays of the unit's first and last segment, and (lanes g = 4 + q) of segment q
      const int64_t first_ray = __shfl_sync(0xffffffffu, my_ray, __ffs(starts) - 1);
      const int64_t last_ray = __shfl_sync(0xffffffffu, my_ray, 31 - __clz(starts));
      uint32_t above = starts;                                // drop the first g - 4 starts
      for (int q = 0; q < g - 4; ++q) above &= above - 1;
      const int64_t seg_ray = __shfl_sync(0xffffffffu, my_ray, above ? __ffs(above) - 1 : 0);
      if (segs_fit) {
        const bool cont = first_ray == open_ray;
        if (g == 4) {
          if (!cont && open_ray >= 0) emit_ray<kW>(grad_view_bias, open_ray, vbc, t);    // the carried ray ended with the last unit
#pragma unroll
          for (int j = 0; j < kNT; ++j) {
            float* v = vbc + 8 * j + 2 * t;
            const float2 o = cont ? *reinterpret_cast<const float2*>(v) : make_float2(0.f, 0.f);
            *reinterpret_cast<float2*>(v) = make_float2(o.x + acc[j][2], o.y + acc[j][3]);
          }
          if (nseg > 1) emit_ray<kW>(grad_view_bias, first_ray, vbc, t);                 // segment 0 ends inside this unit
        }
        if (nseg > 1) {
          if (g > 4 && g - 4 < nseg - 1) {                   // inner segments
#pragma unroll
            for (int j = 0; j < kNT; ++j) red_add2(grad_view_bias + seg_ray * kW + 8 * j + 2 * t, acc[j][2], acc[j][3]);
          }
          __syncwarp();                                       // lanes g == 4 have read vbc
          if (g == 3 + nseg) {                                // the last segment stays open
#pragma unroll
            for (int j = 0; j < kNT; ++j) *reinterpret_cast<float2*>(vbc + 8 * j + 2 * t) = make_float2(acc[j][2], acc[j][3]);
          }
        }
        open_ray = last_ray;
      }
    }
    if (!segs_fit) {                                          // more than 4 rays in 16 samples: per-sample adds
      if (open_ray >= 0 && g == 4) emit_ray<kW>(grad_view_bias, open_ray, vbc, t);
      open_ray = -1;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        if (!live[r]) continue;
        const int64_t ray = ray_id[row[r]];
#pragma unroll
        for (int j = 0; j < kNT; ++j) red_add2(grad_view_bias + ray * kW + 8 * j + 2 * t, d1[j][2 * r], d1[j][2 * r + 1]);
      }
    }
    __syncwarp();
  }
  if (kDz1Out) return;
  if (open_ray >= 0 && g == 4) emit_ray<kW>(grad_view_bias, open_ray, vbc, t);
  if (lane < 3) atomicAdd(grad_b3 + lane, db3);
  __syncthreads();
  // the warps' running sums, added in warp order, go to global once per CTA
  const float* sums = reinterpret_cast<const float*>(smem + bk::oWarp(kW) + bk::tile_bytes(kW));
  auto warp_sum = [&](int r, int c) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) v += sums[w * (kWarpBytes / 4) + r * kStride + c];
    return v;
  };
  for (int i = tid; i < kF * kW; i += kThreads) {                // row f of the sums is column f of dW1k
    const int f = i / kW, c = i % kW;
    atomicAdd(grad_W1k + c * kF + f, warp_sum(f, c));
  }
  for (int i = tid; i < 3 * kW; i += kThreads) atomicAdd(grad_W3 + i, warp_sum(kF + i / kW, i % kW));
  for (int c = tid; c < kW; c += kThreads) {
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) v += sW3[i * kW + c] * warp_sum(kF + 3 + i, c);
    atomicAdd(grad_b2 + c, v);
  }
}

#define UBN_SHADE_BWD_PARAMS                                                                                                    \
  const float* __restrict__ feat, const int64_t* __restrict__ ray_id, const float* __restrict__ W1k, const float* __restrict__ W2, \
      const float* __restrict__ W3, const float* __restrict__ rgb, const float* __restrict__ h1_save,                             \
      const float* __restrict__ h2_save, const float* __restrict__ grad_rgb, int64_t n_pts, float* __restrict__ grad_feat,        \
      float* __restrict__ grad_view_bias, float* __restrict__ grad_W1k, float* __restrict__ grad_b2, float* __restrict__ grad_W3, \
      float* __restrict__ grad_b3, uint32_t* __restrict__ h2_mask, const uint32_t* __restrict__ h1_mask, float* __restrict__ dz1_out
#define UBN_SHADE_BWD_ARGS                                                                                                     \
  feat, ray_id, W1k, W2, W3, rgb, h1_save, h2_save, grad_rgb, n_pts, grad_feat, grad_view_bias, grad_W1k, grad_b2, grad_W3, grad_b3, \
      h2_mask, h1_mask, dz1_out

// the 12-feature kernel keeps its own name; k_shade_bwd_tc_k carries the other feature counts
template <bool kThree, int kWarps, bool kPanel, bool kMask1, bool kDz1Out>
__global__ void __launch_bounds__(32 * kWarps, 1) k_shade_bwd_tc(UBN_SHADE_BWD_PARAMS) {
  shade_bwd_tc<kFeat, kHidden, kThree, kWarps, kPanel, kMask1, kDz1Out>(UBN_SHADE_BWD_ARGS);
}

template <int kF, bool kThree, int kWarps, bool kPanel, bool kMask1, bool kDz1Out>
__global__ void __launch_bounds__(32 * kWarps, 1) k_shade_bwd_tc_k(UBN_SHADE_BWD_PARAMS) {
  shade_bwd_tc<kF, kHidden, kThree, kWarps, kPanel, kMask1, kDz1Out>(UBN_SHADE_BWD_ARGS);
}

// other widths: kCtas resident CTAs per SM
template <int kF, int kW, bool kThree, int kWarps, int kCtas, bool kPanel, bool kMask1>
__global__ void __launch_bounds__(32 * kWarps, kCtas) k_shade_bwd_tc_w(UBN_SHADE_BWD_PARAMS) {
  shade_bwd_tc<kF, kW, kThree, kWarps, kPanel, kMask1, false>(UBN_SHADE_BWD_ARGS);
}
#undef UBN_SHADE_BWD_ARGS
#undef UBN_SHADE_BWD_PARAMS

// ---- backward, launch 2: dW2 += dZ2^T . H1 -------------------------------------------------------------------------------
// A split-K GEMM over samples: each CTA takes 32-sample chunks, stages dZ2 (rebuilt from dz3, W3 and H2 or its ReLU masks) as a
// [32][kStride] fp32 tile and H1 as a [32][kStrideB] tile of ready-split {hi, lo} pairs (split once per element, not once per
// warp), and warp w accumulates output rows 16 w .. 16 w + 15 (at kW = 64, rows 16 (w % 4) .. + 15 and half of the columns).  The tiles are double-buffered and each thread loads the next
// chunk's rows into registers before the MMAs of the current one, so the HBM reads overlap the tensor cores and one barrier
// per chunk suffices.  The MMA accumulator restarts every chunk and is added into an fp32 running sum, so the tensor core
// never carries a long accumulation chain.
namespace dw {
constexpr int kThreads = 256;
constexpr int kK = 32;
__host__ __device__ constexpr int stride_b(int w) { return w + 4; }    // uint2 per element: conflict-free fragment reads
// W3 [3][kW] at offset 0, then two buffers of a dZ2 tile [kK][stride] and an H1 tile [kK][stride_b]
__host__ __device__ constexpr uint32_t buf_a(int w) { return kK * stride(w) * 4; }
__host__ __device__ constexpr uint32_t buf(int w) { return buf_a(w) + kK * stride_b(w) * 8; }
__host__ __device__ constexpr uint32_t oBuf(int w) { return 3 * w * 4; }
__host__ __device__ constexpr uint32_t smem(int w) { return oBuf(w) + 2 * buf(w); }
}  // namespace dw

// one thread's share of a chunk (sample row r, columns 32 q + 4 (tid & 7) .. + 3), straight from global memory
template <int kW>
struct Dw2Rows {
  float4 h1[kW / 32], h2[kW / 32];
  uint32_t m2[kW / 32];
  float y[3], gy[3];
};

template <int kW, bool kPanel, bool kMask2>
__device__ __forceinline__ void dw2_load(Dw2Rows<kW>& d, const float* __restrict__ rgb, const float* __restrict__ h1_save,
                                         const float* __restrict__ h2_save, const uint32_t* __restrict__ h2_mask,
                                         const float* __restrict__ grad_rgb, int64_t r, int64_t n_pts, int c0) {
  const bool ok = r < n_pts;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    d.y[i] = ok ? rgb[r * 3 + i] : 0.f;
    d.gy[i] = ok ? grad_rgb[r * 3 + i] : 0.f;
  }
#pragma unroll
  for (int q = 0; q < kW / 32; ++q) {
    const int c = 32 * q + c0;
    d.h1[q] = ok ? *reinterpret_cast<const float4*>(h1_save + save_idx<kPanel, kW>(r, c)) : zero;
    if (kMask2) d.m2[q] = ok ? h2_mask[mask_idx<kW>(r, q)] : 0u;
    else d.h2[q] = ok ? *reinterpret_cast<const float4*>(h2_save + save_idx<kPanel, kW>(r, c)) : zero;
  }
}

#define UBN_SHADE_DW2_PARAMS                                                                                                 \
  const float* __restrict__ W3, const float* __restrict__ rgb, const float* __restrict__ h1_save,                            \
      const float* __restrict__ h2_save, const uint32_t* __restrict__ h2_mask, const float* __restrict__ grad_rgb, int64_t n_pts, \
      float* __restrict__ grad_W2
#define UBN_SHADE_DW2_ARGS W3, rgb, h1_save, h2_save, h2_mask, grad_rgb, n_pts, grad_W2

template <int kW, bool kThree, bool kPanel, bool kMask2>
__device__ __forceinline__ void shade_dw2_tc(UBN_SHADE_DW2_PARAMS) {
  // output tiles: kMT 16-row m-tiles, each shared by kThreads / 32 / kMT warps that take kNT of its 8-column n-tiles apiece
  constexpr int kMT = kW / 16, kNT = n_tiles(kW) * kMT / (dw::kThreads / 32), kStride = stride(kW), kStrideB = dw::stride_b(kW);
  extern __shared__ __align__(16) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, g = lane >> 2, t = lane & 3, warp = tid >> 5;
  const int mt = kMT == dw::kThreads / 32 ? warp : warp % kMT, j0 = kMT == dw::kThreads / 32 ? 0 : warp / kMT * kNT;
  float* sW3 = reinterpret_cast<float*>(smem);
  for (int i = tid; i < 3 * kW; i += dw::kThreads) sW3[i] = W3[i];
  float sum[kNT][4];
#pragma unroll
  for (int j = 0; j < kNT; ++j) sum[j][0] = sum[j][1] = sum[j][2] = sum[j][3] = 0.f;
  const int sr = tid >> 3, c0 = 4 * (tid & 7);             // staging: sample row, 4 float4 column groups per thread
  const int64_t n_chunks = (n_pts + dw::kK - 1) / dw::kK;
  Dw2Rows<kW> d;
  int64_t ch = blockIdx.x;
  if (ch < n_chunks) dw2_load<kW, kPanel, kMask2>(d, rgb, h1_save, h2_save, h2_mask, grad_rgb, ch * dw::kK + sr, n_pts, c0);
  __syncthreads();                                         // sW3 staged
  for (int buf = 0; ch < n_chunks; ch += gridDim.x, buf ^= 1) {
    float* sA = reinterpret_cast<float*>(smem + dw::oBuf(kW) + buf * dw::buf(kW));                   // dZ2 [sample][unit]
    uint2* sB = reinterpret_cast<uint2*>(smem + dw::oBuf(kW) + buf * dw::buf(kW) + dw::buf_a(kW));   // H1 {hi, lo} [sample][unit]
    float dz3[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) dz3[i] = d.gy[i] * d.y[i] * (1.f - d.y[i]);
#pragma unroll
    for (int q = 0; q < kW / 32; ++q) {
      const int c = 32 * q + c0;
      float hv[4];
      if (kMask2) {
        const uint32_t w = d.m2[q] >> c0;
#pragma unroll
        for (int e = 0; e < 4; ++e) hv[e] = ((w >> e) & 1u) ? 1.f : 0.f;
      } else {
        hv[0] = d.h2[q].x; hv[1] = d.h2[q].y; hv[2] = d.h2[q].z; hv[3] = d.h2[q].w;
      }
      float dv[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float dh = dz3[0] * sW3[c + e] + dz3[1] * sW3[kW + c + e] + dz3[2] * sW3[2 * kW + c + e];
        dv[e] = hv[e] > 0.f ? dh : 0.f;
      }
      *reinterpret_cast<float4*>(sA + sr * kStride + c) = make_float4(dv[0], dv[1], dv[2], dv[3]);
      const float hb[4] = {d.h1[q].x, d.h1[q].y, d.h1[q].z, d.h1[q].w};
      uint32_t hi[4], lo[4];
      split4(hb, hi, lo);
      *reinterpret_cast<uint4*>(sB + sr * kStrideB + c) = make_uint4(hi[0], lo[0], hi[1], lo[1]);
      *reinterpret_cast<uint4*>(sB + sr * kStrideB + c + 2) = make_uint4(hi[2], lo[2], hi[3], lo[3]);
    }
    __syncthreads();                                       // this buffer is complete; the other one is no longer read
    if (ch + gridDim.x < n_chunks)
      dw2_load<kW, kPanel, kMask2>(d, rgb, h1_save, h2_save, h2_mask, grad_rgb, (ch + gridDim.x) * dw::kK + sr, n_pts, c0);
    float acc[kNT][4];
#pragma unroll
    for (int j = 0; j < kNT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
    for (int s = 0; s < dw::kK / 8; ++s) {
      // A[m][k] = dZ2[sample 8 s + k][unit 16 mt + m]
      const float av[4] = {sA[(8 * s + t) * kStride + 16 * mt + g], sA[(8 * s + t) * kStride + 16 * mt + g + 8],
                           sA[(8 * s + t + 4) * kStride + 16 * mt + g], sA[(8 * s + t + 4) * kStride + 16 * mt + g + 8]};
      uint32_t ah[4], al[4];
      split4(av, ah, al);
#pragma unroll
      for (int j = 0; j < kNT; ++j) {
        const uint2 b0 = sB[(8 * s + t) * kStrideB + 8 * (j0 + j) + g], b1 = sB[(8 * s + t + 4) * kStrideB + 8 * (j0 + j) + g];
        mma3<kThree>(acc[j], ah, al, make_uint4(b0.x, b1.x, b0.y, b1.y));
      }
    }
#pragma unroll
    for (int j = 0; j < kNT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) sum[j][e] += acc[j][e];
  }
#pragma unroll
  for (int j = 0; j < kNT; ++j) {
    const int c = 8 * (j0 + j) + 2 * t, m = 16 * mt + g;
    atomicAdd(grad_W2 + m * kW + c, sum[j][0]);
    atomicAdd(grad_W2 + m * kW + c + 1, sum[j][1]);
    atomicAdd(grad_W2 + (m + 8) * kW + c, sum[j][2]);
    atomicAdd(grad_W2 + (m + 8) * kW + c + 1, sum[j][3]);
  }
}

template <bool kThree, bool kPanel, bool kMask2>
__global__ void __launch_bounds__(dw::kThreads, 1) k_shade_dw2_tc(UBN_SHADE_DW2_PARAMS) {
  shade_dw2_tc<kHidden, kThree, kPanel, kMask2>(UBN_SHADE_DW2_ARGS);
}

// other widths: kCtas resident CTAs per SM
template <int kW, bool kThree, int kCtas, bool kPanel, bool kMask2>
__global__ void __launch_bounds__(dw::kThreads, kCtas) k_shade_dw2_tc_w(UBN_SHADE_DW2_PARAMS) {
  shade_dw2_tc<kW, kThree, kPanel, kMask2>(UBN_SHADE_DW2_ARGS);
}

// ---- backward, launch 2 on warpgroup MMA (width 128, panel saves, H2 masks) ---------------------------------------------
// The same split-K GEMM, chunks and numerical policy as shade_dw2_tc, on wgmma.m64n128k8 (TF32): B = H1 is read by the tensor
// cores straight from shared memory, so no warp loads B fragments into registers.  One persistent CTA per SM, three warpgroups:
//   * warpgroup 0 (producer) copies each 32-sample chunk into raw shared-memory slots with cp.async (kRaw - 1 chunks in
//     flight, no registers held for them), then splits H1 into hi / lo and writes it transposed into two K-major
//     [128 units][32 samples] tiles in the 128-byte-swizzle layout of the wgmma descriptor (TF32 wgmma takes K-major
//     operands only; the panel save is unit-minor), plus the chunk's dz3 and H2 mask words, into a ring of kStages stages
//     guarded by full / empty mbarriers;
//   * warpgroups 1 and 2 (consumers) own dW2 rows 64 c .. 64 c + 63 each.  A = dZ2^T is rebuilt in registers from dz3, W3
//     and the masks as shade_dw2_tc builds it, split into hi / lo, and every k-step issues the three mma3 products (al.Bh,
//     ah.Bl, ah.Bh; ah.Bh alone at single_pass).  The accumulator restarts every chunk and is added into an fp32 running sum.
namespace wg {
constexpr int kThreads = 384;
constexpr int kStages = 4;
constexpr int kProducerRegs = 80, kConsumerRegs = 208;          // 128 * 80 + 256 * 208 <= 384 * 168 (launch allotment)
constexpr uint32_t kTile = kHidden * dw::kK * 4;                // one [128][32] fp32 B tile: 16 KB
constexpr uint32_t kExtra = 1024;                               // dz3 [3][32] and H2 mask words [4][32] (keeps 1 KB alignment)
__host__ __device__ constexpr uint32_t stage_bytes(bool three) { return (three ? 2 : 1) * kTile + kExtra; }
// the producer's raw slots: chunks still in flight from global memory (cp.async), kRaw - 1 ahead of the one it converts
constexpr int kRaw = 3;
constexpr uint32_t kRawH1 = 8 * 128 * 16;                       // float4 [8][128 threads]
constexpr uint32_t kRawSlot = kRawH1 + 2 * 6 * 32 * 4;          // + rgb, grad_rgb (warp 0) and mask words (warp 1)
__host__ __device__ constexpr uint32_t oRaw(bool three) { return kStages * stage_bytes(three); }
__host__ __device__ constexpr uint32_t oBar(bool three) { return oRaw(three) + kRaw * kRawSlot; }
// + full and empty barriers, + slack to align the base to the 1 KB the swizzle pattern repeats at
__host__ __device__ constexpr uint32_t smem(bool three) { return oBar(three) + 2 * kStages * 8 + 1024; }
}  // namespace wg

// byte offset of (unit n, sample k) in a K-major [128][32] fp32 tile with the 128-byte swizzle: 16-byte group k / 4 of row n
// lands at group (k / 4) ^ (n % 8)
__device__ __forceinline__ uint32_t sw128_off(int n, int k) { return n * 128 + ((((k >> 2) ^ n) & 7) << 4) + (k & 3) * 4; }

// shared-memory matrix descriptor of a K-major operand in the 128-byte-swizzle layout: 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t sw128_desc(uint32_t addr) {
  return (uint64_t)((addr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// d (64 x 128, fp32, accumulator layout) = (kScaleD ? d : 0) + A (64 x 8, registers, mma.m16n8k8 A layout per warp) . B (desc)
template <int kScaleD>
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
      "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, "
      "%51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "n"(kScaleD));
}

// 16- and 4-byte asynchronous copies global -> shared; ok = false writes zeros and reads nothing
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src, bool ok) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(ok ? 4 : 0) : "memory");
}

// Producer thread tid (warp pw) copies its share of chunk ch into a raw slot: sample row lane of H1 unit quads pw + 4 j as
// float4 [j][tid] (the coalesced 16-byte panel loads of dw2_load), warp 0 also rgb and grad_rgb, warp 1 the four mask words
// ([pw][6][32] words after the H1 part).  Rows >= n_pts are zeros.  Always commits one cp.async group.
__device__ __forceinline__ void dw2_raw_issue(uint8_t* slot, const float* __restrict__ rgb, const float* __restrict__ h1_save,
                                              const uint32_t* __restrict__ h2_mask, const float* __restrict__ grad_rgb,
                                              int64_t ch, int64_t n_chunks, int64_t n_pts, int tid) {
  const int pw = tid >> 5, lane = tid & 31;
  if (ch < n_chunks) {
    const int64_t r = ch * dw::kK + lane;
    const bool ok = r < n_pts;
    const float* src = h1_save + (ok ? save_idx<true, kHidden>(r, 4 * pw) : 0);
    const uint32_t dst = smem_u32(slot) + tid * 16;
#pragma unroll
    for (int j = 0; j < 8; ++j) cp_async16(dst + j * 128 * 16, ok ? src + j * 4 * kPanelRows * 4 : h1_save, ok);
    const uint32_t xd = smem_u32(slot + wg::kRawH1) + (pw * 6 * 32 + lane) * 4;
    if (pw == 0) {
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        cp_async4(xd + i * 128, ok ? rgb + r * 3 + i : rgb, ok);
        cp_async4(xd + (3 + i) * 128, ok ? grad_rgb + r * 3 + i : grad_rgb, ok);
      }
    } else if (pw == 1) {
#pragma unroll
      for (int c = 0; c < kHidden / 32; ++c) cp_async4(xd + c * 128, ok ? h2_mask + mask_idx<kHidden>(r, c) : h2_mask, ok);
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// the same thread's share from the raw slot into a stage: H1 split into hi / lo and transposed into the swizzled tiles,
// dz3 [3][32] and the mask words [4][32] after them
template <bool kThree>
__device__ __forceinline__ void dw2_stage_put(const uint8_t* slot, uint8_t* stage, int tid) {
  const int pw = tid >> 5, lane = tid & 31;
  const float4* h1 = reinterpret_cast<const float4*>(slot);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int q = pw + 4 * j;
    const float4 h = h1[j * 128 + tid];
    const float v[4] = {h.x, h.y, h.z, h.w};
    uint32_t hi[4], lo[4];
    split4(v, hi, lo);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const uint32_t off = sw128_off(4 * q + e, lane);
      *reinterpret_cast<uint32_t*>(stage + off) = hi[e];
      if (kThree) *reinterpret_cast<uint32_t*>(stage + wg::kTile + off) = lo[e];
    }
  }
  const float* x = reinterpret_cast<const float*>(slot + wg::kRawH1) + pw * 6 * 32 + lane;
  float* sx = reinterpret_cast<float*>(stage + (kThree ? 2 : 1) * wg::kTile) + lane;
  if (pw == 0) {
#pragma unroll
    for (int i = 0; i < 3; ++i) sx[i * 32] = x[(3 + i) * 32] * x[i * 32] * (1.f - x[i * 32]);
  } else if (pw == 1) {
#pragma unroll
    for (int c = 0; c < kHidden / 32; ++c) sx[(3 + c) * 32] = x[c * 32];
  }
}

template <bool kThree>
__global__ void __launch_bounds__(wg::kThreads, 1) k_shade_dw2_wgmma(const float* __restrict__ W3, const float* __restrict__ rgb,
                                                                      const float* __restrict__ h1_save,
                                                                      const uint32_t* __restrict__ h2_mask,
                                                                      const float* __restrict__ grad_rgb, int64_t n_pts,
                                                                      float* __restrict__ grad_W2) {
  constexpr int kW = kHidden;
  constexpr uint32_t kStage = wg::stage_bytes(kThree);
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int tid = threadIdx.x, lane = tid & 31;
  const uint32_t full0 = smem_u32(smem + wg::oBar(kThree)), empty0 = full0 + 8 * wg::kStages;
  if (tid == 0) {
    for (int s = 0; s < wg::kStages; ++s) {
      mbar_init(full0 + 8 * s, 128);
      mbar_init(empty0 + 8 * s, 256);
    }
  }
  __syncthreads();
  const int64_t n_chunks = (n_pts + dw::kK - 1) / dw::kK, step = gridDim.x;

  if (tid < 128) {                                          // producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(wg::kProducerRegs));
    uint8_t* raw = smem + wg::oRaw(kThree);
    const int64_t ch0 = blockIdx.x;
    for (int k = 0; k < wg::kRaw - 1; ++k)
      dw2_raw_issue(raw + k * wg::kRawSlot, rgb, h1_save, h2_mask, grad_rgb, ch0 + k * step, n_chunks, n_pts, tid);
    int i = 0;
    for (int64_t ch = ch0; ch < n_chunks; ch += step, ++i) {
      // the slot refilled here was read into the stage at the previous chunk
      dw2_raw_issue(raw + (i + wg::kRaw - 1) % wg::kRaw * wg::kRawSlot, rgb, h1_save, h2_mask, grad_rgb,
                    ch + (wg::kRaw - 1) * step, n_chunks, n_pts, tid);
      asm volatile("cp.async.wait_group %0;" ::"n"(wg::kRaw - 1) : "memory");   // this chunk's copies have landed
      const int s = i % wg::kStages;
      mbar_wait(empty0 + 8 * s, ((i / wg::kStages) & 1) ^ 1);
      dw2_stage_put<kThree>(raw + i % wg::kRaw * wg::kRawSlot, smem + s * kStage, tid);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the generic-proxy stores, before wgmma reads them
      mbar_arrive(full0 + 8 * s);
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(wg::kConsumerRegs));
  const int ct = tid - 128, g = lane >> 2, t = lane & 3;
  const int m0 = 64 * (ct >> 7) + 16 * ((ct >> 5) & 3) + g;     // this thread's rows m0 and m0 + 8 (same 32-unit mask word)
  float w3[3][2];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    w3[i][0] = W3[i * kW + m0];
    w3[i][1] = W3[i * kW + m0 + 8];
  }
  float acc[64], sum[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) acc[e] = sum[e] = 0.f;
  int i = 0;
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += step, ++i) {
    const int s = i % wg::kStages;
    mbar_wait(full0 + 8 * s, (i / wg::kStages) & 1);
    uint8_t* stage = smem + s * kStage;
    const float* sx = reinterpret_cast<const float*>(stage + (kThree ? 2 : 1) * wg::kTile);
    // A[m][k] = dZ2[sample 8 ks + k][unit m], a0 = (m0, t), a1 = (m0 + 8, t), a2 = (m0, t + 4), a3 = (m0 + 8, t + 4)
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int ks = 0; ks < dw::kK / 8; ++ks) {
      float av[4];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int k = 8 * ks + t + 4 * q;
        const float dz3[3] = {sx[k], sx[32 + k], sx[64 + k]};
        const uint32_t w = __float_as_uint(sx[(3 + (m0 >> 5)) * 32 + k]) >> (m0 & 31);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float dh = dz3[0] * w3[0][h] + dz3[1] * w3[1][h] + dz3[2] * w3[2][h];
          av[2 * q + h] = ((w >> (8 * h)) & 1u) ? dh : 0.f;
        }
      }
      split4(av, ah[ks], al[ks]);
    }
    const uint32_t b = smem_u32(stage);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int ks = 0; ks < dw::kK / 8; ++ks) {
      const uint64_t bh = sw128_desc(b + 32 * ks);
      if (kThree) {
        if (ks == 0) wgmma_tf32<0>(acc, al[ks], bh);
        else wgmma_tf32<1>(acc, al[ks], bh);
        wgmma_tf32<1>(acc, ah[ks], sw128_desc(b + wg::kTile + 32 * ks));
        wgmma_tf32<1>(acc, ah[ks], bh);
      } else if (ks == 0) {
        wgmma_tf32<0>(acc, ah[ks], bh);
      } else {
        wgmma_tf32<1>(acc, ah[ks], bh);
      }
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
    for (int e = 0; e < 64; ++e) asm volatile("" : "+f"(acc[e])::"memory");   // no read of acc above the wait
    mbar_arrive(empty0 + 8 * s);
#pragma unroll
    for (int e = 0; e < 64; ++e) sum[e] += acc[e];
  }
  // accumulator element 4 j + e: row m0 + 8 (e / 2), column 8 j + 2 t + e % 2
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) atomicAdd(grad_W2 + (m0 + 8 * (e >> 1)) * kW + 8 * j + 2 * t + (e & 1), sum[4 * j + e]);
}
#undef UBN_SHADE_DW2_ARGS
#undef UBN_SHADE_DW2_PARAMS

// ---- forward on warpgroup MMA (width 128, 12 features) --------------------------------------------------------------------
// The contract of shade_fwd_tc<12, 128, kSave, kThree, 8, kPanel> on wgmma.m64n128k8 (TF32), 64-sample tiles: W1k and W2 are read
// by the tensor cores from shared memory by descriptor, so no warp reloads B fragments per tile.  One persistent CTA per SM:
//   * warpgroup 0 (producer) copies each tile's feature rows and ray ids into a ring of kStages stages with cp.async (zeros past
//     n_pts); the ring's full barrier completes when the copies land (cp.async.mbarrier.arrive), so no producer thread waits on
//     them;
//   * warpgroups 1 and 2 (consumers) take alternate tiles, so one warpgroup's epilogue stores overlap the other's MMAs.  Warp w
//     of a consumer owns rows 16 w + g and 16 w + g + 8 of the tile and, like an mma.sync warp, columns 8 j + 2 t, + 1: the
//     wgmma accumulator of layer 1 is the per-warp m16n8k8 A layout of layer 2 under the k-permutation of shade_fwd_tc
//     (a0..a3 = d[4 s], d[4 s + 2], d[4 s + 1], d[4 s + 3]).  The K-major W2 tile of k-step s therefore holds hidden units
//     8 s + {0, 2, 4, 6, 1, 3, 5, 7} in k order.
// Both weight matrices are staged once per CTA, split into hi / lo, in the 128-byte-swizzle layout of sw128_off (four
// [128][32] tiles per W2 half, one per W1k half with features 12..31 zero).  3xTF32 issues the mma3 products al.Bh, ah.Bl,
// ah.Bh per k-step; single pass ah.Bh.  The epilogues are shade_fwd_tc's (epi_bias_relu, mask_chunk, epi_hidden_layer3, epi_rgb),
// so the saves keep their layout and mask words and rgb differs from the mma.sync kernel only by accumulation order.  All three
// forms (panel saves, row-major saves, no saves) run the same arithmetic, so a no_grad forward gives the training forward's bits.
namespace fg {
constexpr int kThreads = 384;
constexpr int kRows = 64;                                       // samples per tile (the M of one wgmma)
constexpr int kStages = 4;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;          // 128 * 40 + 256 * 232 <= 384 * 168 (launch allotment)
constexpr uint32_t kTile = kHidden * 32 * 4;                    // one [128][32] fp32 tile: 16 KB
constexpr uint32_t kFeatBytes = kRows * kFeat * 4;              // [64][12] fp32 feature rows
constexpr uint32_t kStage = kFeatBytes + kRows * 8;             // + [64] ray ids
constexpr int kChunks = kFeatBytes / 8;                         // 8-byte copies per tile (rows are 8-byte aligned)
__host__ __device__ constexpr uint32_t oW2(int half) { return half * 4 * kTile; }                 // hi, lo
__host__ __device__ constexpr uint32_t oW1(bool three, int half) { return (three ? 8 : 4) * kTile + half * kTile; }
__host__ __device__ constexpr uint32_t oRing(bool three) { return oW1(three, three ? 2 : 1); }
__host__ __device__ constexpr uint32_t oW3(bool three) { return oRing(three) + kStages * kStage; }
__host__ __device__ constexpr uint32_t oB2(bool three) { return oW3(three) + 3 * kHidden * 4; }
__host__ __device__ constexpr uint32_t oBar(bool three) { return oB2(three) + kHidden * 4; }
// + full and empty barriers, + slack to align the base to 1 KB
__host__ __device__ constexpr uint32_t smem(bool three) { return oBar(three) + 2 * kStages * 8 + 1024; }
}  // namespace fg

__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src, bool ok) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(ok ? 8 : 0) : "memory");
}

template <bool kThree, bool kSave, bool kPanel>
__global__ void __launch_bounds__(fg::kThreads, 1) k_shade_fwd_wgmma(UBN_SHADE_FWD_PARAMS) {
  constexpr int kW = kHidden, kF = kFeat, kNT = n_tiles(kHidden);
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int tid = threadIdx.x;
  for (int i = tid; i < kW * kW; i += fg::kThreads) {         // W2[n][unit]: k-step s, k p <- unit 8 s + (p < 4 ? 2 p : 2 p - 7)
    const int n = i >> 7, kk = i & 127, p = kk & 7;
    const float w = W2[n * kW + (kk & ~7) + (p < 4 ? 2 * p : 2 * p - 7)];
    const uint32_t hi = tf32_hi_bits(w), off = (kk >> 5) * fg::kTile + sw128_off(n, kk & 31);
    *reinterpret_cast<uint32_t*>(smem + fg::oW2(0) + off) = hi;
    if (kThree) *reinterpret_cast<uint32_t*>(smem + fg::oW2(1) + off) = __float_as_uint(w - __uint_as_float(hi));
  }
  for (int i = tid; i < kW * 32; i += fg::kThreads) {          // W1k[n][feature], features >= kF zero
    const int n = i >> 5, k = i & 31;
    const float w = k < kF ? W1k[n * kF + k] : 0.f;
    const uint32_t hi = tf32_hi_bits(w), off = sw128_off(n, k);
    *reinterpret_cast<uint32_t*>(smem + fg::oW1(kThree, 0) + off) = hi;
    if (kThree) *reinterpret_cast<uint32_t*>(smem + fg::oW1(kThree, 1) + off) = __float_as_uint(w - __uint_as_float(hi));
  }
  float* sW3 = reinterpret_cast<float*>(smem + fg::oW3(kThree));
  float* sB2 = reinterpret_cast<float*>(smem + fg::oB2(kThree));
  for (int i = tid; i < 3 * kW; i += fg::kThreads) sW3[i] = W3[i];
  for (int i = tid; i < kW; i += fg::kThreads) sB2[i] = b2[i];
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the weight tiles, before wgmma reads them
  const uint32_t full0 = smem_u32(smem + fg::oBar(kThree)), empty0 = full0 + 8 * fg::kStages;
  if (tid == 0) {
    for (int s = 0; s < fg::kStages; ++s) {
      mbar_init(full0 + 8 * s, 128);
      mbar_init(empty0 + 8 * s, 128);
    }
  }
  __syncthreads();
  const int64_t n_tiles = (n_pts + fg::kRows - 1) / fg::kRows, step = gridDim.x;
  uint8_t* ring = smem + fg::oRing(kThree);

  if (tid < 128) {                                          // producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(fg::kProducerRegs));
    int i = 0;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += step, ++i) {
      const int s = i % fg::kStages;
      mbar_wait(empty0 + 8 * s, ((i / fg::kStages) & 1) ^ 1);
      const int64_t r0 = tile * fg::kRows;
      const uint32_t dst = smem_u32(ring + s * fg::kStage);
      for (int q = tid; q < fg::kChunks; q += 128) {
        const bool ok = r0 + q / (kF / 2) < n_pts;
        cp_async8(dst + 8 * q, ok ? feat + r0 * kF + 2 * q : feat, ok);
      }
      if (tid < fg::kRows) cp_async8(dst + fg::kFeatBytes + 8 * tid, r0 + tid < n_pts ? ray_id + r0 + tid : ray_id, r0 + tid < n_pts);
      asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(full0 + 8 * s) : "memory");
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(fg::kConsumerRegs));
  const int c = (tid >> 7) - 1, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int rl = 16 * ((tid >> 5) & 3) + g;                  // this thread's rows rl and rl + 8 of the tile
  const float b3v[3] = {b3[0], b3[1], b3[2]};
  const uint32_t w2 = smem_u32(smem + fg::oW2(0)), w1 = smem_u32(smem + fg::oW1(kThree, 0));
  int i = c;
  for (int64_t tile = blockIdx.x + c * step; tile < n_tiles; tile += 2 * step, i += 2) {
    const int s = i % fg::kStages;
    mbar_wait(full0 + 8 * s, (i / fg::kStages) & 1);
    const float* sf = reinterpret_cast<const float*>(ring + s * fg::kStage);
    const int64_t* sr = reinterpret_cast<const int64_t*>(ring + s * fg::kStage + fg::kFeatBytes);
    // layer-1 A: k-step 0 = features 0..7, k-step 1 = features 8..11 (k = t) and zeros (k = t + 4)
    const float x[2][4] = {{sf[rl * kF + t], sf[(rl + 8) * kF + t], sf[rl * kF + t + 4], sf[(rl + 8) * kF + t + 4]},
                           {sf[rl * kF + 8 + t], sf[(rl + 8) * kF + 8 + t], 0.f, 0.f}};
    const int64_t ray[2] = {sr[rl], sr[rl + 8]};
    mbar_arrive(empty0 + 8 * s);
    const int64_t row[2] = {tile * fg::kRows + rl, tile * fg::kRows + rl + 8};
    const bool live[2] = {row[0] < n_pts, row[1] < n_pts};

    // layer 1
    float h[kNT][4];
    float(&hv)[64] = reinterpret_cast<float(&)[64]>(h);
    {
      uint32_t xh[2][4], xl[2][4];
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) split4(x[ks], xh[ks], xl[ks]);
#pragma unroll
      for (int e = 0; e < 64; ++e) hv[e] = 0.f;
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        const uint64_t bh = sw128_desc(w1 + 32 * ks);
        if (kThree) {
          wgmma_tf32<1>(hv, xl[ks], bh);
          wgmma_tf32<1>(hv, xh[ks], sw128_desc(w1 + fg::kTile + 32 * ks));
        }
        wgmma_tf32<1>(hv, xh[ks], bh);
      }
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
      for (int e = 0; e < 64; ++e) asm volatile("" : "+f"(hv[e])::"memory");
    }
    // epilogue 1: + vb[ray], ReLU, H1 save and mask words
    epi_bias_relu<kNT>(
        h, t, [&](int r, int cc) { return __ldg(reinterpret_cast<const float2*>(vb + ray[r] * kW + cc)); },
        [&](int r, int cc, float v0, float v1) {
          if (kSave && live[r]) *reinterpret_cast<float2*>(h1_out + save_idx<kPanel, kW>(row[r], cc)) = make_float2(v0, v1);
        });
    if (kSave && kPanel && h1_mask) {
#pragma unroll
      for (int cc = 0; cc < kW / 32; ++cc)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const uint32_t w = mask_chunk(h, cc, 2 * r, t);
          if (t == 0 && live[r]) h1_mask[mask_idx<kW>(row[r], cc)] = w;
        }
    }
    // layer 2: A = H1 straight from the accumulator
    float z[kNT][4];
    float(&zv)[64] = reinterpret_cast<float(&)[64]>(z);
    {
      uint32_t ah[kNT][4], al[kNT][4];
#pragma unroll
      for (int ks = 0; ks < kNT; ++ks) {
        const float av[4] = {h[ks][0], h[ks][2], h[ks][1], h[ks][3]};
        split4(av, ah[ks], al[ks]);
      }
#pragma unroll
      for (int e = 0; e < 64; ++e) zv[e] = 0.f;
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int ks = 0; ks < kNT; ++ks) {
        const uint32_t off = (ks >> 2) * fg::kTile + 32 * (ks & 3);
        const uint64_t bh = sw128_desc(w2 + off);
        if (kThree) {
          wgmma_tf32<1>(zv, al[ks], bh);
          wgmma_tf32<1>(zv, ah[ks], sw128_desc(w2 + fg::oW2(1) + off));
        }
        wgmma_tf32<1>(zv, ah[ks], bh);
      }
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
      for (int e = 0; e < 64; ++e) asm volatile("" : "+f"(zv[e])::"memory");
    }
    // epilogue 2: + b2, ReLU, H2 save, layer 3 (CUDA cores), sigmoid
    float p[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    epi_hidden_layer3<kW, kNT>(z, 0, t, sB2, sW3, p, [&](int r, int cc, float a0, float a1) {
      if (kSave && live[r]) *reinterpret_cast<float2*>(h2_out + save_idx<kPanel, kW>(row[r], cc)) = make_float2(a0, a1);
    });
    epi_rgb(p, b3v, t, [&](int r, const float (&v)[3]) {
      if (live[r]) {
        float* o = rgb + row[r] * 3;
#pragma unroll
        for (int k = 0; k < 3; ++k) o[k] = v[k];
      }
    });
  }
}
#undef UBN_SHADE_FWD_PARAMS

// Width 64 (DirectMPIGO, K = 9): warps per CTA and resident CTAs per SM of each launch, from the -Xptxas -v figures of DESIGN §4
namespace w64 {
constexpr int kFwdWarps = 8, kFwdCtas = 2;
constexpr int kBwdWarps = 8, kBwdCtas = 1;               // 3xTF32 needs 230 registers: 2 CTAs (128) or 4 warps x 3 (168) spill
constexpr int kDw2Ctas = 2;
}  // namespace w64

}  // namespace tc
}  // namespace ubn

using namespace ubn;

namespace {

template <typename K>
int set_smem(K kernel, uint32_t bytes) {
  return finish(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
}

// at most ctas CTAs per SM, and no CTA without a unit for each of its warps
unsigned unit_grid(int64_t n_pts, int warps, int ctas = 1) {
  const int64_t n_units = (n_pts + tc::kUnit - 1) / tc::kUnit;
  return (unsigned)std::min<int64_t>((int64_t)kNumSMs * ctas, (n_units + warps - 1) / warps);
}

// kW = 128 runs the kernels that keep their own names; other widths the _w kernels with kCtas resident CTAs per SM
template <int kF, bool kSave, bool kThree, int kWarps, bool kPanel, int kW = tc::kHidden, int kCtas = 1>
int launch_fwd(const float* feat, const float* vb, const int64_t* ray_id, const float* W1k, const float* W2, const float* b2,
               const float* W3, const float* b3, int64_t n, float* rgb, float* h1, float* h2, uint32_t* m1, cudaStream_t st) {
  auto k = [] {
    if constexpr (kW == tc::kHidden) return tc::k_shade_fwd_tc<kF, kSave, kThree, kWarps, kPanel>;
    else return tc::k_shade_fwd_tc_w<kF, kW, kSave, kThree, kWarps, kCtas, kPanel>;
  }();
  constexpr uint32_t bytes = tc::fw::smem(kW);
  if (int e = set_smem(k, bytes)) return e;
  k<<<unit_grid(n, kWarps, kCtas), 32 * kWarps, bytes, st>>>(feat, vb, ray_id, W1k, W2, b2, W3, b3, n, rgb, h1, h2, m1);
  UBN_LAUNCH_CHECK();
  return 0;
}

template <int kF, bool kSave, bool kThree, int kWarps>
int launch_fwd_p(bool panel, const float* feat, const float* vb, const int64_t* ray_id, const float* W1k, const float* W2,
                 const float* b2, const float* W3, const float* b3, int64_t n, float* rgb, float* h1, float* h2, uint32_t* m1,
                 cudaStream_t st) {
  return panel ? launch_fwd<kF, kSave, kThree, kWarps, true>(feat, vb, ray_id, W1k, W2, b2, W3, b3, n, rgb, h1, h2, m1, st)
               : launch_fwd<kF, kSave, kThree, kWarps, false>(feat, vb, ray_id, W1k, W2, b2, W3, b3, n, rgb, h1, h2, nullptr, st);
}

template <int kF, bool kThree, int kWarps, bool kPanel, bool kMask1, bool kDz1Out, int kW = tc::kHidden, int kCtas = 1>
int launch_bwd(const float* feat, const int64_t* ray_id, const float* W1k, const float* W2, const float* W3, const float* rgb,
               const float* h1, const float* h2, const float* grad_rgb, int64_t n, float* grad_feat, float* grad_vb, float* gW1k,
               float* gb2, float* gW3, float* gb3, uint32_t* m2, const uint32_t* m1, float* dz1, cudaStream_t st) {
  auto k = [] {
    if constexpr (kW != tc::kHidden) {
      static_assert(!kDz1Out, "the dZ1 round trip is a width-128 A/B engine");
      return tc::k_shade_bwd_tc_w<kF, kW, kThree, kWarps, kCtas, kPanel, kMask1>;
    } else if constexpr (kF == tc::kFeat) {
      return tc::k_shade_bwd_tc<kThree, kWarps, kPanel, kMask1, kDz1Out>;
    } else {
      return tc::k_shade_bwd_tc_k<kF, kThree, kWarps, kPanel, kMask1, kDz1Out>;
    }
  }();
  const uint32_t bytes = tc::bk::smem_bytes(kWarps, kF, kW);
  if (int e = set_smem(k, bytes)) return e;
  k<<<unit_grid(n, kWarps, kCtas), 32 * kWarps, bytes, st>>>(feat, ray_id, W1k, W2, W3, rgb, h1, h2, grad_rgb, n, grad_feat, grad_vb, gW1k,
                                                      gb2, gW3, gb3, m2, m1, dz1);
  UBN_LAUNCH_CHECK();
  return 0;
}

template <bool kThree, bool kPanel, bool kMask2, int kW = tc::kHidden, int kCtas = 1>
int launch_dw2(const float* W3, const float* rgb, const float* h1, const float* h2, const uint32_t* m2, const float* grad_rgb,
               int64_t n, float* gW2, cudaStream_t st) {
  auto k = [] {
    if constexpr (kW == tc::kHidden) return tc::k_shade_dw2_tc<kThree, kPanel, kMask2>;
    else return tc::k_shade_dw2_tc_w<kW, kThree, kCtas, kPanel, kMask2>;
  }();
  constexpr uint32_t bytes = tc::dw::smem(kW);
  if (int e = set_smem(k, bytes)) return e;
  const int64_t n_chunks = (n + tc::dw::kK - 1) / tc::dw::kK;
  const unsigned grid = (unsigned)std::min<int64_t>((int64_t)kNumSMs * kCtas, n_chunks);
  k<<<grid, tc::dw::kThreads, bytes, st>>>(W3, rgb, h1, h2, m2, grad_rgb, n, gW2);
  UBN_LAUNCH_CHECK();
  return 0;
}

// which engine computes dW2 at width 128 with panel saves and H2 masks: 1 = k_shade_dw2_wgmma (default), 0 = k_shade_dw2_tc
int g_dw2_engine = 1;

template <bool kThree>
int launch_dw2_wgmma(const float* W3, const float* rgb, const float* h1, const uint32_t* m2, const float* grad_rgb, int64_t n,
                     float* gW2, cudaStream_t st) {
  auto k = tc::k_shade_dw2_wgmma<kThree>;
  constexpr uint32_t bytes = tc::wg::smem(kThree);
  if (int e = set_smem(k, bytes)) return e;
  const int64_t n_chunks = (n + tc::dw::kK - 1) / tc::dw::kK;
  k<<<(unsigned)std::min<int64_t>(kNumSMs, n_chunks), tc::wg::kThreads, bytes, st>>>(W3, rgb, h1, m2, grad_rgb, n, gW2);
  UBN_LAUNCH_CHECK();
  return 0;
}

// which kernel runs the width-128, 12-feature forward (8-warp form): 1 = k_shade_fwd_wgmma (default), 0 = k_shade_fwd_tc
int g_fwd_engine = 1;

template <bool kThree, bool kSave, bool kPanel>
int launch_fwd_wgmma(const float* feat, const float* vb, const int64_t* ray_id, const float* W1k, const float* W2, const float* b2,
                     const float* W3, const float* b3, int64_t n, float* rgb, float* h1, float* h2, uint32_t* m1, cudaStream_t st) {
  auto k = tc::k_shade_fwd_wgmma<kThree, kSave, kPanel>;
  constexpr uint32_t bytes = tc::fg::smem(kThree);
  if (int e = set_smem(k, bytes)) return e;
  const int64_t n_tiles = (n + tc::fg::kRows - 1) / tc::fg::kRows;
  k<<<(unsigned)std::min<int64_t>(kNumSMs, n_tiles), tc::fg::kThreads, bytes, st>>>(feat, vb, ray_id, W1k, W2, b2, W3, b3, n, rgb,
                                                                                      h1, h2, m1);
  UBN_LAUNCH_CHECK();
  return 0;
}

template <int kF>
int rgbnet_fwd_tc(const float* feat, const float* view_bias, const int64_t* ray_id, const float* W1k, const float* W2, const float* b2,
                  const float* W3, const float* b3, int64_t n_pts, float* rgb, float* h1_save, float* h2_save, uint32_t* h1_mask,
                  int single_pass, void* stream) {
  if (n_pts <= 0) return 0;
  const bool save = h1_save != nullptr && h2_save != nullptr;
  const bool one = (single_pass & 1) != 0, four = (single_pass & 2) != 0, panel = save && (single_pass & 4) != 0;
  cudaStream_t st = as_stream(stream);
#define UBN_FWD(SAVE, THREE, W) \
  return launch_fwd_p<kF, SAVE, THREE, W>(panel, feat, view_bias, ray_id, W1k, W2, b2, W3, b3, n_pts, rgb, h1_save, h2_save, h1_mask, st)
  if constexpr (kF == tc::kFeat) {
    if (!four && g_fwd_engine == 1) {
#define UBN_FWD_WG(THREE, SAVE, P) \
  return launch_fwd_wgmma<THREE, SAVE, P>(feat, view_bias, ray_id, W1k, W2, b2, W3, b3, n_pts, rgb, h1_save, h2_save, h1_mask, st)
      if (save && panel) { if (one) UBN_FWD_WG(false, true, true); else UBN_FWD_WG(true, true, true); }
      if (save) { if (one) UBN_FWD_WG(false, true, false); else UBN_FWD_WG(true, true, false); }
      if (one) UBN_FWD_WG(false, false, false); else UBN_FWD_WG(true, false, false);
#undef UBN_FWD_WG
    }
  }
  if (save) {
    if (one) { if (four) UBN_FWD(true, false, 4); else UBN_FWD(true, false, 8); }
    if (four) UBN_FWD(true, true, 4); else UBN_FWD(true, true, 8);
  }
  if (one) { if (four) UBN_FWD(false, false, 4); else UBN_FWD(false, false, 8); }
  if (four) UBN_FWD(false, true, 4); else UBN_FWD(false, true, 8);
#undef UBN_FWD
}

template <int kF>
int rgbnet_bwd_tc_fused(const float* feat, const int64_t* ray_id, const float* W1k, const float* W2, const float* W3, const float* rgb,
                        const float* h1_save, const float* h2_save, const float* grad_rgb, int64_t n_pts, float* grad_feat,
                        float* grad_view_bias, float* grad_W1k, float* grad_W2, float* grad_b2, float* grad_W3, float* grad_b3,
                        uint32_t* h2_mask_scratch, const uint32_t* h1_mask, int single_pass, void* stream) {
  if (n_pts <= 0) return 0;
  cudaStream_t st = as_stream(stream);
  // kF = 15: three more sum rows per warp -- 8 warps would need 240 640 B of shared memory (the limit is 232 448 B), so 4 warps
  const bool one = (single_pass & 1) != 0, four = (single_pass & 2) != 0 || kF > 12, panel = (single_pass & 4) != 0;
  const bool mask1 = panel && h1_mask != nullptr, mask2 = panel && h2_mask_scratch != nullptr;
  uint32_t* m2 = mask2 ? h2_mask_scratch : nullptr;
  int e = 0;
#define UBN_BWD(THREE, W, P, M1)                                                                                              \
  e = launch_bwd<kF, THREE, W, P, M1, false>(feat, ray_id, W1k, W2, W3, rgb, h1_save, h2_save, grad_rgb, n_pts, grad_feat,        \
                                         grad_view_bias, grad_W1k, grad_b2, grad_W3, grad_b3, m2, h1_mask, nullptr, st)
#define UBN_BWD_W(THREE, P, M1) \
  do { if (four) UBN_BWD(THREE, 4, P, M1); else if constexpr (kF <= 12) UBN_BWD(THREE, 8, P, M1); } while (0)
#define UBN_BWD_T(P, M1) \
  do { if (one) UBN_BWD_W(false, P, M1); else UBN_BWD_W(true, P, M1); } while (0)
  if (mask1) UBN_BWD_T(true, true);
  else if (panel) UBN_BWD_T(true, false);
  else UBN_BWD_T(false, false);
#undef UBN_BWD_T
#undef UBN_BWD_W
#undef UBN_BWD
  if (e) return e;
#define UBN_DW(THREE, P, M2) return launch_dw2<THREE, P, M2>(W3, rgb, h1_save, h2_save, m2, grad_rgb, n_pts, grad_W2, st)
  if (mask2 && g_dw2_engine == 1) {
    if (one) return launch_dw2_wgmma<false>(W3, rgb, h1_save, m2, grad_rgb, n_pts, grad_W2, st);
    return launch_dw2_wgmma<true>(W3, rgb, h1_save, m2, grad_rgb, n_pts, grad_W2, st);
  }
  if (mask2) { if (one) UBN_DW(false, true, true); else UBN_DW(true, true, true); }
  if (panel) { if (one) UBN_DW(false, true, false); else UBN_DW(true, true, false); }
  if (one) UBN_DW(false, false, false); else UBN_DW(true, false, false);
#undef UBN_DW
}

// hidden width kW != 128: the forward writes its saves in the panel layout only, and the backward runs with both ReLU masks
template <int kF, int kW>
int rgbnet_fwd_tc_w(const float* feat, const float* view_bias, const int64_t* ray_id, const float* W1k, const float* W2,
                    const float* b2, const float* W3, const float* b3, int64_t n_pts, float* rgb, float* h1_save, float* h2_save,
                    uint32_t* h1_mask, int single_pass, void* stream) {
  const bool save = h1_save != nullptr && h2_save != nullptr;
  if (save && (single_pass & 4) == 0) return finish(cudaErrorInvalidValue);
  if (n_pts <= 0) return 0;
  const bool one = (single_pass & 1) != 0;
  cudaStream_t st = as_stream(stream);
  constexpr int W = tc::w64::kFwdWarps, C = tc::w64::kFwdCtas;
#define UBN_FWD_W(SAVE, THREE, M1) \
  return launch_fwd<kF, SAVE, THREE, W, SAVE, kW, C>(feat, view_bias, ray_id, W1k, W2, b2, W3, b3, n_pts, rgb, h1_save, h2_save, M1, st)
  if (save) { if (one) UBN_FWD_W(true, false, h1_mask); else UBN_FWD_W(true, true, h1_mask); }
  if (one) UBN_FWD_W(false, false, nullptr); else UBN_FWD_W(false, true, nullptr);
#undef UBN_FWD_W
}

template <int kF, int kW>
int rgbnet_bwd_tc_fused_w(const float* feat, const int64_t* ray_id, const float* W1k, const float* W2, const float* W3,
                          const float* rgb, const float* h1_save, const float* h2_save, const float* grad_rgb, int64_t n_pts,
                          float* grad_feat, float* grad_view_bias, float* grad_W1k, float* grad_W2, float* grad_b2, float* grad_W3,
                          float* grad_b3, uint32_t* h2_mask_scratch, const uint32_t* h1_mask, int single_pass, void* stream) {
  if (n_pts <= 0) return 0;              // a batch without survivors: its zero-sized mask buffers have no address
  if ((single_pass & 4) == 0 || h1_mask == nullptr || h2_mask_scratch == nullptr) return finish(cudaErrorInvalidValue);
  const bool one = (single_pass & 1) != 0;
  cudaStream_t st = as_stream(stream);
  constexpr int W = tc::w64::kBwdWarps, C = tc::w64::kBwdCtas, C2 = tc::w64::kDw2Ctas;
#define UBN_BWD_W(THREE)                                                                                                        \
  launch_bwd<kF, THREE, W, true, true, false, kW, C>(feat, ray_id, W1k, W2, W3, rgb, h1_save, h2_save, grad_rgb, n_pts, grad_feat, \
                                                     grad_view_bias, grad_W1k, grad_b2, grad_W3, grad_b3, h2_mask_scratch, h1_mask,  \
                                                     nullptr, st)
  if (int e = one ? UBN_BWD_W(false) : UBN_BWD_W(true)) return e;
#undef UBN_BWD_W
  if (one) return launch_dw2<false, true, true, kW, C2>(W3, rgb, h1_save, h2_save, h2_mask_scratch, grad_rgb, n_pts, grad_W2, st);
  return launch_dw2<true, true, true, kW, C2>(W3, rgb, h1_save, h2_save, h2_mask_scratch, grad_rgb, n_pts, grad_W2, st);
}

}  // namespace

extern "C" int ubn_set_dw2_engine(int engine) {
  if (engine < 0 || engine > 1) return finish(cudaErrorInvalidValue);
  g_dw2_engine = engine;
  return 0;
}

extern "C" int ubn_set_fwd_engine(int engine) {
  if (engine < 0 || engine > 1) return finish(cudaErrorInvalidValue);
  g_fwd_engine = engine;
  return 0;
}

extern "C" int ubn_get_fwd_engine(void) { return g_fwd_engine; }

extern "C" int ubn_rgbnet_fwd_tc(const float* feat, const float* view_bias, const int64_t* ray_id, const float* W1k,
                                 const float* W2, const float* b2, const float* W3, const float* b3, int64_t n_pts,
                                 float* rgb, float* h1_save, float* h2_save, uint32_t* h1_mask, int single_pass, void* stream) {
  return rgbnet_fwd_tc<tc::kFeat>(feat, view_bias, ray_id, W1k, W2, b2, W3, b3, n_pts, rgb, h1_save, h2_save, h1_mask, single_pass,
                                  stream);
}

extern "C" int ubn_rgbnet_fwd_tc_k(int n_feat, const float* feat, const float* view_bias, const int64_t* ray_id, const float* W1k,
                                   const float* W2, const float* b2, const float* W3, const float* b3, int64_t n_pts, float* rgb,
                                   float* h1_save, float* h2_save, uint32_t* h1_mask, int single_pass, void* stream) {
#define UBN_FWD_K(F) \
  return rgbnet_fwd_tc<F>(feat, view_bias, ray_id, W1k, W2, b2, W3, b3, n_pts, rgb, h1_save, h2_save, h1_mask, single_pass, stream)
  switch (n_feat) {
    case 3: UBN_FWD_K(3);
    case 12: UBN_FWD_K(12);
    case 15: UBN_FWD_K(15);
    default: return finish(cudaErrorInvalidValue);
  }
#undef UBN_FWD_K
}

extern "C" int ubn_rgbnet_bwd_tc_data(const float* W2, const float* W3, const float* rgb, const float* h1_save,
                                      const float* h2_save, const float* grad_rgb, int64_t n_pts, float* dz1_out,
                                      float* grad_W2, void* stream) {
  if (n_pts <= 0) return 0;
  cudaStream_t st = as_stream(stream);
  if (int e = launch_bwd<tc::kFeat, true, 8, false, false, true>(nullptr, nullptr, nullptr, W2, W3, rgb, h1_save, h2_save, grad_rgb, n_pts,
                                                     nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                                                     dz1_out, st))
    return e;
  return launch_dw2<true, false, false>(W3, rgb, h1_save, h2_save, nullptr, grad_rgb, n_pts, grad_W2, st);
}

extern "C" int ubn_rgbnet_bwd_tc_fused(const float* feat, const int64_t* ray_id, const float* W1k, const float* W2, const float* W3,
                                       const float* rgb, const float* h1_save, const float* h2_save, const float* grad_rgb,
                                       int64_t n_pts, float* grad_feat, float* grad_view_bias, float* grad_W1k, float* grad_W2,
                                       float* grad_b2, float* grad_W3, float* grad_b3, uint32_t* h2_mask_scratch,
                                       const uint32_t* h1_mask, int single_pass, void* stream) {
  return rgbnet_bwd_tc_fused<tc::kFeat>(feat, ray_id, W1k, W2, W3, rgb, h1_save, h2_save, grad_rgb, n_pts, grad_feat, grad_view_bias,
                                        grad_W1k, grad_W2, grad_b2, grad_W3, grad_b3, h2_mask_scratch, h1_mask, single_pass, stream);
}

extern "C" int ubn_rgbnet_bwd_tc_fused_k(int n_feat, const float* feat, const int64_t* ray_id, const float* W1k, const float* W2,
                                         const float* W3, const float* rgb, const float* h1_save, const float* h2_save,
                                         const float* grad_rgb, int64_t n_pts, float* grad_feat, float* grad_view_bias, float* grad_W1k,
                                         float* grad_W2, float* grad_b2, float* grad_W3, float* grad_b3, uint32_t* h2_mask_scratch,
                                         const uint32_t* h1_mask, int single_pass, void* stream) {
#define UBN_BWD_K(F)                                                                                                             \
  return rgbnet_bwd_tc_fused<F>(feat, ray_id, W1k, W2, W3, rgb, h1_save, h2_save, grad_rgb, n_pts, grad_feat, grad_view_bias, \
                                grad_W1k, grad_W2, grad_b2, grad_W3, grad_b3, h2_mask_scratch, h1_mask, single_pass, stream)
  switch (n_feat) {
    case 3: UBN_BWD_K(3);
    case 12: UBN_BWD_K(12);
    case 15: UBN_BWD_K(15);
    default: return finish(cudaErrorInvalidValue);
  }
#undef UBN_BWD_K
}

extern "C" int ubn_rgbnet_fwd_tc_kw(int n_feat, int n_hidden, const float* feat, const float* view_bias, const int64_t* ray_id,
                                    const float* W1k, const float* W2, const float* b2, const float* W3, const float* b3, int64_t n_pts,
                                    float* rgb, float* h1_save, float* h2_save, uint32_t* h1_mask, int single_pass, void* stream) {
  if (n_hidden == tc::kHidden)
    return ubn_rgbnet_fwd_tc_k(n_feat, feat, view_bias, ray_id, W1k, W2, b2, W3, b3, n_pts, rgb, h1_save, h2_save, h1_mask,
                               single_pass, stream);
  if (n_hidden == 64 && n_feat == 9)
    return rgbnet_fwd_tc_w<9, 64>(feat, view_bias, ray_id, W1k, W2, b2, W3, b3, n_pts, rgb, h1_save, h2_save, h1_mask, single_pass,
                                  stream);
  return finish(cudaErrorInvalidValue);
}

extern "C" int ubn_rgbnet_bwd_tc_fused_kw(int n_feat, int n_hidden, const float* feat, const int64_t* ray_id, const float* W1k,
                                          const float* W2, const float* W3, const float* rgb, const float* h1_save, const float* h2_save,
                                          const float* grad_rgb, int64_t n_pts, float* grad_feat, float* grad_view_bias,
                                          float* grad_W1k, float* grad_W2, float* grad_b2, float* grad_W3, float* grad_b3,
                                          uint32_t* h2_mask_scratch, const uint32_t* h1_mask, int single_pass, void* stream) {
  if (n_hidden == tc::kHidden)
    return ubn_rgbnet_bwd_tc_fused_k(n_feat, feat, ray_id, W1k, W2, W3, rgb, h1_save, h2_save, grad_rgb, n_pts, grad_feat,
                                     grad_view_bias, grad_W1k, grad_W2, grad_b2, grad_W3, grad_b3, h2_mask_scratch, h1_mask,
                                     single_pass, stream);
  if (n_hidden == 64 && n_feat == 9)
    return rgbnet_bwd_tc_fused_w<9, 64>(feat, ray_id, W1k, W2, W3, rgb, h1_save, h2_save, grad_rgb, n_pts, grad_feat, grad_view_bias,
                                        grad_W1k, grad_W2, grad_b2, grad_W3, grad_b3, h2_mask_scratch, h1_mask, single_pass, stream);
  return finish(cudaErrorInvalidValue);
}
