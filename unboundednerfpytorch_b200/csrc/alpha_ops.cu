// alpha_ops.cu -- Raw2Alpha / Alphas2Weights kernels of libubnerf_b200.so.
//
// Replaces render_utils_kernel.cu:431-707 of the reference (K10-K16 in SURVEY.md 2a).
//
// raw2alpha*: streaming elementwise, one thread per element, coalesced.
// alpha2weight*: the reference walks each ray with ONE thread (8192 threads total at the benchmark
//   size = 32 blocks on a 132-SM H100, stride-S uncoalesced).  The transmittance recurrence
//   T <- float(double(T) * (1. - double(alpha))) with its early stop at T < 1e-3 is order sensitive, so
//   the sequential evaluation is kept bit-for-bit (i_end is an index output = bit-exact parity target),
//   but re-mapped: one LANE per ray, 32 rays per warp, 32x32 tiles staged through shared memory so all
//   global traffic is coalesced 128-byte rows and the grid covers all SMs.
#include "common.cuh"

namespace ubn {

// ------------------------------------------------------------------------------------------------
// raw2alpha (render_utils_kernel.cu:431-458; raw2alpha_one, common.cuh) / backward (:507-530)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float raw2alpha_bwd_one(float e, float g, float interval) {
  // min(float, 1e10) promotes to double; powf stays float; product in double, stored as float (:515)
  return fmin((double)e, 1e10) * powf(1 + e, -interval - 1) * interval * g;
}

template <bool kNonUni>
__global__ void __launch_bounds__(256) k_raw2alpha(const float* __restrict__ density, float shift, float interval,
                                                   const float* __restrict__ interval_arr, int64_t n,
                                                   float* __restrict__ exp_d, float* __restrict__ alpha) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float e, a;
  raw2alpha_one(density[i], shift, kNonUni ? interval_arr[i] : interval, &e, &a);
  exp_d[i] = e;
  alpha[i] = a;
}

template <bool kNonUni>
__global__ void __launch_bounds__(256) k_raw2alpha_bwd(const float* __restrict__ exp_d,
                                                       const float* __restrict__ grad_back, float interval,
                                                       const float* __restrict__ interval_arr, int64_t n,
                                                       float* __restrict__ grad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  grad[i] = raw2alpha_bwd_one(exp_d[i], grad_back[i], kNonUni ? interval_arr[i] : interval);
}

// ------------------------------------------------------------------------------------------------
// segment bounds (render_utils_kernel.cu:607-617 + the host-side fix-up at :635)
// ------------------------------------------------------------------------------------------------
__global__ void k_init_rays(int64_t n_rays, float* __restrict__ alphainv_last, int64_t* __restrict__ i_start,
                            int64_t* __restrict__ i_end) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  alphainv_last[r] = 1.f;
  i_start[r] = 0;
  i_end[r] = 0;
}

__global__ void k_segment_bounds(const int64_t* __restrict__ ray_id, int64_t n_pts, int64_t* __restrict__ i_start,
                                 int64_t* __restrict__ i_end) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_pts) return;
  const int64_t me = ray_id[idx];
  if (idx > 0) {
    const int64_t prev = ray_id[idx - 1];
    if (me != prev) {
      i_start[me] = idx;
      i_end[prev] = idx;
    }
  }
  if (idx == n_pts - 1) i_end[me] = n_pts;
}

// ------------------------------------------------------------------------------------------------
// alpha2weight forward (render_utils_kernel.cu:577-605)
// ------------------------------------------------------------------------------------------------
constexpr int kA2WWarps = 2;  // 64 rays per block -> 128 blocks at 8192 rays

__global__ void __launch_bounds__(32 * kA2WWarps) k_alpha2weight(
    const float* __restrict__ alpha, int64_t n_rays, float* __restrict__ weight, float* __restrict__ T,
    float* __restrict__ alphainv_last, const int64_t* __restrict__ i_start, int64_t* __restrict__ i_end) {
  __shared__ float s_a[kA2WWarps][32][33];  // alpha in, weight out (in place)
  __shared__ float s_t[kA2WWarps][32][33];  // T out
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t ray0 = ((int64_t)blockIdx.x * kA2WWarps + w) * 32;
  if (ray0 >= n_rays) return;
  const int64_t ray = ray0 + lane;
  const bool live = ray < n_rays;
  const int64_t my_s = live ? i_start[ray] : 0;
  const int my_len = live ? (int)(i_end[ray] - my_s) : 0;
  int max_len = my_len;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) max_len = max(max_len, __shfl_xor_sync(0xffffffffu, max_len, o));

  float T_cum = 1.f;
  bool done = false;
  int stop = my_len;  // number of elements consumed (i_end - i_start after truncation)
  for (int base = 0; base < max_len; base += 32) {
#pragma unroll 4
    for (int rr = 0; rr < 32; ++rr) {
      const int64_t s = __shfl_sync(0xffffffffu, my_s, rr);
      const int l = __shfl_sync(0xffffffffu, my_len, rr);
      const int c = base + lane;
      if (c < l) s_a[w][rr][lane] = alpha[s + c];
    }
    __syncwarp();
    const int ncol = min(32, my_len - base);
    for (int j = 0; j < ncol; ++j) {
      if (!done) {
        const float a = s_a[w][lane][j];
        s_t[w][lane][j] = T_cum;
        s_a[w][lane][j] = T_cum * a;
        T_cum *= (1. - a);          // double intermediate, rounded to float on store (:596)
        if (T_cum < 1e-3) {         // compared in double (:597)
          done = true;
          stop = base + j + 1;
        }
      } else {                      // untouched tail keeps weight = 0, T = 1 (zeros_like / ones_like :624-625)
        s_t[w][lane][j] = 1.f;
        s_a[w][lane][j] = 0.f;
      }
    }
    __syncwarp();
#pragma unroll 4
    for (int rr = 0; rr < 32; ++rr) {
      const int64_t s = __shfl_sync(0xffffffffu, my_s, rr);
      const int l = __shfl_sync(0xffffffffu, my_len, rr);
      const int c = base + lane;
      if (c < l) {
        weight[s + c] = s_a[w][rr][lane];
        T[s + c] = s_t[w][rr][lane];
      }
    }
    __syncwarp();
  }
  if (live) {
    i_end[ray] = my_s + stop;
    alphainv_last[ray] = T_cum;
  }
}

// ------------------------------------------------------------------------------------------------
// alpha2weight backward (render_utils_kernel.cu:654-677)
//   back_cum walks each ray from i_end-1 down to i_start with float fma (order sensitive);
//   grad[i] = gw[i]*T[i] - back_cum / (1 - alpha[i] + 1e-10)  with a double denominator / quotient.
//   Elements outside [i_start, i_end) keep grad = 0 (zeros_like, :684).
// Launch: same 32-rays-per-warp tiling; tiles are visited back to front.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * kA2WWarps) k_alpha2weight_bwd(
    const float* __restrict__ alpha, const float* __restrict__ weight, const float* __restrict__ T,
    const float* __restrict__ alphainv_last, const int64_t* __restrict__ i_start,
    const int64_t* __restrict__ i_end, int64_t n_rays, const float* __restrict__ grad_weights,
    const float* __restrict__ grad_last, float* __restrict__ grad) {
  __shared__ float s_g[kA2WWarps][32][33];  // gw in
  __shared__ float s_b[kA2WWarps][32][33];  // w in, back_cum out
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t ray0 = ((int64_t)blockIdx.x * kA2WWarps + w) * 32;
  if (ray0 >= n_rays) return;
  const int64_t ray = ray0 + lane;
  const bool live = ray < n_rays;
  const int64_t my_s = live ? i_start[ray] : 0;
  const int my_len = live ? (int)(i_end[ray] - my_s) : 0;
  int max_len = my_len;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) max_len = max(max_len, __shfl_xor_sync(0xffffffffu, max_len, o));
  float back_cum = live ? grad_last[ray] * alphainv_last[ray] : 0.f;

  const int n_tiles = (max_len + 31) / 32;
  for (int tile = n_tiles - 1; tile >= 0; --tile) {
    const int base = tile * 32;
#pragma unroll 4
    for (int rr = 0; rr < 32; ++rr) {
      const int64_t s = __shfl_sync(0xffffffffu, my_s, rr);
      const int l = __shfl_sync(0xffffffffu, my_len, rr);
      const int c = base + lane;
      if (c < l) {
        s_g[w][rr][lane] = grad_weights[s + c];
        s_b[w][rr][lane] = weight[s + c];
      }
    }
    __syncwarp();
    const int ncol = min(32, my_len - base);
    for (int j = ncol - 1; j >= 0; --j) {
      const float gw = s_g[w][lane][j];
      const float wt = s_b[w][lane][j];
      s_b[w][lane][j] = back_cum;   // value used by element (base + j)
      back_cum += gw * wt;          // float fma (:674)
    }
    __syncwarp();
#pragma unroll 4
    for (int rr = 0; rr < 32; ++rr) {
      const int64_t s = __shfl_sync(0xffffffffu, my_s, rr);
      const int l = __shfl_sync(0xffffffffu, my_len, rr);
      const int c = base + lane;
      if (c < l) {
        const int64_t i = s + c;
        grad[i] = s_g[w][rr][lane] * T[i] - s_b[w][rr][lane] / (1 - alpha[i] + 1e-10);
      }
    }
    __syncwarp();
  }
}

// zero-fill of grad outside the processed segments: the compact forward guarantees that every point
// belongs to exactly one [i_start, original i_end) segment, but the *truncated* i_end leaves a tail.
__global__ void k_zero_f32(float* __restrict__ p, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 0.f;
}

}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_raw2alpha(const float* density, float shift, float interval, const float* interval_arr, int64_t n_pts,
                  float* exp_d, float* alpha, void* stream) {
  if (n_pts <= 0) return 0;
  if (interval_arr)
    k_raw2alpha<true><<<blocks_for(n_pts, 256), 256, 0, as_stream(stream)>>>(density, shift, interval,
                                                                            interval_arr, n_pts, exp_d, alpha);
  else
    k_raw2alpha<false><<<blocks_for(n_pts, 256), 256, 0, as_stream(stream)>>>(density, shift, interval, nullptr,
                                                                             n_pts, exp_d, alpha);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_raw2alpha_backward(const float* exp_d, const float* grad_back, float interval, const float* interval_arr,
                           int64_t n_pts, float* grad, void* stream) {
  if (n_pts <= 0) return 0;
  if (interval_arr)
    k_raw2alpha_bwd<true><<<blocks_for(n_pts, 256), 256, 0, as_stream(stream)>>>(exp_d, grad_back, interval,
                                                                                interval_arr, n_pts, grad);
  else
    k_raw2alpha_bwd<false><<<blocks_for(n_pts, 256), 256, 0, as_stream(stream)>>>(exp_d, grad_back, interval,
                                                                                 nullptr, n_pts, grad);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_alpha2weight(const float* alpha, const int64_t* ray_id, int64_t n_pts, int64_t n_rays, float* weight,
                     float* T, float* alphainv_last, int64_t* i_start, int64_t* i_end, void* stream) {
  cudaStream_t st = as_stream(stream);
  if (n_rays <= 0) return 0;
  k_init_rays<<<blocks_for(n_rays, 256), 256, 0, st>>>(n_rays, alphainv_last, i_start, i_end);
  UBN_LAUNCH_CHECK();
  if (n_pts <= 0) return 0;
  k_segment_bounds<<<blocks_for(n_pts, 256), 256, 0, st>>>(ray_id, n_pts, i_start, i_end);
  UBN_LAUNCH_CHECK();
  k_alpha2weight<<<blocks_for(n_rays, 32 * kA2WWarps), 32 * kA2WWarps, 0, st>>>(alpha, n_rays, weight, T,
                                                                               alphainv_last, i_start, i_end);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_alpha2weight_backward(const float* alpha, const float* weight, const float* T, const float* alphainv_last,
                              const int64_t* i_start, const int64_t* i_end, int64_t n_pts, int64_t n_rays,
                              const float* grad_weights, const float* grad_last, float* grad, void* stream) {
  cudaStream_t st = as_stream(stream);
  if (n_pts <= 0) return 0;
  // elements past a ray's truncated i_end receive no gradient (zeros_like in the reference)
  k_zero_f32<<<blocks_for(n_pts, 256), 256, 0, st>>>(grad, n_pts);
  UBN_LAUNCH_CHECK();
  if (n_rays <= 0) return 0;
  k_alpha2weight_bwd<<<blocks_for(n_rays, 32 * kA2WWarps), 32 * kA2WWarps, 0, st>>>(
      alpha, weight, T, alphainv_last, i_start, i_end, n_rays, grad_weights, grad_last, grad);
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// segment_sum: out[r, :] = sum over the (sorted) segment of ray r of src[i, :]  -- the reduction the
// reference takes from torch_scatter.segment_coo(reduce='sum') (dvgo.py:401,418; dcvgo.py:345,354,377;
// FourierGrid_model.py:640,666).  One warp per ray: lanes stride over the segment (coalesced rows of K
// floats), per-lane partial sums, xor-shuffle tree -> deterministic (no atomics), any K <= 4.
// ------------------------------------------------------------------------------------------------
namespace ubn {

template <int K>
__global__ void __launch_bounds__(128) k_segment_sum(const float* __restrict__ src, const int64_t* __restrict__ i_start,
                                                     const int64_t* __restrict__ i_end, int64_t n_rays,
                                                     float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const int64_t s = i_start[ray], e = i_end[ray];
  float acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.f;
  for (int64_t i = s + lane; i < e; i += 32) {
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k] += src[i * K + k];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) out[ray * K + k] = acc[k];
  }
}

}  // namespace ubn

extern "C" int ubn_segment_sum(const float* src, int64_t k, const int64_t* ray_id, int64_t n_pts, int64_t n_rays,
                               int64_t* i_start, int64_t* i_end, float* out, void* stream) {
  using namespace ubn;
  cudaStream_t st = as_stream(stream);
  if (n_rays <= 0) return 0;
  if (k < 1 || k > 4) return finish(cudaErrorInvalidValue);
  // bounds (empty rays keep [0,0) -> sum 0); alphainv_last slot of k_init_rays is reused as a dummy via out
  k_init_rays<<<blocks_for(n_rays, 256), 256, 0, st>>>(n_rays, out, i_start, i_end);
  UBN_LAUNCH_CHECK();
  if (n_pts > 0) {
    k_segment_bounds<<<blocks_for(n_pts, 256), 256, 0, st>>>(ray_id, n_pts, i_start, i_end);
    UBN_LAUNCH_CHECK();
  }
  const unsigned nb = blocks_for(n_rays, 4);
  switch (k) {
    case 1: k_segment_sum<1><<<nb, 128, 0, st>>>(src, i_start, i_end, n_rays, out); break;
    case 2: k_segment_sum<2><<<nb, 128, 0, st>>>(src, i_start, i_end, n_rays, out); break;
    case 3: k_segment_sum<3><<<nb, 128, 0, st>>>(src, i_start, i_end, n_rays, out); break;
    default: k_segment_sum<4><<<nb, 128, 0, st>>>(src, i_start, i_end, n_rays, out); break;
  }
  UBN_LAUNCH_CHECK();
  return 0;
}


// ---- composite: rgb_marched[r] = sum_{i in r} weights_i * rgb_i  (FourierGrid_model.py:640-644, dcvgo.py:345-349,
// dvgo.py:401-405) without materialising weights[:,None] * rgb, and its adjoint in one pass -------------------------------
namespace ubn {

__global__ void __launch_bounds__(128) k_composite_fwd(const float* __restrict__ weights, const float* __restrict__ rgb,
                                                       const int64_t* __restrict__ i_start, const int64_t* __restrict__ i_end,
                                                       int64_t n_rays, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const int64_t s = i_start[ray], e = i_end[ray];
  float acc[3] = {0.f, 0.f, 0.f};
  for (int64_t i = s + lane; i < e; i += 32) {
    const float w = weights[i];
#pragma unroll
    for (int k = 0; k < 3; ++k) acc[k] += __fmul_rn(w, rgb[i * 3 + k]);   // product rounded first, like the torch mul
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < 3; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) out[ray * 3 + k] = acc[k];
  }
}

// grad_rgb_i = w_i * g[ray_i];  grad_w_i = sum_c g[ray_i, c] * rgb_i[c]
__global__ void __launch_bounds__(256) k_composite_bwd(const float* __restrict__ weights, const float* __restrict__ rgb,
                                                       const int64_t* __restrict__ ray_id, const float* __restrict__ g,
                                                       int64_t n_pts, float* __restrict__ grad_w, float* __restrict__ grad_rgb) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pts) return;
  const int64_t r = ray_id[i];
  const float g0 = g[3 * r], g1 = g[3 * r + 1], g2 = g[3 * r + 2];
  if (grad_rgb) {
    const float w = weights[i];
    grad_rgb[3 * i] = __fmul_rn(g0, w); grad_rgb[3 * i + 1] = __fmul_rn(g1, w); grad_rgb[3 * i + 2] = __fmul_rn(g2, w);
  }
  if (grad_w)
    grad_w[i] = __fadd_rn(__fadd_rn(__fmul_rn(g0, rgb[3 * i]), __fmul_rn(g1, rgb[3 * i + 1])), __fmul_rn(g2, rgb[3 * i + 2]));
}

}  // namespace ubn

extern "C" int ubn_composite_fwd(const float* weights, const float* rgb, const int64_t* ray_id, int64_t n_pts, int64_t n_rays,
                                 int64_t* i_start, int64_t* i_end, float* out, void* stream) {
  using namespace ubn;
  cudaStream_t st = as_stream(stream);
  if (n_rays <= 0) return 0;
  k_init_rays<<<blocks_for(n_rays, 256), 256, 0, st>>>(n_rays, out, i_start, i_end);
  UBN_LAUNCH_CHECK();
  if (n_pts > 0) {
    k_segment_bounds<<<blocks_for(n_pts, 256), 256, 0, st>>>(ray_id, n_pts, i_start, i_end);
    UBN_LAUNCH_CHECK();
  }
  k_composite_fwd<<<blocks_for(n_rays, 4), 128, 0, st>>>(weights, rgb, i_start, i_end, n_rays, out);
  UBN_LAUNCH_CHECK();
  return 0;
}

extern "C" int ubn_composite_bwd(const float* weights, const float* rgb, const int64_t* ray_id, const float* grad_out,
                                 int64_t n_pts, float* grad_weights, float* grad_rgb, void* stream) {
  using namespace ubn;
  if (n_pts <= 0) return 0;
  k_composite_bwd<<<blocks_for(n_pts, 256), 256, 0, as_stream(stream)>>>(weights, rgb, ray_id, grad_out, n_pts, grad_weights,
                                                                         grad_rgb);
  UBN_LAUNCH_CHECK();
  return 0;
}


// ---- distortion loss (torch_efficient_distloss.flatten_eff_distloss as used at run_train.py:268-274; maths kept in-tree at
// dcvgo.py:387-409):  L = (1/R) sum_rays [ sum_i interval/3 * w_i^2 + 2 sum_i w_i (s_i W_<i - WS_<i) ],  R = max(ray_id)+1,
// W_<i / WS_<i = exclusive prefix sums of w / w*s inside the ray.  One warp per ray: a forward sweep in 32-sample chunks
// (warp scan + carried totals) yields the ray's loss and totals, a second sweep writes
//   dL/dw_i = (1/R) [ 2/3 interval w_i + 2 (s_i W_<i - WS_<i) + 2 ((WS_tot - WS_<=i) - s_i (W_tot - W_<=i)) ].
namespace ubn {

__device__ __forceinline__ float warp_incl_scan(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

__global__ void __launch_bounds__(128) k_distortion_loss(const float* __restrict__ w, const float* __restrict__ s,
                                                         const int64_t* __restrict__ i_start, const int64_t* __restrict__ i_end,
                                                         int64_t n_rays, float interval, const int64_t* __restrict__ last_id,
                                                         float* __restrict__ grad_w, double* __restrict__ ray_loss) {
  const int lane = threadIdx.x & 31;
  const float inv_r = 1.f / (float)(*last_id + 1);     // R = ray_id.max() + 1 = id of the last (sorted) sample + 1, like the library
  const int64_t ray = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const int64_t b = i_start[ray], e = i_end[ray];
  float cw = 0.f, cws = 0.f;        // carried exclusive totals of the chunks done so far
  double loss = 0.0;
  for (int64_t c = b; c < e; c += 32) {
    const int64_t i = c + lane;
    const bool ok = i < e;
    const float wi = ok ? w[i] : 0.f, si = ok ? s[i] : 0.f;
    const float ws = wi * si;
    const float iw = warp_incl_scan(wi, lane), iws = warp_incl_scan(ws, lane);
    const float pw = cw + (iw - wi), pws = cws + (iws - ws);          // exclusive prefixes inside the ray
    if (ok) loss += (double)(interval * (1.f / 3.f) * wi * wi + 2.f * wi * (si * pw - pws));
    cw += __shfl_sync(0xffffffffu, iw, 31);
    cws += __shfl_sync(0xffffffffu, iws, 31);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
  if (lane == 0) ray_loss[ray] = loss;
  if (!grad_w) return;
  const float wt = cw, wst = cws;   // ray totals
  cw = 0.f; cws = 0.f;
  for (int64_t c = b; c < e; c += 32) {
    const int64_t i = c + lane;
    const bool ok = i < e;
    const float wi = ok ? w[i] : 0.f, si = ok ? s[i] : 0.f;
    const float ws = wi * si;
    const float iw = warp_incl_scan(wi, lane), iws = warp_incl_scan(ws, lane);
    const float pw = cw + (iw - wi), pws = cws + (iws - ws);
    const float aw = wt - (cw + iw), aws = wst - (cws + iws);         // strictly-after sums
    if (ok) grad_w[i] = inv_r * (interval * (2.f / 3.f) * wi + 2.f * (si * pw - pws) + 2.f * (aws - si * aw));
    cw += __shfl_sync(0xffffffffu, iw, 31);
    cws += __shfl_sync(0xffffffffu, iws, 31);
  }
}

__global__ void __launch_bounds__(256) k_distortion_finish(const double* __restrict__ ray_loss, int64_t n_rays,
                                                           const int64_t* __restrict__ last_id, float* __restrict__ out) {
  __shared__ double sh[256];
  const float inv_r = 1.f / (float)(*last_id + 1);
  double a = 0;
  for (int64_t r = threadIdx.x; r < n_rays; r += 256) a += ray_loss[r];   // fixed assignment -> deterministic
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = (float)(sh[0] * (double)inv_r);
}

}  // namespace ubn

extern "C" int ubn_distortion_loss(const float* w, const float* s, const int64_t* ray_id, int64_t n_pts, int64_t n_rays,
                                   float interval, int64_t* i_start, int64_t* i_end, float* out1, float* grad_w,
                                   double* scratch, int64_t scratch_len, void* stream) {
  using namespace ubn;
  cudaStream_t st = as_stream(stream);
  if (n_rays <= 0) return finish(cudaErrorInvalidValue);
  if (scratch_len < n_rays) return finish(cudaErrorInvalidValue);
  // segment bounds of the sorted ray_id (empty rays keep [0,0)); out1 doubles as k_init_rays' float slot when n_rays == 1
  float* dummy = reinterpret_cast<float*>(scratch);   // n_rays floats fit in n_rays doubles; overwritten below
  k_init_rays<<<blocks_for(n_rays, 256), 256, 0, st>>>(n_rays, dummy, i_start, i_end);
  UBN_LAUNCH_CHECK();
  if (n_pts > 0) {
    k_segment_bounds<<<blocks_for(n_pts, 256), 256, 0, st>>>(ray_id, n_pts, i_start, i_end);
    UBN_LAUNCH_CHECK();
  }
  if (n_pts <= 0) return finish(cudaErrorInvalidValue);
  const int64_t* last_id = ray_id + (n_pts - 1);      // read on the device: no host sync for R
  k_distortion_loss<<<blocks_for(n_rays, 4), 128, 0, st>>>(w, s, i_start, i_end, n_rays, interval, last_id, grad_w, scratch);
  UBN_LAUNCH_CHECK();
  k_distortion_finish<<<1, 256, 0, st>>>(scratch, n_rays, last_id, out1);
  UBN_LAUNCH_CHECK();
  return 0;
}
