// loss.cu -- the training losses of run_train.py:253-279 and their gradients in two launches
// (SURVEY.md 8f rank 1, "in-kernel losses"):
//   loss = w_main * mse + w_freq * freq + w_entropy * entropy_last + w_nearclip * nearclip + w_rgbper * rgbper
//   mse      = mean_{r,c} (rgb_marched - target)^2                                     F.mse_loss, :254
//   freq     = FourierMSELoss (FourierGrid_model.py:114-130): mse of the REAL part of the length-3 FFT over the colour
//              axis; for d = rgb_marched - target the real parts are X0 = d0+d1+d2 and X1 = X2 = d0 - (d1+d2)/2, so
//              freq = mean_r (X0^2 + 2 X1^2) / 3                                        :255-257 (weight_freq)
//   entropy  = mean_r  -(p log p + (1-p) log(1-p)),  p = clamp(alphainv_last, 1e-6, 1-1e-6)   :258-261
//   nearclip = sum_{m: t_m < near_thres} (density_m - density_m.detach())               :262-268: value 0, d/d density = 1
//   rgbper   = sum_m weights_m * sum_c (raw_rgb_m - target[ray_id_m])^2 / n_rays        :275-278 (weights detached)
// (the distortion term, :269-274, is its own warp-per-ray kernel: ubn_distortion_loss in alpha_ops.cu)
// The reference spends ~25 torch kernels on this (gather target[ray_id] -> 50 MB, sub, pow, sum, mul, sum, clamp, logs,
// means, and their autograd mirrors).  Here one grid-stride kernel reads every operand once, writes the three
// gradients and per-block partial sums (double), and a one-block kernel adds the partials in a fixed order, so the
// loss value is deterministic.
#include "common.cuh"

namespace ubn {

constexpr int kLossBlocks = 592;      // 4 per SM
constexpr int kLossThreads = 256;

__device__ __forceinline__ double block_sum(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) sh[w] = v;
  __syncthreads();
  double t = 0;
  if (threadIdx.x == 0)
    for (int i = 0; i < kLossThreads / 32; ++i) t += sh[i];
  return t;   // valid in thread 0
}

__global__ void __launch_bounds__(kLossThreads) k_render_loss(
    const float* __restrict__ rgb_marched, const float* __restrict__ alphainv_last, const float* __restrict__ raw_rgb,
    const float* __restrict__ weights, const int64_t* __restrict__ ray_id, const float* __restrict__ target,
    const float* __restrict__ t_pts, int64_t n_rays, int64_t n_pts, float w_main, float w_entropy, float w_rgbper, float w_freq,
    float w_nearclip, float near_thres, float* __restrict__ g_rgb_marched, float* __restrict__ g_alphainv,
    float* __restrict__ g_raw_rgb, float* __restrict__ g_raw_density, double* __restrict__ partial) {
  __shared__ double sh[kLossThreads / 32];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double s_mse = 0, s_ent = 0, s_per = 0, s_frq = 0;
  const float inv_n = 1.f / (float)n_rays;
  const float g_mse = w_main * 2.f / (3.f * (float)n_rays);
  const float g_frq = w_freq * 2.f / (3.f * (float)n_rays);
  for (int64_t r = t0; r < n_rays; r += stride) {
    float d[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      d[c] = rgb_marched[3 * r + c] - target[3 * r + c];
      s_mse += (double)(d[c] * d[c]);
    }
    // real part of the 3-point DFT of d: X0 = sum, X1 = X2 = d0 - (d1 + d2) / 2; d/dd0 = 2 X0 + 4 X1, d/dd1 = d/dd2 = 2 X0 - 2 X1
    const float x0 = d[0] + d[1] + d[2], x1 = d[0] - 0.5f * (d[1] + d[2]);
    if (w_freq != 0.f) s_frq += (double)(x0 * x0 + 2.f * x1 * x1);
    if (g_rgb_marched) {
      g_rgb_marched[3 * r] = g_mse * d[0] + g_frq * (x0 + 2.f * x1);
      g_rgb_marched[3 * r + 1] = g_mse * d[1] + g_frq * (x0 - x1);
      g_rgb_marched[3 * r + 2] = g_mse * d[2] + g_frq * (x0 - x1);
    }
    if (alphainv_last) {
      const float a = alphainv_last[r];
      // torch's clamp propagates NaN (fmaxf / fminf would turn it into a bound): a NaN alphainv_last makes the term NaN
      const float p = isnan(a) ? a : fminf(fmaxf(a, 1e-6f), 1.f - 1e-6f);
      const float lp = logf(p), lq = logf(1.f - p);
      s_ent += (double)(-(p * lp + (1.f - p) * lq));
      // d/dp = -(log p - log(1-p)); clamp passes the gradient on [min, max] inclusive
      if (g_alphainv) g_alphainv[r] = (a >= 1e-6f && a <= 1.f - 1e-6f) ? w_entropy * inv_n * (lq - lp) : 0.f;
    }
  }
  if (raw_rgb) {
    const float g_per = w_rgbper * 2.f * inv_n;
    for (int64_t m = t0; m < n_pts; m += stride) {
      const int64_t r = ray_id[m];
      const float w = weights[m];
      float per = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float d = raw_rgb[3 * m + c] - target[3 * r + c];
        per = fmaf(d, d, per);
        if (g_raw_rgb) g_raw_rgb[3 * m + c] = g_per * w * d;
      }
      s_per += (double)(per * w);
    }
  }
  if (g_raw_density)     // nearclip: the loss value is identically 0, its gradient is w_nearclip on the samples closer than near_thres
    for (int64_t m = t0; m < n_pts; m += stride) g_raw_density[m] = (t_pts[m] < near_thres) ? w_nearclip : 0.f;
  const double a = block_sum(s_mse, sh);
  const double b = block_sum(s_ent, sh);
  const double c = block_sum(s_per, sh);
  const double e = block_sum(s_frq, sh);
  if (threadIdx.x == 0) {
    partial[4 * blockIdx.x] = a;
    partial[4 * blockIdx.x + 1] = b;
    partial[4 * blockIdx.x + 2] = c;
    partial[4 * blockIdx.x + 3] = e;
  }
}

__global__ void k_render_loss_finish(const double* __restrict__ partial, int n_blocks, int64_t n_rays, float w_main,
                                     float w_entropy, float w_rgbper, float w_freq, float* __restrict__ out) {
  // one warp, fixed order (lane-strided partial sums, then a fixed shuffle tree): deterministic like the single-thread loop it
  // replaces, whose 592 dependent loads made it one long serial chain
  if (blockIdx.x != 0 || threadIdx.x >= 32) return;
  double a = 0, b = 0, c = 0, e = 0;
  for (int i = threadIdx.x; i < n_blocks; i += 32) { a += partial[4 * i]; b += partial[4 * i + 1]; c += partial[4 * i + 2]; e += partial[4 * i + 3]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_down_sync(0xffffffffu, a, o); b += __shfl_down_sync(0xffffffffu, b, o);
    c += __shfl_down_sync(0xffffffffu, c, o); e += __shfl_down_sync(0xffffffffu, e, o);
  }
  if (threadIdx.x != 0) return;
  const float mse = (float)(a / (3.0 * (double)n_rays));
  const float ent = (float)(b / (double)n_rays);
  const float per = (float)(c / (double)n_rays);
  const float frq = (float)(e / (3.0 * (double)n_rays));
  out[0] = w_main * mse + w_entropy * ent + w_rgbper * per + w_freq * frq;
  out[1] = mse; out[2] = ent; out[3] = per; out[4] = frq;
}

}  // namespace ubn

using namespace ubn;

extern "C" int ubn_render_loss(const float* rgb_marched, const float* alphainv_last, const float* raw_rgb,
                               const float* weights, const int64_t* ray_id, const float* target, const float* t_pts,
                               int64_t n_rays, int64_t n_pts, float w_main, float w_entropy, float w_rgbper, float w_freq,
                               float w_nearclip, float near_thres, float* out5, float* grad_rgb_marched,
                               float* grad_alphainv_last, float* grad_raw_rgb, float* grad_raw_density, double* scratch,
                               int64_t scratch_len, void* stream) {
  if (n_rays <= 0) return finish(cudaErrorInvalidValue);
  if (scratch_len < 4 * kLossBlocks) return finish(cudaErrorInvalidValue);
  cudaStream_t st = as_stream(stream);
  const bool ent = alphainv_last != nullptr && w_entropy != 0.f;
  const bool per = raw_rgb != nullptr && w_rgbper != 0.f && n_pts > 0;
  const bool clip = t_pts != nullptr && grad_raw_density != nullptr && w_nearclip != 0.f && n_pts > 0;
  k_render_loss<<<kLossBlocks, kLossThreads, 0, st>>>(rgb_marched, ent ? alphainv_last : nullptr, per ? raw_rgb : nullptr, weights,
                                                     ray_id, target, t_pts, n_rays, n_pts, w_main, w_entropy, w_rgbper, w_freq,
                                                     w_nearclip, near_thres, grad_rgb_marched, ent ? grad_alphainv_last : nullptr,
                                                     per ? grad_raw_rgb : nullptr, clip ? grad_raw_density : nullptr, scratch);
  UBN_LAUNCH_CHECK();
  k_render_loss_finish<<<1, 32, 0, st>>>(scratch, kLossBlocks, n_rays, w_main, ent ? w_entropy : 0.f, per ? w_rgbper : 0.f, w_freq,
                                         out5);
  UBN_LAUNCH_CHECK();
  return 0;
}

