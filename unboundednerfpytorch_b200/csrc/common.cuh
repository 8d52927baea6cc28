// common.cuh -- shared helpers for libubnerf_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ubnerf_b200.h"

namespace ubn {

constexpr int kNumSMs = 132;  // H100 SXM

extern thread_local cudaError_t g_last_error;
void count_launch();

inline int finish(cudaError_t e) {
  if (e != cudaSuccess) g_last_error = e;
  return (int)e;
}

// Check the launch that was just enqueued (the reference never calls cudaGetLastError).
inline int after_launch() {
  count_launch();
  return finish(cudaGetLastError());
}

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

template <typename T>
__host__ __device__ __forceinline__ T ceil_div(T a, T b) { return (a + b - 1) / b; }

// grid size for a plain elementwise kernel: one thread per element, capped only by int range
inline unsigned blocks_for(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// torch.linspace(start, end, n)[i] as ATen's CUDA kernel evaluates it (RangeFactories.cu): step = (end - start) / (n - 1), then
// start + step * i below the midpoint and end - step * (n - 1 - i) from it on, both contracted to one fma by nvcc.  Shared by the
// lattice kernels of grid_utils.cu and bounds.cu.
__device__ __forceinline__ float linspace_at(float start, float end, int n, int i) {
  if (n <= 1) return start;
  const float step = __fdiv_rn(__fsub_rn(end, start), (float)(n - 1));
  return (i < n / 2) ? fmaf(step, (float)i, start) : fmaf(-step, (float)(n - i - 1), end);
}

// Raw2Alpha of one density (render_utils_kernel.cu:431-458): alpha = 1 - (1 + exp(d + shift))^-interval.  Shared by
// ubn_raw2alpha (alpha_ops.cu) and the coarse-geometry bounds (bounds.cu), so both produce the same bits.
__device__ __forceinline__ void raw2alpha_one(float d, float shift, float interval, float* e_out, float* a_out) {
  const float e = expf(d + shift);  // can be inf
  *e_out = e;
  *a_out = 1 - powf(1 + e, -interval);
}

// ---- shared-memory mbarriers (the TMA brick loads of render_tma.cu, the dW2 pipeline of shade_tc.cu) ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\t"
      "DONE_%=:\n\t}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}

// NDC sample i of n on a forward-facing ray (render_utils_kernel.cu:260-263): p = o + d * (i / (n - 1)), the step as an IEEE
// float division and each coordinate as one fma, the form nvcc gives the reference's `o + d * dist`.  Shared by
// ubn_sample_ndc_pts_on_rays and the fused NDC march, so both produce the same bits.
__device__ __forceinline__ void ndc_point(float ox, float oy, float oz, float dx, float dy, float dz, int i, int n,
                                          float& x, float& y, float& z) {
  const float dist = __fdiv_rn((float)i, (float)(n - 1));
  x = fmaf(dx, dist, ox);
  y = fmaf(dy, dist, oy);
  z = fmaf(dz, dist, oz);
}

// ---- bounded-scene sampling (render_utils_kernel.cu:12-79,167-194) -----------------------------------------------------------
// Shared by ubn_infer_* / ubn_sample_pts_* (ray_ops.cu) and the fused box march (BoxSampler, march_common.cuh), so both produce the
// same bits.  The expressions are kept as the reference writes them: nvcc's default fma contraction then lands on the same operations.
struct RayBox {
  float t_min, t_max;
};

__device__ __forceinline__ RayBox ray_aabb(const float* __restrict__ o, const float* __restrict__ d,
                                           const float* __restrict__ xyz_min,
                                           const float* __restrict__ xyz_max, float near, float far) {
  // zero direction components become 1e-6 (double literal narrowed to float), :23-25
  const float vx = (d[0] == 0) ? (float)1e-6 : d[0];
  const float vy = (d[1] == 0) ? (float)1e-6 : d[1];
  const float vz = (d[2] == 0) ? (float)1e-6 : d[2];
  const float ax = (xyz_max[0] - o[0]) / vx;
  const float ay = (xyz_max[1] - o[1]) / vy;
  const float az = (xyz_max[2] - o[2]) / vz;
  const float bx = (xyz_min[0] - o[0]) / vx;
  const float by = (xyz_min[1] - o[1]) / vy;
  const float bz = (xyz_min[2] - o[2]) / vz;
  RayBox r;
  r.t_min = fmaxf(fminf(fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fminf(az, bz)), far), near);
  r.t_max = fmaxf(fminf(fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fmaxf(az, bz)), far), near);
  return r;
}

__device__ __forceinline__ float ray_norm(const float* __restrict__ d) {
  return sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
}

__device__ __forceinline__ int64_t ray_n_samples(const float* __restrict__ d, float t_min, float t_max,
                                                 float stepdist) {
  const float rnorm = ray_norm(d);
  // max(ceil(float), 1.) is evaluated in double in the reference (:53)
  return (int64_t)fmax((double)ceilf((t_max - t_min) * rnorm / stepdist), 1.);
}

// rays_start = o + d * t_min and rays_dir = d / |d|, each rounded to float as K3 writes them to memory (:72-77)
__device__ __forceinline__ void ray_start_dir(const float* __restrict__ o, const float* __restrict__ d, float t_min, float* start,
                                              float* dir) {
  const float rnorm = ray_norm(d);
  start[0] = o[0] + d[0] * t_min;
  start[1] = o[1] + d[1] * t_min;
  start[2] = o[2] + d[2] * t_min;
  dir[0] = d[0] / rnorm;
  dir[1] = d[1] / rnorm;
  dir[2] = d[2] / rnorm;
}

// sample i of a bounded-scene ray: p = start + dir * (stepdist * i)   (:185-190)
__device__ __forceinline__ void box_point(const float* start, const float* dir, float stepdist, int i, float& x, float& y,
                                          float& z) {
  const float dist = stepdist * i;
  x = start[0] + dir[0] * dist;
  y = start[1] + dir[1] * dist;
  z = start[2] + dir[2] * dist;
}

// the reference's inclusive in-box test: a sample is dropped when (min > p) | (max < p) on any axis (:191-192)
__device__ __forceinline__ bool outside_box(const float* mn, const float* mx, float x, float y, float z) {
  return (mn[0] > x) | (mn[1] > y) | (mn[2] > z) | (mx[0] < x) | (mx[1] < y) | (mx[2] < z);
}

}  // namespace ubn

#define UBN_LAUNCH_CHECK()                 \
  do {                                     \
    int _e = ::ubn::after_launch();        \
    if (_e) return _e;                     \
  } while (0)
