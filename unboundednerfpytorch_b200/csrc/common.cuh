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

}  // namespace ubn

#define UBN_LAUNCH_CHECK()                 \
  do {                                     \
    int _e = ::ubn::after_launch();        \
    if (_e) return _e;                     \
  } while (0)
