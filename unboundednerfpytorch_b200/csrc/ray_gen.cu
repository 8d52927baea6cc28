// ray_gen.cu -- the step either side of the march (SURVEY.md 8f rank 2): camera rays of a view and the per-step
// batch gather, as single launches.
//
// Replaces FourierGrid/dvgo.py:492-555 (get_rays + ndc_rays + get_rays_of_a_view: ~20 torch kernels per view and a
// [H,W,3,3] intermediate) and the four index kernels of run_train.py:204-212 (target / rays_o / rays_d / viewdirs
// = *_tr[sel_i]).  Outputs only: 36 B written per pixel, nothing read but 21 scalars.
#include "ray_gen.cuh"

namespace ubn {

__global__ void __launch_bounds__(256) k_rays_of_a_view(ViewParams v, const float* __restrict__ jitter,
                                                        float* __restrict__ rays_o, float* __restrict__ rays_d,
                                                        float* __restrict__ viewdirs) {
  const int64_t n = (int64_t)v.H * v.W;
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int row = (int)(p / v.W), col = (int)(p - (int64_t)row * v.W);
  float ro[3], rd[3], vd[3];
  pixel_ray(v, row, col, jitter, ro, rd, vd);
  float* w = viewdirs + 3 * p;
  w[0] = vd[0]; w[1] = vd[1]; w[2] = vd[2];
  float* o = rays_o + 3 * p;
  float* d = rays_d + 3 * p;
  o[0] = ro[0]; o[1] = ro[1]; o[2] = ro[2];
  d[0] = rd[0]; d[1] = rd[1]; d[2] = rd[2];
}

// out_a[k] = src_a[idx[k]] for up to four [N,3] fp32 arrays in one launch; thread = (selected ray, array)
struct GatherArgs {
  const float* src[4];
  float* dst[4];
  int n_arrays;
};

__global__ void __launch_bounds__(256) k_gather_rays(GatherArgs a, const int64_t* __restrict__ idx, int64_t n_sel,
                                                     int64_t n_src, int* __restrict__ oob) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t k = t / a.n_arrays;
  const int w = (int)(t - k * a.n_arrays);
  if (k >= n_sel) return;
  int64_t s = idx[k];
  if (s < 0) s += n_src;                    // python-style negative index
  if (s < 0 || s >= n_src) { atomicExch(oob, 1); return; }
  const float* src = a.src[w] + 3 * s;
  float* dst = a.dst[w] + 3 * k;
  dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
}

}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_get_rays_of_a_view(int H, int W, const float* K_host, const float* c2w_host, int c2w_row_stride, int ndc,
                           int inverse_y, int flip_x, int flip_y, int mode, const float* jitter, float* rays_o,
                           float* rays_d, float* viewdirs, void* stream) {
  if (H <= 0 || W <= 0) return 0;
  if (mode < 0 || mode > 2 || (mode == 2 && jitter == nullptr)) return finish(cudaErrorInvalidValue);
  ViewParams v;
  v.fx = K_host[0]; v.cx = K_host[2]; v.fy = K_host[4]; v.cy = K_host[5];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) v.r[r][c] = c2w_host[r * c2w_row_stride + c];
    v.t[r] = c2w_host[r * c2w_row_stride + 3];
  }
  v.H = H; v.W = W; v.ndc = ndc; v.inverse_y = inverse_y; v.flip_x = flip_x; v.flip_y = flip_y;
  v.pix = mode == 1 ? 0.5f : 0.f;
  ndc_scales(H, W, v.fx, v.sw, v.sh);
  const int64_t n = (int64_t)H * W;
  k_rays_of_a_view<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(v, mode == 2 ? jitter : nullptr, rays_o, rays_d, viewdirs);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_gather_rays(const float* const* src, float* const* dst, int n_arrays, const int64_t* idx, int64_t n_sel,
                    int64_t n_src, int* oob_flag, void* stream) {
  if (n_sel <= 0 || n_arrays <= 0) return 0;
  if (n_arrays > 4) return finish(cudaErrorInvalidValue);
  GatherArgs a;
  a.n_arrays = n_arrays;
  for (int i = 0; i < 4; ++i) { a.src[i] = i < n_arrays ? src[i] : nullptr; a.dst[i] = i < n_arrays ? dst[i] : nullptr; }
  k_gather_rays<<<blocks_for(n_sel * n_arrays, 256), 256, 0, as_stream(stream)>>>(a, idx, n_sel, n_src, oob_flag);
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
