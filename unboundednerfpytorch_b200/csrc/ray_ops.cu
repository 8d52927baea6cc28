// ray_ops.cu -- ray / AABB / sampling / mask-cache / cumdist kernels of libubnerf_b200.so.
//
// Replaces FourierGrid/cuda/render_utils_kernel.cu:12-424 and ub360_utils_kernel.cu:13-47 of the
// reference (K1-K9, K21 in SURVEY.md 2a).  Arithmetic is kept expression-for-expression compatible
// (same float/double promotions, same operand order so that nvcc's fma contraction lands on the same
// operations) because the integer / bool outputs (N_steps, ray_id, step_id, mask_outbbox, mask-cache
// hits, cumdist masks) are bit-exact parity targets against the reference's own CUDA build.
#include "common.cuh"

namespace ubn {

thread_local cudaError_t g_last_error = cudaSuccess;
static int64_t g_launches = 0;
void count_launch() { __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED); }

// ------------------------------------------------------------------------------------------------
// ray / AABB  (render_utils_kernel.cu:12-79): ray_aabb, ray_n_samples, ray_start_dir and box_point live in common.cuh, shared
// with the fused box march
// ------------------------------------------------------------------------------------------------
__global__ void k_infer_t_minmax(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                 const float* __restrict__ xyz_min, const float* __restrict__ xyz_max,
                                 float near, float far, int64_t n_rays, float* __restrict__ t_min,
                                 float* __restrict__ t_max) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  const RayBox b = ray_aabb(rays_o + 3 * r, rays_d + 3 * r, xyz_min, xyz_max, near, far);
  t_min[r] = b.t_min;
  t_max[r] = b.t_max;
}

__global__ void k_infer_n_samples(const float* __restrict__ rays_d, const float* __restrict__ t_min,
                                  const float* __restrict__ t_max, float stepdist, int64_t n_rays,
                                  int64_t* __restrict__ n_samples) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  n_samples[r] = ray_n_samples(rays_d + 3 * r, t_min[r], t_max[r], stepdist);
}

__global__ void k_infer_ray_start_dir(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                      const float* __restrict__ t_min, int64_t n_rays,
                                      float* __restrict__ rays_start, float* __restrict__ rays_dir) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  float start[3], dir[3];
  ray_start_dir(rays_o + 3 * r, rays_d + 3 * r, t_min[r], start, dir);
  for (int a = 0; a < 3; ++a) {
    rays_start[3 * r + a] = start[a];
    rays_dir[3 * r + a] = dir[a];
  }
}

// ------------------------------------------------------------------------------------------------
// exclusive scan (replaces the reference's two torch cumsum calls + 2 helper kernels, :144-164,211-219)
// three-phase: per-block (1024 elements) scan -> scan of block totals (one block) -> add back
// ------------------------------------------------------------------------------------------------
constexpr int kScanBlock = 1024;

__device__ __forceinline__ int64_t warp_incl_scan(int64_t v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += n;
  }
  return v;
}

// inclusive scan across a 1024-thread block; returns inclusive value, *total = block sum
__device__ __forceinline__ int64_t block_incl_scan(int64_t v, int64_t* total) {
  __shared__ int64_t warp_sums[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int64_t inc = warp_incl_scan(v);
  if (lane == 31) warp_sums[w] = inc;
  __syncthreads();
  if (w == 0) {
    int64_t s = warp_sums[lane];
    s = warp_incl_scan(s);
    warp_sums[lane] = s;
  }
  __syncthreads();
  if (w > 0) inc += warp_sums[w - 1];
  *total = warp_sums[31];
  __syncthreads();
  return inc;
}

template <typename T>
__global__ void __launch_bounds__(kScanBlock) k_scan_local(const T* __restrict__ in, int64_t n,
                                                           int64_t* __restrict__ offsets,
                                                           int64_t* __restrict__ block_tot) {
  const int64_t i = (int64_t)blockIdx.x * kScanBlock + threadIdx.x;
  const int64_t v = (i < n) ? (int64_t)in[i] : 0;
  int64_t tot;
  const int64_t inc = block_incl_scan(v, &tot);
  if (i < n) offsets[i] = inc - v;
  if (threadIdx.x == 0) block_tot[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kScanBlock) k_scan_block_totals(int64_t* __restrict__ block_tot,
                                                                  int64_t n_blocks) {
  // single block; sequential over tiles of 1024 block totals (n_blocks is tiny: n/1024)
  int64_t carry = 0;
  for (int64_t base = 0; base < n_blocks; base += kScanBlock) {
    const int64_t i = base + threadIdx.x;
    const int64_t v = (i < n_blocks) ? block_tot[i] : 0;
    int64_t tot;
    const int64_t inc = block_incl_scan(v, &tot);
    if (i < n_blocks) block_tot[i] = carry + inc - v;
    carry += tot;
  }
  if (threadIdx.x == 0) block_tot[n_blocks] = carry;  // grand total
}

__global__ void __launch_bounds__(kScanBlock) k_scan_add(int64_t* __restrict__ offsets, int64_t n,
                                                         const int64_t* __restrict__ block_tot,
                                                         int64_t n_blocks) {
  const int64_t i = (int64_t)blockIdx.x * kScanBlock + threadIdx.x;
  if (i < n) offsets[i] += block_tot[blockIdx.x];
  if (i == 0) offsets[n] = block_tot[n_blocks];
}

template <typename T>
static int exclusive_scan(const T* in, int64_t n, int64_t* offsets, int64_t* scratch, cudaStream_t st) {
  if (n <= 0) {
    return finish(cudaMemsetAsync(offsets, 0, sizeof(int64_t), st));
  }
  const int64_t nb = ceil_div<int64_t>(n, kScanBlock);
  k_scan_local<T><<<(unsigned)nb, kScanBlock, 0, st>>>(in, n, offsets, scratch);
  UBN_LAUNCH_CHECK();
  k_scan_block_totals<<<1, kScanBlock, 0, st>>>(scratch, nb);
  UBN_LAUNCH_CHECK();
  k_scan_add<<<(unsigned)nb, kScanBlock, 0, st>>>(offsets, n, scratch, nb);
  UBN_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// ragged sampling (render_utils_kernel.cu:167-242)
// ------------------------------------------------------------------------------------------------
__global__ void k_sample_count(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                               const float* __restrict__ xyz_min, const float* __restrict__ xyz_max,
                               float near, float far, float stepdist, int64_t n_rays,
                               float* __restrict__ t_min, float* __restrict__ t_max,
                               int64_t* __restrict__ n_steps) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  const RayBox b = ray_aabb(rays_o + 3 * r, rays_d + 3 * r, xyz_min, xyz_max, near, far);
  t_min[r] = b.t_min;
  t_max[r] = b.t_max;
  n_steps[r] = ray_n_samples(rays_d + 3 * r, b.t_min, b.t_max, stepdist);
}

__global__ void __launch_bounds__(256) k_sample_emit(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ xyz_min,
    const float* __restrict__ xyz_max, const float* __restrict__ t_min, const int64_t* __restrict__ offsets,
    float stepdist, int64_t n_rays, int64_t total_len, float* __restrict__ rays_pts,
    uint8_t* __restrict__ mask_outbbox, int64_t* __restrict__ ray_id, int64_t* __restrict__ step_id) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total_len) return;
  // upper_bound(offsets, idx) - 1 : the ray whose [offsets[r], offsets[r+1]) contains idx
  int64_t lo = 0, hi = n_rays;  // invariant: offsets[lo] <= idx < offsets[hi]
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (offsets[mid] <= idx) lo = mid; else hi = mid;
  }
  const int64_t r = lo;
  const int i_step = (int)(idx - offsets[r]);
  float start[3], dir[3], px, py, pz;
  ray_start_dir(rays_o + 3 * r, rays_d + 3 * r, t_min[r], start, dir);
  box_point(start, dir, stepdist, i_step, px, py, pz);
  rays_pts[3 * idx] = px;
  rays_pts[3 * idx + 1] = py;
  rays_pts[3 * idx + 2] = pz;
  mask_outbbox[idx] = outside_box(xyz_min, xyz_max, px, py, pz);
  ray_id[idx] = r;
  step_id[idx] = i_step;
}

__global__ void k_sample_ndc(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                             const float* __restrict__ xyz_min, const float* __restrict__ xyz_max,
                             int n_samples, int64_t n_rays, float* __restrict__ rays_pts,
                             uint8_t* __restrict__ mask_outbbox) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_rays * n_samples) return;
  const int64_t r = idx / n_samples;
  const int i_step = (int)(idx % n_samples);
  float px, py, pz;
  ndc_point(rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2], rays_d[3 * r], rays_d[3 * r + 1], rays_d[3 * r + 2], i_step,
            n_samples, px, py, pz);
  rays_pts[3 * idx] = px;
  rays_pts[3 * idx + 1] = py;
  rays_pts[3 * idx + 2] = pz;
  mask_outbbox[idx] = (xyz_min[0] > px) | (xyz_min[1] > py) | (xyz_min[2] > pz) |
                      (xyz_max[0] < px) | (xyz_max[1] < py) | (xyz_max[2] < pz);
}

__global__ void k_sample_bg(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                            const float* __restrict__ t_max, float bg_preserve, int n_samples,
                            int64_t n_rays, float* __restrict__ rays_pts) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_rays * n_samples) return;
  const int64_t r = idx / n_samples;
  const int i_step = (int)(idx % n_samples);
  const float t_inner = t_max[r];
  const float ori_t_outer = t_inner - 1. + 1. / (1. - ((float)i_step) / n_samples);
  const float x = rays_o[3 * r] + rays_d[3 * r] * ori_t_outer;
  const float y = rays_o[3 * r + 1] + rays_d[3 * r + 1] * ori_t_outer;
  const float z = rays_o[3 * r + 2] + rays_d[3 * r + 2] * ori_t_outer;
  const float t_outer = sqrtf(x * x + y * y + z * z);
  const float m = fmaxf(fabsf(x), fmaxf(fabsf(y), fabsf(z)));
  const float R_outer = t_outer / m;
  const float o2i_p = R_outer * R_outer / (t_outer * t_outer) * (1. - bg_preserve) + R_outer / t_outer * bg_preserve;
  rays_pts[3 * idx] = x * o2i_p;
  rays_pts[3 * idx + 1] = y * o2i_p;
  rays_pts[3 * idx + 2] = z * o2i_p;
}

// ------------------------------------------------------------------------------------------------
// mask-cache lookup (render_utils_kernel.cu:367-392)
// ------------------------------------------------------------------------------------------------
__global__ void k_maskcache_lookup(const uint8_t* __restrict__ world, const float* __restrict__ xyz,
                                   const float* __restrict__ scale, const float* __restrict__ shift,
                                   int sz_i, int sz_j, int sz_k, int64_t n_pts, uint8_t* __restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pts) return;
  // round(): half away from zero on the (fma-contracted) float, then int conversion (:385-387)
  const int i = roundf(xyz[3 * p] * scale[0] + shift[0]);
  const int j = roundf(xyz[3 * p + 1] * scale[1] + shift[1]);
  const int k = roundf(xyz[3 * p + 2] * scale[2] + shift[2]);
  uint8_t v = 0;
  if (0 <= i && i < sz_i && 0 <= j && j < sz_j && 0 <= k && k < sz_k)
    v = world[(int64_t)i * sz_j * sz_k + (int64_t)j * sz_k + k];
  out[p] = v;
}

// ------------------------------------------------------------------------------------------------
// cumdist_thres (ub360_utils_kernel.cu:13-32): order-sensitive sequential accumulate-and-reset per ray.
// One lane owns one ray (exact sequential semantics); a warp owns 32 rays and stages 32x32 tiles through
// shared memory so that every global access is a coalesced 128-byte row instead of a stride-S walk.
// ------------------------------------------------------------------------------------------------
constexpr int kTileWarps = 4;

__global__ void __launch_bounds__(32 * kTileWarps) k_cumdist_thres(const float* __restrict__ dist, float thres,
                                                                   int64_t n_rays, int64_t n_pts,
                                                                   uint8_t* __restrict__ mask) {
  __shared__ float s_d[kTileWarps][32][33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t ray0 = ((int64_t)blockIdx.x * kTileWarps + w) * 32;
  if (ray0 >= n_rays) return;
  float cum = 0.f;
  for (int64_t base = 0; base < n_pts; base += 32) {
    // coalesced tile load: row rr = ray ray0+rr, column = lane
#pragma unroll 4
    for (int rr = 0; rr < 32; ++rr) {
      const int64_t r = ray0 + rr, c = base + lane;
      if (r < n_rays && c < n_pts) s_d[w][rr][lane] = dist[r * n_pts + c];
    }
    __syncwarp();
    const int ncol = (int)min((int64_t)32, n_pts - base);
    if (ray0 + lane < n_rays) {
      for (int j = 0; j < ncol; ++j) {
        cum += s_d[w][lane][j];
        const bool over = (cum > thres);
        cum *= float(!over);
        s_d[w][lane][j] = over ? 1.f : 0.f;
      }
    }
    __syncwarp();
#pragma unroll 4
    for (int rr = 0; rr < 32; ++rr) {
      const int64_t r = ray0 + rr, c = base + lane;
      if (r < n_rays && c < n_pts) mask[r * n_pts + c] = (s_d[w][rr][lane] != 0.f);
    }
    __syncwarp();
  }
}

}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_abi_version(void) { return UBN_ABI_VERSION; }
const char* ubn_last_error_string(void) { return cudaGetErrorString(ubn::g_last_error); }
int64_t ubn_launch_count(void) { return __atomic_load_n(&ubn::g_launches, __ATOMIC_RELAXED); }
void ubn_reset_launch_count(void) { __atomic_store_n(&ubn::g_launches, 0, __ATOMIC_RELAXED); }

int ubn_infer_t_minmax(const float* rays_o, const float* rays_d, const float* xyz_min, const float* xyz_max,
                       float near, float far, int64_t n_rays, float* t_min, float* t_max, void* stream) {
  if (n_rays <= 0) return 0;
  k_infer_t_minmax<<<blocks_for(n_rays, 128), 128, 0, as_stream(stream)>>>(rays_o, rays_d, xyz_min, xyz_max,
                                                                          near, far, n_rays, t_min, t_max);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_infer_n_samples(const float* rays_d, const float* t_min, const float* t_max, float stepdist,
                        int64_t n_rays, int64_t* n_samples, void* stream) {
  if (n_rays <= 0) return 0;
  k_infer_n_samples<<<blocks_for(n_rays, 128), 128, 0, as_stream(stream)>>>(rays_d, t_min, t_max, stepdist,
                                                                           n_rays, n_samples);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_infer_ray_start_dir(const float* rays_o, const float* rays_d, const float* t_min, int64_t n_rays,
                            float* rays_start, float* rays_dir, void* stream) {
  if (n_rays <= 0) return 0;
  k_infer_ray_start_dir<<<blocks_for(n_rays, 128), 128, 0, as_stream(stream)>>>(rays_o, rays_d, t_min, n_rays,
                                                                               rays_start, rays_dir);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_sample_pts_count(const float* rays_o, const float* rays_d, const float* xyz_min, const float* xyz_max,
                         float near, float far, float stepdist, int64_t n_rays, float* t_min, float* t_max,
                         int64_t* n_steps, int64_t* offsets, int64_t* scan_scratch, void* stream) {
  cudaStream_t st = as_stream(stream);
  if (n_rays > 0) {
    k_sample_count<<<blocks_for(n_rays, 128), 128, 0, st>>>(rays_o, rays_d, xyz_min, xyz_max, near, far,
                                                           stepdist, n_rays, t_min, t_max, n_steps);
    UBN_LAUNCH_CHECK();
  }
  return exclusive_scan<int64_t>(n_steps, n_rays, offsets, scan_scratch, st);
}

int ubn_sample_pts_emit(const float* rays_o, const float* rays_d, const float* xyz_min, const float* xyz_max,
                        const float* t_min, const int64_t* offsets, float stepdist, int64_t n_rays,
                        int64_t total_len, float* rays_pts, uint8_t* mask_outbbox, int64_t* ray_id,
                        int64_t* step_id, void* stream) {
  if (total_len <= 0) return 0;
  k_sample_emit<<<blocks_for(total_len, 256), 256, 0, as_stream(stream)>>>(
      rays_o, rays_d, xyz_min, xyz_max, t_min, offsets, stepdist, n_rays, total_len, rays_pts, mask_outbbox,
      ray_id, step_id);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_sample_ndc_pts_on_rays(const float* rays_o, const float* rays_d, const float* xyz_min,
                               const float* xyz_max, int64_t n_samples, int64_t n_rays, float* rays_pts,
                               uint8_t* mask_outbbox, void* stream) {
  const int64_t n = n_rays * n_samples;
  if (n <= 0) return 0;
  k_sample_ndc<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(rays_o, rays_d, xyz_min, xyz_max,
                                                                 (int)n_samples, n_rays, rays_pts, mask_outbbox);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_sample_bg_pts_on_rays(const float* rays_o, const float* rays_d, const float* t_max, float bg_preserve,
                              int64_t n_samples, int64_t n_rays, float* rays_pts, void* stream) {
  const int64_t n = n_rays * n_samples;
  if (n <= 0) return 0;
  k_sample_bg<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(rays_o, rays_d, t_max, bg_preserve,
                                                                (int)n_samples, n_rays, rays_pts);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_maskcache_lookup(const uint8_t* world, const float* xyz, const float* xyz2ijk_scale,
                         const float* xyz2ijk_shift, int64_t sz_i, int64_t sz_j, int64_t sz_k, int64_t n_pts,
                         uint8_t* out, void* stream) {
  if (n_pts <= 0) return 0;
  k_maskcache_lookup<<<blocks_for(n_pts, 256), 256, 0, as_stream(stream)>>>(
      world, xyz, xyz2ijk_scale, xyz2ijk_shift, (int)sz_i, (int)sz_j, (int)sz_k, n_pts, out);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_cumdist_thres(const float* dist, float thres, int64_t n_rays, int64_t n_pts, uint8_t* mask,
                      void* stream) {
  if (n_rays <= 0 || n_pts <= 0) return 0;
  const int64_t rays_per_block = 32 * kTileWarps;
  k_cumdist_thres<<<blocks_for(n_rays, (int)rays_per_block), 32 * kTileWarps, 0, as_stream(stream)>>>(
      dist, thres, n_rays, n_pts, mask);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_exclusive_scan_i32(const int32_t* in, int64_t n, int64_t* offsets, int64_t* scratch, void* stream) {
  return exclusive_scan<int32_t>(in, n, offsets, scratch, as_stream(stream));
}

}  // extern "C"
