// grid_utils.cu -- grid-native kernels for the occupancy / progressive-growing utilities (SURVEY.md 8a row a13, 8f rank 3):
//   update_occupancy_cache   FourierGrid_model.py:441-456, dcvgo.py:214-226   -> ubn_lattice_alpha + ubn_maxpool3_gt_and
//   scale_volume_grid        grid.py:63-68, FourierGrid_grid.py:80-85         -> ubn_resample_grid (F.interpolate trilinear, align_corners)
//   voxel_count_views        FourierGrid_model.py:390-420, dvgo.py:238-277    -> ubn_view_scatter_ones + ubn_count_gt
//   update_occupancy_cache_lt_nviews  dcvgo.py:195-213                         -> ubn_view_scatter_ones_contracted + ubn_count_gt
//   maskout_near_cam_vox     FourierGrid_model.py:375-388, dvgo.py:185-196    -> ubn_maskout_near_cam
// The reference runs them as whole-grid torch compositions: a [X,Y,Z,3] meshgrid (100-400 MB at 256^3-320^3), a grid_sample over it,
// an activation, a max_pool3d and a boolean AND for the occupancy update; a [N,S,3] point tensor plus a full autograd backward
// per 10 000 rays for the view count.  Here every utility is one or two kernels that generate lattice / sample coordinates in
// registers.  Lattice coordinates follow torch.linspace's CUDA kernel (start + step * i below the midpoint, end - step * (n-1-i)
// above; both FMA-contracted by nvcc; linspace_at, common.cuh) so that threshold decisions agree with the reference's tensors.
#include <algorithm>

#include "march_common.cuh"

namespace ubn {

// alpha = Raw2Alpha(density(lattice point)) on an [mX, mY, mZ] lattice spanning [lo, hi] inclusive
__global__ void __launch_bounds__(256) k_lattice_alpha(GridView g, float lox, float loy, float loz, float hix, float hiy, float hiz,
                                                       int mX, int mY, int mZ, float shift, float interval, float* __restrict__ alpha) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n = (int64_t)mX * mY * mZ;
  if (idx >= n) return;
  const int k = (int)(idx % mZ), j = (int)((idx / mZ) % mY), i = (int)(idx / ((int64_t)mZ * mY));
  const float x = linspace_at(lox, hix, mX, i), y = linspace_at(loy, hiy, mY, j), z = linspace_at(loz, hiz, mZ, k);
  const float d = grid_density_at(g, x, y, z);
  const float e = expf(d + shift);                       // render_utils_kernel.cu:439-441
  alpha[idx] = 1 - powf(1 + e, -interval);
}

// mask &= max_pool3d(alpha, 3, stride 1, padding 1) > thres     (F.max_pool3d pads with -inf)
// The window maximum is ATen's: `v > m || isnan(v)` takes v, so a NaN in the window pools to NaN, NaN > thres is false and the
// cell is cleared (fmaxf would drop the NaN and keep the cell).
__global__ void __launch_bounds__(256) k_maxpool3_gt_and(const float* __restrict__ alpha, int X, int Y, int Z, float thres,
                                                         uint8_t* __restrict__ mask) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n = (int64_t)X * Y * Z;
  if (idx >= n) return;
  if (!mask[idx]) return;                                // AND with false stays false
  const int k = (int)(idx % Z), j = (int)((idx / Z) % Y), i = (int)(idx / ((int64_t)Z * Y));
  float m = -INFINITY;
  for (int a = max(i - 1, 0); a <= min(i + 1, X - 1); ++a)
    for (int b = max(j - 1, 0); b <= min(j + 1, Y - 1); ++b)
      for (int c = max(k - 1, 0); c <= min(k + 1, Z - 1); ++c) {
        const float v = alpha[((int64_t)a * Y + b) * Z + c];
        if (v > m || isnan(v)) m = v;
      }
  mask[idx] = (m > thres) ? 1 : 0;
}

// F.interpolate(mode='trilinear', align_corners=True) as ATen's upsample_trilinear3d evaluates it (UpSampleTrilinear3d.cu):
// scale = (in - 1) / (out - 1); src = scale * dst; i0 = (int)src; lambda1 = src - i0; lambda0 = 1 - lambda1; nested blend.
struct Resample {
  int P, C, iX, iY, iZ, oX, oY, oZ;
  int64_t isp, isc, isv, osp, osc, osv;   // strides (elements) of slab, channel, voxel: input / output
};

__device__ __forceinline__ void resample_axis(int out_i, int in_size, int out_size, int& i0, int& step1, float& l0, float& l1) {
  const float scale = out_size > 1 ? __fdiv_rn((float)(in_size - 1), (float)(out_size - 1)) : 0.f;
  const float src = __fmul_rn(scale, (float)out_i);
  i0 = (int)src;
  step1 = (i0 < in_size - 1) ? 1 : 0;
  l1 = __fsub_rn(src, (float)i0);
  l0 = __fsub_rn(1.f, l1);
}

__global__ void __launch_bounds__(256) k_resample_grid(const float* __restrict__ in, float* __restrict__ out, Resample r) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n = (int64_t)r.P * r.C * r.oX * r.oY * r.oZ;
  if (idx >= n) return;
  // channel fastest so that channels-last reads / writes coalesce (contiguous grids: C == 1 or a strided walk, rare)
  int64_t t = idx;
  const int c = (int)(t % r.C); t /= r.C;
  const int z = (int)(t % r.oZ); t /= r.oZ;
  const int y = (int)(t % r.oY); t /= r.oY;
  const int x = (int)(t % r.oX);
  const int p = (int)(t / r.oX);
  int x0, xs, y0, ys, z0, zs;
  float t0, t1, h0, h1, w0, w1;
  resample_axis(x, r.iX, r.oX, x0, xs, t0, t1);
  resample_axis(y, r.iY, r.oY, y0, ys, h0, h1);
  resample_axis(z, r.iZ, r.oZ, z0, zs, w0, w1);
  const float* base = in + p * r.isp + c * r.isc;
  auto at = [&](int a, int b, int d) { return __ldg(base + (((int64_t)a * r.iY + b) * r.iZ + d) * r.isv); };
  const float v = t0 * (h0 * (w0 * at(x0, y0, z0) + w1 * at(x0, y0, z0 + zs)) + h1 * (w0 * at(x0, y0 + ys, z0) + w1 * at(x0, y0 + ys, z0 + zs))) +
                  t1 * (h0 * (w0 * at(x0 + xs, y0, z0) + w1 * at(x0 + xs, y0, z0 + zs)) +
                        h1 * (w0 * at(x0 + xs, y0 + ys, z0) + w1 * at(x0 + xs, y0 + ys, z0 + zs)));
  out[p * r.osp + c * r.osc + (((int64_t)x * r.oY + y) * r.oZ + z) * r.osv] = v;
}

// voxel_count_views inner loop: for every (ray, sample) scatter the trilinear weights of a unit gradient into `grad` (the adjoint
// of DenseGrid(1, ...)(rays_pts).sum()), sample positions generated as FourierGrid_model.py:408-415 does with torch ops:
//   vec = d == 0 ? 1e-6 : d;  t_min = clamp(max_axis(min((hi - o) / vec, (lo - o) / vec)), near, far)
//   pts = o + d * (t_min + (step * i) / ||d||)
__global__ void __launch_bounds__(256) k_view_scatter_ones(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                           int64_t n_rays, int n_samples, float near, float far, float step,
                                                           GridView g, float hix, float hiy, float hiz, float* __restrict__ grad) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_rays * n_samples) return;
  const int64_t ray = idx / n_samples;
  const int s = (int)(idx - ray * n_samples);
  const float ox = rays_o[3 * ray], oy = rays_o[3 * ray + 1], oz = rays_o[3 * ray + 2];
  const float dx = rays_d[3 * ray], dy = rays_d[3 * ray + 1], dz = rays_d[3 * ray + 2];
  const float vx = dx == 0.f ? 1e-6f : dx, vy = dy == 0.f ? 1e-6f : dy, vz = dz == 0.f ? 1e-6f : dz;
  const float ax = __fdiv_rn(__fsub_rn(hix, ox), vx), bx = __fdiv_rn(__fsub_rn(g.mn[0], ox), vx);
  const float ay = __fdiv_rn(__fsub_rn(hiy, oy), vy), by = __fdiv_rn(__fsub_rn(g.mn[1], oy), vy);
  const float az = __fdiv_rn(__fsub_rn(hiz, oz), vz), bz = __fdiv_rn(__fsub_rn(g.mn[2], oz), vz);
  float t_min = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fminf(az, bz));
  t_min = fminf(fmaxf(t_min, near), far);
  const float nrm = norm3_torch(dx, dy, dz);
  const float t = __fadd_rn(t_min, __fdiv_rn(__fmul_rn(step, (float)s), nrm));
  const float x = __fadd_rn(ox, __fmul_rn(dx, t)), y = __fadd_rn(oy, __fmul_rn(dy, t)), z = __fadd_rn(oz, __fmul_rn(dz, t));
  const float cx = src_index_guarded(norm_coord(x, g.mn[0], g.len[0]), g.X);
  const float cy = src_index_guarded(norm_coord(y, g.mn[1], g.len[1]), g.Y);
  const float cz = src_index_guarded(norm_coord(z, g.mn[2], g.len[2]), g.Z);
  trilerp1_scatter(grad, 1, g.X, g.Y, g.Z, cx, cy, cz, 1.f);
}

// update_occupancy_cache_lt_nviews inner loop (dcvgo.py:195-213): the same adjoint of a ones grid over the contracted samples.
// Sample s of a ray is the point the fused march and _ContractedBase._sample_dense generate (load_ray + sample_point at
// t_table[s]), bit for bit, so every addend equals the one grid_sample's backward adds for sample_ray's point tensor.  All
// n_rays * S samples count: the reference scatters the full tensor, with no inner-mask, cumdist or mask-cache filter.
__global__ void __launch_bounds__(256) k_view_scatter_ones_contracted(const float* __restrict__ rays_o,
                                                                      const float* __restrict__ rays_d, int64_t n_rays,
                                                                      const float* __restrict__ t_table, MarchParams p, GridView g,
                                                                      float* __restrict__ grad) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_rays * p.S) return;
  const int64_t ray = idx / p.S;
  const int s = (int)(idx - ray * p.S);
  const Ray r = load_ray(rays_o + 3 * ray, rays_d + 3 * ray, p);
  float x, y, z;
  sample_point(r, __ldg(t_table + s), p, x, y, z);
  const float cx = src_index(norm_coord(x, g.mn[0], g.len[0]), g.X);
  const float cy = src_index(norm_coord(y, g.mn[1], g.len[1]), g.Y);
  const float cz = src_index(norm_coord(z, g.mn[2], g.len[2]), g.Z);
  trilerp1_scatter_pairs(grad, g.X, g.Y, g.Z, cx, cy, cz, 1.f);
}

__global__ void __launch_bounds__(256) k_count_gt(const float* __restrict__ grad, float thres, int64_t n, float* __restrict__ count) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && grad[i] > thres) count[i] += 1.f;
}

// maskout_near_cam_vox: grid[idx] = fill where the nearest camera is within near_clip of the lattice point linspace(lo, hi, size)
// per axis -- [-1, 1] in a FourierGrid slab's embedded coordinates, [xyz_min, xyz_max] for DVGO's world lattice -- distances as
// torch evaluates (g - c).pow(2).sum(-1).sqrt() on 3-vectors
__global__ void __launch_bounds__(256) k_maskout_near_cam(float* __restrict__ slab, int64_t sv, int X, int Y, int Z, float lox,
                                                          float loy, float loz, float hix, float hiy, float hiz,
                                                          const float* __restrict__ cams, int n_cams, float near_clip, float fill) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n = (int64_t)X * Y * Z;
  if (idx >= n) return;
  const int k = (int)(idx % Z), j = (int)((idx / Z) % Y), i = (int)(idx / ((int64_t)Z * Y));
  const float gx = linspace_at(lox, hix, X, i), gy = linspace_at(loy, hiy, Y, j), gz = linspace_at(loz, hiz, Z, k);
  float best = INFINITY;
  for (int c = 0; c < n_cams; ++c) {
    const float ex = __fsub_rn(gx, cams[3 * c]), ey = __fsub_rn(gy, cams[3 * c + 1]), ez = __fsub_rn(gz, cams[3 * c + 2]);
    best = fminf(best, norm3_torch(ex, ey, ez));
  }
  if (best <= near_clip) slab[idx * sv] = fill;
}

}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_lattice_alpha(const float* grid, const UbnGridDesc* desc, const float* lattice_min, const float* lattice_max, int64_t mX,
                      int64_t mY, int64_t mZ, float act_shift, float interval, float* alpha, void* stream) {
  const int64_t n = mX * mY * mZ;
  if (n <= 0) return 0;
  const GridView g = make_view(grid, desc);
  k_lattice_alpha<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(g, lattice_min[0], lattice_min[1], lattice_min[2], lattice_max[0],
                                                                     lattice_max[1], lattice_max[2], (int)mX, (int)mY, (int)mZ,
                                                                     act_shift, interval, alpha);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_maxpool3_gt_and(const float* alpha, int64_t X, int64_t Y, int64_t Z, float thres, uint8_t* mask, void* stream) {
  const int64_t n = X * Y * Z;
  if (n <= 0) return 0;
  k_maxpool3_gt_and<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(alpha, (int)X, (int)Y, (int)Z, thres, mask);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_resample_grid(const float* in, const UbnGridDesc* in_desc, float* out, const UbnGridDesc* out_desc, void* stream) {
  if (in_desc->P != out_desc->P || in_desc->C != out_desc->C) return finish(cudaErrorInvalidValue);
  Resample r;
  r.P = in_desc->P; r.C = in_desc->C;
  r.iX = in_desc->X; r.iY = in_desc->Y; r.iZ = in_desc->Z;
  r.oX = out_desc->X; r.oY = out_desc->Y; r.oZ = out_desc->Z;
  r.isp = in_desc->stride_p; r.isc = in_desc->stride_c; r.isv = in_desc->stride_v;
  r.osp = out_desc->stride_p; r.osc = out_desc->stride_c; r.osv = out_desc->stride_v;
  const int64_t n = (int64_t)r.P * r.C * r.oX * r.oY * r.oZ;
  if (n <= 0) return 0;
  k_resample_grid<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(in, out, r);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_view_scatter_ones(const float* rays_o, const float* rays_d, int64_t n_rays, int64_t n_samples, float near, float far,
                          float step, const UbnGridDesc* desc, float* grad, void* stream) {
  if (n_rays <= 0 || n_samples <= 0) return 0;
  if (desc->P != 1 || desc->C != 1) return finish(cudaErrorInvalidValue);
  const GridView g = make_view(nullptr, desc);
  k_view_scatter_ones<<<blocks_for(n_rays * n_samples, 256), 256, 0, as_stream(stream)>>>(
      rays_o, rays_d, n_rays, (int)n_samples, near, far, step, g, desc->xyz_max[0], desc->xyz_max[1], desc->xyz_max[2], grad);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_view_scatter_ones_contracted(const float* rays_o, const float* rays_d, int64_t n_rays, const float* t_table,
                                     const UbnMarchCfg* cfg, const UbnGridDesc* desc, float* grad, void* stream) {
  if (n_rays <= 0 || cfg->n_samples <= 0) return 0;
  if (desc->P != 1 || desc->C != 1 || desc->stride_v != 1) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_params(cfg);
  const GridView g = make_view(nullptr, desc);
  k_view_scatter_ones_contracted<<<blocks_for(n_rays * cfg->n_samples, 256), 256, 0, as_stream(stream)>>>(rays_o, rays_d, n_rays,
                                                                                                          t_table, p, g, grad);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_count_gt(const float* grad, float thres, int64_t n, float* count, void* stream) {
  if (n <= 0) return 0;
  k_count_gt<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(grad, thres, n, count);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_maskout_near_cam(float* slab, int64_t voxel_stride, int64_t X, int64_t Y, int64_t Z, const float* cams, int64_t n_cams,
                         float near_clip, float fill, void* stream) {
  const int64_t n = X * Y * Z;
  if (n <= 0 || n_cams <= 0) return 0;
  k_maskout_near_cam<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(slab, voxel_stride, (int)X, (int)Y, (int)Z, -1.f, -1.f, -1.f,
                                                                        1.f, 1.f, 1.f, cams, (int)n_cams, near_clip, fill);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_maskout_near_cam_lattice(float* slab, int64_t voxel_stride, int64_t X, int64_t Y, int64_t Z, const float* lattice_min,
                                 const float* lattice_max, const float* cams, int64_t n_cams, float near_clip, float fill,
                                 void* stream) {
  const int64_t n = X * Y * Z;
  if (n <= 0 || n_cams <= 0) return 0;
  k_maskout_near_cam<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(slab, voxel_stride, (int)X, (int)Y, (int)Z, lattice_min[0],
                                                                        lattice_min[1], lattice_min[2], lattice_max[0], lattice_max[1],
                                                                        lattice_max[2], cams, (int)n_cams, near_clip, fill);
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
