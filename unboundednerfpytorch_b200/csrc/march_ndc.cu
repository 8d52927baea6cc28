// march_ndc.cu -- pass B of the fused NDC march (DirectMPIGO.forward, dmpigo.py:294-295) and of the fused box march
// (DirectVoxGO.forward, dvgo.py:365-366), and their adjoints.
//
// Pass A and its backward are the contracted march's kernels (march.cu) instantiated with NdcSampler / BoxSampler.  The feature
// read is separate because these models' k0 grids are single-slab with C = 9 (LLFF, and DVGO on the free-dataset lab config),
// 12 (DVGO fine stage) or 3 (rgbnet_dim = 0) channels: a 36- or 12-byte channels-last record is only 4-byte aligned, so the
// float4 quads of the contracted kernels do not apply there; a 48-byte record (C = 12) is 16-byte aligned and is read with
// float4 loads.  The sampling policy is a template
// parameter: the box march's rays stop at their own n_steps.
//
// Lane = sample: each lane that holds a survivor of the current 32-sample chunk reads its 8 corner records with scalar loads and
// accumulates every channel in ATen's corner order (tnw .. bse, z fastest) with the same fma chain as F.grid_sample, so the
// features are bit-identical to it.  In-box NDC points normalise into [-1, 1], where the pre-clamped cell (make_cell) gives the
// same (value, weight) pairs as the bounds-checked read.  The backward adds w * grad into the 8 records with the widest
// reductions each address allows (red.v4 at 16-byte, red.v2 at 8-byte alignment, scalar otherwise).
#include <type_traits>

#include "march_common.cuh"

namespace ubn {

template <class Smp, int kC, bool kBackward>
__global__ void __launch_bounds__(32 * kMarchWarps) k_march_ndc_feature(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, GridView g, MarchParams p, int64_t n_rays,
    const uint8_t* __restrict__ flags, const int64_t* __restrict__ offsets, const float* __restrict__ alpha,
    const float* __restrict__ weight, float* __restrict__ feat /* out (fwd) or grad in (bwd) */, float* __restrict__ grad_grid,
    float* __restrict__ o_alpha, float* __restrict__ o_weight, int64_t* __restrict__ o_ray_id, int64_t* __restrict__ o_step_id) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  int64_t out_base = offsets[ray];
  const int64_t out_end = offsets[ray + 1];
  if (out_base == out_end) return;
  const Ray r = Smp::load(rays_o + 3 * ray, rays_d + 3 * ray, p);
  const int S = p.S;                                   // record stride
  const int n = r.n;                                   // samples of this ray
  const int dY = g.Z * kC, dX = g.Y * g.Z * kC;        // record strides (floats) of +1 in y / x; +1 in z is kC

  for (int base = 0; base < n && out_base < out_end; base += 32) {
    const int s = base + lane;
    const uint8_t f = (s < n) ? flags[ray * S + s] : 0;
    const bool keep = (f & UBN_FLAG_KEEP) != 0;
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (km == 0) continue;
    if (keep) {
      const int64_t row = out_base + __popc(km & ((1u << lane) - 1));
      float x, y, z;
      bool inner;
      Smp::point(r, nullptr, s, p, x, y, z, inner);
      const CellR c = make_cell(src_index(norm_coord(x, g.mn[0], g.len[0]), g.X), src_index(norm_coord(y, g.mn[1], g.len[1]), g.Y),
                                src_index(norm_coord(z, g.mn[2], g.len[2]), g.Z), g.X, g.Y, g.Z);
      if (!kBackward) {
        const float* rec = g.data + (int64_t)c.v * kC;
        float acc[kC];
#pragma unroll
        for (int ch = 0; ch < kC; ++ch) acc[ch] = 0.f;
#pragma unroll
        for (int corner = 0; corner < 8; ++corner) {
          const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
          const float wgt = ((bz ? c.fz : 1.f - c.fz) * (by ? c.fy : 1.f - c.fy)) * (bx ? c.fx : 1.f - c.fx);
          const float* q = rec + bx * dX + by * dY + bz * kC;
          if constexpr (kC % 4 == 0) {                 // 16-byte aligned records: same fma chain, fed by float4 loads
#pragma unroll
            for (int c4 = 0; c4 < kC; c4 += 4) {
              const float4 v = __ldg(reinterpret_cast<const float4*>(q + c4));
              acc[c4] = fmaf(v.x, wgt, acc[c4]);
              acc[c4 + 1] = fmaf(v.y, wgt, acc[c4 + 1]);
              acc[c4 + 2] = fmaf(v.z, wgt, acc[c4 + 2]);
              acc[c4 + 3] = fmaf(v.w, wgt, acc[c4 + 3]);
            }
          } else {
#pragma unroll
            for (int ch = 0; ch < kC; ++ch) acc[ch] = fmaf(__ldg(q + ch), wgt, acc[ch]);
          }
        }
        if constexpr (kC % 4 == 0) {
#pragma unroll
          for (int c4 = 0; c4 < kC; c4 += 4)
            *reinterpret_cast<float4*>(feat + row * kC + c4) = make_float4(acc[c4], acc[c4 + 1], acc[c4 + 2], acc[c4 + 3]);
        } else {
#pragma unroll
          for (int ch = 0; ch < kC; ++ch) feat[row * kC + ch] = acc[ch];
        }
        const int64_t i = ray * S + s;
        if (o_alpha) o_alpha[row] = alpha[i];
        if (o_weight) o_weight[row] = weight[i];
        o_ray_id[row] = ray;
        o_step_id[row] = s;
      } else {
        float gin[kC];
        if constexpr (kC % 4 == 0) {
#pragma unroll
          for (int c4 = 0; c4 < kC; c4 += 4) {
            const float4 v = *reinterpret_cast<const float4*>(feat + row * kC + c4);
            gin[c4] = v.x; gin[c4 + 1] = v.y; gin[c4 + 2] = v.z; gin[c4 + 3] = v.w;
          }
        } else {
#pragma unroll
          for (int ch = 0; ch < kC; ++ch) gin[ch] = feat[row * kC + ch];
        }
        float* rec = grad_grid + (int64_t)c.v * kC;
#pragma unroll
        for (int corner = 0; corner < 8; ++corner) {
          const int bx = corner >> 2, by = (corner >> 1) & 1, bz = corner & 1;
          const float wgt = ((bz ? c.fz : 1.f - c.fz) * (by ? c.fy : 1.f - c.fy)) * (bx ? c.fx : 1.f - c.fx);
          float v[kC];
#pragma unroll
          for (int ch = 0; ch < kC; ++ch) v[ch] = wgt * gin[ch];
          red_add_record<kC>(rec + bx * dX + by * dY + bz * kC, v);
        }
      }
    }
    out_base += __popc(km);
  }
}

// Pass B of the box march for a k0 read elsewhere (the k0 of a TensoRF model, read by its own forward): the compacted records
// alpha, weight, ray_id, step_id and the survivor's point xyz[M, 3] -- box_point, the point ubn_sample_pts_* give the same step --
// in place of the feature read.
__global__ void __launch_bounds__(32 * kMarchWarps) k_march_box_points(
    const float* __restrict__ rays_o, const float* __restrict__ rays_d, MarchParams p, int64_t n_rays,
    const uint8_t* __restrict__ flags, const int64_t* __restrict__ offsets, const float* __restrict__ alpha,
    const float* __restrict__ weight, float* __restrict__ xyz, float* __restrict__ o_alpha, float* __restrict__ o_weight,
    int64_t* __restrict__ o_ray_id, int64_t* __restrict__ o_step_id) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  int64_t out_base = offsets[ray];
  const int64_t out_end = offsets[ray + 1];
  if (out_base == out_end) return;
  const Ray r = BoxSampler::load(rays_o + 3 * ray, rays_d + 3 * ray, p);
  for (int base = 0; base < r.n && out_base < out_end; base += 32) {
    const int s = base + lane;
    const uint8_t f = (s < r.n) ? flags[ray * p.S + s] : 0;
    const bool keep = (f & UBN_FLAG_KEEP) != 0;
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int64_t row = out_base + __popc(km & ((1u << lane) - 1));
      float x, y, z;
      bool inner;
      BoxSampler::point(r, nullptr, s, p, x, y, z, inner);
      xyz[3 * row] = x;
      xyz[3 * row + 1] = y;
      xyz[3 * row + 2] = z;
      const int64_t i = ray * p.S + s;
      if (o_alpha) o_alpha[row] = alpha[i];
      if (o_weight) o_weight[row] = weight[i];
      o_ray_id[row] = ray;
      o_step_id[row] = s;
    }
    out_base += __popc(km);
  }
}

// single slab, channels-last, C in {3, 9}, >= 2 voxels per axis (pre-clamped cells), 32-bit voxel index (make_cell), 4-byte aligned
static bool ndc_feature_grid_ok(const GridView& g) {
  return g.P == 1 && g.sc == 1 && g.sv == g.C && (g.C == 3 || g.C == 9) && g.X >= 2 && g.Y >= 2 && g.Z >= 2 &&
         (int64_t)g.X * g.Y * g.Z < (1ll << 31) && ((uintptr_t)g.data & 3) == 0;
}

// the box march's k0: single slab, channels-last, C in {3, 9, 12}, 16-byte aligned for C = 12 (float4 records), 4-byte otherwise
static bool box_feature_grid_ok(const GridView& g) {
  return g.P == 1 && g.sc == 1 && g.sv == g.C && (g.C == 3 || g.C == 9 || g.C == 12) && g.X >= 2 && g.Y >= 2 && g.Z >= 2 &&
         (int64_t)g.X * g.Y * g.Z < (1ll << 31) && ((uintptr_t)g.data & (g.C == 12 ? 15 : 3)) == 0;
}

template <class Smp, bool kBackward>
static int launch_ndc_feature(const float* rays_o, const float* rays_d, const GridView& g, const MarchParams& p, int64_t n_rays,
                              const uint8_t* flags, const int64_t* offsets, const float* alpha, const float* weight, float* feat,
                              float* grad_grid, float* o_alpha, float* o_weight, int64_t* o_ray_id, int64_t* o_step_id,
                              cudaStream_t st) {
#define UBN_NDC_FEAT(C)                                                                                                    \
  k_march_ndc_feature<Smp, C, kBackward><<<blocks_for(n_rays, kMarchWarps), 32 * kMarchWarps, 0, st>>>(                         \
      rays_o, rays_d, g, p, n_rays, flags, offsets, alpha, weight, feat, grad_grid, o_alpha, o_weight, o_ray_id, o_step_id)
  if constexpr (std::is_same<Smp, BoxSampler>::value) {
    if (g.C == 12) UBN_NDC_FEAT(12);
    else if (g.C == 9) UBN_NDC_FEAT(9);
    else UBN_NDC_FEAT(3);
  } else {
    if (g.C == 9) UBN_NDC_FEAT(9);
    else UBN_NDC_FEAT(3);
  }
#undef UBN_NDC_FEAT
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_march_ndc_feature_fwd(const float* rays_o, const float* rays_d, const float* k0_grid, const UbnGridDesc* k0_desc,
                              const UbnNdcMarchCfg* cfg, int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                              const float* alpha, const float* weight, float* k0_feat, float* out_alpha, float* out_weight,
                              int64_t* ray_id, int64_t* step_id, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(k0_grid, k0_desc);
  if (!ndc_feature_grid_ok(g) || cfg->n_samples < 2) return finish(cudaErrorInvalidValue);
  if ((out_alpha && !alpha) || (out_weight && !weight)) return finish(cudaErrorInvalidValue);
  GridView none{};
  const MarchParams p = make_ndc_params(cfg, none);
  return launch_ndc_feature<NdcSampler, false>(rays_o, rays_d, g, p, n_rays, flags, offsets, alpha, weight, k0_feat, nullptr, out_alpha,
                                   out_weight, ray_id, step_id, as_stream(stream));
}

int ubn_march_ndc_feature_bwd(const float* rays_o, const float* rays_d, const UbnGridDesc* k0_desc, const UbnNdcMarchCfg* cfg,
                              int64_t n_rays, const uint8_t* flags, const int64_t* offsets, const float* grad_feat,
                              float* grad_k0, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(grad_k0, k0_desc);
  if (!ndc_feature_grid_ok(g) || cfg->n_samples < 2) return finish(cudaErrorInvalidValue);
  GridView none{};
  const MarchParams p = make_ndc_params(cfg, none);
  return launch_ndc_feature<NdcSampler, true>(rays_o, rays_d, g, p, n_rays, flags, offsets, nullptr, nullptr, const_cast<float*>(grad_feat),
                                  grad_k0, nullptr, nullptr, nullptr, nullptr, as_stream(stream));
}

int ubn_march_box_feature_fwd(const float* rays_o, const float* rays_d, const float* k0_grid, const UbnGridDesc* k0_desc,
                              const UbnBoxMarchCfg* cfg, int64_t n_rays, const uint8_t* flags, const int64_t* offsets,
                              const float* alpha, const float* weight, float* k0_feat, float* out_alpha, float* out_weight,
                              int64_t* ray_id, int64_t* step_id, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(k0_grid, k0_desc);
  if (!box_feature_grid_ok(g) || cfg->s_max < 1 || ((uintptr_t)k0_feat & 15)) return finish(cudaErrorInvalidValue);
  if ((out_alpha && !alpha) || (out_weight && !weight)) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_box_params(cfg, nullptr);
  return launch_ndc_feature<BoxSampler, false>(rays_o, rays_d, g, p, n_rays, flags, offsets, alpha, weight, k0_feat, nullptr,
                                               out_alpha, out_weight, ray_id, step_id, as_stream(stream));
}

int ubn_march_box_feature_bwd(const float* rays_o, const float* rays_d, const UbnGridDesc* k0_desc, const UbnBoxMarchCfg* cfg,
                              int64_t n_rays, const uint8_t* flags, const int64_t* offsets, const float* grad_feat,
                              float* grad_k0, void* stream) {
  if (n_rays <= 0) return 0;
  const GridView g = make_view(grad_k0, k0_desc);
  if (!box_feature_grid_ok(g) || cfg->s_max < 1 || ((uintptr_t)grad_feat & 15)) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_box_params(cfg, nullptr);
  return launch_ndc_feature<BoxSampler, true>(rays_o, rays_d, g, p, n_rays, flags, offsets, nullptr, nullptr,
                                              const_cast<float*>(grad_feat), grad_k0, nullptr, nullptr, nullptr, nullptr,
                                              as_stream(stream));
}

int ubn_march_box_points_fwd(const float* rays_o, const float* rays_d, const UbnBoxMarchCfg* cfg, int64_t n_rays, const uint8_t* flags,
                             const int64_t* offsets, const float* alpha, const float* weight, float* xyz, float* out_alpha,
                             float* out_weight, int64_t* ray_id, int64_t* step_id, void* stream) {
  if (n_rays <= 0) return 0;
  if (cfg->s_max < 1 || (out_alpha && !alpha) || (out_weight && !weight)) return finish(cudaErrorInvalidValue);
  const MarchParams p = make_box_params(cfg, nullptr);
  k_march_box_points<<<blocks_for(n_rays, kMarchWarps), 32 * kMarchWarps, 0, as_stream(stream)>>>(
      rays_o, rays_d, p, n_rays, flags, offsets, alpha, weight, xyz, out_alpha, out_weight, ray_id, step_id);
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
