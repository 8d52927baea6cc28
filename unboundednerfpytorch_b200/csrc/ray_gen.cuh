// ray_gen.cuh -- the camera ray of one pixel (FourierGrid/dvgo.py:492-557), shared by ubn_get_rays_of_a_view (ray_gen.cu) and
// ubn_frustum_bounds (bounds.cu) so that both produce the same bits.
#pragma once
#include "common.cuh"

namespace ubn {

struct ViewParams {
  float fx, fy, cx, cy;     // K[0][0], K[1][1], K[0][2], K[1][2]
  float r[3][3], t[3];      // c2w[:3,:3], c2w[:3,3]
  int H, W;
  int ndc, inverse_y, flip_x, flip_y;
  float pix;                // 0.5 for mode 'center', 0 for 'lefttop' / 'random' (random offsets come in `jitter`)
  float sw, sh;             // ndc scales -1/(W/(2 focal)), -1/(H/(2 focal)), evaluated in double like Python does
};

// ndc scales of ndc_rays (dvgo.py:532-550, focal = K[0][0]): in double, rounded once to float
__host__ __device__ __forceinline__ void ndc_scales(int H, int W, float fx, float& sw, float& sh) {
  sw = (float)(-1.0 / (W / (2.0 * (double)fx)));
  sh = (float)(-1.0 / (H / (2.0 * (double)fx)));
}

// rays_o, rays_d, viewdirs of pixel (row, col); jitter = [2,H,W] offsets of mode 'random' or nullptr
__device__ __forceinline__ void pixel_ray(const ViewParams& v, int row, int col, const float* __restrict__ jitter, float ro[3],
                                          float rd[3], float vd[3]) {
  // i, j are built BEFORE the flips (dvgo.py:497-513): the flipped image takes the value of the mirrored pixel
  const int sc = v.flip_x ? v.W - 1 - col : col;
  const int sr = v.flip_y ? v.H - 1 - row : row;
  float i = (float)sc + v.pix, j = (float)sr + v.pix;
  if (jitter) {   // mode 'random' (dvgo.py:503-505): i + rand_like(i), j + rand_like(j) drawn BEFORE the flips, and i is
                  // flipped along x only, j along y only; jitter = [2,H,W] (plane 0 for i, plane 1 for j)
    const int64_t n = (int64_t)v.H * v.W;
    i = (float)sc + jitter[(int64_t)row * v.W + sc];
    j = (float)sr + jitter[n + (int64_t)sr * v.W + col];
  }
  float d0 = __fdiv_rn(__fsub_rn(i, v.cx), v.fx);
  float d1 = __fdiv_rn(__fsub_rn(j, v.cy), v.fy);
  float d2 = 1.f;
  if (!v.inverse_y) { d1 = -d1; d2 = -1.f; }
#pragma unroll
  for (int k = 0; k < 3; ++k)   // torch.sum(dirs[..., None, :] * c2w[:3,:3], -1): products first, then a 3-term sum
    rd[k] = __fadd_rn(__fadd_rn(__fmul_rn(d0, v.r[k][0]), __fmul_rn(d1, v.r[k][1])), __fmul_rn(d2, v.r[k][2]));
  const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(rd[0], rd[0]), __fmul_rn(rd[1], rd[1])), __fmul_rn(rd[2], rd[2])));
  ro[0] = v.t[0]; ro[1] = v.t[1]; ro[2] = v.t[2];
  vd[0] = __fdiv_rn(rd[0], nrm); vd[1] = __fdiv_rn(rd[1], nrm); vd[2] = __fdiv_rn(rd[2], nrm);
  if (v.ndc) {   // ndc_rays(H, W, focal = K[0][0], near = 1, ...)  dvgo.py:532-550
    const float near = 1.f;
    const float tt = __fdiv_rn(-__fadd_rn(near, ro[2]), rd[2]);
    ro[0] = __fadd_rn(ro[0], __fmul_rn(tt, rd[0]));
    ro[1] = __fadd_rn(ro[1], __fmul_rn(tt, rd[1]));
    ro[2] = __fadd_rn(ro[2], __fmul_rn(tt, rd[2]));
    const float sw = v.sw, sh = v.sh;
    const float o0 = __fdiv_rn(__fmul_rn(sw, ro[0]), ro[2]);
    const float o1 = __fdiv_rn(__fmul_rn(sh, ro[1]), ro[2]);
    const float o2 = __fadd_rn(1.f, __fdiv_rn(2.f * near, ro[2]));
    const float e0 = __fmul_rn(sw, __fsub_rn(__fdiv_rn(rd[0], rd[2]), __fdiv_rn(ro[0], ro[2])));
    const float e1 = __fmul_rn(sh, __fsub_rn(__fdiv_rn(rd[1], rd[2]), __fdiv_rn(ro[1], ro[2])));
    const float e2 = __fdiv_rn(-2.f * near, ro[2]);
    ro[0] = o0; ro[1] = o1; ro[2] = o2;
    rd[0] = e0; rd[1] = e1; rd[2] = e2;
  }
}

}  // namespace ubn
