/*
 * oracle/ref_ops.c -- TEST INFRASTRUCTURE ONLY.  NOT part of the shipped product.
 *
 * Plain-C (gcc, scalar, single-thread) restatement of the arithmetic of the reference's native
 * layer L0 (sjtuytc/UnboundedNeRFPytorch @ 3d7008d, FourierGrid/cuda/*.cu).  Every function cites
 * the reference file:line whose arithmetic it follows.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference leg may load this library; the product path
 * (unboundednerfpytorch_b200/) never does and fails loudly without its CUDA library.
 *
 * Parity pinning: the reference ships NO tests / golden vectors (SURVEY.md section 4), so this
 * restatement is pinned by (a) running the reference's own Python model files here on CPU on top
 * of these functions (oracle/stubs.py -> tests/golden/, script oracle/make_golden.py) and (b) the
 * reference's own CUDA extension compiled for sm_90a (oracle/_ref/, `make ref`) run on the GPU.
 *
 * Numerics notes (SURVEY.md Appendix A): device code in the reference is compiled by nvcc with
 * default -fmad=true, so `a*b + c` is contracted into one fma; this file is compiled with
 * -ffp-contract=off and spells each contraction explicitly with fmaf() (LLVM rule: for
 * fadd(fmul(a,b), z) the LEFT product is fused).  Expressions that promote to double in the
 * reference (literals `1.`, `1e-3`, `1e10`, `1e-10`) are kept in double here.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define UBO_API __attribute__((visibility("default")))

/* ---- render_utils_kernel.cu:12-35  infer_t_minmax_cuda_kernel ---- */
UBO_API void ubo_infer_t_minmax(const float* rays_o, const float* rays_d,
                                const float* xyz_min, const float* xyz_max,
                                float near, float far, int64_t n_rays,
                                float* t_min, float* t_max) {
  for (int64_t r = 0; r < n_rays; ++r) {
    const float* o = rays_o + 3 * r;
    const float* d = rays_d + 3 * r;
    float vx = (d[0] == 0) ? (float)1e-6 : d[0];
    float vy = (d[1] == 0) ? (float)1e-6 : d[1];
    float vz = (d[2] == 0) ? (float)1e-6 : d[2];
    float ax = (xyz_max[0] - o[0]) / vx, ay = (xyz_max[1] - o[1]) / vy, az = (xyz_max[2] - o[2]) / vz;
    float bx = (xyz_min[0] - o[0]) / vx, by = (xyz_min[1] - o[1]) / vy, bz = (xyz_min[2] - o[2]) / vz;
    t_min[r] = fmaxf(fminf(fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fminf(az, bz)), far), near);
    t_max[r] = fmaxf(fminf(fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fmaxf(az, bz)), far), near);
  }
}

/* rnorm = sqrt(dx*dx + dy*dy + dz*dz), float, fma-contracted (render_utils_kernel.cu:48-51, 68-71) */
static inline float ubo_rnorm(const float* d) {
  return sqrtf(fmaf(d[2], d[2], fmaf(d[1], d[1], d[0] * d[0])));
}

/* ---- render_utils_kernel.cu:38-55  infer_n_samples_cuda_kernel ---- */
UBO_API void ubo_infer_n_samples(const float* rays_d, const float* t_min, const float* t_max,
                                 float stepdist, int64_t n_rays, int64_t* n_samples) {
  for (int64_t r = 0; r < n_rays; ++r) {
    float rnorm = ubo_rnorm(rays_d + 3 * r);
    float c = ceilf((t_max[r] - t_min[r]) * rnorm / stepdist);
    double m = fmax((double)c, 1.);           /* max(float, double literal 1.) is evaluated in double */
    n_samples[r] = (int64_t)m;
  }
}

/* ---- render_utils_kernel.cu:58-79  infer_ray_start_dir_cuda_kernel ---- */
UBO_API void ubo_infer_ray_start_dir(const float* rays_o, const float* rays_d, const float* t_min,
                                     int64_t n_rays, float* rays_start, float* rays_dir) {
  for (int64_t r = 0; r < n_rays; ++r) {
    const float* o = rays_o + 3 * r;
    const float* d = rays_d + 3 * r;
    float rnorm = ubo_rnorm(d);
    for (int a = 0; a < 3; ++a) {
      rays_start[3 * r + a] = fmaf(d[a], t_min[r], o[a]);
      rays_dir[3 * r + a] = d[a] / rnorm;
    }
  }
}

/* ---- render_utils_kernel.cu:144-242  sample_pts_on_rays (K4,K5,K6 + host glue) ----
 * Two-call protocol: (1) ubo_sample_pts_count fills t_min/t_max/N_steps and returns total_len
 * (the reference's N_steps.sum().item(), :212); (2) ubo_sample_pts_emit fills the ragged outputs. */
UBO_API int64_t ubo_sample_pts_count(const float* rays_o, const float* rays_d,
                                     const float* xyz_min, const float* xyz_max,
                                     float near, float far, float stepdist, int64_t n_rays,
                                     float* t_min, float* t_max, int64_t* n_steps) {
  ubo_infer_t_minmax(rays_o, rays_d, xyz_min, xyz_max, near, far, n_rays, t_min, t_max);
  ubo_infer_n_samples(rays_d, t_min, t_max, stepdist, n_rays, n_steps);
  int64_t tot = 0;
  for (int64_t r = 0; r < n_rays; ++r) tot += n_steps[r];
  return tot;
}

UBO_API void ubo_sample_pts_emit(const float* rays_o, const float* rays_d,
                                 const float* xyz_min, const float* xyz_max,
                                 const float* t_min, const int64_t* n_steps,
                                 float stepdist, int64_t n_rays,
                                 float* rays_pts, uint8_t* mask_outbbox,
                                 int64_t* ray_id, int64_t* step_id) {
  int64_t idx = 0;
  for (int64_t r = 0; r < n_rays; ++r) {
    const float* o = rays_o + 3 * r;
    const float* d = rays_d + 3 * r;
    float rnorm = ubo_rnorm(d);
    float st[3], dir[3];
    for (int a = 0; a < 3; ++a) { st[a] = fmaf(d[a], t_min[r], o[a]); dir[a] = d[a] / rnorm; }
    for (int64_t s = 0; s < n_steps[r]; ++s, ++idx) {
      /* :179-180 i_ray/i_step are truncated to int in the reference */
      float dist = stepdist * (float)(int)s;                   /* :184 */
      float px = fmaf(dir[0], dist, st[0]);                    /* :185-187, fma-contracted */
      float py = fmaf(dir[1], dist, st[1]);
      float pz = fmaf(dir[2], dist, st[2]);
      rays_pts[3 * idx] = px; rays_pts[3 * idx + 1] = py; rays_pts[3 * idx + 2] = pz;
      mask_outbbox[idx] = (uint8_t)((xyz_min[0] > px) | (xyz_min[1] > py) | (xyz_min[2] > pz) |
                                    (xyz_max[0] < px) | (xyz_max[1] < py) | (xyz_max[2] < pz));
      ray_id[idx] = r;
      step_id[idx] = s;
    }
  }
}

/* ---- render_utils_kernel.cu:245-270  sample_ndc_pts_on_rays_cuda_kernel ---- */
UBO_API void ubo_sample_ndc_pts_on_rays(const float* rays_o, const float* rays_d,
                                        const float* xyz_min, const float* xyz_max,
                                        int64_t n_samples, int64_t n_rays,
                                        float* rays_pts, uint8_t* mask_outbbox) {
  for (int64_t r = 0; r < n_rays; ++r)
    for (int64_t s = 0; s < n_samples; ++s) {
      int64_t idx = r * n_samples + s;
      float dist = ((float)(int)s) / (float)(int)(n_samples - 1);      /* :260 */
      float px = fmaf(rays_d[3 * r], dist, rays_o[3 * r]);
      float py = fmaf(rays_d[3 * r + 1], dist, rays_o[3 * r + 1]);
      float pz = fmaf(rays_d[3 * r + 2], dist, rays_o[3 * r + 2]);
      rays_pts[3 * idx] = px; rays_pts[3 * idx + 1] = py; rays_pts[3 * idx + 2] = pz;
      mask_outbbox[idx] = (uint8_t)((xyz_min[0] > px) | (xyz_min[1] > py) | (xyz_min[2] > pz) |
                                    (xyz_max[0] < px) | (xyz_max[1] < py) | (xyz_max[2] < pz));
    }
}

/* ---- render_utils_kernel.cu:301-340  sample_bg_pts_on_rays_cuda_kernel (dead export) ---- */
UBO_API void ubo_sample_bg_pts_on_rays(const float* rays_o, const float* rays_d, const float* t_max,
                                       float bg_preserve, int64_t n_samples, int64_t n_rays,
                                       float* rays_pts) {
  for (int64_t r = 0; r < n_rays; ++r)
    for (int64_t s = 0; s < n_samples; ++s) {
      int64_t idx = r * n_samples + s;
      float t_inner = t_max[r];
      float frac = ((float)(int)s) / (float)(int)n_samples;
      float ori_t_outer = (float)((double)t_inner - 1. + 1. / (1. - (double)frac));     /* :325 */
      float x = fmaf(rays_d[3 * r], ori_t_outer, rays_o[3 * r]);
      float y = fmaf(rays_d[3 * r + 1], ori_t_outer, rays_o[3 * r + 1]);
      float z = fmaf(rays_d[3 * r + 2], ori_t_outer, rays_o[3 * r + 2]);
      float t_outer = sqrtf(fmaf(z, z, fmaf(y, y, x * x)));                              /* :296-298 */
      float m = fmaxf(fabsf(x), fmaxf(fabsf(y), fabsf(z)));
      float R = t_outer / m;
      double o2i = (double)(R * R / (t_outer * t_outer)) * (1. - (double)bg_preserve) +
                   (double)(R / t_outer * bg_preserve);                                    /* :332 */
      float o2i_p = (float)o2i;
      rays_pts[3 * idx] = x * o2i_p; rays_pts[3 * idx + 1] = y * o2i_p; rays_pts[3 * idx + 2] = z * o2i_p;
    }
}

/* ---- render_utils_kernel.cu:367-392  maskcache_lookup_cuda_kernel ---- */
UBO_API void ubo_maskcache_lookup(const uint8_t* world, const float* xyz, uint8_t* out,
                                  const float* scale, const float* shift,
                                  int64_t sz_i, int64_t sz_j, int64_t sz_k, int64_t n_pts) {
  for (int64_t p = 0; p < n_pts; ++p) {
    /* round(): C round-half-away-from-zero on the fma-contracted float, then int truncation (:385-387) */
    int i = (int)roundf(fmaf(xyz[3 * p], scale[0], shift[0]));
    int j = (int)roundf(fmaf(xyz[3 * p + 1], scale[1], shift[1]));
    int k = (int)roundf(fmaf(xyz[3 * p + 2], scale[2], shift[2]));
    uint8_t v = 0;                                    /* out is zero-initialised (:405) */
    if (0 <= i && i < sz_i && 0 <= j && j < sz_j && 0 <= k && k < sz_k)
      v = world[(int64_t)i * sz_j * sz_k + (int64_t)j * sz_k + k];
    out[p] = v;
  }
}

/* ---- render_utils_kernel.cu:431-458  raw2alpha(_nonuni)_cuda_kernel ----
 * interval_arr == NULL -> uniform interval. */
UBO_API void ubo_raw2alpha(const float* density, float shift, float interval, const float* interval_arr,
                           int64_t n_pts, float* exp_d, float* alpha) {
  for (int64_t i = 0; i < n_pts; ++i) {
    float e = expf(density[i] + shift);               /* can be inf (:439) */
    float itv = interval_arr ? interval_arr[i] : interval;
    exp_d[i] = e;
    alpha[i] = 1 - powf(1 + e, -itv);
  }
}

/* ---- render_utils_kernel.cu:507-530  raw2alpha(_nonuni)_backward_cuda_kernel ---- */
UBO_API void ubo_raw2alpha_backward(const float* exp_d, const float* grad_back, float interval,
                                    const float* interval_arr, int64_t n_pts, float* grad) {
  for (int64_t i = 0; i < n_pts; ++i) {
    float itv = interval_arr ? interval_arr[i] : interval;
    /* min(float, 1e10) promotes to double; pow(float,float) stays float; product in double (:515) */
    double g = fmin((double)exp_d[i], 1e10) * (double)powf(1 + exp_d[i], -itv - 1) * (double)itv * (double)grad_back[i];
    grad[i] = (float)g;
  }
}

/* ---- render_utils_kernel.cu:607-617,633-635  __set_i_for_segment_start_end + host fix-up ---- */
UBO_API void ubo_segment_bounds(const int64_t* ray_id, int64_t n_pts, int64_t n_rays,
                                int64_t* i_start, int64_t* i_end) {
  memset(i_start, 0, sizeof(int64_t) * (size_t)n_rays);
  memset(i_end, 0, sizeof(int64_t) * (size_t)n_rays);
  if (n_pts == 0) return;
  for (int64_t idx = 1; idx < n_pts; ++idx)
    if (ray_id[idx] != ray_id[idx - 1]) { i_start[ray_id[idx]] = idx; i_end[ray_id[idx - 1]] = idx; }
  i_end[ray_id[n_pts - 1]] = n_pts;
}

/* ---- render_utils_kernel.cu:577-605,619-651  alpha2weight ---- */
UBO_API void ubo_alpha2weight(const float* alpha, const int64_t* ray_id, int64_t n_pts, int64_t n_rays,
                              float* weight, float* T, float* alphainv_last,
                              int64_t* i_start, int64_t* i_end) {
  for (int64_t i = 0; i < n_pts; ++i) { weight[i] = 0.f; T[i] = 1.f; }          /* zeros_like / ones_like :624-625 */
  for (int64_t r = 0; r < n_rays; ++r) alphainv_last[r] = 1.f;                   /* :626 */
  ubo_segment_bounds(ray_id, n_pts, n_rays, i_start, i_end);
  if (n_pts == 0) return;
  for (int64_t r = 0; r < n_rays; ++r) {
    int i_s = (int)i_start[r], i_e_max = (int)i_end[r];
    float T_cum = 1.f;
    int i;
    for (i = i_s; i < i_e_max; ++i) {
      T[i] = T_cum;
      weight[i] = T_cum * alpha[i];
      T_cum = (float)((double)T_cum * (1. - (double)alpha[i]));                  /* :596 double intermediate */
      if ((double)T_cum < 1e-3) { i += 1; break; }                               /* :597-600 */
    }
    i_end[r] = i;
    alphainv_last[r] = T_cum;
  }
}

/* ---- render_utils_kernel.cu:654-677  alpha2weight_backward_cuda_kernel ---- */
UBO_API void ubo_alpha2weight_backward(const float* alpha, const float* weight, const float* T,
                                       const float* alphainv_last, const int64_t* i_start, const int64_t* i_end,
                                       int64_t n_pts, int64_t n_rays,
                                       const float* grad_weights, const float* grad_last, float* grad) {
  for (int64_t i = 0; i < n_pts; ++i) grad[i] = 0.f;                              /* zeros_like :684 */
  for (int64_t r = 0; r < n_rays; ++r) {
    int i_s = (int)i_start[r], i_e = (int)i_end[r];
    float back_cum = grad_last[r] * alphainv_last[r];
    for (int i = i_e - 1; i >= i_s; --i) {
      /* gw*T - back/(1-alpha+1e-10): denominator and quotient in double; the float product gw*T is
       * promoted; nvcc may contract a*b - c into fma only within one precision, so none here (:673) */
      double den = (double)(1 - alpha[i]) + 1e-10;
      grad[i] = (float)((double)(grad_weights[i] * T[i]) - (double)back_cum / den);
      back_cum = fmaf(grad_weights[i], weight[i], back_cum);                      /* :674 contracted */
    }
  }
}

/* ---- adam_upd_kernel.cu:9-58,72  adam / masked adam / per-voxel-lr adam ----
 * mode 0: adam_upd, 1: masked_adam_upd (skip grad==0), 2: adam_upd_with_perlr. */
UBO_API float ubo_adam_step_size(int step, float beta1, float beta2, float lr) {
  /* host-side float arithmetic, adam_upd_kernel.cu:72 */
  return lr * sqrtf(1 - powf(beta2, (float)step)) / (1 - powf(beta1, (float)step));
}

UBO_API void ubo_adam_upd(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                          const float* perlr, int64_t n, int step,
                          float beta1, float beta2, float lr, float eps, int mode) {
  const float step_size = ubo_adam_step_size(step, beta1, beta2, lr);
  for (int64_t i = 0; i < n; ++i) {
    const float g = grad[i];
    if (mode == 1 && g == 0) continue;
    float m = fmaf(beta1, exp_avg[i], (1 - beta1) * g);                           /* :14,:36,:54 */
    float v = fmaf(beta2, exp_avg_sq[i], (1 - beta2) * g * g);                    /* :15 */
    exp_avg[i] = m; exp_avg_sq[i] = v;
    if (mode == 2) param[i] -= step_size * perlr[i] * m / (sqrtf(v) + eps);       /* :56 */
    else           param[i] -= step_size * m / (sqrtf(v) + eps);                  /* :16 */
  }
}

/* ---- total_variation_kernel.cu:8-35,45-47  total_variation_add_grad ----
 * param/grad viewed as [lead, sz_i, sz_j, sz_k]; NOTE the i-axis uses wz and wx is unused (:31-32). */
static inline float ubo_clamp1(float v) { return fminf(fmaxf(v, -1.f), 1.f); }

UBO_API void ubo_total_variation_add_grad(const float* param, float* grad, float wx, float wy, float wz,
                                          int64_t sz_i, int64_t sz_j, int64_t sz_k, int64_t n, int dense_mode) {
  wx /= 6; wy /= 6; wz /= 6;                                                      /* host :45-47 */
  (void)wx;
  float* add = (float*)malloc(sizeof(float) * (size_t)n);
  for (int64_t idx = 0; idx < n; ++idx) {
    add[idx] = 0.f;
    if (!(dense_mode || grad[idx] != 0)) continue;
    int64_t k = idx % sz_k, j = idx / sz_k % sz_j, i = idx / sz_k / sz_j % sz_i;
    float g = 0;
    g += (k == 0        ? 0 : wz * ubo_clamp1(param[idx] - param[idx - 1]));
    g += (k == sz_k - 1 ? 0 : wz * ubo_clamp1(param[idx] - param[idx + 1]));
    g += (j == 0        ? 0 : wy * ubo_clamp1(param[idx] - param[idx - sz_k]));
    g += (j == sz_j - 1 ? 0 : wy * ubo_clamp1(param[idx] - param[idx + sz_k]));
    g += (i == 0        ? 0 : wz * ubo_clamp1(param[idx] - param[idx - sz_k * sz_j]));
    g += (i == sz_i - 1 ? 0 : wz * ubo_clamp1(param[idx] - param[idx + sz_k * sz_j]));
    add[idx] = g;
  }
  /* each element's gate reads its own (pre-add) grad only, so a second pass is equivalent */
  for (int64_t idx = 0; idx < n; ++idx)
    if (dense_mode || grad[idx] != 0) grad[idx] += add[idx];
  free(add);
}

/* ---- ub360_utils_kernel.cu:13-32  cumdist_thres_cuda_kernel ---- */
UBO_API void ubo_cumdist_thres(const float* dist, float thres, int64_t n_rays, int64_t n_pts, uint8_t* mask) {
  for (int64_t r = 0; r < n_rays; ++r) {
    float cum = 0;
    for (int64_t i = r * n_pts; i < (r + 1) * n_pts; ++i) {
      cum += dist[i];
      int over = (cum > thres);
      cum *= (float)(!over);
      mask[i] = (uint8_t)over;
    }
  }
}
