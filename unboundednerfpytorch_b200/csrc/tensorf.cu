// tensorf.cu -- TensoRFGrid, the vector-matrix factorised grid of FourierGrid/grid.py:90-201 (TensoRF, arXiv 2203.09517):
//   forward                    grid.py:111-129, 174-201  -> ubn_tensorf_fwd
//   its adjoint (autograd)                               -> ubn_tensorf_bwd
//   total_variation_add_grad   grid.py:142-154           -> ubn_tensorf_tv_add_grad
//   get_dense_grid             grid.py:156-169           -> ubn_tensorf_dense
// The reference reads each factor with a 2-D F.grid_sample (six launches, six [R, M] outputs), multiplies, concatenates and runs an
// mm.  Here one lane owns one sample: it locates the four plane corners and the two vector nodes of each product group once and
// walks the components, forming the 3R products in registers and folding them straight into the C outputs (f_vec staged in shared
// memory).  A corner's R components are one contiguous record in the channels-last layout, read as 128-bit loads.
//
// Backward: the plane gradients go straight to global memory as vector reductions (planes are a few MB to tens of MB and stay in
// L2).  A vector has only L x R entries that every sample of a step adds into, so its reductions go to vec_copies replicated
// copies (copy = blockIdx % vec_copies) that a closing launch sums in a fixed order.  grad_f_vec = feat^T . grad_out, a sum over
// every sample of the step, follows the long-chain rule of DESIGN.md section 2: each 128-sample tile stages feat and grad_out in
// shared memory, thread k sums row k of the tile's product from zero and adds that partial into its fp32 running sum; the CTAs'
// sums meet once, in CTA order, in the closing launch.
#include "tensorf.cuh"

namespace ubn {
namespace {

constexpr int kTfThreads = 128;   // samples per tile = threads per CTA (the bwd's feat tile is [128][nfeat + 1])

__device__ __forceinline__ void sample_index(const TfView& t, const float* __restrict__ xyz, int64_t m, float* c) {
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = tf_coord(t, a, __ldg(xyz + 3 * m + a));
}

template <int kC>
__device__ __forceinline__ void stage_fvec(const float* __restrict__ fvec, int nfeat, float* sf) {
  if constexpr (kC > 1) {
    for (int i = threadIdx.x; i < nfeat * kC; i += blockDim.x) sf[i] = __ldg(fvec + i);
    __syncthreads();
  }
}

// ---- forward: one lane per sample ------------------------------------------------------------------------------------------
template <int kC, int W>
__global__ void __launch_bounds__(kTfThreads) k_tensorf_fwd(TfView t, const float* __restrict__ fvec, const float* __restrict__ xyz,
                                                            int64_t M, float* __restrict__ out) {
  extern __shared__ float sf[];   // f_vec [nfeat][kC] (kC > 1)
  stage_fvec<kC>(fvec, 2 * t.R + t.Rxy, sf);
  const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float c[3];
  sample_index(t, xyz, m, c);
  float acc[kC];
  tf_read<kC, W>(t, c, sf, acc);
#pragma unroll
  for (int ch = 0; ch < kC; ++ch) out[m * kC + ch] = acc[ch];
}

// ---- backward ----------------------------------------------------------------------------------------------------------------
template <int kC, int W>
__global__ void __launch_bounds__(kTfThreads) k_tensorf_bwd(TfView t, const float* __restrict__ fvec, const float* __restrict__ xyz,
                                                            int64_t M, const float* __restrict__ gout, TfGrads gr,
                                                            float* __restrict__ vcopies, int64_t copy_len, int vec_copies,
                                                            float* __restrict__ fpart) {
  extern __shared__ float sm[];
  const int nfeat = 2 * t.R + t.Rxy;
  const int fs = nfeat + 1;                  // odd row stride: the per-sample feat rows are written without bank conflicts
  float* sf = sm;                            // f_vec [nfeat][kC]
  float* feat = sf + nfeat * kC;             // [128][fs]
  float* gt = feat + kTfThreads * fs;        // grad_out tile [128][kC]
  stage_fvec<kC>(fvec, nfeat, sf);
  float* vc = vcopies + (int64_t)(blockIdx.x % vec_copies) * copy_len;
  const int tid = threadIdx.x;
  float run[kC];                             // thread k < nfeat: running sum of grad_f_vec row k over this CTA's tiles
#pragma unroll
  for (int ch = 0; ch < kC; ++ch) run[ch] = 0.f;
  const int64_t ntiles = (M + kTfThreads - 1) / kTfThreads;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t m = tile * kTfThreads + tid;
    const bool valid = m < M;
    float go[kC];
#pragma unroll
    for (int ch = 0; ch < kC; ++ch) go[ch] = valid ? __ldg(gout + m * kC + ch) : 0.f;
    if constexpr (kC > 1) {
#pragma unroll
      for (int ch = 0; ch < kC; ++ch) gt[tid * kC + ch] = go[ch];
    }
    // a sample with a zero output gradient adds nothing (the density read runs on every in-mask sample; only those that pass
    // the alpha threshold get a gradient)
    bool live = false;
#pragma unroll
    for (int ch = 0; ch < kC; ++ch) live |= go[ch] != 0.f;
    if (live) {
      float c[3];
      sample_index(t, xyz, m, c);
      tf_sample_bwd<kC, W>(t, c, go, sf, feat, tid * fs, gr, vc);
    } else if constexpr (kC > 1) {
      for (int k = 0; k < nfeat; ++k) feat[tid * fs + k] = 0.f;
    }
    if constexpr (kC > 1) {
      __syncthreads();
      if (tid < nfeat) {
        float part[kC];
#pragma unroll
        for (int ch = 0; ch < kC; ++ch) part[ch] = 0.f;
#pragma unroll 4
        for (int s = 0; s < kTfThreads; ++s) {
          const float fv = feat[s * fs + tid];
#pragma unroll
          for (int ch = 0; ch < kC; ++ch) part[ch] = fmaf(fv, gt[s * kC + ch], part[ch]);
        }
#pragma unroll
        for (int ch = 0; ch < kC; ++ch) run[ch] += part[ch];
      }
      __syncthreads();
    }
  }
  if constexpr (kC > 1) {
    if (tid < nfeat) {
#pragma unroll
      for (int ch = 0; ch < kC; ++ch) fpart[((int64_t)blockIdx.x * nfeat + tid) * kC + ch] = run[ch];
    }
  }
}

// ---- total variation: one launch over the elements of all six factors -------------------------------------------------------
struct TfTv {
  int64_t start[7];            // element ranges of the six factors in the launch's index space
  int A[6], B[6], n[6];        // spatial sizes (vectors: B = 1) and components
  float ca[6], cb[6];          // w / 6 of each factor axis
};

__device__ __forceinline__ float huber_d(float d) { return fminf(fmaxf(d, -1.f), 1.f); }   // smooth-L1 (beta 1) derivative

__global__ void __launch_bounds__(256) k_tensorf_tv(TfView t, TfGrads gr, TfTv tv) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= tv.start[6]) return;
  int f = 0;
#pragma unroll
  for (int i = 1; i < 6; ++i) f += (idx >= tv.start[i]) ? 1 : 0;
  int64_t e = idx - tv.start[f];
  const int n = tv.n[f], A = tv.A[f], B = tv.B[f];
  const int r = (int)(e % n);
  e /= n;
  const int b = (int)(e % B), a = (int)(e / B);
  const float* p = t.f[f];
  const int64_t sr = t.sr[f], sa = t.sa[f], sb = t.sb[f];
  const int64_t o = r * sr + a * sa + b * sb;
  const float v = p[o];
  float g = 0.f;
  {
    float h = 0.f;
    if (a > 0) h += huber_d(v - p[o - sa]);
    if (a < A - 1) h -= huber_d(p[o + sa] - v);
    g += tv.ca[f] * h;
  }
  if (B > 1) {
    float h = 0.f;
    if (b > 0) h += huber_d(v - p[o - sb]);
    if (b < B - 1) h -= huber_d(p[o + sb] - v);
    g += tv.cb[f] * h;
  }
  gr.g[f][o] += g;
}

// ---- dense materialisation: node products, one thread per voxel -------------------------------------------------------------
template <int kC>
__global__ void __launch_bounds__(256) k_tensorf_dense(TfView t, const float* __restrict__ fvec, float* __restrict__ out) {
  extern __shared__ float sf[];
  stage_fvec<kC>(fvec, 2 * t.R + t.Rxy, sf);
  const int64_t nv = (int64_t)t.S[0] * t.S[1] * t.S[2];
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  int ijk[3];
  ijk[2] = (int)(v % t.S[2]);
  ijk[1] = (int)((v / t.S[2]) % t.S[1]);
  ijk[0] = (int)(v / ((int64_t)t.S[2] * t.S[1]));
  float acc[kC];
#pragma unroll
  for (int ch = 0; ch < kC; ++ch) acc[ch] = 0.f;
#pragma unroll
  for (int g = 0; g < 3; ++g) {
    const int vf = 5 - g, n = grp_comps(t, g), k0 = grp_feat0(t, g);
    const float* P = t.f[g] + ijk[grp_axis_a(g)] * t.sa[g] + ijk[grp_axis_b(g)] * t.sb[g];
    const float* L = t.f[vf] + ijk[grp_axis_l(g)] * t.sa[vf];
    for (int r = 0; r < n; ++r) {
      const float p = __ldg(P + r * t.sr[g]) * __ldg(L + r * t.sr[vf]);
      if constexpr (kC == 1) {
        acc[0] += p;
      } else {
#pragma unroll
        for (int ch = 0; ch < kC; ++ch) acc[ch] = fmaf(p, sf[(k0 + r) * kC + ch], acc[ch]);
      }
    }
  }
#pragma unroll
  for (int ch = 0; ch < kC; ++ch) out[ch * nv + v] = acc[ch];
}

// ---- host side ----------------------------------------------------------------------------------------------------------------
template <int kC, int W>
int launch_fwd(const TfView& t, const float* fvec, const float* xyz, int64_t M, float* out, cudaStream_t st) {
  const int nfeat = 2 * t.R + t.Rxy;
  const size_t smem = kC > 1 ? (size_t)nfeat * kC * sizeof(float) : 0;
  k_tensorf_fwd<kC, W><<<blocks_for(M, kTfThreads), kTfThreads, smem, st>>>(t, fvec, xyz, M, out);
  UBN_LAUNCH_CHECK();
  return 0;
}

template <int kC, int W>
int launch_bwd(const TfView& t, const float* fvec, const float* xyz, int64_t M, const float* gout, const TfGrads& gr,
               float* vcopies, int64_t copy_len, int vec_copies, float* fpart, int nblk, cudaStream_t st) {
  const int nfeat = 2 * t.R + t.Rxy;
  const size_t smem = kC > 1 ? ((size_t)nfeat * kC + (size_t)kTfThreads * (nfeat + 1) + (size_t)kTfThreads * kC) * sizeof(float) : 0;
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(k_tensorf_bwd<kC, W>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return finish(e);
  }
  k_tensorf_bwd<kC, W><<<nblk, kTfThreads, smem, st>>>(t, fvec, xyz, M, gout, gr, vcopies, copy_len, vec_copies, fpart);
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // namespace
}  // namespace ubn

using namespace ubn;

extern "C" {

int ubn_tensorf_fwd(const float* const* factors, const float* f_vec, const UbnTensorfDesc* desc, const float* xyz, int64_t M,
                    float* out, void* stream) {
  TfView t;
  if (!make_tf_view(factors, desc, t) || (t.C > 1 && !f_vec) || M < 0) return finish(cudaErrorInvalidValue);
  if (M == 0) return 0;
  const cudaStream_t st = as_stream(stream);
  const bool v4 = tf_records4(t, nullptr);
  switch (t.C) {
    case 1: return v4 ? launch_fwd<1, 4>(t, f_vec, xyz, M, out, st) : launch_fwd<1, 1>(t, f_vec, xyz, M, out, st);
    case 3: return v4 ? launch_fwd<3, 4>(t, f_vec, xyz, M, out, st) : launch_fwd<3, 1>(t, f_vec, xyz, M, out, st);
    default: return v4 ? launch_fwd<12, 4>(t, f_vec, xyz, M, out, st) : launch_fwd<12, 1>(t, f_vec, xyz, M, out, st);
  }
}

int ubn_tensorf_bwd(const float* const* factors, const float* f_vec, const UbnTensorfDesc* desc, const float* xyz, int64_t M,
                    const float* grad_out, float* const* grads, float* grad_f_vec, int vec_copies, float* scratch, void* stream) {
  TfView t;
  TfGrads gr;
  if (!make_tf_view(factors, desc, t) || !make_tf_grads(grads, gr) || !scratch || !aligned16(scratch) || M < 0)
    return finish(cudaErrorInvalidValue);
  if (t.C > 1 && (!f_vec || !grad_f_vec)) return finish(cudaErrorInvalidValue);
  if (vec_copies < 1 || vec_copies > 64) return finish(cudaErrorInvalidValue);
  if (M == 0) return 0;
  const cudaStream_t st = as_stream(stream);
  const int nfeat = 2 * t.R + t.Rxy;
  const int64_t copy_len = tf_copy_len(t);
  float* vcopies = scratch;
  float* fpart = scratch + (int64_t)vec_copies * copy_len;
  const int64_t ntiles = (M + kTfThreads - 1) / kTfThreads;
  const int nblk = (int)(ntiles < UBN_TENSORF_BWD_MAX_CTAS ? ntiles : UBN_TENSORF_BWD_MAX_CTAS);
  cudaError_t e = cudaMemsetAsync(vcopies, 0, (size_t)vec_copies * copy_len * sizeof(float), st);
  if (e != cudaSuccess) return finish(e);
  const bool v4 = tf_records4(t, grads);
  int rc;
  switch (t.C) {
    case 1:
      rc = v4 ? launch_bwd<1, 4>(t, f_vec, xyz, M, grad_out, gr, vcopies, copy_len, vec_copies, fpart, nblk, st)
              : launch_bwd<1, 1>(t, f_vec, xyz, M, grad_out, gr, vcopies, copy_len, vec_copies, fpart, nblk, st);
      break;
    case 3:
      rc = v4 ? launch_bwd<3, 4>(t, f_vec, xyz, M, grad_out, gr, vcopies, copy_len, vec_copies, fpart, nblk, st)
              : launch_bwd<3, 1>(t, f_vec, xyz, M, grad_out, gr, vcopies, copy_len, vec_copies, fpart, nblk, st);
      break;
    default:
      rc = v4 ? launch_bwd<12, 4>(t, f_vec, xyz, M, grad_out, gr, vcopies, copy_len, vec_copies, fpart, nblk, st)
              : launch_bwd<12, 1>(t, f_vec, xyz, M, grad_out, gr, vcopies, copy_len, vec_copies, fpart, nblk, st);
      break;
  }
  if (rc) return rc;
  const int nfc = t.C > 1 ? nfeat * t.C : 0;
  const int64_t n = copy_len + nfc;
  k_tensorf_bwd_finish<<<blocks_for(n, 256), 256, 0, st>>>(t, gr, vcopies, copy_len, vec_copies, fpart, nblk, nfc, grad_f_vec);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_tensorf_tv_add_grad(const float* const* factors, float* const* grads, const UbnTensorfDesc* desc, float wx, float wy,
                            float wz, void* stream) {
  TfView t;
  TfGrads gr;
  if (!make_tf_view(factors, desc, t) || !make_tf_grads(grads, gr)) return finish(cudaErrorInvalidValue);
  const int X = t.S[0], Y = t.S[1], Z = t.S[2];
  const float w[3] = {wx / 6.f, wy / 6.f, wz / 6.f};
  TfTv tv;
  const int A[6] = {X, X, Y, X, Y, Z}, B[6] = {Y, Z, Z, 1, 1, 1}, n[6] = {t.Rxy, t.R, t.R, t.R, t.R, t.Rxy};
  const int ax_a[6] = {0, 0, 1, 0, 1, 2}, ax_b[6] = {1, 2, 2, 0, 0, 0};
  tv.start[0] = 0;
  for (int f = 0; f < 6; ++f) {
    tv.A[f] = A[f]; tv.B[f] = B[f]; tv.n[f] = n[f];
    tv.ca[f] = w[ax_a[f]];
    tv.cb[f] = w[ax_b[f]];
    tv.start[f + 1] = tv.start[f] + (int64_t)A[f] * B[f] * n[f];
  }
  k_tensorf_tv<<<blocks_for(tv.start[6], 256), 256, 0, as_stream(stream)>>>(t, gr, tv);
  UBN_LAUNCH_CHECK();
  return 0;
}

int ubn_tensorf_dense(const float* const* factors, const float* f_vec, const UbnTensorfDesc* desc, float* out, void* stream) {
  TfView t;
  if (!make_tf_view(factors, desc, t) || (t.C > 1 && !f_vec) || !out) return finish(cudaErrorInvalidValue);
  const int64_t nv = (int64_t)t.S[0] * t.S[1] * t.S[2];
  const size_t smem = t.C > 1 ? (size_t)(2 * t.R + t.Rxy) * t.C * sizeof(float) : 0;
  const cudaStream_t st = as_stream(stream);
  switch (t.C) {
    case 1: k_tensorf_dense<1><<<blocks_for(nv, 256), 256, smem, st>>>(t, f_vec, out); break;
    case 3: k_tensorf_dense<3><<<blocks_for(nv, 256), 256, smem, st>>>(t, f_vec, out); break;
    default: k_tensorf_dense<12><<<blocks_for(nv, 256), 256, smem, st>>>(t, f_vec, out); break;
  }
  UBN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
