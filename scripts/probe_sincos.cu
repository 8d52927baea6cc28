// Is sincosf(a) bit-identical to (sinf(a), cosf(a)) on this toolchain / GPU for every float |a| <= 8 (the argument range of the
// FourierGrid warps 2^k x, |x| <= 1, k <= 3)?  If so the march kernels may share one range reduction per (axis, frequency).
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a scripts/probe_sincos.cu -o scripts/_bin/probe_sincos && scripts/_bin/probe_sincos
#include <cstdio>
#include <cstdint>
__global__ void k(unsigned long long* bad_s, unsigned long long* bad_c, uint32_t max_bits) {
  unsigned long long bs = 0, bc = 0;
  for (uint64_t b = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; b <= max_bits; b += (uint64_t)gridDim.x * blockDim.x) {
    for (int sgn = 0; sgn < 2; ++sgn) {
      const float a = __uint_as_float((uint32_t)b | (sgn ? 0x80000000u : 0u));
      float s2, c2;
      sincosf(a, &s2, &c2);
      const float s1 = sinf(a), c1 = cosf(a);
      bs += __float_as_uint(s1) != __float_as_uint(s2);
      bc += __float_as_uint(c1) != __float_as_uint(c2);
    }
  }
  atomicAdd(bad_s, bs);
  atomicAdd(bad_c, bc);
}
int main() {
  unsigned long long *d, h[2] = {0, 0};
  cudaMalloc(&d, 16);
  cudaMemcpy(d, h, 16, cudaMemcpyHostToDevice);
  const uint32_t max_bits = 0x41000000u;   // 8.0f
  k<<<132 * 16, 256>>>(d, d + 1, max_bits);
  cudaMemcpy(h, d, 16, cudaMemcpyDeviceToHost);
  printf("{\"probe\": \"sincosf vs sinf/cosf, all floats |a| <= 8\", \"n\": %llu, \"sin_mismatch\": %llu, \"cos_mismatch\": %llu, \"err\": \"%s\"}\n",
         2ull * ((unsigned long long)max_bits + 1), h[0], h[1], cudaGetErrorString(cudaGetLastError()));
  return 0;
}
