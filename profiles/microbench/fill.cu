// Write-stream microbenchmark: what does a pure float4 store stream reach on this
// GPU, for the two output sizes of the bench waves (41 MB, 205 MB)?
// Variants: store flavour (default / .cs / .wt), grid size, bytes per thread-iteration.
#include <cstdio>
#include <cuda_runtime.h>
template <int MODE>
__device__ __forceinline__ void st4(float* p, float4 v) {
  if (MODE == 0) *reinterpret_cast<float4*>(p) = v;
  else if (MODE == 1) asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
  else asm volatile("st.global.wt.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// each CTA gets a contiguous range of `per` tiles of 2048 floats; 256 threads x 2 float4
template <int MODE>
__global__ void __launch_bounds__(256) fill(float* out, const float* __restrict__ base, int tiles, float s) {
  const int per = (tiles + gridDim.x - 1) / gridDim.x;
  const int t0 = blockIdx.x * per, t1 = min(tiles, t0 + per);
  for (int t = t0; t < t1; ++t) {
    const int n0 = (t % 5) * 2048;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int g = threadIdx.x + j * 256;
      float4 b4 = __ldg(reinterpret_cast<const float4*>(base + n0 + g * 4));
      b4.x *= s; b4.y *= s; b4.z *= s; b4.w *= s;
      st4<MODE>(out + (size_t)t * 2048 + g * 4, b4);
    }
  }
}
int main() {
  float *out, *base;
  const size_t maxb = 256u << 20;
  cudaMalloc(&out, maxb); cudaMalloc(&base, 1 << 20); cudaMemset(base, 0, 1 << 20);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  int sm = 132;
  cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, 0);
  for (size_t mb : {41, 205}) {
    const int tiles = (int)(mb * 1000000 / 8192);
    for (int mode = 0; mode < 3; ++mode)
      for (int grid : {sm * 4, sm * 6, sm * 8, sm * 16, tiles}) {
        float best = 1e9;
        for (int it = 0; it < 6; ++it) {
          cudaEventRecord(a);
          if (mode == 0) fill<0><<<grid, 256>>>(out, base, tiles, 2.f);
          if (mode == 1) fill<1><<<grid, 256>>>(out, base, tiles, 2.f);
          if (mode == 2) fill<2><<<grid, 256>>>(out, base, tiles, 2.f);
          cudaEventRecord(b); cudaEventSynchronize(b);
          float ms; cudaEventElapsedTime(&ms, a, b); if (it > 1 && ms < best) best = ms;
        }
        printf("MB=%zu mode=%d grid=%d  %.1f us  %.0f GB/s\n", mb, mode, grid, best * 1e3, mb * 1e-3 / (best * 1e-3));
      }
  }
  return 0;
}
