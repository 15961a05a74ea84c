// Which feature of k_score_emit costs bandwidth?  Progressive variants on the
// bench's output shape: 3072 steps (R = 1,5,1 per group-wave, wave-major) x 10000
// nodes, row stride 10016 floats, 5 chunks of 2048 per step, 6 / 12 / 16 persistent CTAs
// per SM with byte-balanced contiguous ranges.
//   V0 stores only            V1 + base/free loads + compare/select
//   V2 + per-step header/role loads (dependent chain)   V3 = V2 with 128-thread CTAs
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
__device__ __forceinline__ void st4(float* p, float4 v) {
  asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
struct Step { int R, rep_off, role_off, pad; };
template <int V, int THREADS>
__global__ void __launch_bounds__(THREADS) emit(float* out, const float* __restrict__ base, const int* __restrict__ fre,
                                                const Step* __restrict__ steps, const int4* __restrict__ roles,
                                                const int* __restrict__ cta_item, int items) {
  const int item0 = cta_item[blockIdx.x], item1 = min(items, cta_item[blockIdx.x + 1]);
  constexpr int GROUPS = 512, GPT = GROUPS / THREADS;
  for (int item = item0; item < item1; ++item) {
    const int step = item / 5, ch = item % 5;
    int R = 1, rep = step, demand = 1; float need = 2.f;
    if (V >= 2) { Step s = steps[step]; R = s.R; rep = s.rep_off; int4 r = __ldg(roles + s.role_off); demand = r.y; need = (float)r.z; }
    else { const int w = step / 1024; R = w == 1 ? 5 : 1; rep = w == 0 ? step : (w == 1 ? 1024 + (step - 1024) * 5 : 6144 + step - 2048); }
    const int n0 = ch * 2048, n1 = min(n0 + 2048, 10000);
#pragma unroll
    for (int j = 0; j < GPT; ++j) {
      const int g = threadIdx.x + j * THREADS, n = n0 + g * 4;
      if (n < n1) {
        float4 o = make_float4(1.f, 2.f, 3.f, 4.f);
        if (V >= 1) {
          const float4 b4 = __ldg(reinterpret_cast<const float4*>(base + n));
          const int4 a = __ldg(reinterpret_cast<const int4*>(fre + n));
          o.x = a.x >= demand ? need * b4.x : -INFINITY; o.y = a.y >= demand ? need * b4.y : -INFINITY;
          o.z = a.z >= demand ? need * b4.z : -INFINITY; o.w = a.w >= demand ? need * b4.w : -INFINITY;
        }
        float* p = out + (size_t)rep * 10016 + n;
        for (int c = 0; c < R; ++c) { st4(p, o); p += 10016; }
      }
    }
  }
}
int main() {
  const int G = 1024, NS = 3 * G, TR = 7 * G, ITEMS = NS * 5;
  float *out, *base; int *fre, *cta; Step* steps; int4* roles;
  cudaMalloc(&out, (size_t)TR * 10016 * 4); cudaMalloc(&base, 16384 * 4); cudaMalloc(&fre, 16384 * 4);
  cudaMemset(base, 0, 16384 * 4); cudaMemset(fre, 1, 16384 * 4);
  std::vector<Step> hs(NS); std::vector<int4> hr(NS);
  int rep = 0;
  for (int s = 0; s < NS; ++s) { int R = (s / G == 1) ? 5 : 1; hs[s] = {R, rep, s, 0}; rep += R; hr[s] = make_int4(R, 1, 2, 1); }
  cudaMalloc(&steps, NS * sizeof(Step)); cudaMalloc(&roles, NS * 16);
  cudaMemcpy(steps, hs.data(), NS * sizeof(Step), cudaMemcpyHostToDevice); cudaMemcpy(roles, hr.data(), NS * 16, cudaMemcpyHostToDevice);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  int sm = 132;
  cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, 0);
  for (int grid : {sm * 6, sm * 12, sm * 16}) {
    std::vector<int> ci(grid + 1, ITEMS);
    long long total = (long long)TR * 5; int s = 0;
    for (int g = 0; g < grid; ++g) {
      long long target = total * g / grid;
      while (s < NS && (long long)(hs[s].rep_off + hs[s].R) * 5 <= target) ++s;
      if (s >= NS) break;
      long long before = (long long)hs[s].rep_off * 5;
      int ch = target <= before ? 0 : (int)((target - before + hs[s].R - 1) / hs[s].R);
      ci[g] = s * 5 + (ch > 5 ? 5 : ch);
    }
    ci[0] = 0;
    cudaMalloc(&cta, (grid + 1) * 4); cudaMemcpy(cta, ci.data(), (grid + 1) * 4, cudaMemcpyHostToDevice);
    for (int v = 0; v < 4; ++v) {
      float best = 1e9;
      for (int it = 0; it < 6; ++it) {
        cudaEventRecord(a);
        if (v == 0) emit<0, 256><<<grid, 256>>>(out, base, fre, steps, roles, cta, ITEMS);
        if (v == 1) emit<1, 256><<<grid, 256>>>(out, base, fre, steps, roles, cta, ITEMS);
        if (v == 2) emit<2, 256><<<grid, 256>>>(out, base, fre, steps, roles, cta, ITEMS);
        if (v == 3) emit<2, 128><<<grid * 2 > 0 ? grid : grid, 128>>>(out, base, fre, steps, roles, cta, ITEMS);
        cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b); if (it > 1 && ms < best) best = ms;
      }
      printf("grid=%d V%d  %.1f us  %.0f GB/s  (%s)\n", grid, v, best * 1e3, TR * 10000.0 * 4 / 1e9 / (best * 1e-3), cudaGetErrorString(cudaGetLastError()));
    }
    cudaFree(cta);
  }
  return 0;
}
