// TMA bulk-store write-stream ceiling: can ONE small CTA per SM, staging 8 KB tiles in
// shared memory and issuing cp.async.bulk.global.shared::cta stores from one elected thread, keep
// the HBM write stream of the dense-matrix kernel at its ceiling?  (k_score_emit's per-thread
// st.global.cs.v4 stream needs 6 CTAs x 256 threads per SM and most of the issue slots; a bulk-store
// version leaves the SM to the selection kernel running beside it.)
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_fill tma_fill.cu && ./tma_fill
// Work = `tiles` tiles of TILE floats, each stored `reps` times to consecutive rows (the role row
// broadcast to its replicas); segments are taken from a global atomic counter (dynamic balance).
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

constexpr int TILE = 2048;  // floats per tile (8 KB)

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src_smem, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src_smem)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <int STAGES>
__global__ void __launch_bounds__(128) k_tma_fill(float* __restrict__ out, const float* __restrict__ base, int tiles, int reps,
                                                  int* __restrict__ counter) {
  extern __shared__ __align__(128) float smem[];
  __shared__ int s_tile;
  const int tid = threadIdx.x;
  int it = 0;
  while (true) {
    if (tid == 0) {
      s_tile = atomicAdd(counter, 1);
      bulk_wait_read<STAGES - 1>();  // the stores that read this stage STAGES iterations ago are done with it
    }
    __syncthreads();
    const int t = s_tile;
    if (t >= tiles) break;
    float* st = smem + (size_t)(it % STAGES) * TILE;
    // "compute" the tile: need * base, 16 floats per thread
    const float need = (float)(t & 7);
    for (int i = tid; i < TILE / 4; i += 128) {
      float4 b = __ldg(reinterpret_cast<const float4*>(base) + ((t & 3) * (TILE / 4) + i));
      b.x *= need; b.y *= need; b.z *= need; b.w *= need;
      reinterpret_cast<float4*>(st)[i] = b;
    }
    fence_async_smem();
    __syncthreads();
    if (tid == 0) {
      float* dst = out + (size_t)t * reps * TILE;
      for (int r = 0; r < reps; ++r) bulk_s2g(dst + (size_t)r * TILE, st, TILE * 4);
      bulk_commit();
    }
    ++it;
  }
  if (tid == 0) bulk_wait_read<0>();
}

// Per-WARP workers, shaped like the dense-matrix kernel: an item = a sub-chunk of SUB nodes x a block
// of GT role rows ("tiles").  The warp loads the sub-chunk's node operands into registers ONCE
// (SUB/32 floats per lane), prefetches the index of its next item, then per role row only
// computes from registers, writes its private 2 KB stage (ring of STAGES), and lane 0 issues `reps`
// bulk stores.  No block barrier anywhere, only __syncwarp.
template <int STAGES, int SUB>
__global__ void __launch_bounds__(512) k_tma_fill_warp(float* __restrict__ out, const float* __restrict__ base, int tiles, int reps,
                                                       int* __restrict__ counter) {
  extern __shared__ __align__(128) float smem[];
  constexpr int GT = 8;             // role rows per item
  constexpr int V = SUB / 128;      // float4 per lane
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* ring = smem + (size_t)warp * STAGES * SUB;
  const int subs = TILE / SUB;
  const int items = (tiles / GT) * subs;
  int it = 0;
  int next = 0;
  if (lane == 0) next = atomicAdd(counter, 1);
  next = __shfl_sync(0xFFFFFFFFu, next, 0);
  while (next < items) {
    const int t = next;
    if (lane == 0) next = atomicAdd(counter, 1);  // in flight during this item
    const int blk = t / subs, q = t % subs;
    float4 b[V];
#pragma unroll
    for (int j = 0; j < V; ++j)
      b[j] = __ldg(reinterpret_cast<const float4*>(base) + ((blk & 3) * (TILE / 4) + q * (SUB / 4) + lane + 32 * j));
    for (int g = 0; g < GT; ++g) {
      const int tile = blk * GT + g;
      if (lane == 0) bulk_wait_read<STAGES - 1>();
      __syncwarp();
      float* st = ring + (size_t)(it % STAGES) * SUB;
      const float need = (float)(tile & 7);
#pragma unroll
      for (int j = 0; j < V; ++j) {
        float4 o;
        o.x = b[j].x >= 0.f ? need * b[j].x : -1.f;
        o.y = b[j].y >= 0.f ? need * b[j].y : -1.f;
        o.z = b[j].z >= 0.f ? need * b[j].z : -1.f;
        o.w = b[j].w >= 0.f ? need * b[j].w : -1.f;
        reinterpret_cast<float4*>(st)[lane + 32 * j] = o;
      }
      fence_async_smem();
      __syncwarp();
      if (lane == 0) {
        float* dst = out + (size_t)tile * reps * TILE + q * SUB;
        for (int r = 0; r < reps; ++r) bulk_s2g(dst + (size_t)r * TILE, st, SUB * 4);
        bulk_commit();
      }
      ++it;
    }
    next = __shfl_sync(0xFFFFFFFFu, next, 0);
  }
  if (lane == 0) bulk_wait_read<0>();
}

template <int STAGES, int SUB>
float run_tma_warp(float* out, const float* base, int tiles, int reps, int* ctr, int grid, int threads, int iters) {
  const int smem = (threads / 32) * STAGES * SUB * 4;
  cudaFuncSetAttribute(k_tma_fill_warp<STAGES, SUB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  float best = 1e9f;
  for (int i = 0; i < iters; ++i) {
    cudaMemsetAsync(ctr, 0, 4);
    cudaEventRecord(a);
    k_tma_fill_warp<STAGES, SUB><<<grid, threads, smem>>>(out, base, tiles, reps, ctr);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    if (i >= 2 && ms < best) best = ms;
  }
  if (cudaGetLastError() != cudaSuccess) return -1.f;
  return best;
}

// reference: the round-1 pattern (one tile per CTA, st.global.cs.v4 per thread)
__global__ void __launch_bounds__(256) k_st_fill(float* __restrict__ out, const float* __restrict__ base, int reps) {
  const int t = blockIdx.x;
  const float need = (float)(t & 7);
  for (int i = threadIdx.x; i < TILE / 4; i += 256) {
    float4 b = __ldg(reinterpret_cast<const float4*>(base) + ((t & 3) * (TILE / 4) + i));
    b.x *= need; b.y *= need; b.z *= need; b.w *= need;
    float* p = out + (size_t)t * reps * TILE + 4 * i;
    for (int r = 0; r < reps; ++r) {
      asm volatile("st.global.cs.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(b.x), "f"(b.y), "f"(b.z), "f"(b.w) : "memory");
      p += TILE;
    }
  }
}

template <int STAGES>
float run_tma(float* out, const float* base, int tiles, int reps, int* ctr, int grid, int iters) {
  cudaFuncSetAttribute(k_tma_fill<STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGES * TILE * 4);
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  float best = 1e9f;
  for (int i = 0; i < iters; ++i) {
    cudaMemsetAsync(ctr, 0, 4);
    cudaEventRecord(a);
    k_tma_fill<STAGES><<<grid, 128, STAGES * TILE * 4>>>(out, base, tiles, reps, ctr);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    if (i >= 2 && ms < best) best = ms;
  }
  return best;
}

int main(int argc, char** argv) {
  const size_t bytes = argc > 1 ? (size_t)atoll(argv[1]) << 20 : (size_t)287 << 20;
  int sm = 132;
  cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, 0);
  float *out, *base;
  int* ctr;
  cudaMalloc(&out, bytes + (1 << 20));
  cudaMalloc(&base, 4 * TILE * 4);
  cudaMalloc(&ctr, 4);
  cudaMemset(base, 0, 4 * TILE * 4);
  for (int reps : {1, 2, 3}) {
    const int tiles = (int)(bytes / ((size_t)TILE * 4 * reps));
    const double gb = (double)tiles * reps * TILE * 4 / 1e9;
    {
      cudaEvent_t a, b;
      cudaEventCreate(&a);
      cudaEventCreate(&b);
      float best = 1e9f;
      for (int i = 0; i < 8; ++i) {
        cudaEventRecord(a);
        k_st_fill<<<tiles, 256>>>(out, base, reps);
        cudaEventRecord(b);
        cudaEventSynchronize(b);
        float ms;
        cudaEventElapsedTime(&ms, a, b);
        if (i >= 2 && ms < best) best = ms;
      }
      printf("reps %d  st.global.cs.v4, one tile per CTA (%d CTAs x 256 thr): %.1f us  %.0f GB/s\n", reps, tiles, best * 1e3, gb / (best * 1e-3));
    }
    for (int per_sm : {1, 2, 3}) {
      const int grid = sm * per_sm;
      printf("reps %d  TMA bulk store, %d CTA/SM x 128 thr:", reps, per_sm);
      float t4 = run_tma<4>(out, base, tiles, reps, ctr, grid, 8);
      float t8 = run_tma<8>(out, base, tiles, reps, ctr, grid, 8);
      printf("  4 stages %.1f us %.0f GB/s | 8 stages %.1f us %.0f GB/s", t4 * 1e3, gb / (t4 * 1e-3), t8 * 1e3, gb / (t8 * 1e-3));
      if (per_sm <= 2) {
        float t12 = run_tma<12>(out, base, tiles, reps, ctr, grid, 8);
        printf(" | 12 stages %.1f us %.0f GB/s", t12 * 1e3, gb / (t12 * 1e-3));
      }
      if (per_sm == 1) {
        float t24 = run_tma<24>(out, base, tiles, reps, ctr, grid, 8);
        printf(" | 24 stages %.1f us %.0f GB/s", t24 * 1e3, gb / (t24 * 1e-3));
      }
      printf("\n");
    }
  }
  for (int reps : {1, 2}) {
    const int tiles = (int)(bytes / ((size_t)TILE * 4 * reps)) / 8 * 8;
    const double gb = (double)tiles * reps * TILE * 4 / 1e9;
    for (int warps : {2, 4, 8, 12, 16}) {
      printf("reps %d  per-warp TMA workers, %2d warps/SM (1 CTA/SM):", reps, warps);
      float a2 = run_tma_warp<2, 512>(out, base, tiles, reps, ctr, sm, warps * 32, 8);
      float a4 = run_tma_warp<4, 512>(out, base, tiles, reps, ctr, sm, warps * 32, 8);
      float a8 = warps <= 12 ? run_tma_warp<8, 512>(out, base, tiles, reps, ctr, sm, warps * 32, 8) : -1.f;
      float b2 = run_tma_warp<2, 1024>(out, base, tiles, reps, ctr, sm, warps * 32, 8);
      float b4 = warps <= 12 ? run_tma_warp<4, 1024>(out, base, tiles, reps, ctr, sm, warps * 32, 8) : -1.f;
      printf("  2 KB stores: 2 st %.1f us %.0f | 4 st %.1f us %.0f | 8 st %.1f us %.0f GB/s  ||  4 KB stores: 2 st %.1f us %.0f | 4 st %.1f us %.0f GB/s\n",
             a2 * 1e3, gb / (a2 * 1e-3), a4 * 1e3, gb / (a4 * 1e-3), a8 * 1e3, gb / (a8 * 1e-3), b2 * 1e3, gb / (b2 * 1e-3), b4 * 1e3, gb / (b4 * 1e-3));
    }
  }
  cudaError_t e = cudaDeviceSynchronize();
  printf("status: %s\n", cudaGetErrorString(e));
  return e != cudaSuccess;
}
