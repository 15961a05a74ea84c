// emit_tma.cuh — k_emit_tma: the dense (replica x node) matrix of a multi-wave plan written with
// TMA bulk stores from shared memory (cp.async.bulk.global.shared::cta), DESIGN.md §4.2.
//
// Why a second emit kernel.  k_score_emit (score.cuh) streams the matrix with per-thread
// st.global.cs.v4: it needs 6 CTAs x 256 threads per SM (61 K registers) and most of the issue slots
// to keep HBM busy, so nothing else fits on the SM beside it — running the selection kernel
// concurrently made the step slower than running the two in series.  Here one elected lane
// issues a 2 KB bulk store per replica row and the TMA engine moves the bytes: 8 warps per SM
// (one 256-thread CTA, 34 KB of shared memory) come close to the plain-store write bandwidth
// (profiles/microbench/tma_fill.cu measures both),
// and 3/4 of the SM's registers and shared memory are left for k_plan_group, which runs BESIDE this
// kernel on a second stream.
//
// Structure: persistent grid (one CTA per SM), every WARP is an independent worker.
//   item  = a sub-chunk of EMIT_SUB = 512 nodes of this rank's slab x a block of `bsteps` consecutive
//           steps; items are taken from a global atomic counter (dynamic balance: with a static split
//           the slowest SM sets the time), the index of the next item is
//           fetched while the current one is processed;
//   setup = the sub-chunk's node operands (base, free: 16 floats / ints per lane) into registers and
//           the steps' emit records (emit table: 12 words per step, written once when the batch is
//           staged) into the warp's shared memory — one round of loads per item;
//   tile  = one role row of one step over the sub-chunk: S = need * base where the node is feasible
//           (free >= demand, exclusive roles: domain unowned or ours), else -inf, computed from
//           registers into the warp's private ring of EMIT_STAGES x 2 KB, fence.proxy.async,
//           __syncwarp, then lane 0 issues one bulk store per replica of the role and commits the
//           group; cp.async.bulk.wait_group.read frees a stage for reuse.  No block barrier anywhere.
// Bit-identical to k_score_emit<false> (same expression per element; tests/test_gpu_*).
#pragma once
#include "kernels.cuh"

namespace rbgtopo {

constexpr int EMIT_SUB = 512;                 // nodes per item (2 KB per row store)
constexpr int EMIT_WARPS = 8;                 // warps per CTA (one CTA per SM)
constexpr int EMIT_MAX_BSTEPS = 8;

__host__ __device__ inline size_t emit_tma_smem_bytes(int stages) {
  return (size_t)EMIT_WARPS * ((size_t)stages * EMIT_SUB * 4 + EMIT_MAX_BSTEPS * EMIT_TAB_WORDS * 4);
}

__device__ __forceinline__ void bulk_s2g(void* dst, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src_smem)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// One tile of an exclusive role (out of line on purpose, see the call site; it reloads the node
// operands itself so that the caller's register arrays never get an address).
template <int V>
__device__ __noinline__ void emit_tile_excl(const int* __restrict__ free_, const float* __restrict__ base,
                                            const int* __restrict__ owner0, const int* __restrict__ lvl_owner, int ls,
                                            int level, float* st, int n0, int n1, int gid, int demand, float need) {
  const int lane = threadIdx.x & 31;
  // the owner vector of the step's exclusive level (DESIGN.md §3.9), picked here to keep it off the caller's registers
  const int* __restrict__ node_owner = level > 0 ? lvl_owner + (size_t)level * ls : owner0;
  const int len4 = (n1 - n0 + 3) >> 2;
#pragma unroll
  for (int j = 0; j < V; ++j) {
    const int g = lane + 32 * j;
    float4 o4 = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    if (g < len4) {
      const int n = n0 + (g << 2);
      const float4 b4 = __ldg(reinterpret_cast<const float4*>(base + n));
      int4 a = __ldg(reinterpret_cast<const int4*>(free_ + n));
      const int4 ow = __ldg(reinterpret_cast<const int4*>(node_owner + n));
      if (n + 1 >= n1) a.y = -1;  // lanes past the slab are infeasible
      if (n + 2 >= n1) a.z = -1;
      if (n + 3 >= n1) a.w = -1;
      if (!(ow.x == -1 || ow.x == gid)) a.x = -1;
      if (!(ow.y == -1 || ow.y == gid)) a.y = -1;
      if (!(ow.z == -1 || ow.z == gid)) a.z = -1;
      if (!(ow.w == -1 || ow.w == gid)) a.w = -1;
      o4.x = a.x >= demand ? need * b4.x : -INFINITY;
      o4.y = a.y >= demand ? need * b4.y : -INFINITY;
      o4.z = a.z >= demand ? need * b4.z : -INFINITY;
      o4.w = a.w >= demand ? need * b4.w : -INFINITY;
    }
    reinterpret_cast<float4*>(st)[g] = o4;
  }
}

// ctr[0] = item queue, ctr[1] = warps that left the loop (the last one resets both for the next launch)
// STAGES = ring depth per warp; MINB = __launch_bounds__ min blocks (4 caps the kernel at 64 registers so
// that 6 CTAs of k_plan_group fit beside it); CLK = per-warp phase clocks into `clk` (profiling builds of
// the launch: RBGTOPO_EMIT_CLOCKS), [warp][4] = setup, wait, compute, issue cycles.
template <int STAGES, int MINB, bool CLK>
__global__ void __launch_bounds__(32 * EMIT_WARPS, MINB)
k_emit_tma(TopoDev t, BatchDev b, const int* __restrict__ etab, int subs, int items, int* __restrict__ ctr,
           long long* __restrict__ clk) {
  extern __shared__ __align__(128) unsigned char em_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* const ring = reinterpret_cast<float*>(em_smem) + (size_t)warp * STAGES * EMIT_SUB;
  int* const sTab = reinterpret_cast<int*>(em_smem + (size_t)EMIT_WARPS * STAGES * EMIT_SUB * 4) +
                    warp * EMIT_MAX_BSTEPS * EMIT_TAB_WORDS;
  const int BS = b.bsteps;
  const size_t stride = (size_t)t.slab_stride;
  constexpr int V = EMIT_SUB / 128;  // float4 groups per lane
  long long c_setup = 0, c_wait = 0, c_comp = 0, c_issue = 0, c0 = 0;
  int n_items = 0, n_tiles = 0;

  int it = 0;
  int next = 0;
  if (lane == 0) next = atomicAdd(&ctr[0], 1);
  next = __shfl_sync(FULL, next, 0);
  while (next < items) {
    if (CLK) c0 = clock64();
    const int item = next;
    if (lane == 0) next = atomicAdd(&ctr[0], 1);  // in flight while this item is processed
    const int blk = item / subs, sub = item - blk * subs;
    const int step0 = blk * BS;
    const int nst = min(b.n_steps, step0 + BS) - step0;
    const int n0 = t.slab_lo + sub * EMIT_SUB;
    const int n1 = min(n0 + EMIT_SUB, t.slab_hi);
    const int len4 = (n1 - n0 + 3) >> 2;  // float4 groups of the sub-chunk (the last one is padded with -inf)
    // ---- setup: ONE round of loads — the steps' emit records (lanes < 3 * nst, 16 bytes each) and the
    //      node operands are all issued before anything waits on them
    int4 tabv = make_int4(0, 0, 0, 0);
    if (lane < nst * (EMIT_TAB_WORDS / 4))
      tabv = __ldg(reinterpret_cast<const int4*>(etab + (size_t)step0 * EMIT_TAB_WORDS) + lane);
    float4 base4[V];
    int4 av[V];
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const int g = lane + 32 * j;
      base4[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      av[j] = make_int4(-1, -1, -1, -1);
      if (g < len4) {
        const int n = n0 + (g << 2);
        base4[j] = __ldg(reinterpret_cast<const float4*>(t.base + n));
        av[j] = __ldg(reinterpret_cast<const int4*>(t.free_ + n));  // padded past n: safe
        if (n + 4 > n1) {  // only in the slab's last group: lanes past the slab are infeasible
          if (n + 1 >= n1) av[j].y = -1;
          if (n + 2 >= n1) av[j].z = -1;
          av[j].w = -1;
        }
      }
    }
    __syncwarp();  // the previous item's readers of sTab are done
    if (lane < nst * (EMIT_TAB_WORDS / 4)) reinterpret_cast<int4*>(sTab)[lane] = tabv;
    __syncwarp();
    float* const col0 = b.matrix + (n0 - t.slab_lo);
    const uint32_t row_bytes = (uint32_t)len4 * 16u;
    if (CLK) { const long long c1 = clock64(); c_setup += c1 - c0; c0 = c1; ++n_items; }
    for (int si = 0; si < nst; ++si) {
      const int* e = sTab + si * EMIT_TAB_WORDS;
      const int gid = e[0], P = e[2];
      const bool excl_step = (e[1] & RBGTOPO_STEP_EXCLUSIVE) != 0;
      float* rowp = col0 + (size_t)e[3] * stride;
      for (int p = 0; p < P; ++p) {
        const int pr = e[4 + p];
        const int count = pr & 63, demand = pr >> 12;
        const float need = (float)((pr >> 6) & 31);
        const bool rexcl = (pr >> 11) & 1;
        float* const st = ring + (size_t)(it % STAGES) * EMIT_SUB;
        bulk_wait_read<STAGES - 1>();  // this lane's stores that read the stage are done with it (a lane commits <= 1 group per tile)
        __syncwarp();
        if (CLK) { const long long c1 = clock64(); c_wait += c1 - c0; c0 = c1; }
        if (rexcl && excl_step) {
          // rare: exclusive role of an exclusive step — domains owned by another group are infeasible.
          // Kept out of line so that the common path below stays short (inlined and predicated off, it
          // costs issue slots on every tile).
          emit_tile_excl<V>(t.free_, t.base, t.node_owner, t.lvl_owner, level_stride(t.n), step_level(e[1]), st, n0, n1, gid,
                            demand, need);
        } else {
#pragma unroll
          for (int j = 0; j < V; ++j) {
            float4 o4;
            o4.x = av[j].x >= demand ? need * base4[j].x : -INFINITY;
            o4.y = av[j].y >= demand ? need * base4[j].y : -INFINITY;
            o4.z = av[j].z >= demand ? need * base4[j].z : -INFINITY;
            o4.w = av[j].w >= demand ? need * base4[j].w : -INFINITY;
            reinterpret_cast<float4*>(st)[lane + 32 * j] = o4;
          }
        }
        fence_async_smem();
        __syncwarp();
        if (CLK) { const long long c1 = clock64(); c_comp += c1 - c0; c0 = c1; ++n_tiles; }
        // lane c issues the store of replica c (the issue sequence per store — address into uniform
        // registers, UBLKCP — costs ~250 cycles; one lane doing all of them serialised the warp);
        // every lane commits one (possibly empty) bulk group per tile and waits on its own groups
        if (lane < count) bulk_s2g(rowp + (size_t)lane * stride, st, row_bytes);
        bulk_commit();  // every lane, every tile (an empty group completes at once): wait_group counts tiles
        rowp += (size_t)count * stride;
        ++it;
        if (CLK) { const long long c1 = clock64(); c_issue += c1 - c0; c0 = c1; }
      }
    }
    next = __shfl_sync(FULL, next, 0);
  }
  bulk_wait_all();  // every store of this lane has been written
  __syncwarp();
  if (lane == 0) {
    if (CLK) {
      long long* o = clk + (size_t)(blockIdx.x * EMIT_WARPS + warp) * 8;
      o[0] = c_setup; o[1] = c_wait; o[2] = c_comp; o[3] = c_issue; o[4] = n_items; o[5] = n_tiles;
    }
    const int total = (int)(gridDim.x * EMIT_WARPS);
    if (atomicAdd(&ctr[1], 1) == total - 1) {  // everybody left the loop: re-arm the queue
      ctr[0] = 0;
      ctr[1] = 0;
      __threadfence();
    }
  }
}

}  // namespace rbgtopo
