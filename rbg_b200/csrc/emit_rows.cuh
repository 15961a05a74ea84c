// emit_rows.cuh — k_emit_rows: the dense (replica x node) matrix of a multi-wave plan, walked by ROWS
// (DESIGN.md §4.2).  Default dense-matrix kernel of rbgtopo_place_groups / plan batches.
//
// k_score_emit<false, ETAB> (score.cuh) walks steps -> roles -> replicas; on fleets whose waves hold one
// or two replicas per role (cfg3: 1 / 5 / 1 rows per step) that loop nest costs tens of warp instructions
// per 512-byte warp store and the kernel is issue-bound below the HBM peak, while the same kernel comes
// close to it on cfg4 (8 replicas per role).
// Here the unit is the dense row: the plan's row table (kernels.cuh: rtab, written by k_plan_etab on the
// device) says per row what the row needs — need, demand and, for exclusive rows only, the group — and the
// inner loop is  LDS.64 record -> 2 x (4 FMUL + 4 ISETP + 4 FSEL + STG.128)  with nothing per step.
// One CTA (256 threads) = one SEGMENT: `rb` consecutive rows x a chunk of <= 2048 nodes of this rank's
// slab; the node operands (base, free) of a thread's two float4 groups are loaded once per segment.
// All segments form the grid; the hardware scheduler balances them.
// Bit-identical to k_score_emit<false, *>: same operands, same fp32 product, same -inf rule.
#pragma once
#include "score.cuh"

namespace rbgtopo {

constexpr int EMIT_ROWS_MAX = 64;  // upper bound of the rows of a segment (rb)
#ifndef EMIT_ROWS_MIN_CTAS
#define EMIT_ROWS_MIN_CTAS 6
#endif
#ifdef RBGTOPO_PHASE_CLOCKS  // one-off instrumentation: globaltimer at the end of the last CTA of any k_emit_rows launch
__device__ unsigned long long g_emit_end_ns;
#endif

// EXCL = false: no group of the batch is exclusive (the host knows after validating the groups) — the
// owner path is not even compiled in.
template <bool EXCL>
__global__ void __launch_bounds__(SCORE_THREADS, EMIT_ROWS_MIN_CTAS)
k_emit_rows(TopoDev t, float* __restrict__ matrix, const int2* __restrict__ rtab, int n_rows, int lc, int T, int rb) {
  __shared__ int2 sRow[EMIT_ROWS_MAX];  // {need as fp32 bits, demand (bit 31: exclusive row)}
  __shared__ int sGid[EMIT_ROWS_MAX];
  // every segment is scheduled before the dependents may start: k_plan_group's CTAs (launched as a programmatic
  // dependent) fill the SMs as the last segments drain, and wait before they touch the matrix
  pdl_launch_dependents();
  const int tid = threadIdx.x;
  const int seg = blockIdx.x;
  const int blk = seg / lc, ch = seg - blk * lc;
  const int row0 = blk * rb;
  const int nr = min(n_rows - row0, rb);
  if (tid < nr) {
    const int2 r = __ldg(rtab + row0 + tid);
    const int dem = (r.x >> 6) & 0x7FFF;
    // exclusive row: bit 31, and the group's level in bits 24..26 (what the owner test below reads)
    sRow[tid] = make_int2(__float_as_int((float)(r.x & 31)),
                          (EXCL && (r.x & 32)) ? (dem | ((r.x >> 21) & 7) << 24 | (int)0x80000000) : dem);
    if (EXCL) sGid[tid] = r.y;
  }
  // ---- node operands of this thread's two groups (in flight together with the row records)
  const int n0 = t.slab_lo + ch * T;
  const int n1 = min(n0 + T, t.slab_hi);
  const int groups = T >> 2;
  float4 base4[GPT];
  int4 av[GPT];
  bool live[GPT];
#pragma unroll
  for (int j = 0; j < GPT; ++j) {
    const int g = tid + j * SCORE_THREADS;
    const int n = n0 + (g << 2);
    live[j] = g < groups && n < n1;
    base4[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    av[j] = make_int4(-1, -1, -1, -1);
    if (live[j]) {
      base4[j] = __ldg(reinterpret_cast<const float4*>(t.base + n));
      av[j] = __ldg(reinterpret_cast<const int4*>(t.free_ + n));  // padded past n: safe
      if (n + 4 > n1) {  // only in the slab's last group: lanes past the slab are infeasible
        if (n + 1 >= n1) av[j].y = -1;
        if (n + 2 >= n1) av[j].z = -1;
        av[j].w = -1;
      }
    }
  }
  __syncthreads();
  float* rowp = matrix + (size_t)row0 * (size_t)t.slab_stride + (n0 - t.slab_lo) + (tid << 2);
  const size_t stride = (size_t)t.slab_stride;
#pragma unroll 2
  for (int i = 0; i < nr; ++i, rowp += stride) {
    const int2 r = sRow[i];
    const float need = __int_as_float(r.x);
    int dem = r.y;
    if (EXCL && dem < 0) {  // exclusive row: nodes of domains another group owns are infeasible
      const int* const owner = at_level(t, (dem >> 24) & 7).node_owner;
      dem &= 0xFFFFFF;
      const int gid = sGid[i];
#pragma unroll
      for (int j = 0; j < GPT; ++j) {
        if (!live[j]) continue;
        const int4 ow = __ldg(reinterpret_cast<const int4*>(owner + n0 + ((tid + j * SCORE_THREADS) << 2)));
        float4 o4;
        o4.x = (av[j].x >= dem && (ow.x == -1 || ow.x == gid)) ? need * base4[j].x : -INFINITY;
        o4.y = (av[j].y >= dem && (ow.y == -1 || ow.y == gid)) ? need * base4[j].y : -INFINITY;
        o4.z = (av[j].z >= dem && (ow.z == -1 || ow.z == gid)) ? need * base4[j].z : -INFINITY;
        o4.w = (av[j].w >= dem && (ow.w == -1 || ow.w == gid)) ? need * base4[j].w : -INFINITY;
        st_stream_f4(rowp + j * (SCORE_THREADS << 2), o4);
      }
      continue;
    }
#pragma unroll
    for (int j = 0; j < GPT; ++j) {
      float4 o4;
      o4.x = av[j].x >= dem ? need * base4[j].x : -INFINITY;
      o4.y = av[j].y >= dem ? need * base4[j].y : -INFINITY;
      o4.z = av[j].z >= dem ? need * base4[j].z : -INFINITY;
      o4.w = av[j].w >= dem ? need * base4[j].w : -INFINITY;
      if (live[j]) st_stream_f4(rowp + j * (SCORE_THREADS << 2), o4);
    }
  }
  // Chained behind the selection kernel of the PREVIOUS batch (rbgtopo_run_staged_chain) this launch never needed
  // its results; waiting for it here, at the very end, keeps the ordering transitive: when this grid is complete so
  // is everything before it, which the next pass over the previous batch's buffers relies on.  No-op otherwise.
  pdl_wait();
#ifdef RBGTOPO_PHASE_CLOCKS
  __syncthreads();
  if (tid == 0) {
    unsigned long long t_ns;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_ns));
    atomicMax(&g_emit_end_ns, t_ns);
  }
#endif
}

}  // namespace rbgtopo
