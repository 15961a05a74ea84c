// score.cuh — k_score_emit: the dominant kernel of the path (DESIGN.md §4.2).
//
// Emits the dense (replica x node) score matrix as a pure HBM write stream.
// One CTA (256 threads) = one SEGMENT: a chunk of <= 2048 nodes of this rank's slab
// x a block of `bsteps` consecutive steps.  The steps' headers and role records
// are staged in shared memory (two parallel rounds of loads), a thread loads the
// per-node operands of its two float4 groups (base, free: step independent) once,
// and then only the per-step part repeats: 12 ALU ops and the 128-bit streaming
// stores (st.global.cs.v4) per role.  The grid is simply
// all segments: the hardware scheduler balances them (a persistent grid with
// statically byte-balanced ranges was 18 % slower: the slowest SM sets the time).
//   1. background: every role row is  S = need*base[n]  where the node is feasible
//      (free >= demand, and for exclusive roles the domain is unowned or ours),
//      else -inf; written once per replica of the role.  Multi-wave plans stop
//      here (SPARSE = false): their sparse corrections are applied by the kernel
//      that knows the placements (plan_group.cuh).
//   2. step-level batches with anchor pods / consumed capacity: pair*c*w is added
//      onto the just-written, L2-hot scores with fire-and-forget
//      red.global.add.f32 (+ the self term); nodes whose consumed capacity makes
//      them infeasible are overwritten with -inf.  With <= 2 records every warp
//      scans them and applies those inside its own segments (ordered by
//      __syncwarp alone); otherwise one block barrier, then the records are spread
//      over the warps.  All addends are exact integers and -inf absorbs adds, so
//      the result is bit-identical to the oracle's sequential fp32 accumulation
//      in any order.
#pragma once
#include "kernels.cuh"

namespace rbgtopo {

constexpr int GPT = 2;  // float4 groups per thread: chunk <= 256 * 4 * GPT = 2048

__device__ __forceinline__ void red_add_f32(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// Why the loop nest is (chunk outer, steps inner): with one (step, chunk) item per iteration a
// single-replica step cost ~117 instructions per 512-byte warp store (SASS count: node operands,
// tail fix-up and header decode per store); here they are amortised over the block's steps.
//
// SPARSE = false: background rows only (multi-wave plans).  Register cap: 6 CTAs/SM (40 registers,
// 36 bytes of spills) measured best — 0.845 of peak vs 0.826 at 5/SM (no spills), 0.79 at 4 or 8.
#ifndef EMIT_MIN_CTAS_BG
#define EMIT_MIN_CTAS_BG 6
#endif
constexpr int EMIT_MAX_BLOCK = 16;  // upper bound of b.bsteps

// ETAB = true (multi-wave plans, never SPARSE): the per-step metadata comes from the emit table
// (kernels.cuh: 12 words per step, one round of loads) instead of the step blob — the table exists
// before the plan has been expanded, so this launch can overlap the host's plan geometry.
template <bool SPARSE, bool ETAB>
__global__ void __launch_bounds__(SCORE_THREADS, SPARSE ? 6 : EMIT_MIN_CTAS_BG)
k_score_emit(TopoDev t, BatchDev b, int items, const int* __restrict__ etab) {
  const int T = b.chunk, lc = b.lc;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int groups = T >> 2;
  const int* __restrict__ blob = b.blob;
  const size_t stride = (size_t)t.slab_stride;
  (void)lane; (void)warp;

  // segment = blockIdx.x = block * lc + chunk;  `items` = segments * bsteps (host: emit_items)
  const int BS = b.bsteps;
  const int seg = blockIdx.x;
  const int blk = seg / lc, ch = seg - blk * lc;
  if ((seg + 1) * BS > items) return;
  const int step0 = blk * BS;
  const int nst = min(b.n_steps, step0 + BS) - step0;  // the last block may be short
  // per-step metadata of the segment into shared memory: two parallel rounds of loads instead of a
  // dependent header -> role chain in front of every step's stores
  __shared__ int4 sH0[EMIT_MAX_BLOCK];                 // gid flags fixed P
  __shared__ int sRoleOff[EMIT_MAX_BLOCK], sRepOff[EMIT_MAX_BLOCK];
  __shared__ int4 sRoles[EMIT_MAX_BLOCK][MAXP];        // count demand need flags
  if (ETAB) {
    if (tid < nst) {
      const int4 e0 = __ldg(reinterpret_cast<const int4*>(etab + (size_t)(step0 + tid) * EMIT_TAB_WORDS));  // gid flags P rep_off
      sH0[tid] = make_int4(e0.x, e0.y, 0, e0.z);
      sRepOff[tid] = e0.w;
    }
    if (tid >= 32 && tid < 32 + nst * MAXP) {
      const int s = (tid - 32) / MAXP, p = (tid - 32) - s * MAXP;
      const int pr = __ldg(etab + (size_t)(step0 + s) * EMIT_TAB_WORDS + 4 + p);
      sRoles[s][p] = make_int4(pr & 63, pr >> 12, (pr >> 6) & 31, (pr >> 11) & 1);  // count demand need flags
    }
    __syncthreads();
  } else {
    if (tid < nst) {
      const int* __restrict__ hdr = blob + RBGTOPO_HDR_WORDS + (size_t)(step0 + tid) * RBGTOPO_STEP_WORDS;
      sH0[tid] = __ldg(reinterpret_cast<const int4*>(hdr));
      sRoleOff[tid] = __ldg(hdr + 4);
      sRepOff[tid] = __ldg(hdr + 12);
    }
    __syncthreads();
    if (tid < nst * MAXP) {
      const int s = tid / MAXP, p = tid - s * MAXP;
      if (p < sH0[s].w) sRoles[s][p] = __ldg(reinterpret_cast<const int4*>(blob + sRoleOff[s]) + p);
    }
    __syncthreads();
  }
  {
    // ---- node operands of this thread's groups
    const int n0 = t.slab_lo + ch * T;
    const int n1 = min(n0 + T, t.slab_hi);
    float4 base4[GPT];
    int4 av[GPT];
    bool live[GPT];
#pragma unroll
    for (int j = 0; j < GPT; ++j) {
      const int g = tid + j * SCORE_THREADS;
      const int n = n0 + (g << 2);
      live[j] = g < groups && n < n1;
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
    for (int si = 0; si < nst; ++si) {
      const int step = step0 + si;
      const int* __restrict__ hdr = blob + RBGTOPO_HDR_WORDS + (size_t)step * RBGTOPO_STEP_WORDS;
      const int4 h0 = sH0[si];
      const int gid = h0.x, P = h0.w;
      const bool excl_step = (h0.y & RBGTOPO_STEP_EXCLUSIVE) != 0;
      const int4* roles = sRoles[si];
      float* const mrow0 = b.matrix + (size_t)sRepOff[si] * stride + (n0 - t.slab_lo);
      (void)hdr;

      // ---- 1. background rows
#pragma unroll
      for (int j = 0; j < GPT; ++j) {
        if (!live[j]) continue;
        const int g = tid + j * SCORE_THREADS;
        int4 avx = av[j];  // capacity as seen by exclusive roles: blocked domains are infeasible
        if (excl_step) {
          const int4 ow = __ldg(reinterpret_cast<const int4*>(at_level(t, step_level(h0.y)).node_owner + n0 + (g << 2)));
          if (!(ow.x == -1 || ow.x == gid)) avx.x = -1;
          if (!(ow.y == -1 || ow.y == gid)) avx.y = -1;
          if (!(ow.z == -1 || ow.z == gid)) avx.z = -1;
          if (!(ow.w == -1 || ow.w == gid)) avx.w = -1;
        }
        float* rowp = mrow0 + (g << 2);
        for (int p = 0; p < P; ++p) {
          const int4 role = roles[p];  // count demand need flags
          const float need = (float)role.z;
          const int4 a = (role.w & RBGTOPO_ROLE_EXCLUSIVE) ? avx : av[j];
          float4 o4;
          o4.x = a.x >= role.y ? need * base4[j].x : -INFINITY;
          o4.y = a.y >= role.y ? need * base4[j].y : -INFINITY;
          o4.z = a.z >= role.y ? need * base4[j].z : -INFINITY;
          o4.w = a.w >= role.y ? need * base4[j].w : -INFINITY;
          for (int c = 0; c < role.x; ++c) {
            st_stream_f4(rowp, o4);
            rowp += stride;
          }
        }
      }

      // ---- 2. sparse corrections.  Few records: every warp scans them all and
      // applies the ones inside its own segments (ordering by __syncwarp alone).
      // Many records: one block barrier, then the records are spread over warps.
      int4 h1 = make_int4(0, 0, 0, 0), h2 = make_int4(0, 0, 0, 0);
      if (SPARSE) {
        h1 = __ldg(reinterpret_cast<const int4*>(hdr) + 1);  // role_off Q pair_off n_anchors
        h2 = __ldg(reinterpret_cast<const int4*>(hdr) + 2);  // anchor_off n_cons cons_off R
      }
      const bool sparse = SPARSE && (h1.w | h2.y) != 0;
      if (sparse) {
        const bool own = (h1.w + h2.y) <= 2;
        if (own) __syncwarp(); else __syncthreads();  // background stores precede the reductions
        const int* __restrict__ con = blob + h2.z;
        for (int c = own ? lane : tid; c < h2.y; c += own ? 32 : SCORE_THREADS) {  // consumed capacity
          const int m = __ldg(con + 2 * c);
          const int g = (m - n0) >> 2;
          if (m >= n0 && m < n1 && (!own || ((g & (SCORE_THREADS - 1)) >> 5) == warp)) {
            int amt = 0;
            for (int k = 0; k < h2.y; ++k)
              if (__ldg(con + 2 * k) == m) amt += __ldg(con + 2 * k + 1);  // duplicates add up
            const int avail = __ldg(t.free_ + m) - amt;
            float* rowp = mrow0 + (m - n0);
            for (int p = 0; p < P; ++p) {
              const int4 role = roles[p];
              if (avail < role.y)
                for (int k = 0; k < role.x; ++k) rowp[(size_t)k * stride] = -INFINITY;
              rowp += (size_t)role.x * stride;
            }
          }
        }
        const int* __restrict__ anc = blob + h2.x;
        const int Q = h1.y;
        for (int a = own ? 0 : warp; a < h1.w; a += own ? 1 : SCORE_WARPS) {
          const int m = __ldg(anc + 3 * a), q = __ldg(anc + 3 * a + 1), c = __ldg(anc + 3 * a + 2);
          const int rb = __ldg(t.row_ptr + m), re = __ldg(t.row_ptr + m + 1);
          for (int j = rb + lane; j <= re; j += 32) {  // j == re stands for the self term
            int nn, wv;
            if (j < re) {
              nn = __ldg(t.col + j);
              wv = __ldg(t.w + j) * c;
            } else {
              nn = m;
              wv = RBGTOPO_SELF_W * c;
            }
            const int g = (nn - n0) >> 2;
            if (nn >= n0 && nn < n1 && (!own || ((g & (SCORE_THREADS - 1)) >> 5) == warp)) {
              float* rowp = mrow0 + (nn - n0);
              for (int p = 0; p < P; ++p) {
                const int count = __ldg(blob + h1.x + 4 * p);
                const int coef = __ldg(blob + h1.z + p * Q + q);
                if (coef) {
                  const float add = (float)(coef * wv);
                  for (int k = 0; k < count; ++k) red_add_f32(rowp + (size_t)k * stride, add);
                }
                rowp += (size_t)count * stride;
              }
            }
          }
        }
      }
    }
  }
}

}  // namespace rbgtopo
