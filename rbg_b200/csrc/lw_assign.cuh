// lw_assign.cuh — k_lw_assign: selection for leader-worker replicas (rbgtopo_place_groups_lw, DESIGN.md §3.11).
//
// A replica of a role with S pods per replica places all S pods or none, optionally all inside one domain of a
// co-location level C.  The host-driven wave loop stages each wave as a step batch whose role counts are PODS;
// k_score_emit writes the wave's dense rows unchanged, and this kernel reads them directly (as k_alternates does).
// One CTA walks a step at a time (grid-stride over the steps, so the per-domain scratch is sized per resident CTA):
//   * D* of an exclusive step: the fixed domain, else the domain (at the step's level) of the best feasible node of
//     the first participating role — one block-wide u64 arg-max over its row;
//   * per replica, C = -1: S block-wide arg-maxes of key(S[n], n) over the candidates with room for one more pod;
//     C >= 0: one pass that aggregates per level-C domain the pod capacity sum floor(room / demand) (capped at S) and
//     the best candidate key, the arg-max over the domains that hold S pods (D_r), then S arg-maxes inside D_r;
//   * a replica whose S pods do not all fit is placed all or nothing: its pods are -1 and their room is given back.
// Room of node n = free[n] - consumed[n] - taken in this step.  A shared-memory bitmap marks the nodes that have a
// consumed record or a pod of this step; every other node's room is free[n].  S[n] != -inf already implies
// free[n] - consumed[n] >= demand (§3.3), so the C = -1 scans read free[] only for marked nodes.
#pragma once
#include "kernels.cuh"

namespace rbgtopo {

constexpr int LW_THREADS = 256;
constexpr int LW_WARPS = LW_THREADS / 32;

// Per role of a step, the side table word: S | (C + 1) << 8.
__host__ __device__ __forceinline__ int lw_pack_role(int pods, int coloc) { return pods | ((coloc + 1) << 8); }

struct LwLevels {  // domain count of every installed level (level 0 = domain[])
  int nd[RBGTOPO_MAX_EXCL_LEVELS];
};

__device__ __forceinline__ unsigned long long lw_block_max(unsigned long long k, unsigned long long* sRed) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  k = warp_max_u64(k);
  if (lane == 0) sRed[warp] = k;
  __syncthreads();
  unsigned long long m = sRed[0];
#pragma unroll
  for (int i = 1; i < LW_WARPS; ++i) m = max(m, sRed[i]);
  __syncthreads();  // sRed is reused by the next reduction
  return m;
}

// grid: <= n_steps CTAs of LW_THREADS, grid-stride over the steps.  Dynamic shared memory: ceil(n / 32) words.
// lw: [n_steps][MAXP] side table.  dbest / dcap: dstride entries per CTA (level-C domain scratch, C >= 0 only).
// The step's consumed records are sorted by node with one record per node (the host aggregates them).
__global__ void __launch_bounds__(LW_THREADS)
k_lw_assign(TopoDev t, BatchDev b, const int* __restrict__ lw, unsigned long long* dbest, int* dcap, int dstride,
            LwLevels lv) {
  extern __shared__ unsigned int sMark[];
  __shared__ unsigned long long sRed[LW_WARPS];
  __shared__ int sTkNode[RBGTOPO_MAX_STEP_REPLICAS], sTkDem[RBGTOPO_MAX_STEP_REPLICAS];
  const int tid = threadIdx.x;
  const int n = t.n;
  const int words = (n + 31) >> 5;
  const size_t stride = (size_t)t.slab_stride;
  unsigned long long* const my_best = dbest + (size_t)blockIdx.x * dstride;
  int* const my_cap = dcap + (size_t)blockIdx.x * dstride;

  for (int s = blockIdx.x; s < b.n_steps; s += gridDim.x) {
    const int* __restrict__ st = b.blob + RBGTOPO_HDR_WORDS + (size_t)s * RBGTOPO_STEP_WORDS;
    const int flags = st[1], fixed = st[2], P = st[3], nc = st[9];
    const int* __restrict__ roles = b.blob + st[4];
    const int* __restrict__ con = b.blob + st[10];
    const bool excl = (flags & RBGTOPO_STEP_EXCLUSIVE) != 0;
    const int* const dom_e = at_level(t, step_level(flags)).domain;
    int* const out = b.assign + st[12];
    const int drow0 = step_drow(b, s, st[13]);

    for (int i = tid; i < words; i += LW_THREADS) sMark[i] = 0;
    __syncthreads();
    for (int i = tid; i < nc; i += LW_THREADS) {
      const int m = con[2 * i];
      atomicOr(&sMark[m >> 5], 1u << (m & 31));
    }
    __syncthreads();
    int ntk = 0;  // pods of this step taken so far (uniform across the block)

    // room of node m for the pods of this step: free - consumed - taken
    auto room = [&](int m) -> int {
      int r = __ldg(t.free_ + m);
      if ((sMark[m >> 5] >> (m & 31)) & 1u) {
        int lo = 0, hi = nc;  // consumed records: sorted by node, one per node
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (__ldg(con + 2 * mid) < m) lo = mid + 1; else hi = mid;
        }
        if (lo < nc && __ldg(con + 2 * lo) == m) r -= __ldg(con + 2 * lo + 1);
        for (int k = 0; k < ntk; ++k)
          if (sTkNode[k] == m) r -= sTkDem[k];
      }
      return r;
    };

    // ---- D*: fixed, or the domain of the best feasible node of the first participating role
    int dstar = -1;
    if (excl) {
      if (fixed >= 0) {
        dstar = fixed;
      } else {
        int p0 = -1;
        for (int p = 0; p < P && p0 < 0; ++p)
          if (__ldg(roles + 4 * p + 3) & RBGTOPO_ROLE_EXCLUSIVE) p0 = p;
        if (p0 >= 0) {
          const float* row = b.matrix + (size_t)(drow0 + p0) * stride;
          unsigned long long best = 0;
          for (int m = tid; m < n; m += LW_THREADS) {
            const float v = row[m];
            if (v != -INFINITY) best = max(best, make_key(v, m));
          }
          best = lw_block_max(best, sRed);
          if (best != 0) dstar = __ldg(dom_e + key_node(best));
        }
      }
    }

    int pod = 0, unplaced = 0;
    for (int p = 0; p < P; ++p) {
      const int count = __ldg(roles + 4 * p), demand = __ldg(roles + 4 * p + 1);
      const bool part = excl && (__ldg(roles + 4 * p + 3) & RBGTOPO_ROLE_EXCLUSIVE);
      const int word = __ldg(lw + (size_t)s * MAXP + p);
      const int S = word & 0xFF, C = (word >> 8) - 1;
      const float* row = b.matrix + (size_t)(drow0 + p) * stride;
      const int* const dom_c = C >= 0 ? at_level(t, C).domain : nullptr;
      for (int r = 0; r < count / S; ++r, pod += S) {
        const int ntk0 = ntk;
        int dr = -1;
        bool ok = true;
        if (C >= 0) {  // D_r: the level-C domain with the best candidate among those that hold all S pods
          const int nd = lv.nd[C];
          for (int d = tid; d < nd; d += LW_THREADS) {
            __stcg(my_best + d, 0ull);
            __stcg(my_cap + d, 0);
          }
          __syncthreads();
          for (int m = tid; m < n; m += LW_THREADS) {
            const float v = row[m];
            if (v == -INFINITY || (part && __ldg(dom_e + m) != dstar)) continue;
            const int rm = room(m);
            if (rm < demand) continue;
            const int d = __ldg(dom_c + m);
            atomicMax(my_best + d, make_key(v, m));
            atomicAdd(my_cap + d, demand > 0 ? min(rm / demand, S) : S);
          }
          __syncthreads();
          unsigned long long best = 0;
          for (int d = tid; d < nd; d += LW_THREADS)
            if (__ldcg(my_cap + d) >= S) best = max(best, __ldcg(my_best + d));
          best = lw_block_max(best, sRed);
          if (best != 0) dr = __ldg(dom_c + key_node(best));
          else ok = false;
        }
        for (int k = 0; k < S && ok; ++k) {
          unsigned long long best = 0;
          for (int m = tid; m < n; m += LW_THREADS) {
            const float v = row[m];
            if (v == -INFINITY || (part && __ldg(dom_e + m) != dstar) || (C >= 0 && __ldg(dom_c + m) != dr)) continue;
            const unsigned long long key = make_key(v, m);
            if (key <= best) continue;
            if (((sMark[m >> 5] >> (m & 31)) & 1u) && room(m) < demand) continue;
            best = key;
          }
          best = lw_block_max(best, sRed);
          if (best == 0) {
            ok = false;
            break;
          }
          const int node = key_node(best);
          if (tid == 0) {
            sTkNode[ntk] = node;
            sTkDem[ntk] = demand;
            sMark[node >> 5] |= 1u << (node & 31);
            out[pod + k] = node;
          }
          ++ntk;
          __syncthreads();
        }
        if (!ok) {  // all or nothing: the replica's pods give their room back
          ntk = ntk0;
          ++unplaced;
          for (int k = tid; k < S; k += LW_THREADS) out[pod + k] = -1;
        }
      }
    }
    const bool gang = (flags & RBGTOPO_STEP_GANG) != 0;
    if (gang && unplaced)
      for (int i = tid; i < pod; i += LW_THREADS) out[i] = -1;
    if (tid == 0) {
      b.status[s] = unplaced ? (gang ? RBGTOPO_GANG_FAILED : RBGTOPO_PLACED_PART) : RBGTOPO_PLACED_ALL;
      b.domain_out[s] = dstar;
    }
    __syncthreads();  // sMark / sTk* are rebuilt for the next step
  }
}

}  // namespace rbgtopo
