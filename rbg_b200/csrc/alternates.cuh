// alternates.cuh — k_alternates: ranked alternate nodes of every placed replica, read from the dense rows a
// placement pass already wrote (rbgtopo_place_groups_ranked, DESIGN.md §3.10).
//
// Replicas of one role in one wave share their dense row S, so the unit of work is that role row (a JOB):
// one CTA reads the row once with 16-byte loads (and the domain vector of the group's level when the role is held to its
// group's exclusive domain), keeps the top ALT_LIST keys key(S[n], n) of the candidates per thread in
// registers, merges them per warp and across warps, and writes every replica's list: the merged top list
// without the replica's own node, truncated to n_alt.  A candidate n has S[n] != -inf, room for one more
// replica of the role once the group's own placements are taken off free[n], and lies in the required
// domain.  The room test costs one shared-memory bit per node whatever the group's size: the CTA first marks
// the nodes where free[n] - used_g[n] < demand from the group's aggregated placements (node, amount).
// S[n] != -inf already implies free[n] >= demand (§3.3), so free[] is read only for those nodes.
// Bandwidth-bound: 4 bytes per node and job (+ 4 for the domain of exclusive roles).
#pragma once
#include "kernels.cuh"

namespace rbgtopo {

constexpr int ALT_THREADS = 256;
constexpr int ALT_WARPS = ALT_THREADS / 32;
constexpr int ALT_LIST = RBGTOPO_MAX_ALTERNATES + 1;  // the replica's own node may be among the best
constexpr int ALT_DOM_ANY = -1;                        // job.dom: no domain condition
static_assert(ALT_WARPS * ALT_LIST <= 96, "cross-warp merge holds three entries per lane");

struct AltJob {  // one role row of one wave (8 words)
  int row;       // dense row in `rows` (slab_stride floats apart)
  int demand;
  int dom;       // required domain of `level`, ALT_DOM_ANY = none (a negative value other than that: no node)
  int rep0;      // first replica in the compact replica arrays (own[], out)
  int nrep;      // replicas of the role in the wave (<= RBGTOPO_MAX_STEP_REPLICAS)
  int used0;     // the group's placements: used[used0 .. used0 + nused), one entry per node
  int nused;
  int level;     // the group's exclusive level (DESIGN.md §3.9): `dom` is a domain of it
};

__device__ __forceinline__ float key_score(unsigned long long k) {  // inverse of orderable_u32 on the high word
  const uint32_t u = (uint32_t)(k >> 32);
  return __uint_as_float(u ^ ((u >> 31) ? 0x80000000u : 0xFFFFFFFFu));
}

__device__ __forceinline__ void alt_insert(unsigned long long (&top)[ALT_LIST], unsigned long long k) {
#pragma unroll
  for (int j = ALT_LIST - 1; j > 0; --j) {
    if (k > top[j - 1]) top[j] = top[j - 1];
    else if (k > top[j]) top[j] = k;
  }
  if (k > top[0]) top[0] = k;
}

// grid: one CTA per job.  Dynamic shared memory: ceil(n / 32) words (the room bitmap).
// out: per compact replica 1 + 2 * n_alt words — score, n_alt nodes, n_alt scores (fp32 bits).
__global__ void __launch_bounds__(ALT_THREADS)
k_alternates(TopoDev t, const float* __restrict__ rows, const AltJob* __restrict__ jobs, const int2* __restrict__ used,
             const int* __restrict__ own, int n_alt, int* __restrict__ out) {
  extern __shared__ unsigned int sFull[];
  __shared__ unsigned long long sWarp[ALT_WARPS * ALT_LIST];
  __shared__ unsigned long long sTop[ALT_LIST];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const AltJob J = jobs[blockIdx.x];
  const int n = t.n;
  const int words = (n + 31) >> 5;
  for (int i = tid; i < words; i += ALT_THREADS) sFull[i] = 0;
  __syncthreads();
  for (int i = tid; i < J.nused; i += ALT_THREADS) {
    const int2 u = __ldg(used + J.used0 + i);
    if (__ldg(t.free_ + u.x) - u.y < J.demand) atomicOr(&sFull[u.x >> 5], 1u << (u.x & 31));
  }
  __syncthreads();

  // ---- scan: per-thread top list in registers
  const float* row = rows + (size_t)J.row * (size_t)t.slab_stride;
  const bool need_dom = J.dom != ALT_DOM_ANY;
  const int* const dom_l = at_level(t, J.level).domain;
  unsigned long long top[ALT_LIST];
#pragma unroll
  for (int j = 0; j < ALT_LIST; ++j) top[j] = 0;
  const int groups = (n + 3) >> 2;
  for (int g = tid; g < groups; g += ALT_THREADS) {
    const int n0 = g << 2;
    const float4 s4 = __ldcs(reinterpret_cast<const float4*>(row + n0));  // read once: do not keep it in L2
    int4 d4 = make_int4(J.dom, J.dom, J.dom, J.dom);
    if (need_dom) d4 = __ldg(reinterpret_cast<const int4*>(dom_l + n0));  // padded past n: safe
    const float s[4] = {s4.x, s4.y, s4.z, s4.w};
    const int d[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = n0 + j;
      if (m >= n || s[j] == -INFINITY || d[j] != J.dom) continue;
      const unsigned long long k = make_key(s[j], m);
      if (k <= top[ALT_LIST - 1]) continue;
      if ((sFull[m >> 5] >> (m & 31)) & 1u) continue;
      alt_insert(top, k);
    }
  }

  // ---- per warp: ALT_LIST rounds of the warp-wide maximum of the lanes' heads
  for (int r = 0; r < ALT_LIST; ++r) {
    const unsigned long long m = warp_max_u64(top[0]);
    if (m != 0 && top[0] == m) {
#pragma unroll
      for (int j = 0; j < ALT_LIST - 1; ++j) top[j] = top[j + 1];
      top[ALT_LIST - 1] = 0;
    }
    if (lane == 0) sWarp[warp * ALT_LIST + r] = m;
  }
  __syncthreads();
  // ---- across warps: warp 0, three entries per lane
  if (warp == 0) {
    unsigned long long c[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) c[i] = lane + 32 * i < ALT_WARPS * ALT_LIST ? sWarp[lane + 32 * i] : 0;
    for (int r = 0; r < ALT_LIST; ++r) {
      const unsigned long long best = max(c[0], max(c[1], c[2]));
      const unsigned long long m = warp_max_u64(best);
#pragma unroll
      for (int i = 0; i < 3; ++i)
        if (m != 0 && c[i] == m) c[i] = 0;  // keys are distinct: exactly one lane holds m
      if (lane == 0) sTop[r] = m;
    }
  }
  __syncthreads();

  // ---- per replica: the merged list without its own node
  if (tid < J.nrep) {
    const int rep = J.rep0 + tid;
    const int a = own[rep];
    int* o = out + (size_t)rep * (1 + 2 * n_alt);
    o[0] = __float_as_int(a >= 0 ? row[a] : -INFINITY);
    int k = 0;
    if (a >= 0) {
      for (int i = 0; i < ALT_LIST && k < n_alt; ++i) {
        const unsigned long long key = sTop[i];
        if (key == 0) break;
        const int node = key_node(key);
        if (node == a) continue;
        o[1 + k] = node;
        o[1 + n_alt + k] = __float_as_int(key_score(key));
        ++k;
      }
    }
    for (; k < n_alt; ++k) {
      o[1 + k] = -1;
      o[1 + n_alt + k] = __float_as_int(-INFINITY);
    }
  }
}

}  // namespace rbgtopo
