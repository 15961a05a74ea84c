// alternates.cuh — k_alternates: ranked alternate nodes of every placed replica, read from the dense rows a
// placement pass already wrote (rbgtopo_place_groups_ranked, DESIGN.md §3.10).
//
// Replicas of one role in one wave share their dense row S, so the unit of work is that role row (a JOB):
// one CTA reads the row once with 16-byte loads (and the domain vector of the group's level when the role is held to its
// group's exclusive domain), keeps the top ALT_LIST keys key(S[n], n) of the candidates per thread in
// registers, merges them per warp and across warps, and writes every replica's list: the merged top list
// without the replica's own node, truncated to n_alt.  A candidate n has S[n] != -inf, room for one more
// replica of the role once the group's own placements are taken off free[n], and lies in the required
// domain, and in the replicas' co-location domain when the role places leader-worker pods (§3.12: there the replicas
// of a job are the pods of one role row whose replicas chose the same domain D_r).  The room test costs one
// shared-memory bit per node whatever the group's size: the CTA first marks the nodes where free[n] - used_g[n] < demand from the group's aggregated placements (node, amount).
// S[n] != -inf already implies free[n] >= demand (§3.3), so free[] is read only for those nodes.
// Bandwidth-bound: 4 bytes per node and job (+ 4 for each domain condition).
//
// k_alternates_commit ranks the rows of a committed batch (rbgtopo_place_groups_committed_ranked, §3.14): `used` is
// then the whole batch's placements, and a node of a participating job must also pass the owner test every group of the
// batch has left on it (commit_owner with cm.g = n_groups), read only where the room bit is read.
// k_alternates_commit_coloc ranks the pod rows of a committed leader-worker batch
// (rbgtopo_place_groups_lw_committed_ranked, §3.15) that has a co-location domain: both conditions at once;
// k_alternates_commit_coloc_lv the same at exclusive levels (§3.16).
//
// Node-axis shards (rbgtopo_shard_place_groups*_ranked, §3.17): k_alternates_slab ranks a job on this rank's slab of
// its row and writes the job's ALT_LIST best keys of the slab, plus S_r[assign[r]] of every replica whose node lies in
// the slab; after the caller's all-gather, k_alternates_merge merges the world lists of every job into the replicas'
// lists.  The global top ALT_LIST of a job lies in the union of the per-slab top ALT_LIST lists, so the result is the
// world = 1 ranking bit for bit.  k_alternates_slab_coloc does the same for the pod rows of leader-worker forms (§3.18).
#pragma once
#include "kernels.cuh"
#include "plan_group.cuh"

namespace rbgtopo {

constexpr int ALT_THREADS = 256;
constexpr int ALT_WARPS = ALT_THREADS / 32;
constexpr int ALT_LIST = RBGTOPO_MAX_ALTERNATES + 1;  // the replica's own node may be among the best
constexpr int ALT_DOM_ANY = -1;                        // job.dom: no domain condition
static_assert(ALT_WARPS * ALT_LIST <= 96, "cross-warp merge holds three entries per lane");

struct AltJob {  // one role row of one wave, or its pods in one co-location domain (10 words)
  int row;       // dense row in `rows` (slab_stride floats apart)
  int demand;
  int dom;       // required domain of `level`, ALT_DOM_ANY = none (a negative value other than that: no node)
  int rep0;      // first replica in the compact replica arrays (own[], out)
  int nrep;      // replicas (pods) of the job (<= RBGTOPO_MAX_STEP_REPLICAS)
  int used0;     // the group's placements: used[used0 .. used0 + nused), one entry per node
  int nused;
  int level;     // the group's exclusive level (DESIGN.md §3.9): `dom` is a domain of it
  int cdom;      // required domain of `clevel`: the co-location domain D_r of the job's pods, ALT_DOM_ANY = none
  int clevel;
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
// COLOC: some job has a co-location condition.  The <false> form is the ranked placement of one-pod replicas with the
// registers it had before the condition existed (40; the condition costs 5 more, one CTA per SM less).
// COMMIT: gids[job] = the job's group gid; LV: the batch has a group at a level >= 1 (commit_owner<LV>).  COMMIT with
// COLOC: k_alternates_commit_coloc and, at levels, k_alternates_commit_coloc_lv; the other forms keep the registers
// they had without it.
// SLAB (k_alternates_slab, §3.17): the rows are this rank's slab [t.slab_lo, t.slab_hi) of the dense rows (node m at
// m - slab_lo; slab_lo is a multiple of 128, so the domain vectors, read by global node, stay 16-byte aligned), the
// room bitmap covers the slab, and `out` is the job's exchange record: ALT_LIST keys per job (u64, job-major), then one
// score per compact replica at out + 2 * ALT_LIST * gridDim.x (S_r[own] where own lies in the slab, else -inf).
template <bool COLOC, bool COMMIT, bool LV, bool SLAB = false>
__device__ __forceinline__ void alternates_body(TopoDev t, const float* __restrict__ rows,
                                                const AltJob* __restrict__ jobs, const int2* __restrict__ used,
                                                const int* __restrict__ own, int n_alt, int* __restrict__ out,
                                                const CommitDev& cm0, const int* __restrict__ gids) {
  extern __shared__ unsigned int sFull[];
  __shared__ unsigned long long sWarp[ALT_WARPS * ALT_LIST];
  __shared__ unsigned long long sTop[ALT_LIST];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const AltJob J = jobs[blockIdx.x];
  const int lo = SLAB ? t.slab_lo : 0;  // nodes [lo, n) of the row, node m at m - lo
  const int n = SLAB ? t.slab_hi : t.n;
  const int words = (n - lo + 31) >> 5;
  for (int i = tid; i < words; i += ALT_THREADS) sFull[i] = 0;
  __syncthreads();
  for (int i = tid; i < J.nused; i += ALT_THREADS) {
    const int2 u = __ldg(used + J.used0 + i);
    if constexpr (SLAB)
      if (u.x < lo || u.x >= n) continue;
    if (__ldg(t.free_ + u.x) - u.y < J.demand) atomicOr(&sFull[(u.x - lo) >> 5], 1u << ((u.x - lo) & 31));
  }
  __syncthreads();

  // ---- scan: per-thread top list in registers
  const float* row = rows + (size_t)J.row * (size_t)t.slab_stride;
  const bool need_dom = J.dom != ALT_DOM_ANY, need_col = COLOC && J.cdom != ALT_DOM_ANY;
  const int* const dom_l = at_level(t, J.level).domain;
  const int* const dom_c = at_level(t, J.clevel).domain;
  unsigned long long top[ALT_LIST];
#pragma unroll
  for (int j = 0; j < ALT_LIST; ++j) top[j] = 0;
  const int groups = (n - lo + 3) >> 2;
  for (int g = tid; g < groups; g += ALT_THREADS) {
    const int n0 = lo + (g << 2);
    const float4 s4 = __ldcs(reinterpret_cast<const float4*>(row + (n0 - lo)));  // read once: do not keep it in L2
    int4 d4 = make_int4(J.dom, J.dom, J.dom, J.dom);
    if (need_dom) d4 = __ldg(reinterpret_cast<const int4*>(dom_l + n0));  // padded past n: safe
    int4 c4 = make_int4(J.cdom, J.cdom, J.cdom, J.cdom);
    if (need_col) c4 = __ldg(reinterpret_cast<const int4*>(dom_c + n0));
    const float s[4] = {s4.x, s4.y, s4.z, s4.w};
    const int d[4] = {d4.x, d4.y, d4.z, d4.w};
    const int cd[4] = {c4.x, c4.y, c4.z, c4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = n0 + j;
      if (m >= n || s[j] == -INFINITY || d[j] != J.dom || (COLOC && cd[j] != J.cdom)) continue;
      const unsigned long long k = make_key(s[j], m);
      if (k <= top[ALT_LIST - 1]) continue;
      if ((sFull[(m - lo) >> 5] >> ((m - lo) & 31)) & 1u) continue;
      if constexpr (COMMIT)
        if (need_dom) {  // d[j] = dom_{L_g}(m): the owner every group of the batch left on m
          CommitDev cm = cm0;
          cm.level = J.level;
          const int o = commit_owner<LV>(cm, m, d[j], __ldg(at_level(t, J.level).node_owner + m));
          if (!(o == -1 || o == __ldg(gids + blockIdx.x))) continue;
        }
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

  if constexpr (SLAB) {  // the slab's list of the job, and the scores this slab holds
    unsigned long long* const keys = reinterpret_cast<unsigned long long*>(out);
    if (tid < ALT_LIST) keys[(size_t)blockIdx.x * ALT_LIST + tid] = sTop[tid];
    float* const rscore = reinterpret_cast<float*>(out + 2 * ALT_LIST * (size_t)gridDim.x);
    for (int i = tid; i < J.nrep; i += ALT_THREADS) {
      const int a = own[J.rep0 + i];
      rscore[J.rep0 + i] = a >= lo && a < n ? row[a - lo] : -INFINITY;
    }
    return;
  }
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

template <bool COLOC>
__global__ void __launch_bounds__(ALT_THREADS)
k_alternates(TopoDev t, const float* __restrict__ rows, const AltJob* __restrict__ jobs, const int2* __restrict__ used,
             const int* __restrict__ own, int n_alt, int* __restrict__ out) {
  alternates_body<COLOC, false, false>(t, rows, jobs, used, own, n_alt, out, CommitDev{}, nullptr);
}

// cm: the final claims of the committed batch's rounds, cm.g = n_groups (every group's claims count).
template <bool LV>
__global__ void __launch_bounds__(ALT_THREADS)
k_alternates_commit(TopoDev t, const float* __restrict__ rows, const AltJob* __restrict__ jobs,
                    const int2* __restrict__ used, const int* __restrict__ own, int n_alt, int* __restrict__ out,
                    CommitDev cm, const int* __restrict__ gids) {
  alternates_body<false, true, LV>(t, rows, jobs, used, own, n_alt, out, cm, gids);
}

// A committed leader-worker batch with a co-location domain (§3.15): cm holds claim lists the host built from the final
// claims (dhead / dclaim at level 0, cm.g = n_groups).
__global__ void __launch_bounds__(ALT_THREADS)
k_alternates_commit_coloc(TopoDev t, const float* __restrict__ rows, const AltJob* __restrict__ jobs,
                          const int2* __restrict__ used, const int* __restrict__ own, int n_alt, int* __restrict__ out,
                          CommitDev cm, const int* __restrict__ gids) {
  alternates_body<true, true, false>(t, rows, jobs, used, own, n_alt, out, cm, gids);
}

// The same at exclusive levels (§3.16): cm holds the host-built lists in the CommitDev<true> layout (per (level,
// domain) reporters, pods linked at the other levels of lmask), cm.g = n_groups.
__global__ void __launch_bounds__(ALT_THREADS)
k_alternates_commit_coloc_lv(TopoDev t, const float* __restrict__ rows, const AltJob* __restrict__ jobs,
                             const int2* __restrict__ used, const int* __restrict__ own, int n_alt,
                             int* __restrict__ out, CommitDev cm, const int* __restrict__ gids) {
  alternates_body<true, true, true>(t, rows, jobs, used, own, n_alt, out, cm, gids);
}

// A job's slab list for the exchange of §3.17 (one-pod replicas: no co-location condition).  out: see SLAB above.
template <bool COMMIT, bool LV>
__global__ void __launch_bounds__(ALT_THREADS)
k_alternates_slab(TopoDev t, const float* __restrict__ rows, const AltJob* __restrict__ jobs,
                  const int2* __restrict__ used, const int* __restrict__ own, int* __restrict__ out, CommitDev cm,
                  const int* __restrict__ gids) {
  alternates_body<false, COMMIT, LV, true>(t, rows, jobs, used, own, 0, out, cm, gids);
}

// The same for the pod rows of leader-worker forms (§3.18), whose jobs may carry a co-location domain (cdom, clevel).
template <bool COMMIT, bool LV>
__global__ void __launch_bounds__(ALT_THREADS)
k_alternates_slab_coloc(TopoDev t, const float* __restrict__ rows, const AltJob* __restrict__ jobs,
                        const int2* __restrict__ used, const int* __restrict__ own, int* __restrict__ out, CommitDev cm,
                        const int* __restrict__ gids) {
  alternates_body<true, COMMIT, LV, true>(t, rows, jobs, used, own, 0, out, cm, gids);
}

// The merge half of §3.17: one warp per job.  keys_all: `world` exchange buffers of `stride` u64 each, rank-major; in
// each, ALT_LIST keys per job, then one fp32 score per compact replica at word 2 * ALT_LIST * n_jobs.  Keys of
// different slabs are distinct (their nodes are), 0 = no candidate.  xjob[j] = (first compact replica, replicas);
// own[] the replicas' nodes; bounds[0 .. world] the slab bounds (empty slabs allowed).  out: per compact replica
// 1 + 2 * n_alt words, as k_alternates writes them.
constexpr int ALT_MERGE_WARPS = 4;
__global__ void __launch_bounds__(32 * ALT_MERGE_WARPS)
k_alternates_merge(const unsigned long long* __restrict__ keys_all, long long stride, int world, int n_jobs,
                   const int2* __restrict__ xjob, const int* __restrict__ own, const int* __restrict__ bounds,
                   int n_alt, int* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * ALT_MERGE_WARPS + (threadIdx.x >> 5);
  if (j >= n_jobs) return;  // warp-uniform
  unsigned long long top[ALT_LIST];
#pragma unroll
  for (int i = 0; i < ALT_LIST; ++i) top[i] = 0;
  for (int i = lane; i < world * ALT_LIST; i += 32) {
    const int w = i / ALT_LIST;
    const unsigned long long k = __ldg(keys_all + (size_t)w * stride + (size_t)j * ALT_LIST + (i - w * ALT_LIST));
    if (k > top[ALT_LIST - 1]) alt_insert(top, k);
  }
  unsigned long long best[ALT_LIST];  // the job's merged list, the same in every lane
#pragma unroll
  for (int r = 0; r < ALT_LIST; ++r) {
    const unsigned long long m = warp_max_u64(top[0]);
    if (m != 0 && top[0] == m) {
#pragma unroll
      for (int i = 0; i < ALT_LIST - 1; ++i) top[i] = top[i + 1];
      top[ALT_LIST - 1] = 0;
    }
    best[r] = m;
  }
  const int2 J = __ldg(xjob + j);
  for (int e = lane; e < J.y; e += 32) {
    const int rep = J.x + e;
    const int a = __ldg(own + rep);
    int* o = out + (size_t)rep * (1 + 2 * n_alt);
    float sc = -INFINITY;
    if (a >= 0) {  // the rank whose slab holds a: the last w with bounds[w] <= a
      int w0 = 0, w1 = world - 1;
      while (w0 < w1) {
        const int mid = (w0 + w1 + 1) >> 1;
        if (__ldg(bounds + mid) <= a) w0 = mid;
        else w1 = mid - 1;
      }
      sc = __ldg(reinterpret_cast<const float*>(keys_all + (size_t)w0 * stride + (size_t)n_jobs * ALT_LIST) + rep);
    }
    o[0] = __float_as_int(sc);
    int k = 0;
    if (a >= 0) {
#pragma unroll
      for (int i = 0; i < ALT_LIST; ++i) {
        const unsigned long long key = best[i];
        if (k >= n_alt || key == 0) break;
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
