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
// k_lw_assign_repl (§3.18) takes the same decisions on a rank of a node-axis shard, whose dense rows cover its slab
// only: it evaluates every entry from the snapshot and a per-step table of the patched nodes instead of reading rows.
#pragma once
#include "kernels.cuh"
#include "plan_group.cuh"

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

// Where a row entry comes from (DESIGN.md §3.18).  LW_ROWS: the wave's dense rows (k_score_emit wrote them).  The
// replicated forms evaluate the entry from the snapshot every rank holds in full, so that a rank of a node-axis shard
// (whose dense rows cover its slab only) takes the decisions world = 1 takes, over all nodes:
//   v_p(n) = -inf  if free[n] < demand_p, (participating exclusive row) owner(n) not in {-1, gid}, or
//                  free[n] - consumed[n] < demand_p;
//          = need_p·base[n] + delta_p(n)  otherwise, delta_p(n) = sum over anchors (m, q, c) with n in N[m] ∪ {m} of
//                  pair[p][q]·c·w(n, m) (self weight RBGTOPO_SELF_W·c).
// Every term is an exact integer below 2^24 (§3.4), so v_p(n) is bit-identical to what k_score_emit writes.  owner(n)
// as score_emit reads it: LW_REPL the level's node_owner; LW_REPL_CLAIMS the level-0 claim records of earlier groups
// of a committed batch (k_score_emit_claims); LW_REPL_CLAIMS_LV commit_owner<true> (k_score_emit_claims_lv).
enum LwSource { LW_ROWS = 0, LW_REPL = 1, LW_REPL_CLAIMS = 2, LW_REPL_CLAIMS_LV = 3 };

// grid: <= n_steps CTAs of LW_THREADS, grid-stride over the steps.  Dynamic shared memory: ceil(n / 32) words.
// lw: [n_steps][MAXP] side table.  dbest / dcap: dstride entries per CTA (level-C domain scratch, C >= 0 only).
// The step's consumed records are sorted by node with one record per node (the host aggregates them).
// Replicated forms: the step's patch table at b.corr + b.poff[s] * b.corr_w (capacity: the step's patched nodes),
// one record {node, consumed, delta_0 .. delta_{P-1}} per node of the anchors' closed neighbourhoods and the consumed
// records, node-sorted; a node without a bit in the bitmap is unpatched and costs base + free (+ owner, + domain).
// claim_off / claim_rec / occ: LW_REPL_CLAIMS (claim_off: LW_REPL_CLAIMS_LV's step -> group index); cm0: LW_REPL_CLAIMS_LV.
template <int SRC>
__device__ __forceinline__ void lw_assign_body(TopoDev t, BatchDev b, const int* __restrict__ lw,
                                               unsigned long long* dbest, int* dcap, int dstride, LwLevels lv,
                                               const int* __restrict__ claim_off, const int2* __restrict__ claim_rec,
                                               bool occ, const CommitDev* cm0) {
  constexpr bool REPL = SRC != LW_ROWS;
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
    int npat = 0;  // replicated: records of the patch table
    const int W = b.corr_w;
    int* const pat = REPL ? b.corr + (size_t)b.poff[s] * W : nullptr;
    if constexpr (REPL) {
      const int lane = tid & 31, warp = tid >> 5;
      const int na = st[7], Q = st[5];
      const int* __restrict__ anc = b.blob + st[8];
      const int* __restrict__ pair = b.blob + st[6];
      for (int a = warp; a < na; a += LW_WARPS) {  // the anchors' closed neighbourhoods
        const int m = __ldg(anc + 3 * a);
        const int rb = __ldg(t.row_ptr + m), re = __ldg(t.row_ptr + m + 1);
        for (int j = rb + lane; j <= re; j += 32) {
          const int nn = j < re ? __ldg(t.col + j) : m;
          atomicOr(&sMark[nn >> 5], 1u << (nn & 31));
        }
      }
      __syncthreads();
      // the marked nodes in node order: thread tid compacts words [w0, w1) after a block-wide scan of the counts
      const int per = (words + LW_THREADS - 1) / LW_THREADS;
      const int w0 = min(words, tid * per), w1 = min(words, w0 + per);
      int cnt = 0;
      for (int w = w0; w < w1; ++w) cnt += __popc(sMark[w]);
      int incl = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(FULL, incl, o);
        if (lane >= o) incl += v;
      }
      int* const sScan = reinterpret_cast<int*>(sRed);
      if (lane == 31) sScan[warp] = incl;
      __syncthreads();
      int at = incl - cnt;
      for (int i = 0; i < LW_WARPS; ++i) {
        const int v = sScan[i];
        if (i < warp) at += v;
        npat += v;
      }
      for (int w = w0; w < w1; ++w)
        for (unsigned int bits = sMark[w]; bits; bits &= bits - 1, ++at) {
          int* const r = pat + (size_t)at * W;
          r[0] = (w << 5) + __ffs(bits) - 1;
          for (int k = 1; k < W; ++k) r[k] = 0;
        }
      __syncthreads();  // the table's nodes are written; sRed is free again
      auto find = [&](int m) {
        int lo = 0, hi = npat;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (pat[(size_t)mid * W] < m) lo = mid + 1; else hi = mid;
        }
        return lo;
      };
      for (int i = tid; i < nc; i += LW_THREADS) pat[(size_t)find(con[2 * i]) * W + 1] = con[2 * i + 1];
      for (int a = warp; a < na; a += LW_WARPS) {
        const int m = __ldg(anc + 3 * a), q = __ldg(anc + 3 * a + 1), c = __ldg(anc + 3 * a + 2);
        const int rb = __ldg(t.row_ptr + m), re = __ldg(t.row_ptr + m + 1);
        for (int j = rb + lane; j <= re; j += 32) {  // j == re stands for the self term
          const int nn = j < re ? __ldg(t.col + j) : m;
          const int wv = (j < re ? __ldg(t.w + j) : RBGTOPO_SELF_W) * c;
          int* const r = pat + (size_t)find(nn) * W + 2;
          for (int p = 0; p < P; ++p) {
            const int coef = __ldg(pair + p * Q + q);
            if (coef) atomicAdd(r + p, coef * wv);
          }
        }
      }
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

    // replicated: v_p(m) of role p (demand, need; part = a participating row of an exclusive step)
    const int gid = st[0], L = step_level(flags);
    auto value = [&](int p, int m, int demand, int need, bool part) -> float {
      const int f = __ldg(t.free_ + m);
      if (f < demand) return -INFINITY;
      if (part) {
        int o = __ldg(at_level(t, L).node_owner + m);
        if constexpr (SRC == LW_REPL_CLAIMS) {
          int lo = __ldg(claim_off + s), hi = __ldg(claim_off + s + 1);
          while (lo < hi) {  // the step's claim records: sorted by node, one per node
            const int mid = (lo + hi) >> 1;
            if (__ldg(&claim_rec[mid].x) < m) lo = mid + 1; else hi = mid;
          }
          if (lo < __ldg(claim_off + s + 1) && __ldg(&claim_rec[lo].x) == m)
            o = occ ? owner_merge(o, __ldg(&claim_rec[lo].y)) : __ldg(&claim_rec[lo].y);
        } else if constexpr (SRC == LW_REPL_CLAIMS_LV) {
          CommitDev cm = *cm0;
          cm.g = __ldg(claim_off + s);
          cm.level = L;
          o = commit_owner<true>(cm, m, __ldg(dom_e + m), o);
        }
        if (!(o == -1 || o == gid)) return -INFINITY;
      }
      float v = (float)need * __ldg(t.base + m);
      if ((sMark[m >> 5] >> (m & 31)) & 1u) {
        int lo = 0, hi = npat;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (pat[(size_t)mid * W] < m) lo = mid + 1; else hi = mid;
        }
        if (lo < npat && pat[(size_t)lo * W] == m) {  // nodes only this step's pods marked have no record
          if (f - pat[(size_t)lo * W + 1] < demand) return -INFINITY;
          v += (float)pat[(size_t)lo * W + 2 + p];
        }
      }
      return v;
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
          const int dem0 = __ldg(roles + 4 * p0 + 1), need0 = __ldg(roles + 4 * p0 + 2);
          unsigned long long best = 0;
          for (int m = tid; m < n; m += LW_THREADS) {
            float v;
            if constexpr (REPL) v = value(p0, m, dem0, need0, true);
            else v = row[m];
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
      const int need = REPL ? __ldg(roles + 4 * p + 2) : 0;
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
            float v;
            if constexpr (REPL) {
              if (part && __ldg(dom_e + m) != dstar) continue;
              v = value(p, m, demand, need, part);
              if (v == -INFINITY) continue;
            } else {
              v = row[m];
              if (v == -INFINITY || (part && __ldg(dom_e + m) != dstar)) continue;
            }
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
            float v;
            if constexpr (REPL) {
              if ((part && __ldg(dom_e + m) != dstar) || (C >= 0 && __ldg(dom_c + m) != dr)) continue;
              v = value(p, m, demand, need, part);
              if (v == -INFINITY) continue;
            } else {
              v = row[m];
              if (v == -INFINITY || (part && __ldg(dom_e + m) != dstar) || (C >= 0 && __ldg(dom_c + m) != dr)) continue;
            }
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

__global__ void __launch_bounds__(LW_THREADS)
k_lw_assign(TopoDev t, BatchDev b, const int* __restrict__ lw, unsigned long long* dbest, int* dcap, int dstride,
            LwLevels lv) {
  lw_assign_body<LW_ROWS>(t, b, lw, dbest, dcap, dstride, lv, nullptr, nullptr, false, nullptr);
}

// The replicated forms (rbgtopo_place_groups_lw[_committed] at world > 1 on a ctx with RBGTOPO_CFG_LW_SHARDS, and the
// local half of the sharded ranked forms, DESIGN.md §3.18): no dense row is read.
template <int SRC>
__global__ void __launch_bounds__(LW_THREADS)
k_lw_assign_repl(TopoDev t, BatchDev b, const int* __restrict__ lw, unsigned long long* dbest, int* dcap, int dstride,
                 LwLevels lv, const int* __restrict__ claim_off, const int2* __restrict__ claim_rec, bool occ,
                 CommitDev cm) {
  lw_assign_body<SRC>(t, b, lw, dbest, dcap, dstride, lv, claim_off, claim_rec, occ, &cm);
}

}  // namespace rbgtopo
