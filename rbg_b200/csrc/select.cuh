// select.cuh — step header access, the shared pieces of selection / greedy, and the
// kernels that work WITHOUT a shared-memory table (DESIGN.md §4.3-4.4):
//   * k_select_assign: fallback of select_fast.cuh when a step's patched set does not
//     fit a CTA's shared memory — the patched nodes go to a global candidate list and
//     their exact scores are read back from the dense matrix;
//   * k_merge / k_greedy (+ chain_step): the all-gather scheme of node-axis sharding
//     (DESIGN.md §7) and the per-wave plan fallback: merge of the ranks' lists,
//     exclusive domain, greedy, and the chaining of placements into the later waves
//     of a plan through the plan blob.
// A role row is  need*base[n]  except at the step's few PATCHED nodes (closed
// neighbourhoods of its anchor pods, nodes with consumed capacity), so its top-K
// is the merge of (a) the top-K of the patched nodes and (b) the first K feasible,
// unpatched nodes of the per-snapshot background order (slab nodes sorted by
// key(base[n], n) descending; for need == 0 every background score is 0 and the
// order is simply node ascending).  One warp per role row; ballots pick the
// accepted lanes in order, REDUX finds the patch maxima.  Steps are independent
// (snapshot semantics, spec §3.7).
#pragma once
#include "kernels.cuh"
#include "p2p.cuh"

namespace rbgtopo {

constexpr int DOM_ANY = -2;   // no domain restriction
constexpr int DOM_NONE = -1;  // exclusive step without any feasible domain: empty list

constexpr int STEP_SKIP = 4;     // internal step flag: an earlier wave of the gang group failed
constexpr int SEL_CORRECT = 1;   // k_select_assign mode bits: apply the sparse corrections here
constexpr int SEL_CHAIN = 2;     //   and chain the placements into the group's later waves

struct StepHdr {
  int gid, flags, fixed_domain, P, role_off, Q, pair_off, n_anchors, anchor_off, n_cons, cons_off, R, rep_off,
      rolerow_off, next_step, i0;
};
__device__ __forceinline__ StepHdr load_hdr(const BatchDev& b, int step) {
  const int* hdr = b.blob + RBGTOPO_HDR_WORDS + (size_t)step * RBGTOPO_STEP_WORDS;
  StepHdr h;
  h.gid = hdr[0]; h.flags = hdr[1]; h.fixed_domain = hdr[2]; h.P = hdr[3]; h.role_off = hdr[4];
  h.Q = hdr[5]; h.pair_off = hdr[6]; h.n_anchors = hdr[7]; h.anchor_off = hdr[8];
  h.n_cons = hdr[9]; h.cons_off = hdr[10]; h.R = hdr[11]; h.rep_off = hdr[12]; h.rolerow_off = hdr[13];
  h.next_step = hdr[14]; h.i0 = hdr[15];
  return h;
}
// K of role row p = replicas of the step up to and including role p (spec §3.5)
__device__ __forceinline__ int role_k(const BatchDev& b, const StepHdr& h, int p, int n) {
  int k = 0;
  for (int q = 0; q <= p; ++q) k += b.blob[h.role_off + 4 * q];
  return min(k, n);
}
__device__ __forceinline__ int role_rowbase(const BatchDev& b, const StepHdr& h, int p) {
  int k = 0;
  for (int q = 0; q < p; ++q) k += b.blob[h.role_off + 4 * q];
  return k;
}

// The step's patched slab nodes (duplicates allowed) into cand[]; *sCnt counts them.
// Called by every warp of the CTA; the caller zeroes *sCnt before and syncs after.
__device__ __forceinline__ void build_candidates(const TopoDev& t, const BatchDev& b, const StepHdr& h,
                                                 int* cand, int* sCnt) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int* anc = b.blob + h.anchor_off;
  for (int a = warp; a < h.n_anchors; a += nwarps) {
    const int m = anc[3 * a];
    const int rb = t.row_ptr[m], re = t.row_ptr[m + 1];
    for (int j0 = rb; j0 <= re; j0 += 32) {  // j == re stands for the anchor's own node
      const int j = j0 + lane;
      int nn = -1;
      if (j < re) nn = t.col[j];
      else if (j == re) nn = m;
      const bool keep = nn >= t.slab_lo && nn < t.slab_hi;
      const uint32_t msk = __ballot_sync(FULL, keep);
      int base = 0;
      if (lane == 0 && msk) base = atomicAdd(sCnt, __popc(msk));
      base = __shfl_sync(FULL, base, 0);
      if (keep) cand[base + __popc(msk & ((1u << lane) - 1u))] = nn;
    }
  }
  const int* con = b.blob + h.cons_off;
  for (int c = threadIdx.x; c < h.n_cons; c += blockDim.x) {
    const int m = con[2 * c];
    if (m >= t.slab_lo && m < t.slab_hi) cand[atomicAdd(sCnt, 1)] = m;
  }
}

__device__ __forceinline__ void sel_red_add_f32(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// The sparse corrections of one step over this rank's whole slab (the same ones
// k_score_emit applies per chunk, score.cuh): -inf where consumed capacity makes a
// node infeasible, pair*c*w reductions for the anchors' closed neighbourhoods.
// Called by every warp of the CTA after the background rows exist in memory.
__device__ __forceinline__ void correct_step(const TopoDev& t, const BatchDev& b, const StepHdr& h) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const size_t stride = (size_t)t.slab_stride;
  float* const mrow0 = b.matrix + (size_t)h.rep_off * stride - t.slab_lo;  // mrow0[node]
  const int* con = b.blob + h.cons_off;
  for (int c = threadIdx.x; c < h.n_cons; c += blockDim.x) {
    const int m = con[2 * c];
    if (m >= t.slab_lo && m < t.slab_hi && con[2 * c + 1] > 0) {
      int amt = 0;
      for (int k = 0; k < h.n_cons; ++k)
        if (con[2 * k] == m) amt += con[2 * k + 1];
      const int avail = t.free_[m] - amt;
      float* rowp = mrow0 + m;
      for (int p = 0; p < h.P; ++p) {
        const int count = b.blob[h.role_off + 4 * p], demand = b.blob[h.role_off + 4 * p + 1];
        if (avail < demand)
          for (int k = 0; k < count; ++k) rowp[(size_t)k * stride] = -INFINITY;
        rowp += (size_t)count * stride;
      }
    }
  }
  const int* anc = b.blob + h.anchor_off;
  for (int a = warp; a < h.n_anchors; a += nwarps) {
    const int m = anc[3 * a], q = anc[3 * a + 1], c = anc[3 * a + 2];
    if (c == 0) continue;
    const int rb = t.row_ptr[m], re = t.row_ptr[m + 1];
    for (int j = rb + lane; j <= re; j += 32) {  // j == re stands for the self term
      int nn, wv;
      if (j < re) {
        nn = t.col[j];
        wv = t.w[j] * c;
      } else {
        nn = m;
        wv = RBGTOPO_SELF_W * c;
      }
      if (nn >= t.slab_lo && nn < t.slab_hi) {
        float* rowp = mrow0 + nn;
        for (int p = 0; p < h.P; ++p) {
          const int count = b.blob[h.role_off + 4 * p];
          const int coef = b.blob[h.pair_off + p * h.Q + q];
          if (coef) {
            const float add = (float)(coef * wv);
            for (int k = 0; k < count; ++k) sel_red_add_f32(rowp + (size_t)k * stride, add);
          }
          rowp += (size_t)count * stride;
        }
      }
    }
  }
}

// Rank-local top-K of role row p of `step` into out[0..KS) (keys descending, then
// zeros).  sAcc / sPat: per-warp shared scratch of KS keys each.  All 32 lanes call.
// cand/cnt: the step's patched nodes (shared memory when they fit, else the global
// scratch); kcache: per-warp shared array of >= min(cnt, kcap) keys (may be null).
__device__ __forceinline__ void select_role(const TopoDev& t, const BatchDev& b, const StepHdr& h, int p,
                                            int K, int dom, const int* cand, int cnt,
                                            unsigned long long* kcache, int kcap,
                                            unsigned long long* sAcc, unsigned long long* sPat,
                                            unsigned long long* out) {
  const int lane = threadIdx.x & 31;
  if (dom == DOM_NONE || K <= 0) {
    out[lane] = 0;
    return;
  }
  const int demand = b.blob[h.role_off + 4 * p + 1];
  const int need_i = b.blob[h.role_off + 4 * p + 2];
  const bool rexcl = (h.flags & RBGTOPO_STEP_EXCLUSIVE) && (b.blob[h.role_off + 4 * p + 3] & RBGTOPO_ROLE_EXCLUSIVE);
  const float* __restrict__ row =
      b.matrix + (size_t)(h.rep_off + role_rowbase(b, h, p)) * t.slab_stride - t.slab_lo;  // row[node]

  // ---- (a) top-K of the patched nodes (exact scores read back from the matrix,
  // once, into the shared key cache; duplicates of a node give equal keys, which
  // the strictly-below rounds skip)
  int npat = 0;
  {
    const bool cached = kcache != nullptr && cnt <= kcap;
    if (cached) {
      for (int i = lane; i < cnt; i += 32) {
        const int node = cand[i];
        const float x = row[node];
        kcache[i] = (x != -INFINITY && (dom == DOM_ANY || t.domain[node] == dom)) ? make_key(x, node) : 0ull;
      }
      __syncwarp();
    }
    unsigned long long prev = ~0ull;
    for (; npat < K; ++npat) {
      unsigned long long best = 0;
      if (cached) {
        for (int i = lane; i < cnt; i += 32) {
          const unsigned long long k = kcache[i];
          if (k < prev && k > best) best = k;
        }
      } else {
        for (int i = lane; i < cnt; i += 32) {
          const int node = cand[i];
          const float x = row[node];
          if (x != -INFINITY && (dom == DOM_ANY || t.domain[node] == dom)) {
            const unsigned long long k = make_key(x, node);
            if (k < prev && k > best) best = k;
          }
        }
      }
      best = warp_max_u64(best);
      if (best == 0) break;
      if (lane == 0) sPat[npat] = best;
      prev = best;
    }
  }

  // ---- (b) walk the background order
  const int slab_len = t.slab_hi - t.slab_lo;
  const float need = (float)need_i;
  int acc = 0;
  for (int pos = 0; pos < slab_len && acc < K; pos += 32) {
    const int i = pos + lane;
    int node = -1;
    unsigned long long key = 0;
    bool ok = false;
    if (i < slab_len) {
      if (need_i > 0) {
        const unsigned long long ob = t.order[i];
        node = key_node(ob);
        const float base = __uint_as_float((uint32_t)(ob >> 32) ^ 0x80000000u);  // base >= 0
        key = make_key(need * base, node);
      } else {
        node = t.slab_lo + i;
        key = make_key(0.0f, node);
      }
      ok = t.free_[node] >= demand;
      if (ok && rexcl) {
        const int o = t.node_owner[node];
        ok = (o == -1 || o == h.gid);
      }
      if (ok && dom != DOM_ANY) ok = t.domain[node] == dom;
    }
    if (__any_sync(FULL, ok)) {
      // patched nodes are not background: their exact key is in (a)
      for (int e = 0; e < cnt; ++e)
        if (cand[e] == node) ok = false;
    }
    const uint32_t m = __ballot_sync(FULL, ok);
    const int idx = acc + __popc(m & ((1u << lane) - 1u));
    if (ok && idx < K) sAcc[idx] = key;
    acc += __popc(m);
  }
  acc = min(acc, K);
  __syncwarp();

  // ---- merge the two descending lists
  if (lane == 0) {
    int ia = 0, ip = 0;
    for (int r = 0; r < KS; ++r) {
      unsigned long long v = 0;
      if (r < K) {
        const unsigned long long a = ia < acc ? sAcc[ia] : 0ull;
        const unsigned long long c = ip < npat ? sPat[ip] : 0ull;
        if (a > c) { v = a; ++ia; } else if (c) { v = c; ++ip; }
      }
      out[r] = v;
    }
  }
  __syncwarp();
}

// Multi-wave plans (rbgtopo.cu build_plan): write this step's placements into the
// later waves of the same group — anchor record n_static + i and consumed record i
// of every later step, the exclusive domain, and the SKIP flag when a gang group
// failed.  One warp, after the step's assign[] is final.
__device__ __forceinline__ void chain_step(const BatchDev& b, const StepHdr& h, int status, int dstar) {
  const int lane = threadIdx.x & 31;
  __syncwarp();
  int* wb = const_cast<int*>(b.blob);
  const bool excl = (h.flags & RBGTOPO_STEP_EXCLUSIVE) != 0;
  const bool dead = status == RBGTOPO_GANG_FAILED;
  bool any = false;
  for (int i = 0; i < h.R; ++i) any |= b.assign[h.rep_off + i] >= 0;
  const int fixed = excl ? ((dstar >= 0 && any) ? dstar : h.fixed_domain) : -1;
  for (int s2 = h.next_step; s2 > 0;) {
    int* hd = wb + RBGTOPO_HDR_WORDS + (size_t)s2 * RBGTOPO_STEP_WORDS;
    const int n_static = hd[7] - hd[15];  // n_anchors - replicas of the earlier waves
    int rr = 0;
    for (int p = 0; p < h.P; ++p) {
      const int count = b.blob[h.role_off + 4 * p], demand = b.blob[h.role_off + 4 * p + 1];
      const int q = (b.blob[h.role_off + 4 * p + 3] >> 8) & 0xFF;
      for (int c = lane; c < count; c += 32) {
        const int node = b.assign[h.rep_off + rr + c];
        int* ar = wb + hd[8] + 3 * (n_static + h.i0 + rr + c);
        int* cr = wb + hd[10] + 2 * (h.i0 + rr + c);
        ar[0] = node >= 0 ? node : 0;
        ar[1] = q;
        ar[2] = node >= 0 ? 1 : 0;
        cr[0] = node >= 0 ? node : 0;
        cr[1] = node >= 0 ? demand : 0;
      }
      rr += count;
    }
    const int nxt = hd[14];
    if (lane == 0) {
      hd[2] = fixed;
      hd[1] = dead ? (hd[1] | STEP_SKIP) : (hd[1] & ~STEP_SKIP);
    }
    s2 = nxt;
  }
}

// Greedy in replica order on the step's final lists (spec §3.6).  One warp.
// With `chain` the placements are written into the later waves of the same group
// (device-resident multi-wave plans, rbgtopo.cu build_plan): anchor record
// n_static + i and consumed record i of every later step, the exclusive domain,
// and the SKIP flag when a gang group failed.
__device__ __forceinline__ void greedy_step(const TopoDev& t, const BatchDev& b, int step, const StepHdr& h,
                                            const unsigned long long (*sList)[KS], int* sTakenNode,
                                            int* sTakenAmt, int dstar, bool chain = false) {
  const int lane = threadIdx.x & 31;
  const int* con = b.blob + h.cons_off;
  int ntaken = 0, unplaced = 0, r = 0;
  for (int p = 0; p < h.P; ++p) {
    const int count = b.blob[h.role_off + 4 * p], demand = b.blob[h.role_off + 4 * p + 1];
    for (int c = 0; c < count; ++c, ++r) {
      int pick = -1;
      for (int k = 0; k < KS; ++k) {  // the list holds K_p keys, then zeros
        const unsigned long long key = sList[p][k];
        if (key == 0) break;
        const int node = key_node(key);
        int used = 0;
        for (int i = lane; i < h.n_cons; i += 32)
          if (con[2 * i] == node) used += con[2 * i + 1];
        for (int i = lane; i < ntaken; i += 32)
          if (sTakenNode[i] == node) used += sTakenAmt[i];
        used = __reduce_add_sync(FULL, used);
        if (t.free_[node] - used >= demand) {
          pick = node;
          break;
        }
      }
      if (pick >= 0) {
        if (lane == 0) {
          sTakenNode[ntaken] = pick;
          sTakenAmt[ntaken] = demand;
        }
        ++ntaken;
        __syncwarp();
      } else {
        ++unplaced;
      }
      if (lane == 0) b.assign[h.rep_off + r] = pick;
    }
  }
  __syncwarp();
  int status = unplaced ? RBGTOPO_PLACED_PART : RBGTOPO_PLACED_ALL;
  if (unplaced && (h.flags & RBGTOPO_STEP_GANG)) {
    status = RBGTOPO_GANG_FAILED;
    for (int i = lane; i < h.R; i += 32) b.assign[h.rep_off + i] = -1;
  }
  if (lane == 0) {
    b.status[step] = status;
    b.domain_out[step] = dstar;
    b.dstar[step] = dstar;
  }
  if (chain && h.next_step > 0) chain_step(b, h, status, dstar);
}

// ---- world == 1: select + exclusive domain + greedy fused, one CTA per step,
// warp p selects role row p, warp 0 runs the greedy.  blockDim = 32 * PB.
// dynamic shared memory of the selection kernels: cand[CAND_CAP] i32 | keys[PB][CAND_CAP] u64
constexpr int CAND_CAP = 512;
__host__ __device__ inline size_t select_smem_bytes(int PB) { return (size_t)CAND_CAP * 4 + (size_t)PB * CAND_CAP * 8; }

// Builds the patched-node list in shared memory when it fits (the host-computed
// capacity poff[step+1]-poff[step] is an upper bound), else in the global scratch.
struct CandRef { const int* p; int cnt; };
__device__ __forceinline__ CandRef stage_candidates(const TopoDev& t, const BatchDev& b, int step, const StepHdr& h,
                                                    int* sCand, int* sCnt) {
  const int cap = b.poff[step + 1] - b.poff[step];
  int* dst = cap <= CAND_CAP ? sCand : b.cand + b.poff[step];
  if (threadIdx.x == 0) *sCnt = 0;
  __syncthreads();
  build_candidates(t, b, h, dst, sCnt);
  __syncthreads();
  CandRef r;
  r.p = dst;
  r.cnt = *sCnt;
  return r;
}

// LV: the batch has steps at exclusive levels >= 1 (DESIGN.md §3.9).  Level-0 batches launch <false>, whose code is the
// level-0 code: the level's vectors cost registers the <false> instantiation does not pay.
template <bool LV>
__global__ void __launch_bounds__(32 * MAXP) k_select_assign(TopoDev t, BatchDev b, int step_begin, int mode) {
  extern __shared__ __align__(16) unsigned char sel_smem[];
  int* sCand = reinterpret_cast<int*>(sel_smem);
  unsigned long long* sKeys = reinterpret_cast<unsigned long long*>(sel_smem + (size_t)CAND_CAP * 4);
  __shared__ unsigned long long sList[MAXP][KS];
  __shared__ unsigned long long sAcc[MAXP][KS];
  __shared__ unsigned long long sPat[MAXP][KS];
  __shared__ int sTakenNode[KS], sTakenAmt[KS];
  __shared__ int sDstar, sCnt;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int step = step_begin + blockIdx.x;
  const StepHdr h = load_hdr(b, step);
  if constexpr (LV) t = at_level(t, step_level(h.flags));  // domain / owner of the step's exclusive level
  const bool excl_step = (h.flags & RBGTOPO_STEP_EXCLUSIVE) != 0;
  if (h.flags & STEP_SKIP) {  // an earlier wave of this gang group failed: nothing is placed
    if (warp == 0) {
      for (int i = lane; i < h.R; i += 32) b.assign[h.rep_off + i] = -1;
      if (lane == 0) {
        b.status[step] = RBGTOPO_GANG_FAILED;
        b.domain_out[step] = -1;
        b.dstar[step] = -1;
      }
    }
    return;
  }
  if (mode & SEL_CORRECT) {
    correct_step(t, b, h);
    __threadfence();  // the reductions have landed before any read-back below
  }
  const CandRef cr = stage_candidates(t, b, step, h, sCand, &sCnt);
  const int* cand = cr.p;
  const int cnt = cr.cnt;
  int dstar = excl_step ? h.fixed_domain : -1;
  if (excl_step && h.fixed_domain < 0) {
    // D* = domain of the best feasible node of the FIRST participating role (spec §3.5)
    int pstar = -1;
    for (int p = 0; p < h.P; ++p)
      if (b.blob[h.role_off + 4 * p + 3] & RBGTOPO_ROLE_EXCLUSIVE) { pstar = p; break; }
    if (warp == 0) {
      int d = -1;
      if (pstar >= 0) {
        select_role(t, b, h, pstar, 1, DOM_ANY, cand, cnt, sKeys, CAND_CAP, sAcc[0], sPat[0], sList[0]);
        const unsigned long long top = sList[0][0];
        d = top ? t.domain[key_node(top)] : -1;
      }
      if (lane == 0) sDstar = d;
    }
    __syncthreads();
    dstar = sDstar;
  }
  if (warp < h.P) {
    const int p = warp;
    const bool rexcl = excl_step && (b.blob[h.role_off + 4 * p + 3] & RBGTOPO_ROLE_EXCLUSIVE);
    const int dom = rexcl ? (dstar >= 0 ? dstar : DOM_NONE) : DOM_ANY;
    select_role(t, b, h, p, role_k(b, h, p, t.n), dom, cand, cnt, sKeys + (size_t)p * CAND_CAP, CAND_CAP, sAcc[p],
                sPat[p], sList[p]);
    b.merged[(size_t)(h.rolerow_off + p) * KS + lane] = sList[p][lane];
  }
  __syncthreads();
  if (warp == 0) greedy_step(t, b, step, h, sList, sTakenNode, sTakenAmt, dstar, (mode & SEL_CHAIN) != 0);
}

// ---- world > 1, pass 1 (pass2 == 0): rank-local lists of every role row; roles
// of exclusive steps WITHOUT a fixed domain are selected unrestricted (their top-1
// decides D* after the all-gather).  Pass 2 (pass2 == 1): those roles again,
// restricted to D*, into b.excl.
__global__ void __launch_bounds__(32 * MAXP) k_select(TopoDev t, BatchDev b, int pass2) {
  extern __shared__ __align__(16) unsigned char sel_smem[];
  int* sCand = reinterpret_cast<int*>(sel_smem);
  unsigned long long* sKeys = reinterpret_cast<unsigned long long*>(sel_smem + (size_t)CAND_CAP * 4);
  __shared__ unsigned long long sAcc[MAXP][KS];
  __shared__ unsigned long long sPat[MAXP][KS];
  __shared__ int sCnt;
  const int warp = threadIdx.x >> 5;
  const int step = blockIdx.x;
  const StepHdr h = load_hdr(b, step);
  t = at_level(t, step_level(h.flags));  // domain / owner of the step's exclusive level
  const bool excl_step = (h.flags & RBGTOPO_STEP_EXCLUSIVE) != 0;
  const bool unknown = excl_step && h.fixed_domain < 0;
  if (pass2 && !unknown) return;  // CTA-uniform
  const CandRef cr = stage_candidates(t, b, step, h, sCand, &sCnt);
  const int* cand = cr.p;
  const int cnt = cr.cnt;
  if (warp >= h.P) return;
  const int p = warp;
  const bool rexcl = excl_step && (b.blob[h.role_off + 4 * p + 3] & RBGTOPO_ROLE_EXCLUSIVE);
  const int K = role_k(b, h, p, t.n);
  if (!pass2) {
    const int dom = (rexcl && !unknown) ? h.fixed_domain : DOM_ANY;
    select_role(t, b, h, p, K, dom, cand, cnt, sKeys + (size_t)p * CAND_CAP, CAND_CAP, sAcc[p], sPat[p],
                b.lists + (size_t)(h.rolerow_off + p) * KS);
  } else if (rexcl) {
    const int d = b.dstar[step];
    select_role(t, b, h, p, K, d >= 0 ? d : DOM_NONE, cand, cnt, sKeys + (size_t)p * CAND_CAP, CAND_CAP, sAcc[p],
                sPat[p], b.excl + (size_t)(h.rolerow_off + p) * KS);
  }
}

constexpr int SEL_WARPS = 4;
constexpr int SEL_THREADS = SEL_WARPS * 32;

// Top-K of `parts` descending lists of K keys each (src + g*stride), by one warp.
__device__ __forceinline__ int merge_parts(const unsigned long long* src, long long stride, int parts, int K,
                                           unsigned long long* out /* [KS] */) {
  const int lane = threadIdx.x & 31;
  unsigned long long prev = ~0ull;
  int r = 0;
  for (; r < K; ++r) {
    unsigned long long best = 0;
    for (int i = lane; i < parts * K; i += 32) {
      const unsigned long long k = src[(long long)(i / K) * stride + (i % K)];
      if (k < prev && k > best) best = k;
    }
    best = warp_max_u64(best);
    if (best == 0) break;
    if (lane == 0) out[r] = best;
    prev = best;
  }
  for (int q = r + lane; q < KS; q += 32) out[q] = 0;
  __syncwarp();
  return r;
}

// ---- world > 1: merged[rolerow] = top-K over the ranks' lists; D* per step
// pw.world > 1: the lists come from the in-library exchange — wait (acquire) for every source first.
__global__ void __launch_bounds__(SEL_THREADS) k_merge(TopoDev t, BatchDev b, int step_begin, int count, P2PWait pw) {
  p2p_wait_cta(pw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int idx = blockIdx.x * SEL_WARPS + warp;
  if (idx >= count) return;
  const int step = step_begin + idx;
  const StepHdr h = load_hdr(b, step);
  t = at_level(t, step_level(h.flags));  // domain / owner of the step's exclusive level
  const bool excl_step = (h.flags & RBGTOPO_STEP_EXCLUSIVE) != 0;
  int dstar = excl_step ? h.fixed_domain : -1;
  bool dstar_set = !excl_step || h.fixed_domain >= 0;
  for (int p = 0; p < h.P; ++p) {
    unsigned long long* out = b.merged + (size_t)(h.rolerow_off + p) * KS;
    merge_parts(b.lists_all + (size_t)(h.rolerow_off + p) * KS, b.part_stride, b.parts, role_k(b, h, p, t.n), out);
    if (!dstar_set && (b.blob[h.role_off + 4 * p + 3] & RBGTOPO_ROLE_EXCLUSIVE)) {
      const unsigned long long top = out[0];  // the FIRST participating role decides
      dstar = top ? t.domain[key_node(top)] : -1;
      dstar_set = true;
    }
  }
  if (lane == 0) b.dstar[step] = dstar;
}

// ---- world > 1: final lists (restricted ones merged over the ranks) + greedy
__global__ void __launch_bounds__(SEL_THREADS) k_greedy(TopoDev t, BatchDev b, int step_begin, int count, int chain, P2PWait pw) {
  p2p_wait_cta(pw);
  __shared__ unsigned long long sList[SEL_WARPS][MAXP][KS];
  __shared__ int sTakenNode[SEL_WARPS][KS];
  __shared__ int sTakenAmt[SEL_WARPS][KS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int idx = blockIdx.x * SEL_WARPS + warp;
  if (idx >= count) return;
  const int step = step_begin + idx;
  const StepHdr h = load_hdr(b, step);
  if (h.flags & STEP_SKIP) {  // an earlier wave of this gang group failed
    for (int i = lane; i < h.R; i += 32) b.assign[h.rep_off + i] = -1;
    if (lane == 0) {
      b.status[step] = RBGTOPO_GANG_FAILED;
      b.domain_out[step] = -1;
    }
    return;
  }
  const bool unknown = (h.flags & RBGTOPO_STEP_EXCLUSIVE) && h.fixed_domain < 0;
  for (int p = 0; p < h.P; ++p) {
    const bool rexcl = (b.blob[h.role_off + 4 * p + 3] & RBGTOPO_ROLE_EXCLUSIVE) != 0;
    unsigned long long* mg = b.merged + (size_t)(h.rolerow_off + p) * KS;
    if (unknown && rexcl)  // publish the final (restricted) list for rbgtopo_read_topk too
      merge_parts(b.excl_all + (size_t)(h.rolerow_off + p) * KS, b.excl_part_stride, b.parts,
                  role_k(b, h, p, t.n), mg);
    sList[warp][p][lane] = mg[lane];
  }
  __syncwarp();
  greedy_step(t, b, step, h, sList[warp], sTakenNode[warp], sTakenAmt[warp], b.dstar[step], chain != 0);
}

}  // namespace rbgtopo
