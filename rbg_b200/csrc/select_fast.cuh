// select_fast.cuh — k_select_assign_fast: the selection / assignment kernel of
// step-level batches with the step's patched nodes held in a shared-memory hash
// table (DESIGN.md §4.3).  One CTA per step, warp p = role row p.  Selection
// ranges over ALL nodes on every rank (replicated selection, DESIGN.md §7); the
// matrix corrections a rank issues are those of its own column slab.
//
//   1. one pass over the anchors' CSR rows (warp per anchor, coalesced int32 loads)
//      inserts every slab neighbour into the table and accumulates pair*c*w into
//      the per-role delta of its slot (shared-memory float atomics: exact
//      integers, order-free); the same pass issues the fire-and-forget
//      red.global.add.f32 corrections onto the dense matrix when the emit kernel
//      left them to us (multi-wave plans).  Consumed capacity lands in the slot too.
//   2. the slots learn base / free / domain / ownership of their node (one gather);
//      the matrix gets -inf where consumed capacity made a node infeasible.
//   3. warp p: top-K of the patched slots (score = need*base + delta computed
//      in shared memory — no matrix read-back, nothing to wait for), then the walk
//      of the per-snapshot background order with an O(1) table probe as the
//      "is patched" test; ballots pick accepted lanes in order; merge.
//   4. warp 0: greedy from shared memory (every list entry carries its capacity),
//      then the chaining writes for multi-wave plans.
// Falls back to k_select_assign (select.cuh) when a step's patched set does not fit.
#pragma once
#include "select.cuh"
#include "p2p.cuh"

namespace rbgtopo {

struct PatchTab {
  int* node;     // [HT] key, -1 = empty
  int* cons;     // [HT] consumed capacity of the slot's node
  float* delta;  // [PB][HT] per-role score delta of the slot's node
  int mask;      // HT - 1
  // dense view of the occupied slots (built once after the insert pass): rounds
  // iterate cnt entries, not HT slots
  int* dSlot;    // [CAP]
  float* dBase;  // [CAP]
  int* dAvail;   // [CAP] free - consumed
  int* dDom;     // [CAP] domain, bit 31 set = domain owned by another group
  int cnt;
  // nodes selection ranges over: the rank's slab (all-gather scheme, k_shard_select) or all
  // nodes (replicated selection, k_select_assign_fast: identical results on every rank)
  int sel_lo, sel_hi;
  const unsigned long long* sel_order;  // background order of [sel_lo, sel_hi)
};
__host__ __device__ inline size_t fast_smem_bytes(int PB, int HT, int CAP) {
  return (size_t)HT * 4 * (2 + PB) + (size_t)CAP * 16;
}

__device__ __forceinline__ int tab_hash(int n, int mask) { return (int)(((uint32_t)n * 2654435761u) >> 12) & mask; }
__device__ __forceinline__ int tab_insert(const PatchTab& T, int n) {
  int h = tab_hash(n, T.mask);
  while (true) {
    const int old = atomicCAS(&T.node[h], -1, n);
    if (old == -1 || old == n) return h;
    h = (h + 1) & T.mask;
  }
}
__device__ __forceinline__ int tab_find(const PatchTab& T, int n) {
  int h = tab_hash(n, T.mask);
  while (true) {
    const int k = T.node[h];
    if (k == n) return h;
    if (k == -1) return -1;
    h = (h + 1) & T.mask;
  }
}

// Merge of two strictly descending key lists (disjoint: a patched node never appears in the
// background walk) into the first K entries of out[0..KS), zero-padded; capacities follow
// their keys.  Rank = own index + entries of the other list that are larger.  One warp.
__device__ __forceinline__ void merge_lists(const unsigned long long* sAcc, const int* sAccAv, int acc,
                                            const unsigned long long* sPat, const int* sPatAv, int npat, int K,
                                            unsigned long long* out, int* outAvail) {
  const int lane = threadIdx.x & 31;
  out[lane] = 0;
  outAvail[lane] = 0;
  __syncwarp();
  if (lane < acc) {
    const unsigned long long a = sAcc[lane];
    int r = lane;
    for (int j = 0; j < npat; ++j) r += sPat[j] > a;
    if (r < K) { out[r] = a; outAvail[r] = sAccAv[lane]; }
  }
  if (lane < npat) {
    const unsigned long long c = sPat[lane];
    int r = lane;
    for (int j = 0; j < acc; ++j) r += sAcc[j] > c;
    if (r < K) { out[r] = c; outAvail[r] = sPatAv[lane]; }
  }
  __syncwarp();
}

// top-K of role row p into out[0..KS) (+ the capacity of every listed node in
// outAvail); same contract as select_role (select.cuh).
__device__ __forceinline__ void select_role_fast(const TopoDev& t, const BatchDev& b, const StepHdr& h, int p, int K,
                                                 int dom, const PatchTab& T, unsigned long long* sAcc, int* sAccAv,
                                                 unsigned long long* sPat, int* sPatAv, unsigned long long* out,
                                                 int* outAvail) {
  const int lane = threadIdx.x & 31;
  if (dom == DOM_NONE || K <= 0) {
    out[lane] = 0;
    return;
  }
  const int demand = b.blob[h.role_off + 4 * p + 1];
  const int need_i = b.blob[h.role_off + 4 * p + 2];
  const float need = (float)need_i;
  const bool rexcl = (h.flags & RBGTOPO_STEP_EXCLUSIVE) && (b.blob[h.role_off + 4 * p + 3] & RBGTOPO_ROLE_EXCLUSIVE);
  const float* delta = T.delta + (size_t)p * (T.mask + 1);

  // ---- (a) patched slots: keys from shared memory, K strictly-descending rounds
  int npat = 0;
  {
    unsigned long long prev = ~0ull;
    for (; npat < K; ++npat) {
      unsigned long long best = 0;
      int bav = 0;
      for (int i = lane; i < T.cnt; i += 32) {
        const int av = T.dAvail[i], dd = T.dDom[i];
        if (av >= demand && !(rexcl && dd < 0) && (dom == DOM_ANY || (dd & 0x7FFFFFFF) == dom)) {
          const int slot = T.dSlot[i];
          const unsigned long long k = make_key(fmaf(need, T.dBase[i], delta[slot]), T.node[slot]);
          if (k < prev && k > best) { best = k; bav = av; }
        }
      }
      const unsigned long long m = warp_max_u64(best);
      if (m == 0) break;
      const uint32_t who = __ballot_sync(FULL, best == m);
      bav = __shfl_sync(FULL, bav, __ffs(who) - 1);
      if (lane == 0) { sPat[npat] = m; sPatAv[npat] = bav; }
      prev = m;
    }
  }

  // ---- (b) walk the background order; patched nodes are skipped by a table probe
  const int slab_len = T.sel_hi - T.sel_lo;
  int acc = 0;
  for (int pos = 0; pos < slab_len && acc < K; pos += 32) {
    const int i = pos + lane;
    int av = 0;
    unsigned long long key = 0;
    bool ok = false;
    if (i < slab_len) {
      int node;
      if (need_i > 0) {
        const unsigned long long ob = T.sel_order[i];
        node = key_node(ob);
        const float base = __uint_as_float((uint32_t)(ob >> 32) ^ 0x80000000u);  // base >= 0
        key = make_key(need * base, node);
      } else {
        node = T.sel_lo + i;
        key = make_key(0.0f, node);
      }
      av = t.free_[node];
      ok = av >= demand;
      if (ok && rexcl) {
        const int o = t.node_owner[node];
        ok = (o == -1 || o == h.gid);
      }
      if (ok && dom != DOM_ANY) ok = t.domain[node] == dom;
      if (ok) ok = tab_find(T, node) < 0;
    }
    const uint32_t m = __ballot_sync(FULL, ok);
    const int idx = acc + __popc(m & ((1u << lane) - 1u));
    if (ok && idx < K) { sAcc[idx] = key; sAccAv[idx] = av; }
    acc += __popc(m);
  }
  acc = min(acc, K);
  __syncwarp();

  merge_lists(sAcc, sAccAv, acc, sPat, sPatAv, npat, K, out, outAvail);
}

// Steps 0-2 of the kernels below: fill the shared-memory table of the step's patched
// nodes (+ the dense view), optionally issuing the matrix corrections.  Whole CTA.
__device__ __forceinline__ void build_table(const TopoDev& t, const BatchDev& b, const StepHdr& h, PatchTab& T, int HT,
                                            int PB, bool correct, int* sCntp) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nthreads = blockDim.x, nwarps = nthreads >> 5;
  const bool excl_step = (h.flags & RBGTOPO_STEP_EXCLUSIVE) != 0;
  int& sCnt = *sCntp;
  // ---- 0. empty table
  for (int i = tid; i < HT; i += nthreads) {
    T.node[i] = -1;
    T.cons[i] = 0;
  }
  for (int i = tid; i < PB * HT; i += nthreads) T.delta[i] = 0.0f;
  if (tid == 0) sCnt = 0;
  __syncthreads();

  // ---- 1. anchors -> slots (+ matrix corrections when asked), consumed capacity
  const size_t stride = (size_t)t.slab_stride;
  float* const mrow0 = b.matrix + (size_t)h.rep_off * stride - t.slab_lo;  // mrow0[node]
  {
    const int* anc = b.blob + h.anchor_off;
    for (int a = warp; a < h.n_anchors; a += nwarps) {
      const int m = anc[3 * a], q = anc[3 * a + 1], c = anc[3 * a + 2];
      const int rb = t.row_ptr[m], re = t.row_ptr[m + 1];
      for (int j = rb + lane; j <= re; j += 32) {  // j == re stands for the anchor's own node
        int nn, wv;
        if (j < re) {
          nn = t.col[j];
          wv = t.w[j] * c;
        } else {
          nn = m;
          wv = RBGTOPO_SELF_W * c;
        }
        if (nn >= T.sel_lo && nn < T.sel_hi) {
          const int slot = tab_insert(T, nn);
          const bool mine = correct && nn >= t.slab_lo && nn < t.slab_hi;  // this rank's matrix columns
          if (c) {
            float* rowp = mrow0 + nn;
            for (int p = 0; p < h.P; ++p) {
              const int count = b.blob[h.role_off + 4 * p];
              const int coef = b.blob[h.pair_off + p * h.Q + q];
              if (coef) {
                const float add = (float)(coef * wv);
                atomicAdd(&T.delta[(size_t)p * HT + slot], add);
                if (mine)
                  for (int k = 0; k < count; ++k) sel_red_add_f32(rowp + (size_t)k * stride, add);
              }
              rowp += (size_t)count * stride;
            }
          }
        }
      }
    }
    const int* con = b.blob + h.cons_off;
    for (int c = tid; c < h.n_cons; c += nthreads) {
      const int m = con[2 * c], amt = con[2 * c + 1];
      if (m >= T.sel_lo && m < T.sel_hi) atomicAdd(&T.cons[tab_insert(T, m)], amt);
    }
  }
  __syncthreads();

  // ---- 2. dense view + node attributes; -inf where consumed capacity made a node infeasible
  for (int i0 = 0; i0 < HT; i0 += nthreads) {
    const int i = i0 + tid;
    const int node = i < HT ? T.node[i] : -1;
    const bool occ = node >= 0;
    const uint32_t msk = __ballot_sync(FULL, occ);
    int basei = 0;
    if (lane == 0 && msk) basei = atomicAdd(&sCnt, __popc(msk));
    basei = __shfl_sync(FULL, basei, 0);
    if (occ) {
      const int d = basei + __popc(msk & ((1u << lane) - 1u));
      const int av = t.free_[node] - T.cons[i];
      int dd = t.domain[node];
      if (excl_step) {
        const int o = t.node_owner[node];
        if (!(o == -1 || o == h.gid)) dd |= 0x80000000;
      }
      T.dSlot[d] = i;
      T.dBase[d] = t.base[node];
      T.dAvail[d] = av;
      T.dDom[d] = dd;
      if (correct && T.cons[i] > 0 && node >= t.slab_lo && node < t.slab_hi) {
        float* rowp = mrow0 + node;
        for (int p = 0; p < h.P; ++p) {
          const int count = b.blob[h.role_off + 4 * p], demand = b.blob[h.role_off + 4 * p + 1];
          if (av < demand)
            for (int k = 0; k < count; ++k) rowp[(size_t)k * stride] = -INFINITY;
          rowp += (size_t)count * stride;
        }
      }
    }
  }
  __syncthreads();
  T.cnt = sCnt;

}

// LV: as k_select_assign (select.cuh).
template <bool LV>
__global__ void __launch_bounds__(32 * MAXP)
k_select_assign_fast(TopoDev t, BatchDev b, int step_begin, int mode, int HT, int CAP) {
  extern __shared__ __align__(16) unsigned char fs_smem[];
  __shared__ unsigned long long sList[MAXP][KS], sAcc[MAXP][KS], sPat[MAXP][KS];
  __shared__ int sListAv[MAXP][KS], sAccAv[MAXP][KS], sPatAv[MAXP][KS];
  __shared__ int sTakenNode[KS], sTakenAmt[KS];
  __shared__ int sDstar, sCnt;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nthreads = blockDim.x, nwarps = nthreads >> 5;
  const int PB = nwarps;
  PatchTab T;
  T.node = reinterpret_cast<int*>(fs_smem);
  T.cons = T.node + HT;
  T.delta = reinterpret_cast<float*>(T.cons + HT);
  T.mask = HT - 1;
  T.dSlot = reinterpret_cast<int*>(T.delta + (size_t)PB * HT);
  T.dBase = reinterpret_cast<float*>(T.dSlot + CAP);
  T.dAvail = reinterpret_cast<int*>(T.dBase + CAP);
  T.dDom = T.dAvail + CAP;
  T.cnt = 0;
  T.sel_lo = 0;  // replicated selection: all nodes (== the slab when world == 1)
  T.sel_hi = t.n;
  T.sel_order = t.order_all;

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

  build_table(t, b, h, T, HT, PB, (mode & SEL_CORRECT) != 0, &sCnt);

  // ---- 3. exclusive domain, selection
  int dstar = excl_step ? h.fixed_domain : -1;
  if (excl_step && h.fixed_domain < 0) {
    int pstar = -1;
    for (int p = 0; p < h.P; ++p)
      if (b.blob[h.role_off + 4 * p + 3] & RBGTOPO_ROLE_EXCLUSIVE) { pstar = p; break; }
    if (warp == 0) {
      int d = -1;
      if (pstar >= 0) {
        select_role_fast(t, b, h, pstar, 1, DOM_ANY, T, sAcc[0], sAccAv[0], sPat[0], sPatAv[0], sList[0], sListAv[0]);
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
    select_role_fast(t, b, h, p, role_k(b, h, p, t.n), dom, T, sAcc[p], sAccAv[p], sPat[p], sPatAv[p], sList[p],
                     sListAv[p]);
    b.merged[(size_t)(h.rolerow_off + p) * KS + lane] = sList[p][lane];
  }
  __syncthreads();

  // ---- 4. greedy from shared memory (+ chaining for multi-wave plans)
  if (warp == 0) {
    int ntaken = 0, unplaced = 0, r = 0;
    for (int p = 0; p < h.P; ++p) {
      const int count = b.blob[h.role_off + 4 * p], demand = b.blob[h.role_off + 4 * p + 1];
      for (int c = 0; c < count; ++c, ++r) {
        int pick = -1;
        for (int k = 0; k < KS; ++k) {
          const unsigned long long key = sList[p][k];
          if (key == 0) break;
          const int node = key_node(key);
          int used = 0;
          for (int i = lane; i < ntaken; i += 32)
            if (sTakenNode[i] == node) used += sTakenAmt[i];
          used = __reduce_add_sync(FULL, used);
          if (sListAv[p][k] - used >= demand) {
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
    if ((mode & SEL_CHAIN) && h.next_step > 0) chain_step(b, h, status, dstar);
  }
}

// ---- world > 1: rank-local lists of the steps [step_begin, step_begin + gridDim.x).
// pass2 == 0: every role row (exclusive roles of steps WITHOUT a fixed domain are selected
// unrestricted: their top-1 decides D* after the all-gather) into b.lists; the matrix
// corrections of multi-wave plans are issued here (mode & SEL_CORRECT).
// pass2 == 1: those exclusive roles again, restricted to D*, into b.excl.
// px.world > 1: the CTA also stores its rows straight into every rank's exchange buffer (p2p.cuh:
// slot [parity][this rank], row index relative to px_row0) and the last CTA of the grid publishes the
// release flags — the all-gather is fused into the kernel that produces the lists.
template <bool LV>  // as k_select_assign (select.cuh)
__global__ void __launch_bounds__(32 * MAXP)
k_shard_select(TopoDev t, BatchDev b, int step_begin, int pass2, int mode, int HT, int CAP, P2PDev px, int px_row0,
               int px_parity, unsigned long long px_seq, int* __restrict__ px_done) {
  extern __shared__ __align__(16) unsigned char fs_smem[];
  __shared__ unsigned long long sAcc[MAXP][KS], sPat[MAXP][KS], sOut[MAXP][KS];
  __shared__ int sAccAv[MAXP][KS], sPatAv[MAXP][KS], sOutAv[MAXP][KS];
  __shared__ int sCnt;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, PB = blockDim.x >> 5;
  PatchTab T;
  T.node = reinterpret_cast<int*>(fs_smem);
  T.cons = T.node + HT;
  T.delta = reinterpret_cast<float*>(T.cons + HT);
  T.mask = HT - 1;
  T.dSlot = reinterpret_cast<int*>(T.delta + (size_t)PB * HT);
  T.dBase = reinterpret_cast<float*>(T.dSlot + CAP);
  T.dAvail = reinterpret_cast<int*>(T.dBase + CAP);
  T.dDom = T.dAvail + CAP;
  T.cnt = 0;
  T.sel_lo = t.slab_lo;  // all-gather scheme: rank-local lists
  T.sel_hi = t.slab_hi;
  T.sel_order = t.order;
  const int step = step_begin + blockIdx.x;
  const StepHdr h = load_hdr(b, step);
  if constexpr (LV) t = at_level(t, step_level(h.flags));  // domain / owner of the step's exclusive level
  const bool excl_step = (h.flags & RBGTOPO_STEP_EXCLUSIVE) != 0;
  const bool unknown = excl_step && h.fixed_domain < 0;
  // what this warp's row is worth to the peers: the selected list, or zeros (skipped step, role not reselected)
  unsigned long long mine = 0ull;
  const bool idle = (h.flags & STEP_SKIP) || (pass2 && !unknown);  // CTA-uniform
  if (idle) {
    if (!pass2 && warp < h.P) b.lists[(size_t)(h.rolerow_off + warp) * KS + lane] = 0;
  } else {
    build_table(t, b, h, T, HT, PB, !pass2 && (mode & SEL_CORRECT) != 0, &sCnt);
    if (warp < h.P) {
      const int p = warp;
      const bool rexcl = excl_step && (b.blob[h.role_off + 4 * p + 3] & RBGTOPO_ROLE_EXCLUSIVE);
      const int K = role_k(b, h, p, t.n);
      if (!pass2) {
        const int dom = (rexcl && !unknown) ? h.fixed_domain : DOM_ANY;
        select_role_fast(t, b, h, p, K, dom, T, sAcc[p], sAccAv[p], sPat[p], sPatAv[p], sOut[p], sOutAv[p]);
        mine = sOut[p][lane];
        b.lists[(size_t)(h.rolerow_off + p) * KS + lane] = mine;
      } else if (rexcl) {
        const int d = b.dstar[step];
        select_role_fast(t, b, h, p, K, d >= 0 ? d : DOM_NONE, T, sAcc[p], sAccAv[p], sPat[p], sPatAv[p], sOut[p], sOutAv[p]);
        mine = sOut[p][lane];
        b.excl[(size_t)(h.rolerow_off + p) * KS + lane] = mine;
      }
    }
  }
  if (px.world > 1) {  // fused all-gather: rows -> every rank's buffer, then the last CTA raises the flags
    if (warp < h.P) {
      const long long off = ((long long)px_parity * px.world + px.rank) * px.slot_stride +
                            (long long)(h.rolerow_off + warp - px_row0) * KS + lane;
      for (int g = 0; g < px.world; ++g) px.peer[g][off] = mine;
    }
    __threadfence_system();
    __syncthreads();
    if (tid == 0) {
      const int prev = atomicAdd(px_done, 1);
      if (prev == (int)gridDim.x - 1) {
        __threadfence_system();
        for (int g = 0; g < px.world; ++g)
          st_release_sys_u64(px.peer[g] + px.flags_off + ((long long)px_parity * px.world + px.rank) * P2P_FLAG_STRIDE, px_seq);
        *px_done = 0;
      }
    }
  }
}

}  // namespace rbgtopo
