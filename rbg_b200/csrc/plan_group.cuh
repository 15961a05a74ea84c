// plan_group.cuh — k_plan_group: every wave of a group in ONE launch (world == 1
// multi-wave plans, DESIGN.md §4.4).
//
// Waves of one group depend only on each other (batch = snapshot semantics, spec
// §3.7), so one CTA walks its group's steps through the `next_step` links and
// carries the group's state in shared memory instead of chaining it through HBM
// and three launches:
//   * the hash table of patched nodes is INCREMENTAL: wave w only inserts the
//     closed neighbourhoods of the replicas wave w-1 placed.  A slot keeps, per
//     GROUP role q, aw[q] = sum of c*w over the anchor pods of role q next to the
//     node, and the capacity consumed on it; the score delta of a role row is
//     sum_q pair[p][q] * aw[q] (exact integers, spec §3.4), evaluated where needed;
//   * placements, the exclusive domain and a failed gang never leave the CTA;
//   * the dense matrix gets its sparse corrections per wave from the table: one
//     red.global.add.f32 per (patched node, role row) with the summed delta,
//     -inf where consumed capacity made the node infeasible.
// Node-axis sharding (world > 1): selection is REPLICATED — it is O(K + patches) per role,
// independent of the node count, so every rank runs it over ALL nodes (table, background
// order `order_all`, greedy) and reaches the identical placement without exchanging
// anything; only the HBM-bound dense matrix is sharded, and a rank applies the
// corrections that fall into its column slab.  No collective on the step path.
// Selection (patched slots merged with the walk of the background order) and the
// greedy are the ones of select_fast.cuh.  Steps are read from the expanded plan
// blob; the chained anchor / consumed records of later steps are neither written
// nor read here.
#pragma once
#include "select_fast.cuh"

namespace rbgtopo {

struct GroupTab {
  int* node;        // [HT] key, -1 = empty
  int* cons;        // [HT] capacity consumed on the slot's node by earlier waves
  float* aw;        // [QB][HT] anchor weight per group role
  int mask, HT;
  int* cnt;         // occupied slots; the thread whose CAS claims a slot appends it to dSlot
  int* dSlot;       // [CAP] dense view of the occupied slots (insertion order)
  float* dBase;     // [CAP]
  int* dFree;       // [CAP] free capacity of the node in the snapshot
  int* dDom;        // [CAP] domain, bit 31 set = domain owned by another group
};
struct GroupRole {  // role row of the current wave, staged in shared memory
  int count, demand, need, flags;
};

// Dynamic shared memory of k_plan_group.  Every array is sized by the batch (QB roles per group, PB warps >= role rows
// of any wave), not by the ABI maxima: at cfg3's geometry (QB 5, PB 4, HT 512, CAP 448) it is 26 356 B, which with the
// kernel's static shared memory and the 1 KB the hardware reserves per CTA lets 8 CTAs share an H100 SM (228 KB).
__host__ __device__ inline size_t group_smem_bytes(int QB, int PB, int HT, int CAP) {
  return (size_t)HT * 4 * (2 + QB) + (size_t)CAP * 16 +                          // table + dense view
         (size_t)PB * KS * (3 * 8 + 3 * 4) +                                      // per-role key lists + capacities
         (size_t)PB * 16 + (size_t)PB * QB * 4 +                                  // staged roles + pair rows
         (size_t)QB * 5 * 4;                                                      // DIRECT: role table + placed counts
}

// capacity left on dense entry i after the consumption of earlier waves
__device__ __forceinline__ int gtab_avail(const GroupTab& T, int i) { return T.dFree[i] - T.cons[T.dSlot[i]]; }

__device__ __forceinline__ int gtab_insert(const GroupTab& T, int n) {
  int h = tab_hash(n, T.mask);
  while (true) {
    const int old = atomicCAS(&T.node[h], -1, n);
    if (old == -1) T.dSlot[atomicAdd(T.cnt, 1)] = h;  // claimed: the capacity bound keeps this below CAP
    if (old == -1 || old == n) return h;
    h = (h + 1) & T.mask;
  }
}
__device__ __forceinline__ bool gtab_has(const GroupTab& T, int n) {
  int h = tab_hash(n, T.mask);
  while (true) {
    const int k = T.node[h];
    if (k == n) return true;
    if (k == -1) return false;
    h = (h + 1) & T.mask;
  }
}
__device__ __forceinline__ float gtab_delta(const GroupTab& T, const float* pair_row, int Q, int slot) {
  float d = 0.0f;
  const float* aw = T.aw + slot;
  for (int q = 0; q < Q; ++q, aw += T.HT) d = fmaf(pair_row[q], *aw, d);
  return d;
}

#ifdef RBGTOPO_PHASE_CLOCKS  // one-off instrumentation: per-CTA phase timestamps
__device__ long long g_phase_clk[2048 * 32];
__device__ int g_dbg_skip;  // timing experiments only: bit 0 = no corrections, bit 1 = no patched-slot pass
__device__ long long g_cta_ns[2048 * 4];  // globaltimer at CTA start / end, table entries, SM id
__device__ __forceinline__ long long pg_gtime() { long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ int pg_smid() { int v; asm volatile("mov.u32 %0, %%smid;" : "=r"(v)); return v; }
#define PCLK(k) do { if (tid == 0 && blockIdx.x < 2048 && (k) < 32) g_phase_clk[blockIdx.x * 32 + (k)] = clock64(); } while (0)
#define PCLKL(k) do { if ((k) >= 0 && (threadIdx.x & 31) == 0 && blockIdx.x < 2048 && (k) < 32) g_phase_clk[blockIdx.x * 32 + (k)] = clock64(); } while (0)
#else
#define PCLK(k) do {} while (0)
#define PCLKL(k) do {} while (0)
#endif

// Lane `lane`'s candidate at position pos + lane of the background order (spec §3.3: for
// need == 0 every background score is 0, so the order is node-ascending), with the node
// attributes selection filters on.  Loaded early (before the table passes of a wave) for
// pos == 0 so that the two dependent round trips are off the critical path.
struct BgCand {
  unsigned long long ob;  // order entry (need > 0) — key(base, node)
  int node, free_, owner, dom;
};
// second half of a candidate load: `ob` = t.order[i] is already in a register
__device__ __forceinline__ BgCand bg_attrs(const TopoDev& t, int need_i, int i, int n_sel, unsigned long long ob) {
  BgCand c;
  c.ob = ob;
  c.node = -1;
  c.free_ = 0;
  c.owner = -1;
  c.dom = -1;
  if (i < n_sel) {
    c.node = need_i > 0 ? key_node(ob) : i;
    c.free_ = t.free_[c.node];
    c.owner = t.node_owner[c.node];
    c.dom = t.domain[c.node];
  }
  return c;
}
__device__ __forceinline__ BgCand bg_load(const TopoDev& t, int need_i, int i, int n_sel) {
  return bg_attrs(t, need_i, i, n_sel, (i < n_sel && need_i > 0) ? t.order_all[i] : 0ull);
}

// ---- committed batch (rbgtopo_place_groups_committed, DESIGN.md §3.8) -----------------------------------------------
// Group g of a committed batch sees what the groups before it took: capacity on the nodes their replicas were placed
// on, and the exclusive domains they reported.  Both are kept as short linked lists that k_commit_claims rebuilds from
// the results of every round; a node or domain nobody claimed costs one load.  The selection reads them exactly where
// it reads the node's attributes (the table's dense view, the background candidates) and records that it did, so that
// k_commit_diff can tell which later groups a changed claim can affect.
struct CommitDev {
  const int* head;     // [nodes] first claim on the node (the dense row of the replica), -1 = none
  const int4* claim;   // [rows] {group index, demand, next claim on the same node, 0}
  const int* dhead;    // [domains] first exclusive group that reported the domain, -1 = none
  const int2* dclaim;  // [groups] {gid, next group that reported the same domain}
  int* reader;         // [nodes] largest group index whose selection read the node this round
  int* dreader;        // [domains] the same for the owner of the domain (exclusive groups)
  int g;               // the group this CTA places (set by the kernel)
  bool excl;           // ... and whether it is exclusive
  bool occ;            // occupancy mode (§3.9): owners are per node, derived from the pods' records
  // Batches with a group at a level >= 1 (the <true> variants, §3.9): dhead / dreader are indexed by
  // doff[L] + (domain of level L), and the placed participating pods of exclusive groups are linked per (level, domain)
  // into phead / pclaim for every level of `lmask` other than their group's.  Unused by the <false> variants.
  const int* ldom;     // level L's domain of node n at L * lstride + n (row 0 = level 0)
  const int* doff;     // [levels + 1] first head of level L in dhead / dreader / phead
  int* phead;          // first pod claim in (L, d), -1 = none
  int4* pclaim;        // [rows][popc(lmask)] {group index, gid, next pod claim in the same (L, d), 0}
  int lstride;
  int lmask;           // levels of the batch's exclusive groups
  int level;           // cm.g's exclusive level (set by the kernel)
};
// capacity the groups before cm.g took on `node`
__device__ __forceinline__ int commit_ext(const CommitDev& cm, int node) {
  int s = 0;
  for (int i = cm.head[node]; i >= 0;) {
    const int4 c = cm.claim[i];
    if (c.x < cm.g) s += c.y;
    i = c.z;
  }
  return s;
}
// owner of a node of domain `dom` for group cm.g, given the snapshot's `owner`: the gid of the LAST earlier exclusive
// group that reported the domain, else `owner`.  In occupancy mode `owner` is the node's own derived owner_0, which the
// records may block inside a domain another node of which is free: the claim is merged into it, so that a claim never
// unblocks what the records block.
//
// LV (a batch with a group at a level >= 1, occupancy mode): `owner` is owner_{L_g}[node] and `dom` = dom_{L_g}(node),
// L_g = cm.level.  The owner is owner ⊕ K ⊕ P (§3.9): K merges, for every level L of the batch's exclusive groups, the
// gid of the last earlier group that reported dom_L(node) at level L; P merges the gid of every pod an earlier exclusive
// group of another level placed in dom_{L_g}(node) (pods of cm.g's own level lie in their group's reported domain, which
// K covers).
__device__ __forceinline__ int commit_dom(const CommitDev& cm, int L, int node, int dom) {
  return L == cm.level ? dom : cm.ldom[(size_t)L * cm.lstride + node];
}
template <bool LV = false>
__device__ __forceinline__ int commit_owner(const CommitDev& cm, int node, int dom, int owner) {
  if constexpr (!LV) {
    int last = -1, claim = -1;
    for (int i = cm.dhead[dom]; i >= 0;) {
      const int2 c = cm.dclaim[i];
      if (i < cm.g && i > last) { last = i; claim = c.x; }
      i = c.y;
    }
    return last < 0 ? owner : cm.occ ? owner_merge(owner, claim) : claim;
  } else {
    for (int m = cm.lmask; m; m &= m - 1) {
      const int L = __ffs(m) - 1;
      const int d = cm.doff[L] + commit_dom(cm, L, node, dom);
      int last = -1, claim = -1;
      for (int i = cm.dhead[d]; i >= 0;) {
        const int2 c = cm.dclaim[i];
        if (i < cm.g && i > last) { last = i; claim = c.x; }
        i = c.y;
      }
      if (last >= 0) owner = owner_merge(owner, claim);
      if (L == cm.level)
        for (int i = cm.phead[d]; i >= 0;) {
          const int4 c = cm.pclaim[i];
          if (c.x < cm.g) owner = owner_merge(owner, c.y);
          i = c.z;
        }
    }
    return owner;
  }
}
// The marks only grow within a round, so a plain L2 load that already shows cm.g or more makes the atomic redundant; the
// CTAs of a round all read the head of the background order, and this keeps them from queueing on the same addresses.
// LV: an exclusive group marks the node's domain at every level of the batch's exclusive groups (what commit_owner reads).
template <bool LV = false>
__device__ __forceinline__ void commit_note_read(const CommitDev& cm, int node, int dom) {
  if (__ldcg(&cm.reader[node]) < cm.g) atomicMax(&cm.reader[node], cm.g);
  if constexpr (!LV) {
    if (cm.excl && __ldcg(&cm.dreader[dom]) < cm.g) atomicMax(&cm.dreader[dom], cm.g);
  } else if (cm.excl) {
    for (int m = cm.lmask; m; m &= m - 1) {
      const int L = __ffs(m) - 1;
      int* const p = &cm.dreader[cm.doff[L] + commit_dom(cm, L, node, dom)];
      if (__ldcg(p) < cm.g) atomicMax(p, cm.g);
    }
  }
}
// a background candidate as group cm.g sees it (the selection notes the read where the candidate's capacity or owner
// can decide anything: not where its domain alone rules it out)
template <bool LV = false>
__device__ __forceinline__ void commit_adjust(BgCand& c, const CommitDev& cm) {
  if (c.node < 0) return;
  c.free_ -= commit_ext(cm, c.node);
  if (cm.excl) c.owner = commit_owner<LV>(cm, c.node, c.dom, c.owner);
}

// top-K of a role row into out[0..KS) (+ capacities): select_role_fast with the
// delta evaluated from the per-group-role planes.  `first` = bg_load(..., lane, ...) when
// have_first.  One warp.  COMMIT: the background candidates it loads are seen through `cm` (`first` already is).
template <bool COMMIT = false, bool CLV = false>
__device__ __forceinline__ void select_role_group(const TopoDev& t, int gid, bool excl_step, const GroupRole& role,
                                                  const float* pair_row, int Q, int K, int dom, const GroupTab& T,
                                                  int cnt, bool have_first, const BgCand& first, int dbg,
                                                  unsigned long long* sAcc, int* sAccAv,
                                                  unsigned long long* sPat, int* sPatAv, unsigned long long* out,
                                                  int* outAvail, const CommitDev* cm = nullptr) {
  const int lane = threadIdx.x & 31;
  if (dom == DOM_NONE || K <= 0) {
    out[lane] = 0;
    outAvail[lane] = 0;
    __syncwarp();
    return;
  }
  const int demand = role.demand;
  const float need = (float)role.need;
  const bool rexcl = excl_step && (role.flags & RBGTOPO_ROLE_EXCLUSIVE);

  // ---- (a) patched slots, K strictly-descending rounds.  The keys of the first 32 * EREG
  //      entries are evaluated once and stay in registers; entries past that are re-evaluated
  //      per round.
  constexpr int EREG = 8;
  auto entry_key = [&](int i) -> unsigned long long {
    const int av = gtab_avail(T, i), dd = T.dDom[i];
    if constexpr (COMMIT)
      if (dom == DOM_ANY || (dd & 0x7FFFFFFF) == dom) commit_note_read<CLV>(*cm, T.node[T.dSlot[i]], dd & 0x7FFFFFFF);
    if (av >= demand && !(rexcl && dd < 0) && (dom == DOM_ANY || (dd & 0x7FFFFFFF) == dom)) {
      const int slot = T.dSlot[i];
      return make_key(fmaf(need, T.dBase[i], gtab_delta(T, pair_row, Q, slot)), T.node[slot]);
    }
    return 0ull;
  };
  unsigned long long kreg[EREG];
#ifdef RBGTOPO_PHASE_CLOCKS
  if (g_dbg_skip & 2) cnt = 0;
#endif
#pragma unroll
  for (int j = 0; j < EREG; ++j) {
    kreg[j] = 0ull;
    if (32 * j < cnt) {  // warp-uniform: small tables skip the tail of the unrolled body
      const int i = lane + 32 * j;
      if (i < cnt) kreg[j] = entry_key(i);
    }
  }
  int npat = 0;
  {
    unsigned long long prev = ~0ull;
    for (; npat < K; ++npat) {
      unsigned long long best = 0;
      int bi = 0;
#pragma unroll
      for (int j = 0; j < EREG; ++j)
        if (32 * j < cnt && kreg[j] < prev && kreg[j] > best) { best = kreg[j]; bi = lane + 32 * j; }
      for (int i = lane + 32 * EREG; i < cnt; i += 32) {
        const unsigned long long k = entry_key(i);
        if (k < prev && k > best) { best = k; bi = i; }
      }
      const unsigned long long m = warp_max_u64(best);
      if (m == 0) break;
      if (best == m) { sPat[npat] = m; sPatAv[npat] = gtab_avail(T, bi); }  // keys are unique: one lane
      prev = m;
    }
  }
  __syncwarp();
  PCLKL(dbg);

  // ---- (b) walk the background order; patched nodes are skipped by a table probe
  int acc = 0;
  for (int pos = 0; pos < t.n && acc < K; pos += 32) {
    BgCand c = (pos == 0 && have_first) ? first : bg_load(t, role.need, pos + lane, t.n);
    if constexpr (COMMIT) {
      if (!(pos == 0 && have_first)) commit_adjust<CLV>(c, *cm);
      if (c.node >= 0 && (dom == DOM_ANY || c.dom == dom)) commit_note_read<CLV>(*cm, c.node, c.dom);
    }
    bool ok = c.node >= 0 && c.free_ >= demand;
    if (ok && rexcl) ok = (c.owner == -1 || c.owner == gid);
    if (ok && dom != DOM_ANY) ok = c.dom == dom;
    if (ok) ok = !gtab_has(T, c.node);
    const uint32_t m = __ballot_sync(FULL, ok);
    const int idx = acc + __popc(m & ((1u << lane) - 1u));
    if (ok && idx < K) {
      // need > 0: base >= 0 is the high word of the order entry
      const float base = __uint_as_float((uint32_t)(c.ob >> 32) ^ 0x80000000u);
      sAcc[idx] = role.need > 0 ? make_key(need * base, c.node) : make_key(0.0f, c.node);
      sAccAv[idx] = c.free_;
    }
    acc += __popc(m);
  }
  acc = min(acc, K);
  __syncwarp();
  PCLKL(dbg < 0 ? -1 : dbg + 1);

  merge_lists(sAcc, sAccAv, acc, sPat, sPatAv, npat, K, out, outAvail);
}

// Inserts the closed neighbourhood of anchor pod(s) (node m, group role q, count c) and the
// capacity `dem` consumed on m.  One warp.
__device__ __forceinline__ void gtab_add_anchor(const TopoDev& t, const GroupTab& T, int m, int q, int c, int dem) {
  const int lane = threadIdx.x & 31;
  if (lane == 0 && dem > 0) atomicAdd(&T.cons[gtab_insert(T, m)], dem);
  if (c <= 0) return;
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
    atomicAdd(&T.aw[(size_t)q * T.HT + gtab_insert(T, nn)], (float)wv);
  }
}

// Next wave of a group from its role table (level, pending, demand, flags per role): the rule of walk_waves
// (rbgtopo.cu) / plan_wave_at (plan.cuh), one wave per call with the cursor (cr, taken) carried by the caller.
// Fills role[] / count[] and returns the number of role rows (0 = no wave left).  One thread.
__device__ __forceinline__ int wave_next(const int* roles, int q, int& cr, int& taken, int* role, int* count) {
  while (cr < q && roles[4 * cr + 1] - taken <= 0) { ++cr; taken = 0; }
  if (cr >= q) return 0;
  const int level = roles[4 * cr];
  int n = 0, P = 0;
  while (cr < q && roles[4 * cr] == level && n < RBGTOPO_MAX_STEP_REPLICAS && P < RBGTOPO_MAX_STEP_ROLES) {
    const int left = roles[4 * cr + 1] - taken;
    if (left <= 0) { ++cr; taken = 0; continue; }
    const int take = min(left, RBGTOPO_MAX_STEP_REPLICAS - n);
    role[P] = cr;
    count[P] = take;
    ++P;
    n += take;
    taken += take;
    if (taken == roles[4 * cr + 1]) { ++cr; taken = 0; }
  }
  return P;
}

// Dense role rows of the direct path, part 1: cnt[g] = the role rows of group g (one thread per group replays its wave
// rule).  The first dense role row of group g (step_drow, kernels.cuh) is the exclusive prefix of cnt, which the host
// takes with a saturating device scan (rbgtopo.cu: launch_group_rows).  Like k_group_rtab it runs on the not yet
// validated blob: a group that fails a range check has no rows, and a count is clamped to `n_rows`.
constexpr int RRCOUNT_THREADS = 256;
__global__ void __launch_bounds__(RRCOUNT_THREADS) k_group_rrcount(const int* __restrict__ grp, int words, int n_groups, int n_rows,
                                                                   int* __restrict__ cnt) {
  const int g = blockIdx.x * RRCOUNT_THREADS + threadIdx.x;
  if (g >= n_groups) return;
  const int* rec = grp + RBGTOPO_HDR_WORDS + (size_t)g * RBGTOPO_GROUP_WORDS;  // the host checked that the group table fits the blob
  const int q = rec[3];
  const long long roff = rec[4];
  int rr = 0;
  if (q >= 1 && q <= RBGTOPO_MAX_GROUP_ROLES && roff >= 0 && roff + 4 * q <= words && rec[9] > 0) {
    int cr = 0, tk = 0, role[RBGTOPO_MAX_STEP_ROLES], count[RBGTOPO_MAX_STEP_ROLES];
    for (int P; rr < n_rows && (P = wave_next(grp + roff, q, cr, tk, role, count)) > 0;) rr += P;
  }
  cnt[g] = min(rr, n_rows);
}
// a + b capped at n: associative on [0, n], and a + b <= 2n < 2^31 never overflows (n <= 2^30)
struct SatAdd {
  int n;
  __host__ __device__ __forceinline__ int operator()(int a, int b) const { return min(a + b, n); }
};

// Row table of k_emit_rows (kernels.cuh) straight from the GROUPS blob, one warp per group: the group's dense role
// rows are [drow[g], + its role rows) in role order within a wave, waves in order (launch_group_rows) — the rows of a
// group are a function of the blob alone, so the dense matrix needs nothing the host computes per step.
// rbgtopo_place_groups' direct path launches both kernels right behind the upload of the blob, i.e. BEFORE the host
// has validated the blob (the validation runs meanwhile and the result is only used if it passes): every offset and
// count read from the blob is range-checked against `words` / `n_rows` here, a group that fails a check writes
// nothing, and the wave loop ends when the rows run out — garbage in, bounded garbage out, no out-of-range access.
constexpr int RTAB_WARPS = 4;
__global__ void __launch_bounds__(32 * RTAB_WARPS) k_group_rtab(const int* __restrict__ grp, int words, int n_groups, int n_rows,
                                                              const int* __restrict__ drow, int2* __restrict__ rtab) {
  __shared__ int sR[RTAB_WARPS][4 * RBGTOPO_MAX_GROUP_ROLES], sP[RTAB_WARPS][RBGTOPO_MAX_GROUP_ROLES * RBGTOPO_MAX_GROUP_ROLES];
  __shared__ int sPl[RTAB_WARPS][RBGTOPO_MAX_GROUP_ROLES], sRole[RTAB_WARPS][RBGTOPO_MAX_STEP_ROLES], sCount[RTAB_WARPS][RBGTOPO_MAX_STEP_ROLES];
  __shared__ int sNP[RTAB_WARPS];
  const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
  const int g = blockIdx.x * RTAB_WARPS + wi;
  if (g >= n_groups) return;
  const int* rec = grp + RBGTOPO_HDR_WORDS + (size_t)g * RBGTOPO_GROUP_WORDS;  // the host checked that the group table fits the blob
  const int gid = rec[0], q = rec[3];
  const long long roff = rec[4], poff = rec[5];
  const bool excl = (rec[1] & RBGTOPO_STEP_EXCLUSIVE) != 0;
  if (q < 1 || q > RBGTOPO_MAX_GROUP_ROLES || roff < 0 || roff + 4 * q > words || poff < 0 || poff + q * q > words) return;
  if (rec[9] <= 0) return;  // nothing pending: no rows
  for (int i = lane; i < 4 * q; i += 32) sR[wi][i] = grp[roff + i];
  for (int i = lane; i < q * q; i += 32) sP[wi][i] = grp[poff + i];
  if (lane < RBGTOPO_MAX_GROUP_ROLES) sPl[wi][lane] = 0;
  __syncwarp();
  int cr = 0, tk = 0;
  long long row = drow[g];
  while (row < n_rows) {
    if (lane == 0) sNP[wi] = wave_next(sR[wi], q, cr, tk, sRole[wi], sCount[wi]);  // the cursor lives in lane 0
    __syncwarp();
    const int P = sNP[wi];
    if (P == 0) break;
    if (lane < P) {  // one role row per lane: its record
      const int ri = sRole[wi][lane];
      int need = 0;
      for (int j = 0; j < q; ++j)
        if (sP[wi][ri * q + j] > 0) need += sR[wi][4 * j + 1] - sPl[wi][j];
      const bool rexcl = excl && (sR[wi][4 * ri + 3] & RBGTOPO_ROLE_EXCLUSIVE);
      if (row + lane < n_rows)
        rtab[row + lane] = make_int2(emit_pack_row(sR[wi][4 * ri + 2], max(0, min(need, RBGTOPO_NEED_CAP)), rexcl, rec[10] & 7), gid);
    }
    __syncwarp();
    row += P;
    if (lane < P) sPl[wi][sRole[wi][lane]] += sCount[wi][lane];
    __syncwarp();
  }
}

// grid = groups with at least one pending replica = the steps of wave 0; CTA g starts at step g.
// QB = largest role count of a group in the batch, PB = warps per CTA (>= roles of any wave).
// record == 0: the sparse corrections of the dense matrix are applied here (the kernel must run
//   AFTER k_score_emit wrote the background rows: serial pipeline).
// record == 1: the kernel never touches the matrix — selection and the greedy need only the table —
//   and leaves, per step, a compact list of corrections (node, one value per role row: the summed
//   delta, or -inf) in b.corr / b.corr_cnt for k_plan_correct.  It then runs CONCURRENTLY with
//   k_score_emit on a second stream; the step's critical path becomes max(emit, select) + correct.
//
// DIRECT = true (rbgtopo_place_groups, the host-buffer entry point): there is no expanded plan.  b.blob is the GROUPS
// blob as the caller passed it, b.perm[blockIdx.x] the group this CTA places; the CTA replays the group's wave rule
// itself (wave_next), derives every wave's role records (count, demand, predicted need) and pair rows from the
// group's role table, and reports per GROUP: b.status[g] = worst wave status, b.domain_out[g] = the exclusive
// domain.  The host then computes nothing per step — no step numbering, section sizes or prefixes — and launches
// this kernel right behind the dense-matrix kernel (DESIGN.md §4.4).
//
// COMMIT = true (k_plan_group_commit, rbgtopo_place_groups_committed; implies DIRECT): one round of a committed batch
// (DESIGN.md §3.8).  The CTA's group sees the claims of the groups before it through `cm` where it reads node
// attributes — free capacity minus what they took, the owner of a domain they reported — and records what it read.
// No dense matrix exists: the kernel never touches one.  `need` counts the replicas actually placed by earlier
// waves (not the planned ones), so every group is exact without the host-driven loop.
template <bool DIRECT, bool COMMIT, bool CLV = false>
__device__ __forceinline__ void plan_group_body(TopoDev t, BatchDev b, int QB, int HT, int CAP, int record, CommitDev cm) {
  extern __shared__ __align__(16) unsigned char pg_smem[];
  __shared__ int sTakenNode[KS], sTakenAmt[KS], sTakenRole[KS];
  __shared__ int sDstar, sCnt, sNew, sStatus, sAny, sCorrN;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nthreads = blockDim.x, nwarps = nthreads >> 5;
  const int PB = nwarps;
  GroupTab T;
  T.node = reinterpret_cast<int*>(pg_smem);
  T.cons = T.node + HT;
  T.aw = reinterpret_cast<float*>(T.cons + HT);
  T.mask = HT - 1;
  T.HT = HT;
  T.cnt = &sCnt;
  T.dSlot = reinterpret_cast<int*>(T.aw + (size_t)QB * HT);
  T.dBase = reinterpret_cast<float*>(T.dSlot + CAP);
  T.dFree = reinterpret_cast<int*>(T.dBase + CAP);
  T.dDom = T.dFree + CAP;
  // per-role lists (8-byte aligned: everything before is a multiple of 8 bytes when CAP, HT are multiples of 32)
  unsigned long long* sList = reinterpret_cast<unsigned long long*>(T.dDom + CAP);
  unsigned long long* sAcc = sList + (size_t)PB * KS;
  unsigned long long* sPat = sAcc + (size_t)PB * KS;
  int* sListAv = reinterpret_cast<int*>(sPat + (size_t)PB * KS);
  int* sAccAv = sListAv + (size_t)PB * KS;
  int* sPatAv = sAccAv + (size_t)PB * KS;
  GroupRole* sRole = reinterpret_cast<GroupRole*>(sPatAv + (size_t)PB * KS);  // [PB]
  float* sPair = reinterpret_cast<float*>(sRole + PB);                         // [PB][QB]
  int* sGR = reinterpret_cast<int*>(sPair + (size_t)PB * QB);                  // DIRECT: role table of the group [4 * QB]
  int* sPlaced = sGR + 4 * QB;                                                 // DIRECT: replicas of a role in earlier waves [QB]
  // CSR row bounds of the previous wave's placements: live only in phase A, in warp 0's selection scratch (which
  // phase D alone uses)
  int* const sRowB = reinterpret_cast<int*>(sAcc);
  int* const sRowN = sRowB + KS;

  // A dense-matrix kernel of ANOTHER batch may be chained behind this launch as a programmatic dependent
  // (rbgtopo_run_staged_chain): it touches none of this batch's buffers, and its CTAs can only become resident
  // where this kernel leaves registers free — on SMs it does not fill, and everywhere as its CTAs retire.  The
  // trigger comes after this CTA's own wait for the dense-matrix kernel of ITS batch (below), so that "a chained
  // kernel has started" implies "everything up to this batch's dense matrix is complete"; in record mode nothing
  // is waited for.
  if (record) pdl_launch_dependents();
  PCLK(30);
#ifdef RBGTOPO_PHASE_CLOCKS
  if (tid == 0 && blockIdx.x < 2048) { g_cta_ns[blockIdx.x * 4] = pg_gtime(); g_cta_ns[blockIdx.x * 4 + 3] = pg_smid(); }
#endif
  int wave_i = 0;
  int step = b.perm ? b.perm[blockIdx.x] : blockIdx.x;  // launch order: heavy groups dealt across the SMs (rbgtopo.cu)
  // DIRECT: `step` is the group's index in the GROUPS blob; the header is the group record
  __shared__ int sWRole[DIRECT ? RBGTOPO_MAX_STEP_ROLES : 1], sWCount[DIRECT ? RBGTOPO_MAX_STEP_ROLES : 1];
  __shared__ int sWP, sWN, sCr, sTk;
  // DIRECT: first assign index, pending replicas, replicas of earlier waves, first dense role row of the next wave, results
  int g_rep0 = 0, g_pend = 0, g_i0 = 0, g_drow = 0, g_stat = 0, g_dom = -1;
  StepHdr h;
  if (DIRECT) {
    const int* rec = b.blob + RBGTOPO_HDR_WORDS + (size_t)step * RBGTOPO_GROUP_WORDS;
    h.gid = rec[0];
    h.flags = rec[1] & (RBGTOPO_STEP_EXCLUSIVE | RBGTOPO_STEP_GANG);
    h.fixed_domain = (rec[1] & RBGTOPO_STEP_EXCLUSIVE) ? rec[2] : -1;
    h.Q = rec[3];
    h.role_off = rec[4];
    h.pair_off = rec[5];
    h.n_anchors = rec[6];
    h.anchor_off = rec[7];
    h.i0 = 0;
    g_rep0 = rec[8];  // place_groups passes the whole fleet as one batch: assign_off is the assign index
    g_pend = rec[9];
    if (!COMMIT) g_drow = step_drow(b, step, 0);
    h.P = 0; h.R = 0; h.rep_off = g_rep0; h.rolerow_off = 0; h.next_step = 0; h.n_cons = 0; h.cons_off = 0;
  } else {
    h = load_hdr(b, step);  // in flight while the table is cleared
  }
  // every wave of the group is placed at its exclusive level (in a committed batch: level 0 unless CLV)
  const int level = DIRECT ? b.blob[RBGTOPO_HDR_WORDS + (size_t)step * RBGTOPO_GROUP_WORDS + 10] : step_level(h.flags);
  t = at_level(t, level);
  for (int i = tid; i < HT; i += nthreads) {
    T.node[i] = -1;
    T.cons[i] = 0;
  }
  for (int i = tid; i < QB * HT; i += nthreads) T.aw[i] = 0.0f;
  if (tid == 0) sCnt = 0;
  if (DIRECT) {
    for (int i = tid; i < 4 * h.Q; i += nthreads) sGR[i] = b.blob[h.role_off + i];
    if (tid < h.Q) sPlaced[tid] = 0;
    if (tid == 0) { sCr = 0; sTk = 0; }
  }
  const bool excl_step = (h.flags & RBGTOPO_STEP_EXCLUSIVE) != 0;
  const bool gang = (h.flags & RBGTOPO_STEP_GANG) != 0;
  const int gid = h.gid, Q = h.Q;
  if constexpr (COMMIT) {
    cm.g = step;
    cm.excl = excl_step;
    if constexpr (CLV) cm.level = level;
  }
  int fixed = excl_step ? h.fixed_domain : -1;
  g_dom = fixed;  // DIRECT: an exclusive group confirms the domain it already occupies
  const size_t stride = (size_t)t.slab_stride;
  __syncthreads();

  // the group's scheduled pods (anchor records of its first step)
  {
    const int* anc = b.blob + h.anchor_off;
    for (int a = warp; a < h.n_anchors - h.i0; a += nwarps) gtab_add_anchor(t, T, anc[3 * a], anc[3 * a + 1], anc[3 * a + 2], 0);
  }
  int n_new = 0;     // replicas placed by the previous wave: sTaken*[0, n_new)
  int cnt_done = 0;  // dense entries whose node attributes are loaded

  while (true) {
    PCLK(wave_i * 8 + 0);
    // head of the background order for this warp's candidates: in flight during A (used when need > 0)
    const unsigned long long ob0 = lane < t.n ? t.order_all[lane] : 0ull;
    // ---- A. this wave's roles; consumption + CSR row bounds of the previous wave's placements
    if (DIRECT) {
      // the wave itself: role rows and counts from the group's role table (one thread), then the records
      // k_expand_plan would have written: (count, demand, predicted need, flags | group role << 8) and the pair rows
      if (tid == 0) {
        int cr = sCr, tk = sTk;
        const int P = wave_next(sGR, Q, cr, tk, sWRole, sWCount);
        int n = 0;
        for (int k = 0; k < P; ++k) n += sWCount[k];
        sCr = cr;
        sTk = tk;
        sWP = P;
        sWN = n;
      }
      __syncthreads();
      h.P = sWP;
      h.R = sWN;
      h.rep_off = g_rep0 + g_i0;
      h.drow = g_drow;
      if (h.P == 0) break;  // no wave left (a group with pending replicas always has a first one)
      if (tid < h.P) {
        const int ri = sWRole[tid];
        int need = 0;
        for (int j = 0; j < Q; ++j)
          if (b.blob[h.pair_off + ri * Q + j] > 0) need += sGR[4 * j + 1] - sPlaced[j];
        sRole[tid] = GroupRole{sWCount[tid], sGR[4 * ri + 2], min(need, RBGTOPO_NEED_CAP), (sGR[4 * ri + 3] & 0xFF) | (ri << 8)};
      }
      for (int i = tid; i < h.P * Q; i += nthreads)
        sPair[(i / Q) * QB + i % Q] = (float)b.blob[h.pair_off + sWRole[i / Q] * Q + i % Q];
    } else {
      if (tid < h.P) {
        const int4 r = *reinterpret_cast<const int4*>(b.blob + h.role_off + 4 * tid);
        sRole[tid] = GroupRole{r.x, r.y, r.z, r.w};
      }
      for (int i = tid; i < h.P * Q; i += nthreads)
        sPair[(i / Q) * QB + i % Q] = (float)b.blob[h.pair_off + i];
    }
    if (tid == 0) sCorrN = 0;
    if (tid < n_new) {
      const int m = sTakenNode[tid];
      const int rb = t.row_ptr[m], re = t.row_ptr[m + 1];
      sRowB[tid] = rb;
      sRowN[tid] = re - rb + 1;  // + the node itself
      atomicAdd(&T.cons[gtab_insert(T, m)], sTakenAmt[tid]);
    }
    __syncthreads();
    // background candidates of this warp's role: two dependent round trips, consumed in D
    BgCand first;
    const bool have_first = warp < h.P;
    if (have_first) first = bg_attrs(t, sRole[warp].need, lane, t.n, ob0);
    if constexpr (COMMIT)
      if (have_first) commit_adjust<CLV>(first, cm);
    // closed neighbourhoods of the placements: one flat pass over all their CSR entries
    {
      int total = 0;
      for (int a = 0; a < n_new; ++a) total += sRowN[a];
      for (int e = tid; e < total; e += nthreads) {
        int a = 0, off = e;
        while (off >= sRowN[a]) off -= sRowN[a++];
        const int m = sTakenNode[a], q = sTakenRole[a];
        int nn, wv;
        if (off < sRowN[a] - 1) {
          nn = t.col[sRowB[a] + off];
          wv = t.w[sRowB[a] + off];
        } else {
          nn = m;
          wv = RBGTOPO_SELF_W;
        }
        atomicAdd(&T.aw[(size_t)q * HT + gtab_insert(T, nn)], (float)wv);
      }
    }
    __syncthreads();
    PCLK(wave_i * 8 + 1);

    // ---- B. node attributes of the slots claimed since the last wave, capacities of all
    const int cnt = sCnt;
    for (int d = cnt_done + tid; d < cnt; d += nthreads) {
      const int node = T.node[T.dSlot[d]];
      int dd = t.domain[node];
      if (excl_step) {
        int o = t.node_owner[node];
        if constexpr (COMMIT) o = commit_owner<CLV>(cm, node, dd, o);
        if (!(o == -1 || o == gid)) dd |= 0x80000000;
      }
      T.dBase[d] = t.base[node];
      T.dFree[d] = t.free_[node];
      if constexpr (COMMIT) T.dFree[d] -= commit_ext(cm, node);  // the selection notes the read (select_role_group)
      T.dDom[d] = dd;
    }
    cnt_done = cnt;
    __syncthreads();
    PCLK(wave_i * 8 + 2);

    PCLK(wave_i * 8 + 3);
    // ---- D. exclusive domain, selection (warp p = role row p)
    int dstar = excl_step ? fixed : -1;
    if (excl_step && fixed < 0) {
      int pstar = -1;
      for (int p = 0; p < h.P; ++p)
        if (sRole[p].flags & RBGTOPO_ROLE_EXCLUSIVE) { pstar = p; break; }
      if (warp == 0) {
        int d = -1;
        if (pstar >= 0) {
          select_role_group<COMMIT, CLV>(t, gid, excl_step, sRole[pstar], sPair + pstar * QB, Q, 1, DOM_ANY, T,
                                    cnt, pstar == 0, first, 29, sAcc, sAccAv, sPat, sPatAv, sList, sListAv, &cm);
          const unsigned long long top = sList[0];
          d = top ? t.domain[key_node(top)] : -1;
        }
        if (lane == 0) sDstar = d;
      }
      __syncthreads();
      dstar = sDstar;
    }
    if (warp < h.P) {
      const int p = warp;
      const bool rexcl = excl_step && (sRole[p].flags & RBGTOPO_ROLE_EXCLUSIVE);
      const int dom = rexcl ? (dstar >= 0 ? dstar : DOM_NONE) : DOM_ANY;
      int K = 0;
      for (int q = 0; q <= p; ++q) K += sRole[q].count;
      K = min(K, t.n);
      select_role_group<COMMIT, CLV>(t, gid, excl_step, sRole[p], sPair + p * QB, Q, K, dom, T, cnt, true, first,
                                warp == 0 ? wave_i * 8 + 6 : -1, sAcc + p * KS, sAccAv + p * KS, sPat + p * KS,
                                sPatAv + p * KS, sList + p * KS, sListAv + p * KS, &cm);
      if (!DIRECT) b.merged[(size_t)(h.rolerow_off + p) * KS + lane] = sList[p * KS + lane];
    }
    __syncthreads();
    PCLK(wave_i * 8 + 4);

    // ---- C. sparse corrections of this step's matrix rows (fire and forget), by the warps the
    //         greedy does not use (nwarps >= 4)
#ifdef RBGTOPO_PHASE_CLOCKS
    if (!(g_dbg_skip & 1))
#endif
    if (warp != 0 && record && !COMMIT) {
      // one record per patched node of this rank's slab whose rows differ from the background:
      // [node, value of role row 0 .. P-1] (the summed delta, or -inf); region of step s =
      // b.corr + poff[s] * b.corr_w, never more than the step's patch capacity
      int* const reg = b.corr + (size_t)b.poff[step] * b.corr_w;
      for (int d = tid - 32; d < cnt; d += nthreads - 32) {
        const int slot = T.dSlot[d];
        const int node = T.node[slot];
        if (node < t.slab_lo || node >= t.slab_hi) continue;  // another rank's columns
        const int av = gtab_avail(T, d);
        const bool consumed = T.cons[slot] > 0;
        float v[MAXP];
        bool any = false;
#pragma unroll
        for (int p = 0; p < MAXP; ++p) {
          v[p] = 0.0f;
          if (p < h.P) {
            v[p] = (consumed && av < sRole[p].demand) ? -INFINITY
                                                      : gtab_delta(T, sPair + p * QB, Q, slot);
            any |= v[p] != 0.0f;
          }
        }
        if (any) {
          int* e = reg + (size_t)atomicAdd(&sCorrN, 1) * b.corr_w;
          e[0] = node;
#pragma unroll
          for (int p = 0; p < MAXP; ++p)
            if (p < h.P) e[1 + p] = __float_as_int(v[p]);
        }
      }
    } else if (warp != 0 && !COMMIT) {
      // first touch of the matrix: as a programmatic dependent of the dense-matrix kernel, everything up to
      // here (table, selection of wave 0) ran while that kernel was draining; warp 0 (greedy) never waits
      if (wave_i == 0) {
        pdl_wait();
        pdl_launch_dependents();
      }
      float* const mrow0 = b.matrix + (size_t)h.drow * stride - t.slab_lo;  // mrow0[node]
      for (int d = tid - 32; d < cnt; d += nthreads - 32) {
        const int slot = T.dSlot[d];
        const int node = T.node[slot];
        if (node < t.slab_lo || node >= t.slab_hi) continue;  // another rank's columns
        const int av = gtab_avail(T, d);
        const bool consumed = T.cons[slot] > 0;
        float* rowp = mrow0 + node;
        for (int p = 0; p < h.P; ++p, rowp += stride) {
          if (consumed && av < sRole[p].demand) {
            *rowp = -INFINITY;
          } else {
            const float add = gtab_delta(T, sPair + p * QB, Q, slot);
            if (add != 0.0f) sel_red_add_f32(rowp, add);
          }
        }
      }
    }

    // ---- E. greedy (spec §3.6), candidates across lanes: lane k judges list entry k, lane i keeps
    //         placement i; the placements stay in sTaken* for the next wave
    if (warp == 0) {
      int tnode = -1, tamt = 0, trole = 0;
      int ntaken = 0, unplaced = 0, r = 0;
      for (int p = 0; p < h.P; ++p) {
        const int count = sRole[p].count, demand = sRole[p].demand;
        const int grole = (sRole[p].flags >> 8) & 0xFF;
        const unsigned long long key = sList[p * KS + lane];  // descending, zero-padded
        const int node = key ? key_node(key) : -1;
        const int av = sListAv[p * KS + lane];
        for (int c = 0; c < count; ++c, ++r) {
          int used = 0;
          for (int i = 0; i < ntaken; ++i) {
            const int n_i = __shfl_sync(FULL, tnode, i), a_i = __shfl_sync(FULL, tamt, i);
            used += n_i == node ? a_i : 0;
          }
          const uint32_t okm = __ballot_sync(FULL, key != 0 && av - used >= demand);
          const int pick = okm ? __shfl_sync(FULL, node, __ffs(okm) - 1) : -1;
          if (pick >= 0) {
            if (lane == ntaken) { tnode = pick; tamt = demand; trole = grole; }
            ++ntaken;
          } else {
            ++unplaced;
          }
          if (lane == 0) b.assign[h.rep_off + r] = pick;
          if constexpr (COMMIT)
            if (lane == 0 && pick >= 0) sPlaced[grole] += 1;  // placed, not planned: `need` of the next wave is exact
        }
      }
      int status = unplaced ? RBGTOPO_PLACED_PART : RBGTOPO_PLACED_ALL;
      if (unplaced && gang) {
        status = RBGTOPO_GANG_FAILED;
        for (int i = lane; i < h.R; i += 32) b.assign[h.rep_off + i] = -1;
        ntaken = 0;
      }
      if (lane < ntaken) {
        sTakenNode[lane] = tnode;
        sTakenAmt[lane] = tamt;
        sTakenRole[lane] = trole;
      }
      if (lane == 0) {
        if (!DIRECT) {
          b.status[step] = status;
          b.domain_out[step] = dstar;
          b.dstar[step] = dstar;
        }
        sNew = ntaken;
        sStatus = status;
        sAny = ntaken > 0;
      }
    }
    if (DIRECT && !COMMIT && tid < h.P) sPlaced[sWRole[tid]] += sWCount[tid];  // planned, as the host's wave rule counts them
    __syncthreads();
    if (record && tid == 0) b.corr_cnt[step] = sCorrN;
    PCLK(wave_i * 8 + 5);
    ++wave_i;
    if (DIRECT) {  // per-group result (what plan_results derives from the per-step outputs of the expanded plan)
      g_stat = max(g_stat, sStatus);
      // COMMIT: like the host-driven loop, a wave that placed nothing does not move the reported domain (the
      // snapshot path re-runs such groups through that loop)
      if (dstar >= 0 && (!COMMIT || sAny)) g_dom = dstar;
      g_i0 += h.R;
      g_drow += h.P;
      n_new = sNew;
      if (excl_step && dstar >= 0 && sAny) fixed = dstar;
      if (sStatus == RBGTOPO_GANG_FAILED) break;
      continue;  // the next wave, if the role table has one
    }
    if (h.next_step <= 0) break;
    n_new = sNew;
    if (excl_step && dstar >= 0 && sAny) fixed = dstar;
    if (sStatus == RBGTOPO_GANG_FAILED) {  // nothing of the group is placed: its later waves report the failure
      if (warp == 0)
        for (int s2 = h.next_step; s2 > 0;) {
          const StepHdr h2 = load_hdr(b, s2);
          for (int i = lane; i < h2.R; i += 32) b.assign[h2.rep_off + i] = -1;
          if (lane == 0) {
            b.status[s2] = RBGTOPO_GANG_FAILED;
            b.domain_out[s2] = -1;
            b.dstar[s2] = -1;
            if (record) b.corr_cnt[s2] = 0;
          }
          s2 = h2.next_step;
        }
      break;
    }
    step = h.next_step;
    h = load_hdr(b, step);
  }
  if (DIRECT) {
    // a gang group is placed completely or not at all (plan_results does this on the host for expanded plans)
    if (g_stat == RBGTOPO_GANG_FAILED || (gang && g_stat != RBGTOPO_PLACED_ALL)) {
      for (int i = tid; i < g_pend; i += nthreads) b.assign[g_rep0 + i] = -1;
      g_stat = RBGTOPO_GANG_FAILED;
      g_dom = -1;
    }
    if (tid == 0) {
      b.status[step] = g_stat;
      b.domain_out[step] = excl_step ? g_dom : -1;
    }
  }
  PCLK(31);
#ifdef RBGTOPO_PHASE_CLOCKS
  if (tid == 0 && blockIdx.x < 2048) { g_cta_ns[blockIdx.x * 4 + 1] = pg_gtime(); g_cta_ns[blockIdx.x * 4 + 2] = sCnt; }
#endif
}

template <bool DIRECT>
__global__ void __launch_bounds__(32 * MAXP, 4) k_plan_group(TopoDev t, BatchDev b, int QB, int HT, int CAP, int record) {
  plan_group_body<DIRECT, false>(t, b, QB, HT, CAP, record, CommitDev{});
}

// One round of a committed batch (DESIGN.md §3.8): b.perm[0 .. gridDim.x) = the groups of the round (ascending).
// LV: a batch with a group at an exclusive level >= 1 (claims across levels, §3.9); <false> is the level-0 code.
template <bool LV>
__global__ void __launch_bounds__(32 * MAXP, 4) k_plan_group_commit(TopoDev t, BatchDev b, int QB, int HT, int CAP, CommitDev cm) {
  plan_group_body<true, true, LV>(t, b, QB, HT, CAP, 0, cm);
}

// Claims of a committed batch, one warp per group, from the results of the last round (assign / domain_out of the
// plan kernel, the blob for groups with nothing pending): every placed replica links its dense row into the list of
// its node, every exclusive group that reports a domain links itself into the list of the domain.  head / dhead are
// -1 on entry.  A failed gang has no placements and reports no domain.
// LV: the domain is linked at (group level L_h, D), i.e. into dhead[doff[L_h] + D], and every placed replica of a
// participating role of an exclusive group also links into the pod list of (L, dom_L(node)) for every level L of
// cm.lmask other than L_h (slot k = L's rank in lmask; cm.phead is -1 on entry).
template <bool LV>
__global__ void __launch_bounds__(32 * RTAB_WARPS) k_commit_claims(const int* __restrict__ grp, int n_groups,
                                                                 const int* __restrict__ assign, const int* __restrict__ domain,
                                                                 int* head, int4* claim, int* dhead, int2* dclaim, CommitDev cm) {
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * RTAB_WARPS + (threadIdx.x >> 5);
  if (g >= n_groups) return;
  const int* rec = grp + RBGTOPO_HDR_WORDS + (size_t)g * RBGTOPO_GROUP_WORDS;
  const int q = rec[3], roff = rec[4], row0 = rec[8], pend = rec[9];
  const bool excl = (rec[1] & RBGTOPO_STEP_EXCLUSIVE) != 0;
  if (lane == 0 && excl) {
    const int d = pend > 0 ? domain[g] : rec[2];  // nothing pending: the group confirms the domain it occupies
    if (d >= 0) dclaim[g] = make_int2(rec[0], atomicExch(&dhead[(LV ? cm.doff[rec[10]] : 0) + d], g));
  }
  const int nl = LV ? __popc(cm.lmask) : 0;
  int pre = 0;  // a group's rows are its roles' pending replicas in role order
  for (int r = 0; r < q; ++r) {
    const int pr = grp[roff + 4 * r + 1], dem = grp[roff + 4 * r + 2];
    const bool pod = LV && excl && (grp[roff + 4 * r + 3] & RBGTOPO_ROLE_EXCLUSIVE);
    for (int i = lane; i < pr; i += 32) {
      const int row = row0 + pre + i, node = assign[row];
      if (node < 0) continue;
      claim[row] = make_int4(g, dem, atomicExch(&head[node], row), 0);
      if constexpr (LV)
        if (pod) {
          int k = 0;
          for (int m = cm.lmask; m; m &= m - 1, ++k) {
            const int L = __ffs(m) - 1;
            if (L == rec[10]) continue;
            const int e = row * nl + k;
            int* const ph = cm.phead + cm.doff[L] + cm.ldom[(size_t)L * cm.lstride + node];
            cm.pclaim[e] = make_int4(g, rec[0], atomicExch(ph, e), 0);
          }
        }
    }
    pre += pr;
  }
}

// The claim lists of a committed leader-worker batch at levels (DESIGN.md §3.16) are built on the host; their heads
// are dense arrays, so each round only the heads that change are written: heads[set[i].x] = set[i].y.
__global__ void k_set_heads(int* heads, const int2* __restrict__ set, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) heads[set[i].x] = set[i].y;
}

// After a round of a committed batch: which later groups can a changed claim affect?  One warp per group of the round
// (b.perm order).  A group's claims changed when a placement or its reported domain differs from the previous round's
// (`prev`, which is then updated).  A changed claim on node n matters only when a later group read n this round
// (reader[n] > g), a changed domain only when a later exclusive group read a node of it.  *cmin = the lowest group with
// a claim that matters: groups up to it saw exactly the claims they will see from now on, the next round re-runs the
// groups above it.
// LV: a changed domain is (L_h, D); a changed placement of a participating role of an exclusive group also matters when
// a later exclusive group read a node of (L, dom_L) of its old or new node at a level L != L_h of cm.lmask (the pod
// claims of k_commit_claims).  Marks may over-report (a re-run round); they never under-report.
template <bool LV>
__global__ void __launch_bounds__(32 * RTAB_WARPS) k_commit_diff(const int* __restrict__ grp, const int* __restrict__ groups,
                                                               int n_run, const int* __restrict__ assign,
                                                               const int* __restrict__ domain, int* prev_assign,
                                                               int* prev_domain, const int* __restrict__ reader,
                                                               const int* __restrict__ dreader, int* cmin, CommitDev cm) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * RTAB_WARPS + (threadIdx.x >> 5);
  if (k >= n_run) return;
  const int g = groups[k];
  const int* rec = grp + RBGTOPO_HDR_WORDS + (size_t)g * RBGTOPO_GROUP_WORDS;
  const int row0 = rec[8], pend = rec[9];
  bool hit = false;
  if constexpr (!LV) {
    for (int i = lane; i < pend; i += 32) {
      const int a = assign[row0 + i], o = prev_assign[row0 + i];
      if (a != o) {
        hit |= (a >= 0 && reader[a] > g) || (o >= 0 && reader[o] > g);
        prev_assign[row0 + i] = a;
      }
    }
  } else {
    const int q = rec[3], roff = rec[4], lh = rec[10];
    const bool excl = (rec[1] & RBGTOPO_STEP_EXCLUSIVE) != 0;
    auto dread = [&](int node) {  // a later exclusive group read (L, dom_L(node)), L != L_h
      bool r = false;
      for (int m = cm.lmask; m; m &= m - 1) {
        const int L = __ffs(m) - 1;
        if (L != lh) r |= dreader[cm.doff[L] + cm.ldom[(size_t)L * cm.lstride + node]] > g;
      }
      return r;
    };
    int pre = 0;
    for (int r = 0; r < q; ++r) {
      const int pr = grp[roff + 4 * r + 1];
      const bool pod = excl && (grp[roff + 4 * r + 3] & RBGTOPO_ROLE_EXCLUSIVE);
      for (int i = lane; i < pr; i += 32) {
        const int row = row0 + pre + i, a = assign[row], o = prev_assign[row];
        if (a != o) {
          hit |= (a >= 0 && reader[a] > g) || (o >= 0 && reader[o] > g);
          if (pod) hit |= (a >= 0 && dread(a)) || (o >= 0 && dread(o));
          prev_assign[row] = a;
        }
      }
      pre += pr;
    }
  }
  if (lane == 0) {
    const int d = domain[g], od = prev_domain[g];
    if (d != od) {
      const int* const dr = LV ? dreader + cm.doff[rec[10]] : dreader;
      hit |= (d >= 0 && dr[d] > g) || (od >= 0 && dr[od] > g);
      prev_domain[g] = d;
    }
  }
  if (__any_sync(FULL, hit) && lane == 0) atomicMin(cmin, g);
}

// Applies the correction records k_plan_group(record = 1) left: one warp per step, one lane per
// record; a value is added onto the dense row of its role with red.global.add.f32 (exact
// integers, spec §3.4), -inf is stored.  Runs after k_score_emit AND k_plan_group finished.
constexpr int CORRECT_WARPS = 4;
__global__ void __launch_bounds__(32 * CORRECT_WARPS) k_plan_correct(TopoDev t, BatchDev b) {
  const int lane = threadIdx.x & 31;
  const int step = blockIdx.x * CORRECT_WARPS + (threadIdx.x >> 5);
  if (step >= b.n_steps) return;
  const int cnt = b.corr_cnt[step];
  if (cnt <= 0) return;
  const int* __restrict__ hdr = b.blob + RBGTOPO_HDR_WORDS + (size_t)step * RBGTOPO_STEP_WORDS;
  const int P = hdr[3];
  const size_t stride = (size_t)t.slab_stride;
  float* const mrow0 = b.matrix + (size_t)step_drow(b, step, hdr[13]) * stride - t.slab_lo;  // mrow0[node]
  const int* const reg = b.corr + (size_t)b.poff[step] * b.corr_w;
  for (int e = lane; e < cnt; e += 32) {
    const int* rec = reg + (size_t)e * b.corr_w;
    float* rowp = mrow0 + rec[0];
    for (int p = 0; p < P; ++p, rowp += stride) {
      const float v = __int_as_float(rec[1 + p]);
      if (v == -INFINITY) *rowp = -INFINITY;
      else if (v != 0.0f) sel_red_add_f32(rowp, v);
    }
  }
}

}  // namespace rbgtopo
