// kernels.cuh — shared device types and helpers + the per-snapshot kernels of the
// placement hot path (DESIGN.md §4).
//
// Algebra (DESIGN.md §4.1): the spec's score  S_rho = W·A_rho  with
// A_rho = sum_q pair[rho][q]·anchor[q] + need_rho·min(free,F)  is linear in A, so
//     S_rho[n] = need_rho · base[n]  +  sum over anchor pods (m,q,c) of
//                pair[rho][q]·c·W[n][m]
// with base = W·min(free,F) shared by EVERY step of a snapshot (one CSR pass per
// snapshot, k_base below: TMA-staged SpMV) and the anchor term sparse (<= deg+1
// entries per pod).  All terms are exact integers below 2^24 (spec §3.4), so
// this is bit-identical to the oracle's sequential fp32 accumulation.  The dense
// (replica x node) matrix is then a pure HBM write stream (score.cuh) plus
// sparse red.global.add.f32 corrections; selection works from `base`, the
// per-snapshot sorted `order` and the few patched nodes (select_fast.cuh,
// plan_group.cuh) and never scans the matrix.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/rbgtopo.h"

namespace rbgtopo {

constexpr int KS = RBGTOPO_MAX_STEP_REPLICAS;  // list stride (= KMAX = 32)
constexpr int MAXP = RBGTOPO_MAX_STEP_ROLES;
constexpr int MAXQ = RBGTOPO_MAX_GROUP_ROLES;
constexpr int SCORE_THREADS = 256;
constexpr int SCORE_WARPS = SCORE_THREADS / 32;
constexpr int BASE_THREADS = 256;
constexpr int BASE_TILE_ROWS = 256;
constexpr int BASE_TILE_NNZ = 6144;       // 2 x 24 KB staged by TMA bulk copies
constexpr int FMIN_SMEM_MAX = 131072;     // nodes whose u8 fmin vector is staged
constexpr uint32_t FULL = 0xFFFFFFFFu;

struct TopoDev {
  int n;                 // nodes
  int slab_lo, slab_hi;  // node-axis shard of this rank
  int slab_stride;       // floats per matrix row (slab length rounded up to 32)
  const int* row_ptr;
  const int* col;
  const int* w;
  const int* free_;
  const int* domain;
  const int* node_owner;      // owner[domain[n]]
  const unsigned char* fmin;  // min(free, F) as u8, padded to 16 B
  const float* base;          // W·fmin, padded to slab_stride past slab_hi
  // slab nodes sorted by key(base[n], n) descending (one radix sort per snapshot):
  // the "background" order every unpatched row shares (DESIGN.md §4.3)
  const unsigned long long* order;
  const unsigned long long* order_all;  // the same over ALL nodes (== order when world == 1)
  // exclusive levels (occupancy mode, DESIGN.md §3.9): level L's domain / owner vector at L * level_stride(n).  The
  // struct keeps its size (the stride is derived from n): a larger kernel parameter block costs the selection kernels
  // registers
  const int* lvl_domain;
  const int* lvl_owner;
};

// ---- exclusive level of a step or group (DESIGN.md §3.9): bits 8..10 of the step flags on the device (a caller's
// step blob carries it in word +14, which plans use for the wave link), bits 21..23 of a row-table record
constexpr int STEP_LEVEL_SHIFT = 8;
__host__ __device__ __forceinline__ int step_level(int flags) { return (flags >> STEP_LEVEL_SHIFT) & 7; }
__host__ __device__ __forceinline__ int level_stride(int n) { return (n + 31) & ~31; }
// The snapshot as a group at level L sees it: domain / node_owner are level L's vectors.  Level 0 keeps the
// pointers it has (row 0 of lvl_domain / lvl_owner is the same data).
__device__ __forceinline__ TopoDev at_level(TopoDev t, int L) {
  if (L > 0) {
    t.domain = t.lvl_domain + (size_t)L * level_stride(t.n);
    t.node_owner = t.lvl_owner + (size_t)L * level_stride(t.n);
  }
  return t;
}

struct BatchDev {
  const int* blob;
  int n_steps;
  int lc;           // chunks per step on this rank (work items of k_score_emit)
  int chunk;        // nodes per chunk (multiple of 128)
  int parts;        // ranks (list parts to merge)
  int bsteps;       // steps per block of k_score_emit's work order (score.cuh)
  int emit_matrix;
  float* matrix;              // [total R][slab_stride]
  int* cand;                  // per-step scratch: patched slab nodes (select.cuh)
  const int* poff;            // [n_steps + 1] scratch offsets (host prefix of the caps)
  const int* perm;            // [groups with pending replicas] first step of the group CTA i of k_plan_group places, or nullptr
  unsigned long long* lists;  // [rolerows][KS] rank-local top-K per role row
  const unsigned long long* lists_all;  // [parts][rolerows][KS]
  long long part_stride;                // u64 elements between parts
  unsigned long long* merged;  // [rolerows][KS]
  unsigned long long* excl;    // [rolerows][KS] local restricted reselect
  const unsigned long long* excl_all;  // [parts][rolerows][KS]
  long long excl_part_stride;
  int* dstar;    // [n_steps]
  int* assign;   // [total R]
  int* status;   // [n_steps]
  int* domain_out;  // [n_steps]
  // correction records of multi-wave plans (plan_group.cuh: k_plan_group(record) -> k_plan_correct)
  int* corr;      // [patch_cap][corr_w]: node, one value per role row
  int* corr_cnt;  // [n_steps]
  int corr_w;     // 1 + largest role count of a step in the batch
};

// ---- emit table of a multi-wave plan: what the dense-matrix kernels need per step, 12 words —
// gid, step flags, P, first dense row, 8 packed role rows (count | need << 6 | exclusive << 11 | demand << 12;
// count <= 32, need <= 16, demand <= 32767).  Written by k_plan_etab (plan.cuh) straight from the GROUPS
// blob, before the rest of the plan geometry exists, so the matrix can be emitted while the host still
// computes section offsets and patch capacities (DESIGN.md §4.4).
constexpr int EMIT_TAB_WORDS = 12;
__host__ __device__ __forceinline__ int emit_pack_role(int count, int demand, int need, int flags) {
  return count | (need << 6) | ((flags & RBGTOPO_ROLE_EXCLUSIVE) << 11) | (demand << 12);
}

// ---- row table of a multi-wave plan (emit_rows.cuh): per dense row {need | exclusive << 5 | demand << 6 | level << 21,
// gid} (need <= RBGTOPO_NEED_CAP < 32, demand <= 32767).  `exclusive` = the step and the role are exclusive: only then
// does a background row depend on the group (nodes another group owns at the group's level are infeasible).
__host__ __device__ __forceinline__ int emit_pack_row(int demand, int need, bool rexcl, int level) {
  return need | ((rexcl ? 1 : 0) << 5) | (demand << 6) | (level << 21);
}

// ---------------------------------------------------------------- helpers
__device__ __forceinline__ uint32_t orderable_u32(float x) {
  uint32_t b = __float_as_uint(x);
  return b ^ ((b >> 31) ? 0xFFFFFFFFu : 0x80000000u);
}
__device__ __forceinline__ unsigned long long make_key(float s, int node) {
  return ((unsigned long long)orderable_u32(s) << 32) |
         (unsigned long long)(0xFFFFFFFFu - (uint32_t)node);
}
__device__ __forceinline__ int key_node(unsigned long long k) {
  return (int)(0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFull));
}
// warp-wide max of a u64 with two REDUX ops (hi word, then lo among the ties)
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long k) {
  uint32_t hi = (uint32_t)(k >> 32);
  uint32_t mhi = __reduce_max_sync(FULL, hi);
  uint32_t lo = (hi == mhi) ? (uint32_t)k : 0u;
  uint32_t mlo = __reduce_max_sync(FULL, lo);
  return ((unsigned long long)mhi << 32) | mlo;
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
// streaming 128-bit store: the dense matrix is written once and not re-read by
// this kernel, keep it out of L1 and mark it evict-first in L2.
__device__ __forceinline__ void st_stream_f4(float* p, float4 v) {
  asm volatile("st.global.cs.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}

// ---- programmatic dependent launch (griddepcontrol, sm_90+): the primary grid lets its dependents become
// resident early; a dependent blocks in pdl_wait() until the primary grid has completed and its writes are visible.
// Both are no-ops for a kernel launched without the programmatic attribute / with no dependents.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- mbarrier + TMA 1-D bulk copy (cp.async.bulk), sm_90+ -----------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(dst_smem)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ============================================================= k_prep / k_base
// fmin[n] = min(free[n], F) (u8) and node_owner[n] = owner[domain[n]].
__global__ void k_prep(int n, const int* __restrict__ free_, const int* __restrict__ domain,
                       const int* __restrict__ owner, unsigned char* __restrict__ fmin,
                       int* __restrict__ node_owner) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    int f = free_[i];
    fmin[i] = (unsigned char)(f < RBGTOPO_F_CAP ? f : RBGTOPO_F_CAP);
    node_owner[i] = owner[domain[i]];
  }
}

// ============================================================= k_level_owner
// Owner vectors of occupancy mode (DESIGN.md §3.9, rbgtopo_set_exclusive_levels).  Level L's vectors live at
// [L * ls, L * ls + n) of `dom` / `owner` (ls = level_stride(n): the dense-matrix kernels load owners as int4);
// the per-level domain tables are tab[doff[L] + d] (present) and tab[total_d + doff[L] + d] (keyed).  Owner
// values merge with  -1 (+) x = x,  x (+) x = x,  anything else -2  (blocked for every group).
// phase 0: clear the tables; 1: scatter the records (node, gid, level); 2: one gather per node.
__device__ __forceinline__ int owner_merge(int a, int b) { return a == -1 ? b : (b == -1 || a == b) ? a : -2; }
__device__ __forceinline__ void owner_merge_at(int* p, int g) {
  const int old = atomicCAS(p, -1, g);
  if (old != -1 && old != g && old != -2) atomicExch(p, -2);  // -2 absorbs: nothing can leave it afterwards
}
__global__ void k_level_owner(int phase, int n, int n_lv, const int* __restrict__ dom, const int* __restrict__ doff,
                              int total_d, int* __restrict__ tab, const int* __restrict__ occ, int n_occ,
                              int* __restrict__ owner) {
  const int ls = level_stride(n);
  const int stride = gridDim.x * blockDim.x;
  const int i0 = blockIdx.x * blockDim.x + threadIdx.x;
  if (phase == 0) {
    for (int i = i0; i < 2 * total_d; i += stride) tab[i] = -1;
  } else if (phase == 1) {
    for (int r = i0; r < n_occ; r += stride) {
      const int node = occ[3 * r], gid = occ[3 * r + 1], lv = occ[3 * r + 2];
      for (int L = 0; L < n_lv; ++L) {
        const int d = doff[L] + dom[(size_t)L * ls + node];
        owner_merge_at(tab + d, gid);                       // present: records count at every level
        if (L == lv) owner_merge_at(tab + total_d + d, gid);  // keyed: only at the record's own level
      }
    }
  } else {
    for (int v = i0; v < n; v += stride) {
      int k = -1;
      for (int L = 0; L < n_lv; ++L) k = owner_merge(k, tab[total_d + doff[L] + dom[(size_t)L * ls + v]]);
      for (int L = 0; L < n_lv; ++L) owner[(size_t)L * ls + v] = owner_merge(tab[doff[L] + dom[(size_t)L * ls + v]], k);
    }
  }
}

// base[n] = sum_j w_j * fmin[col_j] + SELF_W * fmin[n]   for the rows of one tile.
// The tile's contiguous col_idx / edge_w segment and (when it fits) the whole u8
// fmin vector are staged into shared memory with TMA bulk copies completing on
// one mbarrier; 8 lanes walk one row (vector of int32 gathers from smem, fp32
// accumulate), reduced with warp shuffles.  tiles[] = (row0, row1) pairs built on
// the host so that nnz <= BASE_TILE_NNZ (a single over-long row is its own tile
// and reads global memory directly).
__global__ void __launch_bounds__(BASE_THREADS)
k_base(TopoDev t, const int2* __restrict__ tiles, int fmin_staged, int fmin_bytes,
       float* __restrict__ base_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t bar;
  int* s_col = reinterpret_cast<int*>(smem_raw);
  int* s_w = s_col + (BASE_TILE_NNZ + 8);
  unsigned char* s_fmin = reinterpret_cast<unsigned char*>(s_w + (BASE_TILE_NNZ + 8));

  const int2 tile = tiles[blockIdx.x];
  const int r0 = tile.x, r1 = tile.y;
  const int e0 = t.row_ptr[r0], e1 = t.row_ptr[r1];
  const int a0 = e0 & ~3;  // 16-byte aligned segment start
  const int seg = e1 - a0;
  const bool staged = seg <= BASE_TILE_NNZ + 4;
  const uint32_t seg_bytes = (uint32_t)(((seg * 4) + 15) & ~15);

  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t total = (staged ? 2u * seg_bytes : 0u) + (fmin_staged ? (uint32_t)fmin_bytes : 0u);
    mbar_expect_tx(&bar, total);
    if (staged && seg_bytes) {
      bulk_g2s(s_col, t.col + a0, seg_bytes, &bar);
      bulk_g2s(s_w, t.w + a0, seg_bytes, &bar);
    }
    if (fmin_staged) bulk_g2s(s_fmin, t.fmin, (uint32_t)fmin_bytes, &bar);
  }
  mbar_wait(&bar, 0);

  const unsigned char* fm = fmin_staged ? s_fmin : t.fmin;
  const int sub = threadIdx.x & 7;
  const int iters = (r1 - r0 + (BASE_THREADS / 8) - 1) / (BASE_THREADS / 8);
  for (int it = 0; it < iters; ++it) {
    const int r = r0 + it * (BASE_THREADS / 8) + (threadIdx.x >> 3);
    float acc = 0.0f;
    if (r < r1) {
      const int rb = t.row_ptr[r], re = t.row_ptr[r + 1];
      if (staged) {
        for (int j = rb + sub; j < re; j += 8)
          acc += (float)s_w[j - a0] * (float)fm[s_col[j - a0]];
      } else {
        for (int j = rb + sub; j < re; j += 8) acc += (float)t.w[j] * (float)fm[t.col[j]];
      }
    }
    acc += __shfl_xor_sync(FULL, acc, 4);
    acc += __shfl_xor_sync(FULL, acc, 2);
    acc += __shfl_xor_sync(FULL, acc, 1);
    if (r < r1 && sub == 0) base_out[r] = acc + (float)RBGTOPO_SELF_W * (float)fm[r];
  }
}

// ======================================================= background order, small snapshots
// order[0 .. hi-lo) = the nodes [lo, hi) sorted by key(base[n], n) descending, for slabs of at most
// ORDER_SMALL_MAX nodes: ONE CTA, bitonic network in shared memory (keys are unique, so the order is the
// same total order a radix sort gives), instead of a 4-pass library radix sort plus its key build /
// expansion kernels; larger slabs keep the library sort.
constexpr int ORDER_SMALL_MAX = 16384;
constexpr int ORDER_SMALL_THREADS = 1024;
__global__ void __launch_bounds__(ORDER_SMALL_THREADS) k_order_sort_small(const float* __restrict__ base, int lo, int hi,
                                                                          unsigned long long* __restrict__ order) {
  extern __shared__ __align__(16) unsigned long long so_keys[];
  const int n = hi - lo;
  int p2 = 32;
  while (p2 < n) p2 <<= 1;
  for (int i = threadIdx.x; i < p2; i += ORDER_SMALL_THREADS) so_keys[i] = i < n ? make_key(base[lo + i], lo + i) : 0ull;  // 0 sorts last
  __syncthreads();
  for (int k = 2; k <= p2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (p2 >> 1); t += ORDER_SMALL_THREADS) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // lower index of the t-th pair at distance j
        const int l = i | j;
        const unsigned long long a = so_keys[i], b2 = so_keys[l];
        const bool desc = (i & k) == 0;  // final pass (k == p2): every pair descending
        if ((a < b2) == desc) {
          so_keys[i] = b2;
          so_keys[l] = a;
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < n; i += ORDER_SMALL_THREADS) order[i] = so_keys[i];
}

// ================================================== incremental snapshot refresh (SURVEY.md §8f rank 3)
// A few nodes changed their free capacity (a pod was bound / deleted).  base = W * min(free, F) is linear in
// fmin, so  base[n] += w(n, m) * delta_m  over the closed neighbourhood of every changed node m — exact
// integer arithmetic below 2^24, hence bit-identical to a full recomputation in any order — and the
// background order is REPAIRED: the affected entries are taken out and merged back at their new rank
// instead of sorting all N keys again.  pos[node] = the node's position in `order` is kept beside it.
constexpr int DELTA_MAX_AFFECTED = 2048;  // affected nodes one repair handles (above: full refresh)

// order -> pos (after every full sort)
__global__ void k_order_pos(const unsigned long long* __restrict__ order, int n, int* __restrict__ pos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) pos[key_node(order[i])] = i;
}

// One warp per changed node: new capacity, delta onto the neighbourhood's base, affected nodes appended once.
// `changed` = (node, free) pairs, host-deduplicated.  aff[0] = counter, aff[1 ..] = affected nodes.
__global__ void k_delta_apply(TopoDev t, int* __restrict__ free_w, unsigned char* __restrict__ fmin_w, float* __restrict__ base_w,
                              const int* __restrict__ changed, int n_changed, int* __restrict__ flag, int* __restrict__ aff) {
  const int lane = threadIdx.x & 31;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (c >= n_changed) return;
  const int m = changed[2 * c], f_new = changed[2 * c + 1];
  const int f_old = free_w[m];
  const int d = min(f_new, RBGTOPO_F_CAP) - min(f_old, RBGTOPO_F_CAP);
  if (lane == 0) {
    free_w[m] = f_new;
    fmin_w[m] = (unsigned char)min(f_new, RBGTOPO_F_CAP);
  }
  if (d == 0) return;  // the scores only see min(free, F): nothing else moves (capacity itself is read live)
  const int rb = t.row_ptr[m], re = t.row_ptr[m + 1];
  for (int j = rb + lane; j <= re; j += 32) {  // j == re stands for m itself
    const int nn = j < re ? t.col[j] : m;
    const int wv = j < re ? t.w[j] : RBGTOPO_SELF_W;
    atomicAdd(&base_w[nn], (float)(wv * d));
    if (atomicExch(&flag[nn], 1) == 0) {
      const int k = atomicAdd(&aff[0], 1);
      if (k < DELTA_MAX_AFFECTED) aff[1 + k] = nn;
    }
  }
}

// One CTA: the affected nodes' new keys (descending) and old positions (ascending), both sorted in shared
// memory by a bitonic network (<= 2048 elements: 66 short rounds); flags cleared for the next delta.
__global__ void __launch_bounds__(1024) k_delta_sort(const float* __restrict__ base, const int* __restrict__ pos,
                                                     int* __restrict__ flag, int* __restrict__ aff,
                                                     unsigned long long* __restrict__ new_keys, int* __restrict__ old_pos) {
  __shared__ unsigned long long sk[DELTA_MAX_AFFECTED];
  __shared__ int sp[DELTA_MAX_AFFECTED];
  const int A = min(aff[0], DELTA_MAX_AFFECTED);
  int p2 = 32;
  while (p2 < A) p2 <<= 1;
  for (int i = threadIdx.x; i < p2; i += blockDim.x) {
    if (i < A) {
      const int node = aff[1 + i];
      sk[i] = make_key(base[node], node);
      sp[i] = pos[node];
      flag[node] = 0;
    } else {
      sk[i] = 0ull;        // sorts last (descending)
      sp[i] = 0x7FFFFFFF;  // sorts last (ascending)
    }
  }
  __syncthreads();
  for (int k = 2; k <= p2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int tt = threadIdx.x; tt < (p2 >> 1); tt += blockDim.x) {
        const int i = ((tt & ~(j - 1)) << 1) | (tt & (j - 1)), l = i | j;
        const bool up = (i & k) == 0;
        const unsigned long long a = sk[i], b2 = sk[l];
        if ((a < b2) == up) { sk[i] = b2; sk[l] = a; }   // keys: descending
        const int pa = sp[i], pb = sp[l];
        if ((pa > pb) == up) { sp[i] = pb; sp[l] = pa; }  // positions: ascending
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < A; i += blockDim.x) {
    new_keys[i] = sk[i];
    old_pos[i] = sp[i];
  }
}

// Merge: every kept entry of the old order moves by (new keys above it) - (removed entries before it);
// every affected node is inserted at (its rank among the new keys) + (kept entries above it).
__global__ void k_delta_merge(const unsigned long long* __restrict__ order_old, int n, const int* __restrict__ aff,
                              const unsigned long long* __restrict__ new_keys, const int* __restrict__ old_pos,
                              unsigned long long* __restrict__ order_new, int* __restrict__ pos) {
  const int A = min(aff[0], DELTA_MAX_AFFECTED);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  auto removed_before = [&](int p) {  // old positions < p that were taken out
    int lo = 0, hi = A;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (old_pos[mid] < p) lo = mid + 1; else hi = mid; }
    return lo;
  };
  if (i < n) {
    const unsigned long long key = order_old[i];
    const int rb = removed_before(i);
    const bool removed = rb < A && old_pos[rb] == i;
    if (!removed) {
      int lo = 0, hi = A;  // new keys greater than key (new_keys is descending)
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (new_keys[mid] > key) lo = mid + 1; else hi = mid; }
      const int np = i - rb + lo;
      order_new[np] = key;
      pos[key_node(key)] = np;
    }
  }
  if (i < A) {
    const unsigned long long key = new_keys[i];
    int lo = 0, hi = n;  // old entries greater than key (order_old is descending); the node's own old entry may count: it is removed below
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (order_old[mid] > key) lo = mid + 1; else hi = mid; }
    const int np = i + lo - removed_before(lo);
    order_new[np] = key;
    pos[key_node(key)] = np;
  }
}

}  // namespace rbgtopo
