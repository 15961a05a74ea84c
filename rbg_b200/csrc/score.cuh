// score.cuh — k_score_emit: the dominant kernel of the path (DESIGN.md §4.2).
//
// Emits the dense score matrix of a step-level batch (one row per role row: step_drow) as a pure HBM write stream.
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
//      else -inf; written once for all replicas of the role.  (Multi-wave plans
//      take k_emit_rows, emit_rows.cuh, and their corrections are applied by the
//      kernel that knows the placements, plan_group.cuh.)
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
#include "plan_group.cuh"

namespace rbgtopo {

constexpr int GPT = 2;  // float4 groups per thread: chunk <= 256 * 4 * GPT = 2048

__device__ __forceinline__ void red_add_f32(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// Why the loop nest is (chunk outer, steps inner): with one (step, chunk) item per iteration a
// single-replica step cost ~117 instructions per 512-byte warp store (SASS count: node operands,
// tail fix-up and header decode per store); here they are amortised over the block's steps.
constexpr int EMIT_MAX_BLOCK = 16;  // upper bound of b.bsteps

// CLAIMS (k_score_emit_claims, rbgtopo_place_groups_lw_committed, DESIGN.md §3.13): exclusive domains earlier groups of a
// committed batch reported.  Per step, claim_rec[claim_off[step] .. claim_off[step + 1]) = {node, claim gid} for every
// node of a claimed level-0 domain.  The effective owner is the claim gid (map mode) or owner_merge(node_owner[n], gid)
// (occupancy, `occ`); participating rows of exclusive steps are rewritten to need·base[n] or -inf there, BEFORE the
// consumed and anchor passes (-inf absorbs their adds, and an unblocked node must exist before them).  The step's
// consumed records are then sorted by node with one record per node, so a record is its node's whole amount.
// LV (k_score_emit_claims_lv, a batch with a group at an exclusive level >= 1, DESIGN.md §3.16): no records.  The
// background pass of an exclusive step reads each node's owner as commit_owner<true> gives it to group
// step_grp[step] at the step's level (owner_L ⊕ K ⊕ P, the claim lists `cm0` the host built from the previous round).
// ELIG (k_score_emit_elig, rbgtopo_place_groups_eligible[_ranked], DESIGN.md §3.19): node classes.  cls[n] = the class
// of node n (u8, padded past the last node like free_); admit[step * MAXP + p] = the classes role row p of the step may
// use.  A node whose class bit is clear counts as having no room (-1) for that row, so its background entry is -inf and
// the sparse pass, which only adds onto entries or sets them to -inf, keeps it there.  With CLAIMS as well
// (k_score_emit_claims[_lv]_elig, rbgtopo_place_groups_eligible_committed[_ranked], DESIGN.md §3.20): LV masks after
// commit_owner like any other owner; the level-0 rewrite of claimed nodes tests the class bit too.
template <bool CLAIMS, bool LV = false, bool ELIG = false>
__device__ __forceinline__ void score_emit(TopoDev t, BatchDev b, int items, const int* __restrict__ claim_off,
                                           const int2* __restrict__ claim_rec, bool occ,
                                           const int* __restrict__ step_grp = nullptr, const CommitDev* cm0 = nullptr,
                                           const unsigned char* __restrict__ cls = nullptr,
                                           const unsigned long long* __restrict__ admit = nullptr) {
  const int T = b.chunk, lc = b.lc;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int groups = T >> 2;
  const int* __restrict__ blob = b.blob;
  const size_t stride = (size_t)t.slab_stride;

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
  __shared__ int sRoleOff[EMIT_MAX_BLOCK], sDrow[EMIT_MAX_BLOCK];
  __shared__ int4 sRoles[EMIT_MAX_BLOCK][MAXP];        // count demand need flags
  if (tid < nst) {
    const int* __restrict__ hdr = blob + RBGTOPO_HDR_WORDS + (size_t)(step0 + tid) * RBGTOPO_STEP_WORDS;
    sH0[tid] = __ldg(reinterpret_cast<const int4*>(hdr));
    sRoleOff[tid] = __ldg(hdr + 4);
    sDrow[tid] = step_drow(b, step0 + tid, __ldg(hdr + 13));
  }
  __syncthreads();
  __shared__ unsigned long long sAdmit[ELIG ? EMIT_MAX_BLOCK : 1][ELIG ? MAXP : 1];
  if (tid < nst * MAXP) {
    const int s = tid / MAXP, p = tid - s * MAXP;
    if (p < sH0[s].w) sRoles[s][p] = __ldg(reinterpret_cast<const int4*>(blob + sRoleOff[s]) + p);
    if constexpr (ELIG)
      if (p < sH0[s].w) sAdmit[s][p] = __ldg(admit + (size_t)(step0 + s) * MAXP + p);
  }
  __syncthreads();
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
      float* const mrow0 = b.matrix + (size_t)sDrow[si] * stride + (n0 - t.slab_lo);

      // ---- 1. background rows
#pragma unroll
      for (int j = 0; j < GPT; ++j) {
        if (!live[j]) continue;
        const int g = tid + j * SCORE_THREADS;
        int4 avx = av[j];  // capacity as seen by exclusive roles: blocked domains are infeasible
        if (excl_step) {
          int4 ow = __ldg(reinterpret_cast<const int4*>(at_level(t, step_level(h0.y)).node_owner + n0 + (g << 2)));
          if constexpr (LV) {
            const int n = n0 + (g << 2);
            const int4 dm = __ldg(reinterpret_cast<const int4*>(at_level(t, step_level(h0.y)).domain + n));
            CommitDev cm = *cm0;
            cm.g = __ldg(step_grp + step);
            cm.level = step_level(h0.y);
            ow.x = commit_owner<true>(cm, n, dm.x, ow.x);  // n < n1: live
            if (n + 1 < n1) ow.y = commit_owner<true>(cm, n + 1, dm.y, ow.y);
            if (n + 2 < n1) ow.z = commit_owner<true>(cm, n + 2, dm.z, ow.z);
            if (n + 3 < n1) ow.w = commit_owner<true>(cm, n + 3, dm.w, ow.w);
          }
          if (!(ow.x == -1 || ow.x == gid)) avx.x = -1;
          if (!(ow.y == -1 || ow.y == gid)) avx.y = -1;
          if (!(ow.z == -1 || ow.z == gid)) avx.z = -1;
          if (!(ow.w == -1 || ow.w == gid)) avx.w = -1;
        }
        float* rowp = mrow0 + (g << 2);
        // ELIG: the classes of the group's four nodes, one per byte (n % 4 == 0, padded: safe).  Loaded per step
        // (L1-hot after the first) rather than held across the step loop, which would cost two more live registers.
        unsigned cls4 = 0;
        if constexpr (ELIG) cls4 = __ldg(reinterpret_cast<const unsigned*>(cls + n0 + (g << 2)));
        for (int p = 0; p < P; ++p) {
          const int4 role = roles[p];  // count demand need flags
          const float need = (float)role.z;
          int4 a = (role.w & RBGTOPO_ROLE_EXCLUSIVE) ? avx : av[j];
          if constexpr (ELIG) {
            const unsigned long long m = sAdmit[si][p];
            if (!((m >> (cls4 & 0xFF)) & 1)) a.x = -1;
            if (!((m >> ((cls4 >> 8) & 0xFF)) & 1)) a.y = -1;
            if (!((m >> ((cls4 >> 16) & 0xFF)) & 1)) a.z = -1;
            if (!((m >> (cls4 >> 24)) & 1)) a.w = -1;
          }
          float4 o4;
          o4.x = a.x >= role.y ? need * base4[j].x : -INFINITY;
          o4.y = a.y >= role.y ? need * base4[j].y : -INFINITY;
          o4.z = a.z >= role.y ? need * base4[j].z : -INFINITY;
          o4.w = a.w >= role.y ? need * base4[j].w : -INFINITY;
          st_stream_f4(rowp, o4);
          rowp += stride;
        }
      }

      if constexpr (CLAIMS && !LV) {
        const int c0 = __ldg(claim_off + step), c1 = __ldg(claim_off + step + 1);
        if (excl_step && c1 > c0) {
          __syncthreads();  // the background stores precede the rewrite
          for (int i = c0 + tid; i < c1; i += SCORE_THREADS) {
            const int2 cl = __ldg(claim_rec + i);
            const int m = cl.x;
            if (m < n0 || m >= n1) continue;
            const int ow = occ ? owner_merge(__ldg(t.node_owner + m), cl.y) : cl.y;
            const int a = (ow == -1 || ow == gid) ? __ldg(t.free_ + m) : -1;
            const float bm = __ldg(t.base + m);
            if constexpr (ELIG) {  // the rewrite must not turn a class-excluded node back into a finite entry
              const unsigned k = __ldg(cls + m);
              for (int p = 0; p < P; ++p)
                if (roles[p].w & RBGTOPO_ROLE_EXCLUSIVE)
                  mrow0[(size_t)p * stride + (m - n0)] =
                      a >= roles[p].y && ((sAdmit[si][p] >> k) & 1) ? (float)roles[p].z * bm : -INFINITY;
            } else {
              for (int p = 0; p < P; ++p)
                if (roles[p].w & RBGTOPO_ROLE_EXCLUSIVE)
                  mrow0[(size_t)p * stride + (m - n0)] = a >= roles[p].y ? (float)roles[p].z * bm : -INFINITY;
            }
          }
          __syncthreads();  // ... and the consumed and anchor passes follow it
        }
      }

      // ---- 2. sparse corrections.  Few records: every warp scans them all and
      // applies the ones inside its own segments (ordering by __syncwarp alone).
      // Many records: one block barrier, then the records are spread over warps.
      const int4 h1 = __ldg(reinterpret_cast<const int4*>(hdr) + 1);  // role_off Q pair_off n_anchors
      const int4 h2 = __ldg(reinterpret_cast<const int4*>(hdr) + 2);  // anchor_off n_cons cons_off R
      if ((h1.w | h2.y) != 0) {
        const bool own = (h1.w + h2.y) <= 2;
        if (own) __syncwarp(); else __syncthreads();  // background stores precede the reductions
        const int* __restrict__ con = blob + h2.z;
        for (int c = own ? lane : tid; c < h2.y; c += own ? 32 : SCORE_THREADS) {  // consumed capacity
          const int m = __ldg(con + 2 * c);
          const int g = (m - n0) >> 2;
          if (m >= n0 && m < n1 && (!own || ((g & (SCORE_THREADS - 1)) >> 5) == warp)) {
            int amt = 0;
            if constexpr (CLAIMS) {
              amt = __ldg(con + 2 * c + 1);  // one record per node
            } else {
              for (int k = 0; k < h2.y; ++k)
                if (__ldg(con + 2 * k) == m) amt += __ldg(con + 2 * k + 1);  // duplicates add up
            }
            const int avail = __ldg(t.free_ + m) - amt;
            for (int p = 0; p < P; ++p)
              if (avail < roles[p].y) mrow0[(size_t)p * stride + (m - n0)] = -INFINITY;
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
              for (int p = 0; p < P; ++p) {
                const int coef = __ldg(blob + h1.z + p * Q + q);
                if (coef) red_add_f32(mrow0 + (size_t)p * stride + (nn - n0), (float)(coef * wv));
              }
            }
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(SCORE_THREADS, 6)
k_score_emit(TopoDev t, BatchDev b, int items) {
  score_emit<false>(t, b, items, nullptr, nullptr, false);
}

// Only rbgtopo_place_groups_lw_committed launches this variant.
__global__ void __launch_bounds__(SCORE_THREADS, 6)
k_score_emit_claims(TopoDev t, BatchDev b, int items, const int* __restrict__ claim_off,
                    const int2* __restrict__ claim_rec, bool occ) {
  score_emit<true>(t, b, items, claim_off, claim_rec, occ);
}

// rbgtopo_place_groups_lw_committed[_ranked] on a batch with a group at a level >= 1 (DESIGN.md §3.16): step_grp[step]
// = the step's group index in the batch; cm = the claim lists of the groups' previous-round results.
__global__ void __launch_bounds__(SCORE_THREADS, 6)
k_score_emit_claims_lv(TopoDev t, BatchDev b, int items, const int* __restrict__ step_grp, CommitDev cm) {
  score_emit<true, true>(t, b, items, nullptr, nullptr, true, step_grp, &cm);
}

// rbgtopo_place_groups_eligible[_ranked] (DESIGN.md §3.19): the waves of the leader-worker loop with node classes;
// admit = the mask section of the wave's side table, MAXP entries per step.
__global__ void __launch_bounds__(SCORE_THREADS, 6)
k_score_emit_elig(TopoDev t, BatchDev b, int items, const unsigned char* __restrict__ cls,
                  const unsigned long long* __restrict__ admit) {
  score_emit<false, false, true>(t, b, items, nullptr, nullptr, false, nullptr, nullptr, cls, admit);
}

// rbgtopo_place_groups_eligible_committed[_ranked] (DESIGN.md §3.20): k_score_emit_claims with node classes (a batch at
// level 0) ...
__global__ void __launch_bounds__(SCORE_THREADS, 6)
k_score_emit_claims_elig(TopoDev t, BatchDev b, int items, const int* __restrict__ claim_off,
                         const int2* __restrict__ claim_rec, bool occ, const unsigned char* __restrict__ cls,
                         const unsigned long long* __restrict__ admit) {
  score_emit<true, false, true>(t, b, items, claim_off, claim_rec, occ, nullptr, nullptr, cls, admit);
}

// ... and k_score_emit_claims_lv with node classes (a batch with a group at a level >= 1).
__global__ void __launch_bounds__(SCORE_THREADS, 6)
k_score_emit_claims_lv_elig(TopoDev t, BatchDev b, int items, const int* __restrict__ step_grp, CommitDev cm,
                            const unsigned char* __restrict__ cls, const unsigned long long* __restrict__ admit) {
  score_emit<true, true, true>(t, b, items, nullptr, nullptr, true, step_grp, &cm, cls, admit);
}

}  // namespace rbgtopo
