// Device-side expansion of a GROUPS blob into the wave-major step blob of a
// multi-wave plan (DESIGN.md §4.4).  The host only computes the per-step
// geometry (which group / wave a step is, where its section starts, its replica
// and role-row prefixes); the ~4x larger step blob itself — headers, role
// records with the predicted `need`, pair rows, anchor records, the placeholder
// records the waves fill in — never exists on the host and never crosses PCIe.
//
// `grp` = device copy of the GROUPS blob exactly as the caller passed it (include/rbgtopo.h);
// it is the head of the staging buffer `src`, or the one an earlier batch of the same call
// uploaded.  Staging buffer (device copy of what the host wrote into pinned memory):
//   [0, gwords)               the GROUPS blob (absent when `grp` points elsewhere)
//   [aux_off, +8*ns)          per step: group, wave, sec_off, sec_end, rep_off, row_off, next_step, i0
//   [tail_off, +tail_words)   poff[ns + 1], copied behind the plan
//
// The wave rule is the one of plugin.py / place_groups_slow (a wave = the next
// <= 32 replicas of <= 8 roles of one dependency level); it is replayed per step
// from the group's role table, so the host does not ship the wave table either.
#pragma once
#include <cstdint>

#include "../../include/rbgtopo.h"
#include "kernels.cuh"

namespace rbgtopo {

constexpr int PLAN_AUX_WORDS = 8;

constexpr int PLAN_WARPS = 4;  // warps (= steps) per CTA of k_expand_plan

// Per-warp scratch: the group's record, role table and pair matrix (one coalesced round of
// loads), then the wave of this step and the per-role placed-before counts.
struct PlanScratch {
  int rec[RBGTOPO_GROUP_WORDS];
  int roles[4 * RBGTOPO_MAX_GROUP_ROLES];
  int pair[RBGTOPO_MAX_GROUP_ROLES * RBGTOPO_MAX_GROUP_ROLES];
  int placed[RBGTOPO_MAX_GROUP_ROLES];
  int cum[RBGTOPO_MAX_GROUP_ROLES + 1];  // prefix of placed[]: replicas of earlier waves, group order
  int n;                                 // roles of this wave
  int role[RBGTOPO_MAX_STEP_ROLES], count[RBGTOPO_MAX_STEP_ROLES];
};

// Replays the wave rule of a group up to wave `w` (one lane, shared-memory operands):
// S->role/count/n = that wave, S->placed[j] = replicas of role j placed by the waves before it.
__device__ __forceinline__ void plan_wave_at(PlanScratch* S, int q, int w) {
  const int* roles = S->roles;
  int cr = 0, taken = 0, idx = 0;
  for (int j = 0; j < RBGTOPO_MAX_GROUP_ROLES; ++j) S->placed[j] = 0;
  S->n = 0;
  while (cr < q) {
    if (roles[4 * cr + 1] - taken <= 0) { ++cr; taken = 0; continue; }
    const int level = roles[4 * cr];
    int n = 0, P = 0;
    while (cr < q && roles[4 * cr] == level && n < RBGTOPO_MAX_STEP_REPLICAS && P < RBGTOPO_MAX_STEP_ROLES) {
      const int left = roles[4 * cr + 1] - taken;
      if (left <= 0) { ++cr; taken = 0; continue; }
      const int take = min(left, RBGTOPO_MAX_STEP_REPLICAS - n);
      S->role[P] = cr; S->count[P] = take;
      ++P;
      n += take;
      taken += take;
      if (taken == roles[4 * cr + 1]) { ++cr; taken = 0; }
    }
    S->n = P;
    if (idx == w) break;
    for (int k = 0; k < P; ++k) S->placed[S->role[k]] += S->count[k];
    ++idx;
  }
  int acc = 0;
  for (int j = 0; j < RBGTOPO_MAX_GROUP_ROLES; ++j) { S->cum[j] = acc; acc += S->placed[j]; }
  S->cum[RBGTOPO_MAX_GROUP_ROLES] = acc;
}

// Emit table of the plan (kernels.cuh), one warp per step, from the GROUPS blob and the step numbering
// alone: sgw = (group, wave) per step.  The role rows (count, demand, predicted need) are those
// k_expand_plan writes into the step blob later; the first dense row of a step is the group's offset in
// the batch (assign_off - row_base) plus the replicas of the group's earlier waves — GROUP order, no
// prefix over steps needed.  Runs right after the first H2D of rbgtopo_place_groups.
//
// rtab (emit_rows.cuh) is the same information per DENSE ROW: {need | exclusive << 5 | demand << 6, gid} for every
// replica row of the step, `exclusive` set only when the step AND the role are exclusive (the one case in
// which the row depends on the group) — k_emit_rows walks rows, not steps.
__global__ void __launch_bounds__(32 * PLAN_WARPS) k_plan_etab(const int* __restrict__ grp, const int* __restrict__ sgw, int ns,
                                                               int row_base, int* __restrict__ etab, int2* __restrict__ rtab) {
  __shared__ PlanScratch scratch[PLAN_WARPS];
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * PLAN_WARPS + (threadIdx.x >> 5);
  if (s >= ns) return;
  PlanScratch* S = &scratch[threadIdx.x >> 5];
  const int g = sgw[2 * s], w = sgw[2 * s + 1];
  if (lane < RBGTOPO_GROUP_WORDS) S->rec[lane] = grp[RBGTOPO_HDR_WORDS + (long long)g * RBGTOPO_GROUP_WORDS + lane];
  __syncwarp();
  const int q = S->rec[3];
  const int* g_roles = grp + S->rec[4];
  const int* g_pair = grp + S->rec[5];
  for (int i = lane; i < 4 * q; i += 32) S->roles[i] = g_roles[i];
  for (int i = lane; i < q * q; i += 32) S->pair[i] = g_pair[i];
  __syncwarp();
  if (lane == 0) plan_wave_at(S, q, w);
  __syncwarp();
  const int P = S->n;
  int* e = etab + (size_t)s * EMIT_TAB_WORDS;
  if (lane < RBGTOPO_MAX_STEP_ROLES) {
    int packed = 0;
    if (lane < P) {
      const int ri = S->role[lane];
      int need = 0;
      for (int j = 0; j < q; ++j)
        if (S->pair[ri * q + j] > 0) need += S->roles[4 * j + 1] - S->placed[j];
      need = min(need, RBGTOPO_NEED_CAP);
      packed = emit_pack_role(S->count[lane], S->roles[4 * ri + 2], need, S->roles[4 * ri + 3]);
      int r0 = S->rec[8] - row_base + S->cum[RBGTOPO_MAX_GROUP_ROLES];  // first dense row of the step
      for (int k = 0; k < lane; ++k) r0 += S->count[k];
      const bool rexcl = (S->rec[1] & RBGTOPO_STEP_EXCLUSIVE) && (S->roles[4 * ri + 3] & RBGTOPO_ROLE_EXCLUSIVE);
      const int2 rr = make_int2(emit_pack_row(S->roles[4 * ri + 2], need, rexcl, S->rec[10]), S->rec[0]);
      for (int k = 0; k < S->count[lane]; ++k) rtab[r0 + k] = rr;
    }
    e[4 + lane] = packed;
  } else if (lane == 8) {
    e[0] = S->rec[0];
    e[1] = (S->rec[1] & (RBGTOPO_STEP_EXCLUSIVE | RBGTOPO_STEP_GANG)) | S->rec[10] << STEP_LEVEL_SHIFT;
    e[2] = P;
    e[3] = S->rec[8] - row_base + S->cum[RBGTOPO_MAX_GROUP_ROLES];
  }
}

// One warp per step (+ warps for the tail words and the blob header).  Writes every word of
// its step's header and section, so the plan buffer needs no clearing.
__global__ void __launch_bounds__(32 * PLAN_WARPS) k_expand_plan(const int* __restrict__ grp, const int* __restrict__ src,
                                                                 int* __restrict__ out, int ns, int plan_words,
                                                                 int aux_off, int tail_off, int tail_words, int racc,
                                                                 int rowacc) {
  __shared__ PlanScratch scratch[PLAN_WARPS];
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * PLAN_WARPS + (threadIdx.x >> 5);
  if (s >= ns) {
    const int i = (s - ns) * 32 + lane;
    if (i < tail_words) out[plan_words + i] = src[tail_off + i];
    if (i == tail_words) {
      out[0] = RBGTOPO_BLOB_MAGIC;
      out[1] = RBGTOPO_ABI_VERSION;
      out[2] = ns;
      out[3] = plan_words;
      out[4] = racc;
      out[5] = rowacc;
      out[6] = 0;
      out[7] = 0;
    }
    return;
  }
  PlanScratch* S = &scratch[threadIdx.x >> 5];
  const int av = lane < PLAN_AUX_WORDS ? src[aux_off + s * PLAN_AUX_WORDS + lane] : 0;
  const int g = __shfl_sync(0xFFFFFFFFu, av, 0), w = __shfl_sync(0xFFFFFFFFu, av, 1);
  const int sec = __shfl_sync(0xFFFFFFFFu, av, 2), sec_end = __shfl_sync(0xFFFFFFFFu, av, 3);
  const int rep = __shfl_sync(0xFFFFFFFFu, av, 4), row = __shfl_sync(0xFFFFFFFFu, av, 5);
  const int next = __shfl_sync(0xFFFFFFFFu, av, 6), i0 = __shfl_sync(0xFFFFFFFFu, av, 7);
  if (lane < RBGTOPO_GROUP_WORDS) S->rec[lane] = grp[RBGTOPO_HDR_WORDS + (long long)g * RBGTOPO_GROUP_WORDS + lane];
  __syncwarp();
  const int gid = S->rec[0], gflags = S->rec[1], gfixed = S->rec[2], q = S->rec[3], na = S->rec[6];
  const int* g_roles = grp + S->rec[4];
  const int* g_pair = grp + S->rec[5];
  const int* g_anc = grp + S->rec[7];
  for (int i = lane; i < 4 * q; i += 32) S->roles[i] = g_roles[i];
  for (int i = lane; i < q * q; i += 32) S->pair[i] = g_pair[i];
  __syncwarp();
  if (lane == 0) plan_wave_at(S, q, w);
  __syncwarp();
  const int P = S->n;
  const int pair_off = sec + 4 * P, anchor_off = pair_off + P * q;
  const int place_off = anchor_off + 3 * na, cons_off = place_off + 3 * i0;
  if (lane < P) {  // role record `lane`
    const int ri = S->role[lane];
    int need = 0;
    for (int j = 0; j < q; ++j)
      if (S->pair[ri * q + j] > 0) need += S->roles[4 * j + 1] - S->placed[j];
    *reinterpret_cast<int4*>(out + sec + 4 * lane) =
        make_int4(S->count[lane], S->roles[4 * ri + 2], min(need, RBGTOPO_NEED_CAP), (S->roles[4 * ri + 3] & 0xFF) | (ri << 8));
  }
  for (int i = lane; i < P * q; i += 32) out[pair_off + i] = S->pair[S->role[i / q] * q + i % q];
  for (int i = lane; i < 3 * na; i += 32) out[anchor_off + i] = g_anc[i];
  // one record per replica of the earlier waves (group order = role-ascending), filled on the
  // device by the wave that places it; count 1 is what the host's exactness bound assumed
  for (int r = lane; r < i0; r += 32) {
    int j = 0;
    while (S->cum[j + 1] <= r) ++j;
    out[place_off + 3 * r] = 0;
    out[place_off + 3 * r + 1] = j;
    out[place_off + 3 * r + 2] = 1;
  }
  for (int i = cons_off + lane; i < sec_end; i += 32) out[i] = 0;  // consumed records + pad
  if (lane < 4) {
    int n = 0;
    for (int k = 0; k < P; ++k) n += S->count[k];
    int4 v;
    if (lane == 0)
      v = make_int4(gid, (gflags & (RBGTOPO_STEP_EXCLUSIVE | RBGTOPO_STEP_GANG)) | S->rec[10] << STEP_LEVEL_SHIFT,
                    (gflags & RBGTOPO_STEP_EXCLUSIVE) ? gfixed : -1, P);
    else if (lane == 1) v = make_int4(sec, q, pair_off, na + i0);
    else if (lane == 2) v = make_int4(anchor_off, i0, cons_off, n);
    else v = make_int4(rep, row, next, i0);
    reinterpret_cast<int4*>(out + RBGTOPO_HDR_WORDS + (long long)s * RBGTOPO_STEP_WORDS)[lane] = v;
  }
}

}  // namespace rbgtopo
