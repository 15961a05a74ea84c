// rbgtopo.cu — host runtime behind the C ABI of include/rbgtopo.h: context,
// snapshot upload + validation + refresh pipeline, batch ("blob") validation,
// multi-wave plan geometry (the plan itself is expanded on the device: plan.cuh),
// slot pool, launches, timing.  Kernels: kernels.cuh (snapshot), score.cuh (dense
// matrix), plan_group.cuh / select_fast.cuh / select.cuh (selection + greedy).
// No CPU fallback exists: every entry point needs a CUDA device (sm_90).
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <map>
#include <mutex>
#include <optional>
#include <shared_mutex>
#include <string>
#include <vector>

#include "kernels.cuh"
#include "plan.cuh"
#include "score.cuh"
#include "emit_rows.cuh"
#include "select.cuh"
#include "select_fast.cuh"
#include "plan_group.cuh"
#include "p2p.cuh"
#include "alternates.cuh"
#include "lw_assign.cuh"

using namespace rbgtopo;

namespace {

// Error text.  The failing call stores it for the calling THREAD (g_err) and, thread-agnostic, as
// the library's most recent error (g_last_err): a cgo caller whose goroutine migrated to another
// OS thread between the failing call and rbgtopo_last_error still gets the text.  The Go shim
// fetches it inside the same C helper as the call (go/pkg/scheduler/b200topo/cgo_bridge.go), where
// no migration can happen; the fallback is for callers that do not.
thread_local std::string g_err;
thread_local int g_err_code = 0;
std::mutex g_last_err_mu;
std::string g_last_err;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  g_err_code = code;
  {
    std::lock_guard<std::mutex> g(g_last_err_mu);
    g_last_err = buf;
  }
  return code;
}

// NVTX range of a host-side phase (SURVEY.md §5 tracing row): visible in nsys / ncu timelines, free otherwise.
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

#define CK(expr)                                                                      \
  do {                                                                                \
    cudaError_t e__ = (expr);                                                         \
    if (e__ != cudaSuccess)                                                           \
      return fail(RBGTOPO_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
                  __FILE__, __LINE__);                                                \
  } while (0)

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;  // elements
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = n + n / 4 + 64;
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
};
template <typename T>
struct PinBuf {
  T* p = nullptr;
  size_t cap = 0;
  bool pageable = false;  // host-only inspection (rbgtopo_plan_describe): plain malloc, no CUDA call
  ~PinBuf() { release(); }
  void release() {
    if (!p) return;
    if (pageable) free(p); else cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    release();
    size_t want = n + n / 4 + 64;
    if (pageable) {
      p = static_cast<T*>(malloc(want * sizeof(T)));
      if (!p) return cudaErrorMemoryAllocation;
      cap = want;
      return cudaSuccess;
    }
    cudaError_t e = cudaMallocHost(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
};

struct Topology {
  bool valid = false;
  int n = 0, n_domains = 0;
  long long e = 0;
  long long wsum_max = 0;  // max over rows of sum_j w_j (exactness bound)
  uint64_t generation = 0;
  DevBuf<int> row_ptr, col, w, free_, domain, owner, node_owner, dom_ptr, dom_nodes;
  DevBuf<unsigned char> fmin;
  DevBuf<float> base;
  DevBuf<unsigned long long> okeys, order;  // background order of the slab (score.cuh / select.cuh)
  DevBuf<unsigned long long> okeys_all, order_all;  // world > 1: the order over all nodes (plan_group.cuh)
  DevBuf<unsigned char> sort_tmp;
  // incremental refresh (rbgtopo_update_nodes_delta, world == 1): position of every node in `order`, the scratch
  // of one repair, and whether pos matches order (set by every full refresh)
  DevBuf<int> pos, flag, aff, old_pos, d_changed;
  DevBuf<unsigned long long> new_keys, order_alt;
  bool pos_valid = false;
  int key_nb = 0, key_bits = 64;           // compact sort key of the background order (prepare_refresh)
  cudaGraphExec_t refresh_exec = nullptr;  // captured refresh chain of this topology (run_base): k_prep + k_base ...
  cudaGraphExec_t order_exec = nullptr;    // ... and the order sorts, so that base_ready can be recorded between them
  bool refresh_ready = false;              // buffers sized / graph built for the current topology
  std::vector<int> h_degp1;  // deg(n) + 1, for the patch-list capacity of a step
  int max_degp1 = 1;
  DevBuf<int2> tiles;
  int n_tiles = 0;
  std::vector<int> h_domain;  // kept for update_nodes validation
  float base_ms = 0.f;
  // occupancy mode (rbgtopo_set_exclusive_levels, DESIGN.md §3.9): levels 0..n_levels, level L's domain / owner
  // vector at [L * level_stride(n), + n) of lvl_domain / lvl_owner (row 0 of lvl_domain = domain); the selection
  // kernels then read lvl_owner's row 0 instead of node_owner (topo_dev)
  bool occ = false;
  int n_levels = 0;
  int lvl_total_d = 0;                      // sum of the levels' domain counts
  std::vector<int> lvl_nd;                  // [n_levels + 1] domain count of every level (fixed_domain checks)
  std::vector<int> h_lvl_domain;            // [n_levels][n] levels 1..n_levels on the host (co-located alternates)
  DevBuf<int> lvl_domain, lvl_owner, lvl_doff, lvl_tab, occ_rec;
  // node classes (rbgtopo_set_node_classes, DESIGN.md §3.19): class of every node as u8, zero-padded to 16 B past n
  // (k_score_emit_elig loads four nodes' classes as one word); n_classes = 0: none installed
  int n_classes = 0;
  DevBuf<unsigned char> cls;
};

struct BatchMeta {
  int n_steps = 0, total_r = 0, total_p = 0, max_p = 1, max_k = 1, max_q = 1;
  bool any_excl_unknown = false;
  bool any_level = false;    // a step at an exclusive level >= 1: the <true> selection kernels (a caller's blob: stage_into
                             // moves the level from word +14 into the step flags)
  long long words = 0;
  long long h2d_words = 0;   // what staging actually uploaded
  long long scores = 0;      // sum R * N
  long long algo_bytes = 0;  // DESIGN.md §5
  long long patch_cap = 0;   // sum of the per-step patch-list capacities
  int max_cap = 0;           // largest per-step capacity (sizes the shared-memory hash table)
  std::vector<int> poff;     // [n_steps + 1] patch-list offsets
  std::vector<int> rowmap;   // step batches: [total_r] dense role row of every replica (rbgtopo_read_scores)
};

// Ranked alternates on node-axis shards (rbgtopo_shard_place_groups*_ranked, DESIGN.md §3.17): what a handle carries
// from the local call to the merge.  The jobs are those run_alternates made, in the order it made them (the same on
// every rank: they follow from replicated placements); the merge reads nothing else, no snapshot state.
struct AltExchange {
  int n_alt = 0;
  int64_t total_r = 0;                   // replicas of the call's assign vector
  std::vector<int> bounds;               // [world + 1] slab bounds of every rank
  std::vector<int2> job;                 // per job: first compact replica, replicas
  std::vector<int> own, idx;             // per compact replica: node, index in assign
  std::vector<unsigned long long> keys;  // per job ALT_LIST keys of this rank's slab (collected by run_alternates)
  std::vector<float> rscore;             // per compact replica: S_r[own] where own lies in this slab, else -inf
  int64_t bytes = 0;                     // the exchange buffer: keys, then rscore, padded to 8 bytes
  DevBuf<unsigned long long> buf;
  void reset(int n) {
    n_alt = n;
    total_r = bytes = 0;
    bounds.clear(); job.clear(); own.clear(); idx.clear(); keys.clear(); rscore.clear();
  }
};

struct Batch {
  bool in_use = false;    // reserved by a call or a stage handle
  bool staged = false;    // holds a staged blob (handle alive)
  bool xchg = false;      // holds an exchange of rbgtopo_shard_place_groups*_ranked (handle alive until the merge)
  bool ran = false;
  bool early_emit = false;    // plan_stage already enqueued the dense-matrix kernel of the next pass (+ its two events)
  bool d2h_enqueued = false;  // enqueue_d2h ran for the last pass; fetch_batch only has to wait
  uint64_t epoch = 0;         // topology epoch the batch was validated / sized against (set_topology bumps it)
  uint64_t lvl_epoch = 0;     // partition install the batch's levels >= 1 (b->m.any_level) were validated against
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;  // selection of multi-wave plans, concurrent with the dense-matrix kernel
  cudaEvent_t ev[8] = {};          // 0/1 staging, 2/3 fork/join of stream2, 4/5 D2H, 6 snapshot fence
  std::vector<cudaEvent_t> it_ev;  // triples (before score, after score, after select) per pass
  int passes = 0, pend_launches = 0, untimed_or_timed_passes = 0;  // since the last harvest
  bool shard_timed = false;
  BatchMeta m;
  DevBuf<int> blob;
  DevBuf<float> matrix;
  DevBuf<unsigned long long> lists, merged, excl;
  DevBuf<int> cand;  // patched-node scratch of the selection kernels
  DevBuf<int2> rtab;           // row table of a plan (emit_rows.cuh)
  // dense role rows (step_drow, kernels.cuh): first row per plan step (direct path: per group), and per replica of a
  // plan the row rbgtopo_read_scores returns (step batches: BatchMeta::rowmap)
  DevBuf<int> drow, rowmap;
  DevBuf<int> rrcnt;                 // direct path: role rows per group (k_group_rrcount), scanned into drow
  DevBuf<unsigned char> scan_tmp;    // ... by the device scan's temporary storage
  bool any_excl = false;       // a group of the plan is exclusive: k_emit_rows<true>
  int perm_n = 0;              // > 0: the plan's tail holds the CTA -> first-step order of k_plan_group (plan_geometry)
  std::vector<char> pass_mid;  // per pending pass: was the event between the two kernels recorded?
  // host-buffer entry point: the GROUPS blob was copied to the pinned staging and its upload enqueued BEFORE validation
  // (bytes only; no kernel reads them unless the validation passes), valid while both buffers stay where they were
  const int32_t* prestaged_h = nullptr;
  const int* prestaged_d = nullptr;
  size_t prestaged_hcap = 0, prestaged_dcap = 0;  // a re-allocation changes the capacity even when the address comes back
  bool tev = false;            // timing events (ev[0], ev[1], ev[4], ev[5], the early emit's) recorded since the staging
  DevBuf<int> corr, corr_cnt;  // correction records of a plan: k_plan_group(record) -> k_plan_correct
  // device-resident multi-wave plan (rbgtopo_stage_groups / place_groups): steps are
  // wave-major; wave w = steps [wave_begin[w], wave_begin[w + 1])
  std::vector<int> wave_begin, wave_maxp;
  std::vector<int> step_group;   // plan step -> group
  std::vector<int> step_row;     // [n_steps + 1] role-row prefix
  // device-expanded plans: the staging buffer (GROUPS blob | per-step geometry | poff)
  DevBuf<int> gsrc;
  long long aux_off = -1;        // word offset of the per-step geometry in h_in; -1: host-built plan
  int g_lo = 0;                  // first group of the GROUPS blob this plan covers
  std::vector<int> grp_flags, grp_assign_off, grp_pending, grp_fixed;
  DevBuf<int> out;  // assign[total_r] | status[n] | domain[n] | dstar[n]
  PinBuf<int> h_in, h_out;
  // committed batches (place_groups_committed): head[nodes] | dhead[domains] | phead[domains] | reader[nodes] |
  // dreader[domains] | previous round's assign[total_r] and domain[n] | lowest group whose changed claims matter; the
  // claim lists.  Domains are level 0's, or (a group at a level >= 1) those of every installed level; phead and the
  // pod claims exist only then.
  DevBuf<int> cm_int;
  DevBuf<int4> cm_claim, cm_pclaim;
  DevBuf<int2> cm_dclaim;
  // ranked placement (place_groups_ranked): jobs | placements | own nodes, then the per-replica lists
  DevBuf<int> alt;
  PinBuf<int> h_alt;
  // leader-worker placement (place_groups_lw): the wave's (S, C) side table, the per-CTA level-C domain scratch
  DevBuf<int> lw, lw_cap;
  PinBuf<int> h_lw;
  // ... committed at levels (§3.16): the changed heads, dclaim and pclaim of the round's claim lists (heads in cm_int)
  DevBuf<int> lwc;
  PinBuf<int> h_lwc;
  DevBuf<unsigned long long> lw_best;
  // ranked host-driven wave loops (run_waves): the dense rows of every (wave, role), kept
  // across calls like the matrix
  DevBuf<float> kept;
  AltExchange x;  // xchg: the exchange; the merge's tables and outputs are in alt / h_alt
  ~Batch() {
    if (stream) cudaStreamDestroy(stream);
    if (stream2) cudaStreamDestroy(stream2);
    for (auto& e : ev) if (e) cudaEventDestroy(e);
    for (auto& e : it_ev) cudaEventDestroy(e);
  }
};

}  // namespace

struct rbgtopo_ctx {
  rbgtopo_config cfg{};
  int sm_count = 132;
  int slab_lo = 0, slab_hi = 0, slab_stride = 0, lc = 1, chunk = 2048;
  std::shared_mutex topo_mu;  // update = exclusive, score calls = shared
  uint64_t topo_epoch = 0;    // bumped by set_topology: handles staged against an older topology are stale
  uint64_t lvl_epoch = 0;     // bumped by every partition install: handles with steps at levels >= 1 staged before it
                              // are stale (their level ids and fixed domains belong to the old partitions)
  std::mutex pool_mu;
  Topology topo;
  std::vector<std::unique_ptr<Batch>> batches;
  cudaStream_t ext_stream = nullptr;
  bool use_ext_stream = false;
  // Per-kernel CUDA events inside a pass (rbgtopo_set_kernel_timing).  Off (default): a pass records only its
  // start / end, and k_plan_group is launched as a PROGRAMMATIC DEPENDENT of the dense-matrix kernel — its CTAs
  // become resident while the last dense-matrix CTAs drain and wait (griddepcontrol.wait) before they touch the
  // matrix.  On: an event sits between the two kernels, which serialises them (that is what it measures).
  std::atomic<bool> kernel_timing{false};
  // snapshot refresh pipeline: update_nodes enqueues on topo_stream and returns; every batch
  // stream waits on topo_ready before it touches the snapshot
  cudaStream_t topo_stream = nullptr;
  // base_ready: free / node_owner / fmin / base of the latest refresh are written (what the dense-matrix kernel
  // reads); topo_ready: the background order too (what selection reads).  The sort overlaps the emit.
  cudaEvent_t base_ready = nullptr;
  cudaEvent_t topo_ready = nullptr, ev_base_a = nullptr, ev_base_b = nullptr, fence_ev = nullptr;
  bool base_timing_pending = false;
  // update_nodes staging, double buffered: the copy of update k leaves h_free[k & 1]; the host only
  // waits for update k - 2's H2D (long finished) before overwriting it, not for the refresh chain
  PinBuf<int> h_free[2], h_owner[2], h_occ[2];
  PinBuf<unsigned char> h_cls[2];
  cudaEvent_t stage_ev[2] = {nullptr, nullptr};
  unsigned stage_idx = 0;
  std::mutex stat_mu;
  // in-library all-gather over peer memory (p2p.cuh); SPMD: every rank makes the same calls in the same order
  DevBuf<unsigned long long> xbuf;
  DevBuf<int> p2p_ctr;  // [0] = CTA counter of k_p2p_push, [1] = timeout flag of k_p2p_wait
  P2PDev p2p{};
  int p2p_rows_cap = 0;
  bool p2p_ready = false;
  unsigned long long p2p_seq = 0;
  long long p2p_bytes_last = 0;  // bytes this rank stored into PEER buffers during the last pass
  std::vector<void*> p2p_opened;
  // recorded on its stream by every rbgtopo_run_staged_p2p; the next one waits for it.  Batches run on streams of their
  // own, and two exchange passes in flight at once would share the parity slots, the flags and the CTA counter
  cudaEvent_t p2p_done = nullptr;
  rbgtopo_timing last{};
  std::vector<float> last_score_ms, last_select_ms;  // per pass, harvested by the last fetch (rbgtopo_last_pass_times)
  long long calls = 0, scores_total = 0, launches = 0;
  long long delta_repairs = 0;  // incremental repairs of update_nodes_delta since the last set_topology
  // occupancy of k_plan_group: per instantiation (DIRECT) the launch shape last asked about and its CTAs per SM;
  // the last launch's grid and CTAs per SM (rbgtopo_plan_occupancy)
  struct PlanOcc { int nth = 0; size_t smem = 0; int per_sm = 0; } plan_occ[2];
  int plan_ctas = 0, plan_ctas_per_sm = 0;
};

namespace {

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// Exclusive level of a group (word +10) or caller-built step (word +14), DESIGN.md §3.9.  n_levels = the installed
// levels (0 outside occupancy mode), -1 when unknown (the describe calls accept any level >= 0).  Level 0 is placed
// everywhere; an installed level >= 1 only where `place` (a ctx created with RBGTOPO_CFG_LEVEL_PLACEMENT, and not
// for committed batches): elsewhere it is a documented limit, which hosts read as "no hint".
inline int level_code(int level, int n_levels, bool place) {
  if (level == 0) return RBGTOPO_OK;
  if (level < 0 || (n_levels >= 0 && level > n_levels)) return RBGTOPO_EINVAL;
  return (n_levels < 0 || place) ? RBGTOPO_OK : RBGTOPO_ELIMIT;
}
inline int installed_levels(const rbgtopo_ctx* c) { return c->topo.occ ? c->topo.n_levels : 0; }
inline bool places_levels(const rbgtopo_ctx* c) { return (c->cfg.flags & RBGTOPO_CFG_LEVEL_PLACEMENT) != 0; }
// committed batches at levels >= 1 (create accepts the flag only together with RBGTOPO_CFG_LEVEL_PLACEMENT)
inline bool commits_levels(const rbgtopo_ctx* c) { return (c->cfg.flags & RBGTOPO_CFG_COMMIT_LEVELS) != 0; }
// rbgtopo_place_groups_lw[_committed] at world > 1 (DESIGN.md §3.18)
inline bool lw_shards(const rbgtopo_ctx* c) { return (c->cfg.flags & RBGTOPO_CFG_LW_SHARDS) != 0; }
// Domain count of installed level L (level_code accepted it): the range of a fixed domain at that level.
inline int level_domains(const Topology& T, int L) { return L == 0 ? T.n_domains : T.lvl_nd[L]; }
constexpr size_t kFastSmemMax = 200 * 1024;
constexpr int kMaxExactTerm = 1 << 24;  // pair weights and anchor counts above this can never satisfy spec §3.4
// Switches, read once when the library loads (INTEGRATION.md §5).
const bool kPerWavePlan = getenv("RBGTOPO_PER_WAVE_PLAN") != nullptr;  // one launch per wave instead of k_plan_group
// Multi-wave plans, default: the dense-matrix kernel, then k_plan_group applying the corrections itself.
// RBGTOPO_CONCURRENT_PLAN=1: k_plan_group (record mode: it never touches the matrix) on a second stream
// beside the dense-matrix kernel, corrections applied afterwards by k_plan_correct.  Opt-in: the write
// stream inflates the latency of the selection's dependent loads and the two kernels fight for registers.
const bool kSerialPlan = getenv("RBGTOPO_CONCURRENT_PLAN") == nullptr;
const bool kNoPdl = getenv("RBGTOPO_NO_PDL") != nullptr;                // plain stream order between the two plan kernels
const bool kKernelTimingEnv = getenv("RBGTOPO_KERNEL_TIMING") != nullptr;  // initial value of rbgtopo_set_kernel_timing
const bool kProfileHost = getenv("RBGTOPO_PROFILE_HOST") != nullptr;
const bool kSelectHighPriority = getenv("RBGTOPO_SELECT_LOW_PRIO") == nullptr;
const bool kSelectFirst = getenv("RBGTOPO_SELECT_FIRST") != nullptr;  // launch order of the two concurrent kernels
// Residency cap of k_plan_group beside the dense-matrix kernel: its CTAs REQUEST this much dynamic shared
// memory (they use ~26 KB on cfg3), so at most floor(227 KB / request) of them share an SM and the rest of the
// register file stays with the emit kernel (DESIGN.md §4.5).  0 = no inflation.
const int kSelectSmemKB = getenv("RBGTOPO_SELECT_SMEM_KB") ? std::max(0, atoi(getenv("RBGTOPO_SELECT_SMEM_KB"))) : 0;
// Dense rows of a plan: k_emit_rows (emit_rows.cuh, row-major walk of the plan's row table); RBGTOPO_EMIT_ROWS = rows
// per segment.
const int kEmitRowsBlock = getenv("RBGTOPO_EMIT_ROWS") ? std::min(EMIT_ROWS_MAX, std::max(1, atoi(getenv("RBGTOPO_EMIT_ROWS")))) : 6;
const int kEmitBlockSteps =
    getenv("RBGTOPO_EMIT_BLOCK") ? std::min(EMIT_MAX_BLOCK, std::max(1, atoi(getenv("RBGTOPO_EMIT_BLOCK")))) : 4;
// place_groups can pipeline a fleet as two halves (host geometry of half 2 under the device work of
// half 1).  Opt-in: at 1 024 groups it does not pay — the step is device-bound and the latency-bound
// k_plan_group takes as long for half the groups as for all of them.
const int kSplitMinGroups =
    getenv("RBGTOPO_SPLIT_MIN_GROUPS") ? std::max(2, atoi(getenv("RBGTOPO_SPLIT_MIN_GROUPS"))) : (1 << 30);
const bool kCompactSortKey = getenv("RBGTOPO_WIDE_SORT_KEY") == nullptr;
const bool kRefreshGraph = getenv("RBGTOPO_NO_REFRESH_GRAPH") == nullptr;
// RBGTOPO_SMALL_SORT=1: single-CTA bitonic sort of the order for slabs <= 16 384 nodes instead of the library
// radix sort.  Opt-in: 105 barrier rounds at 10 000 nodes make it slower than the radix sort.
const bool kSmallSort = getenv("RBGTOPO_SMALL_SORT") != nullptr;
const bool kVerifyPlan = getenv("RBGTOPO_VERIFY_PLAN") != nullptr;  // self-check: device-expanded plan == host-built plan
const int kHostThreads = getenv("RBGTOPO_HOST_THREADS") ? std::max(1, atoi(getenv("RBGTOPO_HOST_THREADS"))) : 4;
// With the per-shape caches a group costs little host time: below a few thousand groups an OpenMP region costs more
// than it saves (the 1 024-group bench fleet is faster on one thread than on 2 or 4).
const int kHostParallelMinGroups = getenv("RBGTOPO_HOST_PARALLEL_MIN") ? std::max(1, atoi(getenv("RBGTOPO_HOST_PARALLEL_MIN"))) : 4096;

// Events that only measure (staging, early emit, D2H, refresh) are recorded with kernel timing on or under
// RBGTOPO_PROFILE_HOST: each costs stream time, and the host-buffer entry points are latency-bound.
inline bool timing_events(const rbgtopo_ctx* c) { return kProfileHost || c->kernel_timing.load(std::memory_order_relaxed); }

// First node of rank g's slab (g = W: n): g * n / W rounded down to 128, so a slab may be empty.
int slab_bound(int n, int W, int g) {
  if (g <= 0) return 0;
  if (g >= W) return n;
  long long b = (long long)g * n / W;
  return (int)(b / 128 * 128);
}

void compute_slab(rbgtopo_ctx* c, int n) {
  const int W = c->cfg.world, r = c->cfg.rank;
  auto bound = [&](int g) { return slab_bound(n, W, g); };
  c->slab_lo = bound(r);
  c->slab_hi = bound(r + 1);
  int max_len = 0;
  for (int g = 0; g < W; ++g) max_len = std::max(max_len, bound(g + 1) - bound(g));
  int tcfg = c->cfg.chunk_nodes > 0 ? c->cfg.chunk_nodes : 2048;
  tcfg = std::min(2048, std::max(128, round_up(tcfg, 128)));
  c->lc = std::max(1, (max_len + tcfg - 1) / tcfg);
  c->chunk = std::min(2048, std::max(128, round_up((max_len + c->lc - 1) / c->lc, 128)));
  c->slab_stride = round_up(std::max(1, c->lc * c->chunk), 32);
}

TopoDev topo_dev(const rbgtopo_ctx* c) {
  TopoDev t;
  const Topology& T = c->topo;
  t.n = T.n;
  t.slab_lo = c->slab_lo;
  t.slab_hi = c->slab_hi;
  t.slab_stride = c->slab_stride;
  t.row_ptr = T.row_ptr.p;
  t.col = T.col.p;
  t.w = T.w.p;
  t.free_ = T.free_.p;
  t.domain = T.domain.p;
  t.node_owner = T.occ ? T.lvl_owner.p : T.node_owner.p;  // occupancy mode: owner_0 derived from the pods
  t.fmin = T.fmin.p;
  t.base = T.base.p;
  t.order = T.order.p;
  t.order_all = c->cfg.world > 1 ? T.order_all.p : T.order.p;
  t.lvl_domain = T.lvl_domain.p;
  t.lvl_owner = T.lvl_owner.p;
  return t;
}

// Sort keys of the background order.  base is a non-negative integer-valued float (sums of
// int weights x fmin), so  (int(base) << nb) | (2^nb - 1 - node)  orders exactly like
// make_key(base, node) and needs only nb + bits(max base) <= ~32 of the 64 key bits: the radix
// sort runs 4 passes instead of 8.  nb == 0 selects the plain 64-bit key.
__global__ void k_order_keys(TopoDev t, int lo, int hi, int nb, unsigned long long* keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hi - lo) return;
  const int node = lo + i;
  if (nb == 0)
    keys[i] = make_key(t.base[node], node);
  else
    keys[i] = ((unsigned long long)(long long)t.base[node] << nb) | (unsigned long long)(((1u << nb) - 1u) - (uint32_t)node);
}
// compact sorted keys -> the key(base, node) form the selection kernels read
__global__ void k_order_expand(unsigned long long* keys, int n, int nb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  const uint32_t mask = (1u << nb) - 1u;
  keys[i] = make_key((float)(long long)(k >> nb), (int)(mask - (uint32_t)(k & mask)));
}

// prep + base kernels on `s`; records base_ms.
void harvest_base_ms(rbgtopo_ctx* c) {
  if (!c->base_timing_pending) return;
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, c->ev_base_a, c->ev_base_b) == cudaSuccess) {
    c->topo.base_ms = ms;
    c->base_timing_pending = false;
  } else {
    (void)cudaGetLastError();  // not finished yet
  }
}

// The snapshot refresh chain (k_prep, k_base, order keys + radix sort[s]): 12-21 launches.
// prepare_refresh sizes every buffer (allocations are not allowed under stream capture);
// enqueue_refresh only launches.
int prepare_refresh(rbgtopo_ctx* c) {
  Topology& T = c->topo;
  {  // compact sort key: node bits + bits of the largest possible base = (wsum_max + self) * F
    auto bits = [](unsigned long long v) { int b = 0; while (v) { ++b; v >>= 1; } return std::max(1, b); };
    const int nb = bits((unsigned long long)std::max(1, T.n - 1));
    // From 2^24 on, base is an fp32 sum that is no longer exact (such a snapshot only admits need = 0 steps): a
    // rounded sum can reach the power of two above the bound (bound 2^28 - 8 sums to 2^28), so reserve one more bit.
    const unsigned long long bound = (unsigned long long)(T.wsum_max + RBGTOPO_SELF_W) * RBGTOPO_F_CAP;
    const int bb = bits(bound) + (bound >= (1ull << 24) ? 1 : 0);
    if (kCompactSortKey && nb + bb <= 62 && nb <= 31) {
      T.key_nb = nb;
      T.key_bits = nb + bb;
    } else {
      T.key_nb = 0;
      T.key_bits = 64;
    }
  }
  const int fmin_bytes = round_up(T.n, 16);
  const int staged = T.n <= FMIN_SMEM_MAX ? 1 : 0;
  const size_t smem = (size_t)2 * (BASE_TILE_NNZ + 8) * 4 + (staged ? fmin_bytes : 0);
  CK(cudaFuncSetAttribute(k_base, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int slab_len = c->slab_hi - c->slab_lo;
  size_t tmp_bytes = 0, need = 0;
  if (slab_len > 0) {
    CK(T.okeys.reserve(slab_len));
    CK(T.order.reserve(slab_len));
    CK(cub::DeviceRadixSort::SortKeysDescending(nullptr, tmp_bytes, T.okeys.p, T.order.p, slab_len, 0, 64, nullptr));
    need = std::max(need, tmp_bytes);
  }
  if (c->cfg.world > 1 && T.n > 0) {
    CK(T.okeys_all.reserve(T.n));
    CK(T.order_all.reserve(T.n));
    CK(cub::DeviceRadixSort::SortKeysDescending(nullptr, tmp_bytes, T.okeys_all.p, T.order_all.p, T.n, 0, 64, nullptr));
    need = std::max(need, tmp_bytes);
  }
  CK(T.sort_tmp.reserve(need + 256));
  if (c->cfg.world == 1) {
    CK(T.pos.reserve((size_t)T.n));
    CK(T.flag.reserve((size_t)T.n));
    CK(cudaMemset(T.flag.p, 0, T.flag.cap * 4));
    CK(T.aff.reserve(1 + DELTA_MAX_AFFECTED));
    CK(T.old_pos.reserve(DELTA_MAX_AFFECTED));
    CK(T.new_keys.reserve(DELTA_MAX_AFFECTED));
    CK(T.order_alt.reserve((size_t)T.n));
  }
  return RBGTOPO_OK;
}

// part: 1 = k_prep + k_base, 2 = the background order(s), 3 = both (base_ready recorded in between)
int enqueue_refresh(rbgtopo_ctx* c, cudaStream_t s, int part) {
  Topology& T = c->topo;
  if (part & 1) {
  k_prep<<<(T.n + 255) / 256, 256, 0, s>>>(T.n, T.free_.p, T.domain.p, T.owner.p, T.fmin.p,
                                           T.node_owner.p);
  const int fmin_bytes = round_up(T.n, 16);
  const int staged = T.n <= FMIN_SMEM_MAX ? 1 : 0;
  const size_t smem = (size_t)2 * (BASE_TILE_NNZ + 8) * 4 + (staged ? fmin_bytes : 0);
  const TopoDev td = topo_dev(c);
  k_base<<<T.n_tiles, BASE_THREADS, smem, s>>>(td, T.tiles.p, staged, fmin_bytes, T.base.p);
  }
  // what the dense-matrix kernel reads is complete here; the order below is only read by selection
  if (part == 3) CK(cudaEventRecord(c->base_ready, s));
  if (!(part & 2)) {
    CK(cudaGetLastError());
    return RBGTOPO_OK;
  }
  const TopoDev td = topo_dev(c);
  // background order: slab nodes by key(base, node) descending, once per snapshot
  const int slab_len = c->slab_hi - c->slab_lo;
  auto p2_bytes = [](int n) { int p2 = 32; while (p2 < n) p2 <<= 1; return (size_t)p2 * 8; };
  if (slab_len > 0 && slab_len <= ORDER_SMALL_MAX && kSmallSort) {
    k_order_sort_small<<<1, ORDER_SMALL_THREADS, p2_bytes(slab_len), s>>>(T.base.p, c->slab_lo, c->slab_hi, T.order.p);
  } else if (slab_len > 0) {
    k_order_keys<<<(slab_len + 255) / 256, 256, 0, s>>>(td, c->slab_lo, c->slab_hi, T.key_nb, T.okeys.p);
    size_t tmp_bytes = T.sort_tmp.cap;
    CK(cub::DeviceRadixSort::SortKeysDescending(T.sort_tmp.p, tmp_bytes, T.okeys.p, T.order.p, slab_len, 0, T.key_bits, s));
    if (T.key_nb) k_order_expand<<<(slab_len + 255) / 256, 256, 0, s>>>(T.order.p, slab_len, T.key_nb);
  }
  if (c->cfg.world == 1 && slab_len > 0)  // node -> position, for the incremental repair of the order
    k_order_pos<<<(slab_len + 255) / 256, 256, 0, s>>>(T.order.p, slab_len, T.pos.p);
  if (c->cfg.world > 1 && T.n > 0 && T.n <= ORDER_SMALL_MAX && kSmallSort) {
    k_order_sort_small<<<1, ORDER_SMALL_THREADS, p2_bytes(T.n), s>>>(T.base.p, 0, T.n, T.order_all.p);
  } else if (c->cfg.world > 1 && T.n > 0) {  // replicated selection (plan_group.cuh) walks the order of ALL nodes
    k_order_keys<<<(T.n + 255) / 256, 256, 0, s>>>(td, 0, T.n, T.key_nb, T.okeys_all.p);
    size_t tmp_bytes = T.sort_tmp.cap;
    CK(cub::DeviceRadixSort::SortKeysDescending(T.sort_tmp.p, tmp_bytes, T.okeys_all.p, T.order_all.p, T.n, 0, T.key_bits, s));
    if (T.key_nb) k_order_expand<<<(T.n + 255) / 256, 256, 0, s>>>(T.order_all.p, T.n, T.key_nb);
  }
  CK(cudaGetLastError());
  return RBGTOPO_OK;
}

// Refresh of the per-snapshot vectors on `s`; records base_ms.  The chain is captured once per
// topology into a CUDA graph and replayed (one launch instead of 12+ from update_nodes);
// RBGTOPO_NO_REFRESH_GRAPH or a failed capture fall back to the plain launches.
int run_base(rbgtopo_ctx* c, cudaStream_t s, bool sync) {
  NvtxRange nv("rbgtopo:run_base");
  Topology& T = c->topo;
  if (!T.refresh_ready) {
    int rc = prepare_refresh(c);
    if (rc) return rc;
    for (cudaGraphExec_t* e : {&T.refresh_exec, &T.order_exec})
      if (*e) {
        cudaGraphExecDestroy(*e);
        *e = nullptr;
      }
    // two graphs — (k_prep, k_base) and the order sorts — so that base_ready can be recorded between them with a
    // plain cudaEventRecord: the dense-matrix kernel of the next batch then overlaps the sort
    auto capture = [&](int part, cudaGraphExec_t* out) {
      if (!kRefreshGraph || cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) != cudaSuccess) return;
      const int erc = enqueue_refresh(c, s, part);
      cudaGraph_t g = nullptr;
      const cudaError_t ce = cudaStreamEndCapture(s, &g);
      if (erc != RBGTOPO_OK || ce != cudaSuccess || !g || cudaGraphInstantiate(out, g, 0) != cudaSuccess) *out = nullptr;
      if (g) cudaGraphDestroy(g);
      (void)cudaGetLastError();
    };
    capture(1, &T.refresh_exec);
    if (T.refresh_exec) capture(2, &T.order_exec);
    if (!T.order_exec && T.refresh_exec) {
      cudaGraphExecDestroy(T.refresh_exec);
      T.refresh_exec = nullptr;
    }
    T.refresh_ready = true;
  }
  const bool tev = timing_events(c);
  if (tev) CK(cudaEventRecord(c->ev_base_a, s));
  if (T.refresh_exec) {
    CK(cudaGraphLaunch(T.refresh_exec, s));
    CK(cudaEventRecord(c->base_ready, s));
    CK(cudaGraphLaunch(T.order_exec, s));
  } else {
    int rc = enqueue_refresh(c, s, 3);
    if (rc) return rc;
  }
  if (tev) CK(cudaEventRecord(c->ev_base_b, s));
  CK(cudaEventRecord(c->topo_ready, s));
  T.pos_valid = c->cfg.world == 1;
  c->base_timing_pending = tev;
  CK(cudaGetLastError());
  if (sync) {
    CK(cudaStreamSynchronize(s));
    harvest_base_ms(c);
  }
  std::lock_guard<std::mutex> g(c->stat_mu);
  c->launches += 3;
  return RBGTOPO_OK;
}

// ---- blob validation (host, O(words)) ----------------------------------------
// `trusted`: the blob was built by build_plan from an already validated GROUPS blob — the
// per-record range checks are skipped, the derived metadata and the exactness bound are not.
// Work items of k_score_emit (score.cuh): idx = (block * lc + chunk) * bsteps + step_in_block;
// one CTA per (block, chunk) segment, scheduled by the hardware.
inline long long emit_items(int ns, int lc) {
  return (long long)((ns + kEmitBlockSteps - 1) / kEmitBlockSteps) * lc * kEmitBlockSteps;
}

int validate_blob(const rbgtopo_ctx* c, const int32_t* blob, int64_t words, BatchMeta* m, bool trusted = false) {
  const Topology& T = c->topo;
  if (!blob || words < RBGTOPO_HDR_WORDS) return fail(RBGTOPO_EINVAL, "blob too short");
  if (blob[0] != RBGTOPO_BLOB_MAGIC) return fail(RBGTOPO_EINVAL, "bad blob magic");
  if (blob[1] != RBGTOPO_ABI_VERSION) return fail(RBGTOPO_EINVAL, "blob version %d", blob[1]);
  const int ns = blob[2];
  if (ns < 0 || blob[3] != words || words > 0x7FFFFFFFLL)
    return fail(RBGTOPO_EINVAL, "blob header: n_steps=%d words=%d/%lld", ns, blob[3], (long long)words);
  if ((int64_t)RBGTOPO_HDR_WORDS + (int64_t)ns * RBGTOPO_STEP_WORDS > words)
    return fail(RBGTOPO_EINVAL, "step table exceeds blob");
  const long long row_w = T.wsum_max + RBGTOPO_SELF_W;
  long long racc = 0, pacc = 0;
  *m = BatchMeta{};
  m->poff.assign((size_t)ns + 1, 0);
  int* const pcs = m->poff.data() + 1;  // per-step patch capacity first, prefix-summed below
  auto in = [&](long long off, long long cnt) { return off >= 0 && cnt >= 0 && off + cnt <= words; };
#define STEP_FAIL(code, ...) return report ? fail(code, __VA_ARGS__) : (int)(code)
  // Everything about step s that does not depend on the steps before it.  report=false: code only
  // (called from worker threads); report=true: also formats the message.
  auto check_step = [&](int s, bool report) -> int {
    const int32_t* st = blob + RBGTOPO_HDR_WORDS + (int64_t)s * RBGTOPO_STEP_WORDS;
    const int P = st[3], Q = st[5], na = st[7], nc = st[9], R = st[11];
    if (st[0] < 0) STEP_FAIL(RBGTOPO_EINVAL, "step %d: gid < 0", s);
    if (P < 1 || P > RBGTOPO_MAX_STEP_ROLES) STEP_FAIL(RBGTOPO_ELIMIT, "step %d: %d roles", s, P);
    if (Q < 0 || Q > RBGTOPO_MAX_GROUP_ROLES) STEP_FAIL(RBGTOPO_ELIMIT, "step %d: q=%d", s, Q);
    if (R < 1 || R > RBGTOPO_MAX_STEP_REPLICAS) STEP_FAIL(RBGTOPO_ELIMIT, "step %d: %d replicas", s, R);
    if (!in(st[4], 4LL * P) || !in(st[6], (long long)P * Q) || !in(st[8], 3LL * na) || !in(st[10], 2LL * nc))
      STEP_FAIL(RBGTOPO_EINVAL, "step %d: section out of bounds", s);
    // exclusive level: word +14 of a caller's step, the step flags of a plan (whose word +14 is the wave link)
    const int lv = trusted ? step_level(st[1]) : st[14];
    if (!trusted) {
      if (const int lc = level_code(lv, installed_levels(c), places_levels(c)))
        STEP_FAIL(lc, "step %d: exclusive level %d (%d installed%s)", s, lv, installed_levels(c),
                  places_levels(c) ? "" : "; placement at level 0 only");
    }
    if (st[2] < -1 || st[2] >= level_domains(T, lv)) STEP_FAIL(RBGTOPO_EINVAL, "step %d: fixed_domain %d (level %d)", s, st[2], lv);
    const int32_t* roles = blob + st[4];
    const int32_t* pair = blob + st[6];
    const int32_t* anc = blob + st[8];
    const int32_t* con = blob + st[10];
    int rsum = 0;
    for (int p = 0; p < P; ++p) {
      if (roles[4 * p] < 1 || roles[4 * p + 1] < 0 || roles[4 * p + 1] > RBGTOPO_MAX_FREE ||
          roles[4 * p + 2] < 0 || roles[4 * p + 2] > RBGTOPO_NEED_CAP)
        STEP_FAIL(RBGTOPO_EINVAL, "step %d role %d: count/demand/need", s, p);
      rsum += roles[4 * p];
    }
    if (rsum != R) STEP_FAIL(RBGTOPO_EINVAL, "step %d: role counts sum to %d, R=%d", s, rsum, R);
    if (!trusted) {
      // flag words: only the documented bits (bit 4 of the step flags is the internal STEP_SKIP, bits
      // 8.. of the role flags carry the group role index in plans); wave links belong to plans only
      if (st[1] & ~(RBGTOPO_STEP_EXCLUSIVE | RBGTOPO_STEP_GANG)) STEP_FAIL(RBGTOPO_EINVAL, "step %d: unknown step flags 0x%x", s, st[1]);
      for (int p = 0; p < P; ++p)
        if (roles[4 * p + 3] & ~RBGTOPO_ROLE_EXCLUSIVE) STEP_FAIL(RBGTOPO_EINVAL, "step %d role %d: unknown role flags", s, p);
      if (st[15] != 0) STEP_FAIL(RBGTOPO_EINVAL, "step %d: reserved word 15 must be 0", s);
      for (int i = 0; i < P * Q; ++i)
        if (pair[i] < 0 || pair[i] > kMaxExactTerm) STEP_FAIL(RBGTOPO_EINVAL, "step %d: pair weight out of [0, 2^24]", s);
      for (int a = 0; a < na; ++a) {
        if (anc[3 * a] < 0 || anc[3 * a] >= T.n || anc[3 * a + 1] < 0 || anc[3 * a + 1] >= Q ||
            anc[3 * a + 2] < 0 || anc[3 * a + 2] > kMaxExactTerm)
          STEP_FAIL(RBGTOPO_EINVAL, "step %d anchor %d out of range", s, a);
      }
      for (int i = 0; i < nc; ++i)
        if (con[2 * i] < 0 || con[2 * i] >= T.n || con[2 * i + 1] < 0 || con[2 * i + 1] > RBGTOPO_MAX_FREE)
          STEP_FAIL(RBGTOPO_EINVAL, "step %d consumed %d out of range", s, i);
    }
    // exactness contract (spec §3.4), conservative: every anchor on one node.  Terms are bounded by
    // 2^24 each and the sum saturates as soon as the bound is violated: no signed overflow.
    const long long amax_limit = ((1LL << 24) + row_w - 1) / row_w;  // amax * row_w >= 2^24  <=>  amax >= limit
    for (int p = 0; p < P; ++p) {
      long long amax = (long long)roles[4 * p + 2] * RBGTOPO_F_CAP;
      for (int a = 0; a < na && amax < amax_limit; ++a) amax += (long long)pair[p * Q + anc[3 * a + 1]] * anc[3 * a + 2];
      if (amax >= amax_limit)
        STEP_FAIL(RBGTOPO_EINEXACT, "step %d role %d: max score bound >= 2^24 (anchor weight %lld x row weight %lld)", s, p, amax, row_w);
    }
    if (st[4] & 3) STEP_FAIL(RBGTOPO_EINVAL, "step %d: role_off must be a multiple of 4 words", s);
    if (trusted && (st[15] < 0 || st[15] > na || (st[14] != 0 && (st[14] <= s || st[14] >= ns))))
      STEP_FAIL(RBGTOPO_EINVAL, "step %d: bad wave links", s);
    // patched-node scratch: closed neighbourhoods of the anchors + consumed nodes.  Records of
    // earlier waves (the last st[15]) are filled on the device: any node.
    long long pc = nc;
    for (int a = 0; a < na; ++a) pc += a < na - st[15] ? T.h_degp1[anc[3 * a]] : T.max_degp1;
    if (pc > 0x7FFFFFF0LL) STEP_FAIL(RBGTOPO_ELIMIT, "step %d: patch list exceeds 2^31 entries", s);
    pcs[s] = (int)pc;
    return RBGTOPO_OK;
  };
#undef STEP_FAIL
  int first_bad = ns;
#pragma omp parallel for schedule(static) num_threads(kHostThreads) reduction(min : first_bad) if (ns >= 256 && kHostThreads > 1)
  for (int s = 0; s < ns; ++s)
    if (check_step(s, false) != RBGTOPO_OK) first_bad = std::min(first_bad, s);
  if (first_bad < ns) return check_step(first_bad, true);
  if (!trusted) m->rowmap.clear();
  for (int s = 0; s < ns; ++s) {  // the prefix-dependent part
    const int32_t* st = blob + RBGTOPO_HDR_WORDS + (int64_t)s * RBGTOPO_STEP_WORDS;
    if ((!trusted && st[12] != racc) || st[13] != pacc) return fail(RBGTOPO_EINVAL, "step %d: bad prefix offsets", s);
    if (trusted && (st[12] < 0 || st[12] + st[11] > blob[4])) return fail(RBGTOPO_EINVAL, "step %d: replica rows out of range", s);
    const long long pc = pcs[s];
    if (m->patch_cap + pc > 0x7FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "patch lists exceed 2^31 entries");
    m->patch_cap += pc;
    m->max_cap = (int)std::max<long long>(m->max_cap, std::min<long long>(pc, 1 << 30));
    pcs[s] = (int)m->patch_cap;
    if (!trusted)  // a step batch's steps are its groups: role p of step s is dense role row pacc + p
      for (int p = 0; p < st[3]; ++p) m->rowmap.insert(m->rowmap.end(), blob[st[4] + 4 * p], (int)pacc + p);
    racc += st[11];
    pacc += st[3];
    m->max_p = std::max(m->max_p, st[3]);
    m->max_k = std::max(m->max_k, st[11]);
    m->max_q = std::max(m->max_q, st[5]);
    if ((st[1] & RBGTOPO_STEP_EXCLUSIVE) && st[2] < 0) m->any_excl_unknown = true;
    if (trusted ? step_level(st[1]) != 0 : st[14] != 0) m->any_level = true;
  }
  if (blob[4] != racc || blob[5] != pacc) return fail(RBGTOPO_EINVAL, "blob totals mismatch");
  if (emit_items(ns, c->lc) > 0x7FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "steps x chunks exceed 2^31 work items");
  m->n_steps = ns;
  m->total_r = (int)racc;
  m->total_p = (int)pacc;
  m->words = words;
  const long long slab = c->slab_hi - c->slab_lo;
  m->scores = racc * slab;
  // DESIGN.md §5: bytes k_score_emit must move for this rank's slab: the dense
  // matrix write (one row per role row) + the batch blob read + the per-snapshot base/free
  // vectors once (they are L2-resident across the steps of a launch).  The sparse corrections
  // (a few dozen 4-byte reductions per step) are deliberately NOT counted.
  m->algo_bytes = 4LL * pacc * slab + 4LL * words + 8LL * slab;
  return RBGTOPO_OK;
}

int acquire_batch(rbgtopo_ctx* c, Batch** out) {
  std::lock_guard<std::mutex> g(c->pool_mu);
  for (auto& b : c->batches)
    if (!b->in_use) {
      b->in_use = true;
      *out = b.get();
      return RBGTOPO_OK;
    }
  auto nb = std::make_unique<Batch>();
  CK(cudaStreamCreateWithFlags(&nb->stream, cudaStreamNonBlocking));
  {
    int lo = 0, hi = 0;  // numerically lower = higher priority
    CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    CK(cudaStreamCreateWithPriority(&nb->stream2, cudaStreamNonBlocking, kSelectHighPriority ? hi : lo));
  }
  for (auto& e : nb->ev) CK(cudaEventCreate(&e));
  nb->in_use = true;
  *out = nb.get();
  c->batches.push_back(std::move(nb));
  return RBGTOPO_OK;
}
void release_batch(rbgtopo_ctx* c, Batch* b) {
  std::lock_guard<std::mutex> g(c->pool_mu);
  b->wave_begin.clear();
  b->d2h_enqueued = false;
  b->in_use = false;
  b->staged = false;
  b->xchg = false;
  b->ran = false;
}

cudaStream_t stream_of(rbgtopo_ctx* c, Batch* b) { return c->use_ext_stream ? c->ext_stream : b->stream; }

// device scratch + result buffers sized from b->m
int reserve_batch_buffers(rbgtopo_ctx* c, Batch* b) {
  const BatchMeta& m = b->m;
  CK(b->matrix.reserve((size_t)std::max(1, m.total_p) * c->slab_stride));
  CK(b->cand.reserve((size_t)m.patch_cap + 1));
  CK(b->lists.reserve((size_t)std::max(1, m.total_p) * KS));
  CK(b->merged.reserve((size_t)std::max(1, m.total_p) * KS));
  CK(b->excl.reserve((size_t)std::max(1, m.total_p) * KS));
  if (!b->wave_begin.empty()) {
    CK(b->corr.reserve((size_t)m.patch_cap * (size_t)(1 + m.max_p) + 1));
    CK(b->corr_cnt.reserve((size_t)m.n_steps + 1));
  }
  const size_t out_n = (size_t)m.total_r + 3 * (size_t)m.n_steps + 4;
  CK(b->out.reserve(out_n));
  CK(b->h_out.reserve(out_n));
  return RBGTOPO_OK;
}

// validate + size buffers + H2D.  Caller holds topo_mu shared.
// blob == b->h_in.p: the (trusted) plan was built in place in the pinned staging buffer.
int stage_into(rbgtopo_ctx* c, Batch* b, const int32_t* blob, int64_t words) {
  NvtxRange nv("rbgtopo:stage_into");
  if (!c->topo.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
  const bool in_place = blob == b->h_in.p;
  int rc = validate_blob(c, blob, words, &b->m, in_place);
  if (rc) return rc;
  const BatchMeta& m = b->m;
  cudaStream_t s = stream_of(c, b);
  const size_t in_words = (size_t)words + (size_t)m.n_steps + 1;  // blob | poff
  CK(b->blob.reserve(in_words));
  if (in_place) {
    if (b->h_in.cap < in_words) return fail(RBGTOPO_EINVAL, "internal: in-place plan without tail room");
  } else {
    CK(b->h_in.reserve(in_words));
  }
  rc = reserve_batch_buffers(c, b);
  if (rc) return rc;
  b->m.h2d_words = (long long)in_words;
  b->epoch = c->topo_epoch;
  b->lvl_epoch = c->lvl_epoch;
  b->tev = timing_events(c);
  b->perm_n = 0;
  if (b->tev) CK(cudaEventRecord(b->ev[0], s));  // staging touches the batch's own buffers only; run_batch waits for a pending refresh
  if (!in_place) memcpy(b->h_in.p, blob, (size_t)words * 4);
  if (m.any_level && !in_place)  // the kernels read a step's level from its flags: word +14 is the wave link of plans
    for (int s2 = 0; s2 < m.n_steps; ++s2) {
      int32_t* st = b->h_in.p + RBGTOPO_HDR_WORDS + (size_t)s2 * RBGTOPO_STEP_WORDS;
      st[1] |= st[14] << STEP_LEVEL_SHIFT;
      st[14] = 0;
    }
  memcpy(b->h_in.p + words, m.poff.data(), ((size_t)m.n_steps + 1) * 4);
  CK(cudaMemcpyAsync(b->blob.p, b->h_in.p, in_words * 4, cudaMemcpyHostToDevice, s));
  if (b->tev) CK(cudaEventRecord(b->ev[1], s));
  b->staged = true;
  b->ran = false;
  return RBGTOPO_OK;
}

BatchDev batch_dev(rbgtopo_ctx* c, Batch* b) {
  BatchDev d;
  d.blob = b->blob.p;
  d.n_steps = b->m.n_steps;
  d.lc = c->lc;
  d.chunk = c->chunk;
  d.parts = 1;
  {
    d.emit_matrix = b->wave_begin.empty() ? 1 : 3;  // plans: background only, corrections per wave

  }
  d.matrix = b->matrix.p;
  d.drow = b->wave_begin.empty() ? nullptr : b->drow.p;
  d.cand = b->cand.p;
  d.poff = b->blob.p + b->m.words;
  d.perm = (b->perm_n > 0 && !b->wave_begin.empty() && b->perm_n == b->wave_begin[1]) ? d.poff + b->m.n_steps + 1 : nullptr;
  d.bsteps = kEmitBlockSteps;
  d.lists = b->lists.p;
  d.lists_all = b->lists.p;
  d.part_stride = 0;
  d.merged = b->merged.p;
  d.excl = b->excl.p;
  d.excl_all = b->excl.p;
  d.excl_part_stride = 0;
  d.assign = b->out.p;
  d.status = b->out.p + b->m.total_r;
  d.domain_out = d.status + b->m.n_steps;
  d.dstar = d.domain_out + b->m.n_steps;
  d.corr = b->corr.p;
  d.corr_cnt = b->corr_cnt.p;
  d.corr_w = 1 + b->m.max_p;
  return d;
}

// Dense role rows of a multi-wave plan from its row table (b->rtab, one entry per role row): needs neither the
// expanded plan blob nor b->m, so plan_stage can launch it while the host still computes the rest of the geometry.
// pdl: launch k_emit_rows as a programmatic dependent of the kernel before it on s (run_chain: the selection kernel of
// another batch)
int launch_emit_plan(rbgtopo_ctx* c, Batch* b, cudaStream_t s, long long n_rows, bool pdl = false) {
  const long long segs = ((n_rows + kEmitRowsBlock - 1) / kEmitRowsBlock) * c->lc;
  if (segs > 0x7FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "rows x chunks exceed 2^31 segments");
  if (segs > 0) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)segs);
    cfg.blockDim = dim3(SCORE_THREADS);
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    const int2* rt = b->rtab.p;
    if (b->any_excl)
      CK(cudaLaunchKernelEx(&cfg, k_emit_rows<true>, topo_dev(c), b->matrix.p, rt, (int)n_rows, (int)c->lc, (int)c->chunk, (int)kEmitRowsBlock));
    else
      CK(cudaLaunchKernelEx(&cfg, k_emit_rows<false>, topo_dev(c), b->matrix.p, rt, (int)n_rows, (int)c->lc, (int)c->chunk, (int)kEmitRowsBlock));
  }
  return RBGTOPO_OK;
}

// claim_off != nullptr (step batches of rbgtopo_place_groups_lw_committed only): k_score_emit_claims with the owner
// claims of earlier groups per step (score.cuh).  cm != nullptr (the same call at levels, §3.16):
// k_score_emit_claims_lv with the group index of every step.  admit != nullptr (step batches of
// rbgtopo_place_groups_eligible[_ranked], §3.19): k_score_emit_elig with MAXP class masks per step; with claim_off or
// cm as well (rbgtopo_place_groups_eligible_committed[_ranked], §3.20): k_score_emit_claims[_lv]_elig.  The claims are
// tested first: masks alone must never stand in for a committed wave's owner claims.
int launch_score(rbgtopo_ctx* c, Batch* b, cudaStream_t s, const int* claim_off = nullptr,
                 const int2* claim_rec = nullptr, const int* step_grp = nullptr, const CommitDev* cm = nullptr,
                 const unsigned long long* admit = nullptr) {
  const BatchMeta& m = b->m;
  if (m.n_steps == 0) return RBGTOPO_OK;
  if (!b->wave_begin.empty()) return launch_emit_plan(c, b, s, m.total_p);  // multi-wave plan: background rows from the row table
  const int items = (int)emit_items(m.n_steps, c->lc);
  const int grid = items / kEmitBlockSteps;  // one CTA per (block of steps, chunk of nodes)
  const unsigned char* cls = c->topo.cls.p;
  if (cm && admit)
    k_score_emit_claims_lv_elig<<<grid, SCORE_THREADS, 0, s>>>(topo_dev(c), batch_dev(c, b), items, step_grp, *cm, cls,
                                                               admit);
  else if (cm)
    k_score_emit_claims_lv<<<grid, SCORE_THREADS, 0, s>>>(topo_dev(c), batch_dev(c, b), items, step_grp, *cm);
  else if (claim_off && admit)
    k_score_emit_claims_elig<<<grid, SCORE_THREADS, 0, s>>>(topo_dev(c), batch_dev(c, b), items, claim_off, claim_rec,
                                                            c->topo.occ, cls, admit);
  else if (claim_off)
    k_score_emit_claims<<<grid, SCORE_THREADS, 0, s>>>(topo_dev(c), batch_dev(c, b), items, claim_off, claim_rec, c->topo.occ);
  else if (admit)
    k_score_emit_elig<<<grid, SCORE_THREADS, 0, s>>>(topo_dev(c), batch_dev(c, b), items, cls, admit);
  else
    k_score_emit<<<grid, SCORE_THREADS, 0, s>>>(topo_dev(c), batch_dev(c, b), items);  // step batch: rows + sparse corrections
  return RBGTOPO_OK;
}

// Launch geometry of k_plan_group for a multi-wave plan; false when the plan has to take the
// per-wave path (RBGTOPO_PER_WAVE_PLAN, or a group's table exceeds a CTA's shared memory).
struct PlanGroupCfg { int nth, HT, CAP, n0; size_t smem; };
bool plan_group_cfg(const Batch* b, PlanGroupCfg* o) {
  if (b->wave_begin.empty() || kPerWavePlan) return false;
  o->nth = std::max(128, 32 * b->m.max_p);
  o->CAP = std::max(32, round_up(b->m.max_cap, 32));
  o->HT = 64;
  while (o->HT <= o->CAP && o->HT < (1 << 20)) o->HT <<= 1;  // > CAP: probes always meet an empty slot
  o->smem = group_smem_bytes(b->m.max_q, o->nth / 32, o->HT, o->CAP);
  o->n0 = b->wave_begin.size() > 1 ? b->wave_begin[1] : 0;  // groups with pending replicas
  return o->smem <= kFastSmemMax;
}

// Records the occupancy of a k_plan_group launch (`ctas` CTAs of `nth` threads with `smem` bytes of dynamic shared
// memory).  Its launch order assumes that every CTA is resident from the start — one round — which holds while
// ctas <= CTAs per SM x SMs (group_smem_bytes); rbgtopo_plan_occupancy reports it.  The occupancy query runs only when
// the launch shape changes.
int note_plan_occupancy(rbgtopo_ctx* c, bool direct, int nth, size_t smem, int ctas) {
  std::lock_guard<std::mutex> g(c->stat_mu);
  auto& o = c->plan_occ[direct];
  if (o.nth != nth || o.smem != smem) {
    int n = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, direct ? k_plan_group<true> : k_plan_group<false>, nth, smem));
    o.nth = nth;
    o.smem = smem;
    o.per_sm = n;
  }
  c->plan_ctas = ctas;
  c->plan_ctas_per_sm = o.per_sm;
  return RBGTOPO_OK;
}

// world == 1: one fused kernel (select + exclusive domain + greedy), one CTA per step
int launch_select_assign(rbgtopo_ctx* c, Batch* b, cudaStream_t s, const BatchDev& d, int* launches, bool pdl = false) {
  const int ns = b->m.n_steps;
  if (ns == 0) return RBGTOPO_OK;
  // shared-memory hash table for the patched nodes of a step: power of two >= 1.5 x the
  // largest capacity among the launch's steps; >= 4 warps per CTA for the table passes
  auto table = [&](int s0, int s1, int* CAP, int* HT) {
    int mc = 0;
    for (int s2 = s0; s2 < s1; ++s2) mc = std::max(mc, b->m.poff[s2 + 1] - b->m.poff[s2]);
    *CAP = std::max(32, round_up(mc, 32));
    *HT = 64;
    while (2 * *HT < 3 * *CAP && *HT < (1 << 20)) *HT <<= 1;
  };
  int CAP, HT;
  table(0, ns, &CAP, &HT);
  // the table has one delta row per warp of the CTA as launched (>= 4 warps), not per role: sized by max_p alone, a
  // batch of 1-2 role steps would pass this check and then ask for more than kFastSmemMax at launch.  Per-wave launches
  // below take at most this many warps and table slots.
  const int nth = std::max(128, 32 * b->m.max_p);
  const bool fast = fast_smem_bytes(nth / 32, HT, CAP) <= kFastSmemMax;
  if (b->wave_begin.empty()) {
    if (fast)
      (b->m.any_level ? k_select_assign_fast<true> : k_select_assign_fast<false>)<<<ns, nth, fast_smem_bytes(nth / 32, HT, CAP), s>>>(topo_dev(c), d, 0, 0, HT, CAP);
    else if (c->cfg.world != 1)
      return fail(RBGTOPO_ELIMIT, "a step's patched set exceeds shared memory: world > 1 must use the shard calls");
    else
      (b->m.any_level ? k_select_assign<true> : k_select_assign<false>)<<<ns, 32 * b->m.max_p, select_smem_bytes(b->m.max_p), s>>>(topo_dev(c), d, 0, 0);
    ++*launches;
    return RBGTOPO_OK;
  }
  // multi-wave plan, preferred: every wave of a group in one CTA of ONE launch (plan_group.cuh)
  PlanGroupCfg pg;
  if (plan_group_cfg(b, &pg)) {
    if (pg.n0 > 0) {
      int rc = note_plan_occupancy(c, false, pg.nth, pg.smem, pg.n0);
      if (rc) return rc;
      if (pdl) {  // programmatic dependent of the dense-matrix kernel just launched on s
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3((unsigned)pg.n0);
        cfg.blockDim = dim3((unsigned)pg.nth);
        cfg.dynamicSmemBytes = pg.smem;
        cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        CK(cudaLaunchKernelEx(&cfg, k_plan_group<false>, topo_dev(c), d, (int)b->m.max_q, pg.HT, pg.CAP, 0));
      } else {
        k_plan_group<false><<<pg.n0, pg.nth, pg.smem, s>>>(topo_dev(c), d, b->m.max_q, pg.HT, pg.CAP, 0);
      }
      ++*launches;
    }
    return RBGTOPO_OK;
  }
  if (c->cfg.world != 1)
    return fail(RBGTOPO_ELIMIT, "plan does not fit k_plan_group's shared memory: world > 1 must use the shard_wave calls");
  // fallback: one launch per wave, placements chained through the plan blob in HBM
  const int wave_mode = SEL_CORRECT | SEL_CHAIN;
  for (size_t w = 0; w + 1 < b->wave_begin.size(); ++w) {
    const int n = b->wave_begin[w + 1] - b->wave_begin[w];
    if (n <= 0) continue;
    if (fast) {
      const int nth = std::max(128, 32 * b->wave_maxp[w]);
      table(b->wave_begin[w], b->wave_begin[w + 1], &CAP, &HT);
      (b->m.any_level ? k_select_assign_fast<true> : k_select_assign_fast<false>)<<<n, nth, fast_smem_bytes(nth / 32, HT, CAP), s>>>(
          topo_dev(c), d, b->wave_begin[w], wave_mode, HT, CAP);
    } else
      (b->m.any_level ? k_select_assign<true> : k_select_assign<false>)<<<n, 32 * b->wave_maxp[w], select_smem_bytes(b->wave_maxp[w]), s>>>(
          topo_dev(c), d, b->wave_begin[w], wave_mode);
    ++*launches;
  }
  return RBGTOPO_OK;
}

constexpr int kMaxTimedPasses = 512;

int ensure_pass_events(Batch* b, int passes) {
  while ((int)b->it_ev.size() < 3 * passes) {
    cudaEvent_t e;
    CK(cudaEventCreate(&e));
    b->it_ev.push_back(e);
  }
  return RBGTOPO_OK;
}

// full single-rank pipeline, `iters` times, ENQUEUE ONLY; results stay on the
// device.  Every pass gets three events (before score, after score, after
// select) until kMaxTimedPasses passes are pending harvest.
int run_batch(rbgtopo_ctx* c, Batch* b, int iters) {
  NvtxRange nv("rbgtopo:run_batch");
  cudaStream_t s = stream_of(c, b);
  int launches = 0;
  BatchDev d = batch_dev(c, b);
  for (int it = 0; it < iters; ++it) {
    const bool early = b->early_emit;  // the staging enqueued this pass's dense-matrix kernel and its events already
    b->early_emit = false;
    // per-pass events only with kernel timing on (or for the pass the staging started): an event record between two
    // kernels costs microseconds of stream time, as much as it measures
    const bool timed = early ? b->tev : (b->passes < kMaxTimedPasses && c->kernel_timing.load(std::memory_order_relaxed));
    const int e0 = 3 * b->passes;
    if (timed && !early) {
      int rc = ensure_pass_events(b, b->passes + 1);
      if (rc) return rc;
      CK(cudaEventRecord(b->it_ev[e0], s));
    }
    int rc;
    PlanGroupCfg pg;
    bool has_mid = true;
    if (it == 0) {  // a pending snapshot refresh: the dense-matrix kernel needs base / free, selection also the order
      if (!early) CK(cudaStreamWaitEvent(s, c->base_ready, 0));
      if (!kSerialPlan || b->wave_begin.empty()) CK(cudaStreamWaitEvent(s, c->topo_ready, 0));
    }
    if (!kSerialPlan && plan_group_cfg(b, &pg)) {
      // Concurrent pipeline: the selection + greedy of every group (k_plan_group, record mode: it never
      // touches the matrix) on stream2 beside the dense-matrix kernel on s; the corrections follow both.
      cudaStream_t s2 = b->stream2;
      CK(cudaEventRecord(b->ev[2], s));
      CK(cudaStreamWaitEvent(s2, b->ev[2], 0));  // after the staging / the previous pass's k_plan_correct
      const size_t pg_smem = std::min(kFastSmemMax, std::max(pg.smem, (size_t)kSelectSmemKB * 1024));
      if (pg.n0 > 0) {
        rc = note_plan_occupancy(c, false, pg.nth, pg_smem, pg.n0);
        if (rc) return rc;
      }
      if (kSelectFirst && pg.n0 > 0) k_plan_group<false><<<pg.n0, pg.nth, pg_smem, s2>>>(topo_dev(c), d, b->m.max_q, pg.HT, pg.CAP, 1);
      rc = launch_score(c, b, s);
      if (rc) return rc;
      ++launches;
      if (timed) CK(cudaEventRecord(b->it_ev[e0 + 1], s));
      if (!kSelectFirst && pg.n0 > 0) k_plan_group<false><<<pg.n0, pg.nth, pg_smem, s2>>>(topo_dev(c), d, b->m.max_q, pg.HT, pg.CAP, 1);
      if (pg.n0 > 0) {
        CK(cudaEventRecord(b->ev[3], s2));
        CK(cudaStreamWaitEvent(s, b->ev[3], 0));
        k_plan_correct<<<(b->m.n_steps + CORRECT_WARPS - 1) / CORRECT_WARPS, 32 * CORRECT_WARPS, 0, s>>>(topo_dev(c), d);
        launches += 2;
      }
    } else {
      // no event (and no wait) between the two kernels unless asked for: k_plan_group is then a programmatic
      // dependent of the dense-matrix kernel
      const bool mid = early || c->kernel_timing.load(std::memory_order_relaxed);
      const bool pdl = !mid && !kNoPdl && !b->wave_begin.empty();
      has_mid = mid;
      if (it == 0 && !mid) CK(cudaStreamWaitEvent(s, c->topo_ready, 0));  // the background order of the refresh
      if (!early) {
        rc = launch_score(c, b, s);
        if (rc) return rc;
        if (timed && mid) CK(cudaEventRecord(b->it_ev[e0 + 1], s));
      }
      ++launches;
      if (it == 0 && mid) CK(cudaStreamWaitEvent(s, c->topo_ready, 0));
      rc = launch_select_assign(c, b, s, d, &launches, pdl);
      if (rc) return rc;
    }
    if (timed) {
      CK(cudaEventRecord(b->it_ev[e0 + 2], s));
      if ((int)b->pass_mid.size() <= b->passes) b->pass_mid.resize(b->passes + 1, 1);
      b->pass_mid[b->passes] = has_mid;
      b->passes += 1;
    }
    b->untimed_or_timed_passes += 1;
  }
  CK(cudaGetLastError());
  b->ran = true;
  b->pend_launches += launches;
  std::lock_guard<std::mutex> g(c->stat_mu);
  c->launches += launches;
  return RBGTOPO_OK;
}

// Pipeline of staged PLAN batches on one stream, ENQUEUE ONLY: `passes` passes, pass k over batch k % n.  Batches are
// independent (own matrix, plan, outputs), so every dense-matrix kernel but the first is chained behind the selection
// kernel of the batch before it as a programmatic dependent: its CTAs fill the SMs while the slowest groups of that
// selection are still being placed (their CTA lifetimes spread widely on cfg3), instead of after the launch gap.
// Falls back to plain passes when the chain does not apply (kernel timing on, other dense-matrix kernels, world > 1's
// per-wave paths, batches on different streams).
int run_chain(rbgtopo_ctx* c, Batch** bs, int n, int passes) {
  NvtxRange nv("rbgtopo:run_chain");
  cudaStream_t s = stream_of(c, bs[0]);
  bool chain = !kNoPdl && kSerialPlan && !c->kernel_timing.load(std::memory_order_relaxed) && n > 1;
  PlanGroupCfg pg;
  for (int i = 0; i < n; ++i) chain = chain && stream_of(c, bs[i]) == s && !bs[i]->early_emit && plan_group_cfg(bs[i], &pg);
  if (!chain) {
    for (int k = 0; k < passes; ++k) {
      int rc = run_batch(c, bs[k % n], 1);
      if (rc) return rc;
    }
    return RBGTOPO_OK;
  }
  CK(cudaStreamWaitEvent(s, c->base_ready, 0));  // a pending snapshot refresh: base / free, and the background order
  CK(cudaStreamWaitEvent(s, c->topo_ready, 0));
  int launches = 0;
  for (int k = 0; k < passes; ++k) {
    Batch* b = bs[k % n];
    int rc = launch_emit_plan(c, b, s, b->m.total_p, /*pdl=*/k > 0);
    if (rc) return rc;
    ++launches;
    rc = launch_select_assign(c, b, s, batch_dev(c, b), &launches, /*pdl=*/true);
    if (rc) return rc;
    b->ran = true;
    b->untimed_or_timed_passes += 1;
  }
  CK(cudaGetLastError());
  for (int i = 0; i < n; ++i) bs[i]->pend_launches += 2 * ((passes - i + n - 1) / n);
  std::lock_guard<std::mutex> g(c->stat_mu);
  c->launches += launches;
  return RBGTOPO_OK;
}

// synchronise, copy the last pass's results out, harvest the timing of every
// pass enqueued since the previous harvest.
// The D2H half of fetch_batch, enqueue only (place_groups pipelines two batches).
int enqueue_d2h(rbgtopo_ctx* c, Batch* b) {
  cudaStream_t s = stream_of(c, b);
  const BatchMeta& m = b->m;
  const size_t out_n = (size_t)m.total_r + 2 * (size_t)m.n_steps;
  if (b->tev) CK(cudaEventRecord(b->ev[4], s));
  if (out_n) CK(cudaMemcpyAsync(b->h_out.p, b->out.p, out_n * 4, cudaMemcpyDeviceToHost, s));
  if (b->tev) CK(cudaEventRecord(b->ev[5], s));
  b->d2h_enqueued = true;
  return RBGTOPO_OK;
}

int fetch_batch(rbgtopo_ctx* c, Batch* b, int32_t* assign, int32_t* status, int32_t* domain) {
  NvtxRange nv("rbgtopo:fetch_batch");
  cudaStream_t s = stream_of(c, b);
  const BatchMeta& m = b->m;
  if (!b->d2h_enqueued) {
    int rc = enqueue_d2h(c, b);
    if (rc) return rc;
  }
  b->d2h_enqueued = false;
  const auto f0 = std::chrono::steady_clock::now();
  CK(cudaStreamSynchronize(s));
  const auto f1 = std::chrono::steady_clock::now();
  CK(cudaGetLastError());
  if (assign && m.total_r) memcpy(assign, b->h_out.p, (size_t)m.total_r * 4);
  if (status && m.n_steps) memcpy(status, b->h_out.p + m.total_r, (size_t)m.n_steps * 4);
  if (domain && m.n_steps) memcpy(domain, b->h_out.p + m.total_r + m.n_steps, (size_t)m.n_steps * 4);
#ifdef RBGTOPO_PHASE_CLOCKS
  if (!b->wave_begin.empty() && b->wave_begin.size() > 1) {
    const int n0 = std::min(2048, b->wave_begin[1]);
    std::vector<long long> clk((size_t)2048 * 32);
    if (cudaMemcpyFromSymbol(clk.data(), g_phase_clk, clk.size() * 8) == cudaSuccess) {
      const char* names[6] = {"start", "A anchors", "B attrs", "C corrections", "D select", "E greedy"};
      double tot = 0;
      long long t0min = LLONG_MAX, t1max = 0;
      for (int g = 0; g < n0; ++g) { tot += (double)(clk[g * 32 + 31] - clk[g * 32 + 30]); t0min = std::min(t0min, clk[g * 32 + 30]); t1max = std::max(t1max, clk[g * 32 + 31]); }
      fprintf(stderr, "[phase clocks] CTA lifetime avg %.0f cycles; first start -> last end %lld cycles\n", tot / n0, t1max - t0min);
      std::vector<long long> ns((size_t)2048 * 4);
      if (cudaMemcpyFromSymbol(ns.data(), g_cta_ns, ns.size() * 8) == cudaSuccess) {  // global-timer timeline of the launch
        long long g0 = LLONG_MAX, g1 = 0;
        for (int g = 0; g < n0; ++g) { g0 = std::min(g0, ns[g * 4]); g1 = std::max(g1, ns[g * 4 + 1]); }
        std::vector<long long> st, life, cn;
        for (int g = 0; g < n0; ++g) { st.push_back(ns[g * 4] - g0); life.push_back(ns[g * 4 + 1] - ns[g * 4]); cn.push_back(ns[g * 4 + 2]); }
        std::sort(st.begin(), st.end()); std::sort(life.begin(), life.end()); std::sort(cn.begin(), cn.end());
        auto q = [&](const std::vector<long long>& v, double f) { return v[std::min(v.size() - 1, (size_t)(f * v.size()))]; };
        {  // per SM: when its last CTA ended, and the anchors-class mix (group index mod 4 in the bench fleet)
          std::map<int, std::pair<long long, int>> sm;  // smid -> (last end, CTAs)
          std::map<int, std::vector<int>> cls;
          for (int g = 0; g < n0; ++g) {
            auto& e = sm[(int)ns[g * 4 + 3]];
            e.first = std::max(e.first, ns[g * 4 + 1] - g0);
            e.second += 1;
            cls[(int)ns[g * 4 + 3]].push_back(g & 3);
          }
          std::vector<long long> ends;
          for (auto& kv : sm) ends.push_back(kv.second.first);
          std::sort(ends.begin(), ends.end());
          int pure = 0;
          for (auto& kv : cls) { bool same = true; for (int c2 : kv.second) same = same && c2 == kv.second[0]; pure += same; }
          {
            std::map<int, std::vector<int>> blk;
            for (int g = 0; g < n0; ++g) blk[(int)ns[g * 4 + 3]].push_back(g);
            int shown = 0;
            for (auto& kv : blk) {
              if (shown++ >= 4) break;
              fprintf(stderr, "[cta timeline] SM %d runs blocks:", kv.first);
              for (int g : kv.second) fprintf(stderr, " %d", g);
              fprintf(stderr, "\n");
            }
          }
          fprintf(stderr, "[cta timeline] per SM (%zu SMs): last CTA ends at ns min %lld p50 %lld p90 %lld max %lld; SMs whose CTAs all have the same (group mod 4): %d\n",
                  ends.size(), ends.front(), q(ends, .5), q(ends, .9), ends.back(), pure);
        }
        fprintf(stderr, "[cta timeline] first start -> last end %lld ns; start offset ns p50 %lld p90 %lld max %lld; lifetime ns min %lld p50 %lld p90 %lld max %lld; table entries min %lld p50 %lld p90 %lld max %lld\n",
                g1 - g0, q(st, .5), q(st, .9), st.back(), life.front(), q(life, .5), q(life, .9), life.back(), cn.front(), q(cn, .5), q(cn, .9), cn.back());
        {  // second round: CTAs that started only after another CTA of the launch retired; the tail behind the dense matrix
          long long first_end = LLONG_MAX;
          for (int g = 0; g < n0; ++g) first_end = std::min(first_end, ns[g * 4 + 1]);
          int late = 0;
          for (int g = 0; g < n0; ++g) late += ns[g * 4] > first_end;
          unsigned long long emit_end = 0;
          std::map<int, long long> cls_end;  // group mod 4 -> last end
          for (int g = 0; g < n0; ++g) cls_end[g & 3] = std::max(cls_end[g & 3], ns[g * 4 + 1] - g0);
          if (cudaMemcpyFromSymbol(&emit_end, g_emit_end_ns, 8) == cudaSuccess && emit_end)
            fprintf(stderr, "[cta timeline] dense matrix ends at %lld ns (after the first plan CTA start); tail after it %lld ns\n",
                    (long long)emit_end - g0, g1 - (long long)emit_end);
          fprintf(stderr, "[cta timeline] %d of %d CTAs started after the first CTA retired (at %lld ns); last end by group mod 4:",
                  late, n0, first_end - g0);
          for (auto& kv : cls_end) fprintf(stderr, " %d: %lld", kv.first, kv.second);
          fprintf(stderr, "\n");
        }
      }
      for (int w = 0; w < 3; ++w) {
        double d[6] = {0};
        for (int g = 0; g < n0; ++g) {
          const long long* c0 = &clk[g * 32 + w * 8];
          d[0] += (double)(c0[0] - (w ? clk[g * 32 + (w - 1) * 8 + 5] : clk[g * 32 + 30]));
          for (int k = 1; k < 6; ++k) d[k] += (double)(c0[k] - c0[k - 1]);
        }
        double da = 0, db = 0, dm = 0;
        for (int g = 0; g < n0; ++g) {
          const long long* c0 = &clk[g * 32 + w * 8];
          da += (double)(c0[6] - c0[3]); db += (double)(c0[7] - c0[6]); dm += (double)(c0[4] - c0[7]);
        }
        fprintf(stderr, "[phase clocks] wave %d:", w);
        for (int k = 0; k < 6; ++k) fprintf(stderr, " %s %.0f", names[k], d[k] / n0);
        fprintf(stderr, " | D: patched %.0f, background %.0f, merge+sync %.0f", da / n0, db / n0, dm / n0);
        fprintf(stderr, "\n");
      }
    }
  }
#endif
  static const bool prof_dev = getenv("RBGTOPO_PROFILE_HOST") != nullptr;
  if (prof_dev && b->tev && b->passes == 1 && !b->wave_begin.empty()) {  // device timeline of a place_groups call, us after the staging began
    float t[6] = {0, 0, 0, 0, 0, 0};
    cudaEvent_t evs[6] = {b->it_ev[0], b->it_ev[1], b->ev[1], b->it_ev[2], b->ev[4], b->ev[5]};
    for (int i = 0; i < 6; ++i)
      if (cudaEventElapsedTime(&t[i], b->ev[0], evs[i]) != cudaSuccess) t[i] = -1.f;
    fprintf(stderr, "[rbgtopo fetch] stream sync returned after %.0f us\n", std::chrono::duration<double, std::micro>(f1 - f0).count());
    fprintf(stderr, "[rbgtopo device] us after staging began: emit start %.0f, emit end %.0f, plan expanded %.0f, selection end %.0f, D2H start %.0f, D2H end %.0f\n",
            t[0] * 1e3, t[1] * 1e3, t[2] * 1e3, t[3] * 1e3, t[4] * 1e3, t[5] * 1e3);
    (void)cudaGetLastError();
  }
  rbgtopo_timing tm{};
  float x = 0.f;
  if (b->tev && cudaEventElapsedTime(&x, b->ev[0], b->ev[1]) == cudaSuccess) tm.h2d_ms = x;
  float score = 0.f, sel = 0.f;
  std::vector<float> pass_score, pass_sel;
  int mids = 0;
  for (int it = 0; it < b->passes; ++it) {
    if (it < (int)b->pass_mid.size() && !b->pass_mid[it]) continue;  // pass without the event between its kernels
    ++mids;
    if (cudaEventElapsedTime(&x, b->it_ev[3 * it], b->it_ev[3 * it + 1]) == cudaSuccess) { score += x; pass_score.push_back(x); }
    if (cudaEventElapsedTime(&x, b->it_ev[3 * it + 1], b->it_ev[3 * it + 2]) == cudaSuccess) { sel += x; pass_sel.push_back(x); }
  }
  if (mids > 0) {
    tm.score_ms = score / mids;
    tm.select_ms = sel / mids;
  }
  if (b->tev && cudaEventElapsedTime(&x, b->ev[4], b->ev[5]) == cudaSuccess) tm.d2h_ms = x;
  float whole = 0.f;  // passes timed as a whole (kernel timing off)
  for (int it = 0; it < b->passes; ++it)
    if (it < (int)b->pass_mid.size() && !b->pass_mid[it] && cudaEventElapsedTime(&x, b->it_ev[3 * it], b->it_ev[3 * it + 2]) == cudaSuccess) whole += x;
  tm.total_ms = tm.h2d_ms + score + sel + whole + tm.d2h_ms;
  harvest_base_ms(c);
  tm.base_ms = c->topo.base_ms;
  tm.scores = m.scores;
  tm.algo_bytes = m.algo_bytes;
  tm.launches = b->pend_launches;
  tm.h2d_words = (int32_t)m.h2d_words;
  (void)cudaGetLastError();  // events recorded under stream capture have no timestamps: not an error here
  const int total_passes = b->untimed_or_timed_passes;
  b->passes = 0;
  b->pass_mid.clear();
  b->pend_launches = 0;
  b->untimed_or_timed_passes = 0;
  std::lock_guard<std::mutex> g(c->stat_mu);
  c->last = tm;
  c->last_score_ms.swap(pass_score);
  c->last_select_ms.swap(pass_sel);
  c->calls += 1;
  c->scores_total += m.scores * std::max(1, total_passes);
  return RBGTOPO_OK;
}

// any_epoch: rbgtopo_release only — a handle staged against an older topology can still be released, and so can an
// exchange handle (§3.17).
Batch* batch_of(rbgtopo_ctx* c, int handle, bool any_epoch = false) {
  std::lock_guard<std::mutex> g(c->pool_mu);
  if (handle < 0 || handle >= (int)c->batches.size()) return nullptr;
  Batch* b = c->batches[handle].get();
  if (!(b->in_use && (b->staged || (any_epoch && b->xchg)))) return nullptr;
  if (!any_epoch && b->epoch != c->topo_epoch) return nullptr;  // sizes / offsets belong to the old topology
  if (!any_epoch && b->m.any_level && b->lvl_epoch != c->lvl_epoch) return nullptr;  // levels of old partitions
  return b;
}

// Orders the snapshot writers behind everything already enqueued on the batch streams: the refresh
// chain (topo_stream) must not rewrite free / owner / base / order while a batch enqueued by
// run_staged / shard_* (asynchronous, lock released) still reads them.  Caller holds topo_mu
// exclusively, so nothing new is enqueued meanwhile.  sync = also wait on the host (set_topology
// frees and reallocates the buffers).
int fence_batches(rbgtopo_ctx* c, bool sync) {
  std::lock_guard<std::mutex> g(c->pool_mu);
  if (c->use_ext_stream) {
    if (sync) CK(cudaStreamSynchronize(c->ext_stream));
    else {
      CK(cudaEventRecord(c->fence_ev, c->ext_stream));
      CK(cudaStreamWaitEvent(c->topo_stream, c->fence_ev, 0));
    }
  }
  for (auto& b : c->batches) {
    if (!b->in_use || !b->stream) continue;
    if (sync) {
      CK(cudaStreamSynchronize(b->stream));
      CK(cudaStreamSynchronize(b->stream2));
    } else {
      // an idle batch (staged and fetched, nothing enqueued since) has nothing in flight that could read the old snapshot
      const bool idle = cudaStreamQuery(b->stream) == cudaSuccess && (!b->stream2 || cudaStreamQuery(b->stream2) == cudaSuccess);
      (void)cudaGetLastError();  // cudaErrorNotReady is the answer, not an error
      if (idle) continue;
      CK(cudaEventRecord(b->ev[6], b->stream));
      CK(cudaStreamWaitEvent(c->topo_stream, b->ev[6], 0));
    }
  }
  return RBGTOPO_OK;
}
int handle_of(rbgtopo_ctx* c, Batch* b) {
  std::lock_guard<std::mutex> g(c->pool_mu);
  for (size_t i = 0; i < c->batches.size(); ++i)
    if (c->batches[i].get() == b) return (int)i;
  return -1;
}

}  // namespace

// ============================================================== C ABI
extern "C" {

int32_t rbgtopo_abi_version(void) { return RBGTOPO_ABI_VERSION; }

int32_t rbgtopo_last_error(rbgtopo_ctx*, char* buf, int32_t len) {
  std::string text = g_err;
  if (text.empty()) {  // another OS thread made the failing call (goroutine migration)
    std::lock_guard<std::mutex> g(g_last_err_mu);
    text = g_last_err;
  }
  if (buf && len > 0) {
    int n = (int)std::min<size_t>(text.size(), (size_t)len - 1);
    memcpy(buf, text.data(), n);
    buf[n] = 0;
  }
  return (int32_t)text.size();
}

int32_t rbgtopo_create(const rbgtopo_config* cfg, rbgtopo_ctx** out) {
  if (!cfg || !out) return fail(RBGTOPO_EINVAL, "null argument");
  *out = nullptr;
  if (cfg->world < 1 || cfg->rank < 0 || cfg->rank >= cfg->world)
    return fail(RBGTOPO_EINVAL, "rank %d / world %d", cfg->rank, cfg->world);
  if (cfg->flags & ~(RBGTOPO_CFG_LEVEL_PLACEMENT | RBGTOPO_CFG_COMMIT_LEVELS | RBGTOPO_CFG_LW_COMMIT_LEVELS |
                     RBGTOPO_CFG_LW_SHARDS))
    return fail(RBGTOPO_EINVAL, "unknown config flags 0x%x", cfg->flags);
  if ((cfg->flags & RBGTOPO_CFG_COMMIT_LEVELS) && !(cfg->flags & RBGTOPO_CFG_LEVEL_PLACEMENT))
    return fail(RBGTOPO_EINVAL, "RBGTOPO_CFG_COMMIT_LEVELS needs RBGTOPO_CFG_LEVEL_PLACEMENT (flags 0x%x)", cfg->flags);
  if ((cfg->flags & RBGTOPO_CFG_LW_COMMIT_LEVELS) && !(cfg->flags & RBGTOPO_CFG_COMMIT_LEVELS))
    return fail(RBGTOPO_EINVAL, "RBGTOPO_CFG_LW_COMMIT_LEVELS needs RBGTOPO_CFG_COMMIT_LEVELS (flags 0x%x)", cfg->flags);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev <= 0)
    return fail(RBGTOPO_ENODEVICE, "no CUDA device (%s); rbgtopo has no CPU path",
                e == cudaSuccess ? "count=0" : cudaGetErrorString(e));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(RBGTOPO_ENODEVICE, "device %d of %d", cfg->device, ndev);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(RBGTOPO_ENODEVICE, "device %d is sm_%d%d; kernels are built for sm_90a only", cfg->device,
                prop.major, prop.minor);
  CK(cudaSetDevice(cfg->device));
  auto c = std::make_unique<rbgtopo_ctx>();
  c->cfg = *cfg;
  c->cfg.emit_matrix = 1;  // the dense matrix is always materialised (it is the product; rbgtopo_read_scores)
  c->sm_count = prop.multiProcessorCount;
  c->kernel_timing.store(kKernelTimingEnv);
  CK(cudaStreamCreateWithFlags(&c->topo_stream, cudaStreamNonBlocking));
  CK(cudaEventCreateWithFlags(&c->topo_ready, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&c->base_ready, cudaEventDisableTiming));
  CK(cudaFuncSetAttribute(k_order_sort_small, cudaFuncAttributeMaxDynamicSharedMemorySize, ORDER_SMALL_MAX * 8));
  CK(cudaEventCreate(&c->ev_base_a));
  CK(cudaEventCreate(&c->ev_base_b));
  CK(cudaEventCreateWithFlags(&c->fence_ev, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&c->p2p_done, cudaEventDisableTiming));
  for (auto& e : c->stage_ev) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (auto* f : {k_select_assign_fast<false>, k_select_assign_fast<true>})
    CK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFastSmemMax));
  for (auto* f : {k_shard_select<false>, k_shard_select<true>})
    CK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFastSmemMax));
  CK(cudaFuncSetAttribute(k_plan_group<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFastSmemMax));
  CK(cudaFuncSetAttribute(k_plan_group<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFastSmemMax));
  CK(cudaFuncSetAttribute(k_plan_group<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  for (auto* f : {k_plan_group_commit<false>, k_plan_group_commit<true>}) {
    CK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFastSmemMax));
    CK(cudaFuncSetAttribute(f, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  }
  for (auto* f : {k_alternates<false>, k_alternates<true>})
    CK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFastSmemMax));
  for (auto* f : {k_alternates_commit<false>, k_alternates_commit<true>, k_alternates_commit_coloc,
                  k_alternates_commit_coloc_lv})
    CK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFastSmemMax));
  for (auto* f : {k_alternates_slab<false, false>, k_alternates_slab<true, false>, k_alternates_slab<true, true>,
                  k_alternates_slab_coloc<false, false>, k_alternates_slab_coloc<true, false>,
                  k_alternates_slab_coloc<true, true>})
    CK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFastSmemMax));
  CK(cudaFuncSetAttribute(k_lw_assign, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFastSmemMax));
  for (auto* f : {k_lw_assign_repl<LW_REPL>, k_lw_assign_repl<LW_REPL_CLAIMS>, k_lw_assign_repl<LW_REPL_CLAIMS_LV>})
    CK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFastSmemMax));
  CK(cudaFuncSetAttribute(k_plan_group<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
#ifdef RBGTOPO_PHASE_CLOCKS
  {
    const int skip = getenv("RBGTOPO_DBG_SKIP") ? atoi(getenv("RBGTOPO_DBG_SKIP")) : 0;
    CK(cudaMemcpyToSymbol(g_dbg_skip, &skip, sizeof skip));
  }
#endif
  *out = c.release();
  return RBGTOPO_OK;
}

int32_t rbgtopo_destroy(rbgtopo_ctx* c) {
  if (!c) return RBGTOPO_OK;
  cudaSetDevice(c->cfg.device);
  cudaDeviceSynchronize();
  for (void* q : c->p2p_opened) cudaIpcCloseMemHandle(q);
  if (c->topo.refresh_exec) cudaGraphExecDestroy(c->topo.refresh_exec);
  if (c->topo.order_exec) cudaGraphExecDestroy(c->topo.order_exec);
  if (c->topo_stream) cudaStreamDestroy(c->topo_stream);
  if (c->topo_ready) cudaEventDestroy(c->topo_ready);
  if (c->base_ready) cudaEventDestroy(c->base_ready);
  if (c->ev_base_a) cudaEventDestroy(c->ev_base_a);
  if (c->ev_base_b) cudaEventDestroy(c->ev_base_b);
  if (c->fence_ev) cudaEventDestroy(c->fence_ev);
  if (c->p2p_done) cudaEventDestroy(c->p2p_done);
  for (auto& e : c->stage_ev) if (e) cudaEventDestroy(e);
  delete c;
  return RBGTOPO_OK;
}

int32_t rbgtopo_set_topology(rbgtopo_ctx* c, int32_t n, int64_t e, const int32_t* row_ptr,
                             const int32_t* col, const int32_t* w, const int32_t* free_slots,
                             const int32_t* domain, int32_t n_domains, const int32_t* owner,
                             uint64_t generation) {
  if (!c || !row_ptr || !free_slots || !domain || !owner || (e > 0 && (!col || !w)))
    return fail(RBGTOPO_EINVAL, "null argument");
  if (n < 1 || e < 0 || e > 0x7FFFFFF0LL || n_domains < 1) return fail(RBGTOPO_EINVAL, "n=%d e=%lld", n, (long long)e);
  if (row_ptr[0] != 0 || row_ptr[n] != e) return fail(RBGTOPO_EINVAL, "row_ptr ends");
  // ---- validation (spec §3.1)
  long long wsum_max = 0;
  for (int i = 0; i < n; ++i) {
    if (row_ptr[i + 1] < row_ptr[i]) return fail(RBGTOPO_EINVAL, "row_ptr not monotone at %d", i);
    if (free_slots[i] < 0 || free_slots[i] > RBGTOPO_MAX_FREE) return fail(RBGTOPO_EINVAL, "free[%d]", i);
    if (domain[i] < 0 || domain[i] >= n_domains) return fail(RBGTOPO_EINVAL, "domain[%d]", i);
    long long ws = 0;
    for (int j = row_ptr[i]; j < row_ptr[i + 1]; ++j) {
      const int cj = col[j];
      if (cj < 0 || cj >= n || cj == i) return fail(RBGTOPO_EINVAL, "col_idx[%d]=%d in row %d", j, cj, i);
      if (j > row_ptr[i] && col[j - 1] >= cj) return fail(RBGTOPO_EINVAL, "row %d not strictly ascending", i);
      if (w[j] < 0 || w[j] > RBGTOPO_MAX_EDGE_W) return fail(RBGTOPO_EINVAL, "edge_w[%d]", j);
      ws += w[j];
      const int32_t* lo = col + row_ptr[cj];
      const int32_t* hi = col + row_ptr[cj + 1];
      const int32_t* it = std::lower_bound(lo, hi, i);
      if (it == hi || *it != i || w[it - col] != w[j])
        return fail(RBGTOPO_EINVAL, "CSR not symmetric at edge (%d,%d)", i, cj);
    }
    wsum_max = std::max(wsum_max, ws);
  }
  for (int d = 0; d < n_domains; ++d)
    if (owner[d] < -1) return fail(RBGTOPO_EINVAL, "domain_owner[%d]", d);

  std::unique_lock<std::shared_mutex> lk(c->topo_mu);
  CK(cudaSetDevice(c->cfg.device));
  Topology& T = c->topo;
  // every batch already enqueued finishes before its snapshot buffers are freed / resized, and
  // the handles staged so far become stale (their sizes and offsets belong to the old topology)
  {
    int frc = fence_batches(c, true);
    if (frc) return frc;
    CK(cudaStreamSynchronize(c->topo_stream));
    c->topo_epoch += 1;
  }
  T.valid = false;
  compute_slab(c, n);
  // base-kernel tiles
  std::vector<int2> tiles;
  for (int r = 0; r < n;) {
    int r1 = r;
    const int a0 = row_ptr[r] & ~3;
    while (r1 < n && r1 - r < BASE_TILE_ROWS && row_ptr[r1 + 1] - a0 <= BASE_TILE_NNZ) ++r1;
    if (r1 == r) r1 = r + 1;  // over-long row: its own (unstaged) tile
    tiles.push_back(make_int2(r, r1));
    r = r1;
  }
  // nodes grouped by domain
  std::vector<int> dom_ptr(n_domains + 1, 0), dom_nodes(n);
  for (int i = 0; i < n; ++i) dom_ptr[domain[i] + 1]++;
  for (int d = 0; d < n_domains; ++d) dom_ptr[d + 1] += dom_ptr[d];
  {
    std::vector<int> cur(dom_ptr.begin(), dom_ptr.end() - 1);
    for (int i = 0; i < n; ++i) dom_nodes[cur[domain[i]]++] = i;
  }
  const size_t pad = 64;
  CK(T.row_ptr.reserve(n + 1 + pad));
  CK(T.col.reserve((size_t)e + pad));
  CK(T.w.reserve((size_t)e + pad));
  CK(T.free_.reserve(n + pad));
  CK(T.domain.reserve(n + pad));
  CK(T.owner.reserve(n_domains + pad));
  CK(T.node_owner.reserve(n + pad));
  CK(T.dom_ptr.reserve(n_domains + 1 + pad));
  CK(T.dom_nodes.reserve(n + pad));
  CK(T.fmin.reserve((size_t)round_up(n, 16) + pad));
  CK(T.base.reserve((size_t)n + 4096));
  CK(T.tiles.reserve(tiles.size()));
  CK(cudaMemset(T.col.p, 0, T.col.cap * 4));
  CK(cudaMemset(T.w.p, 0, T.w.cap * 4));
  CK(cudaMemset(T.fmin.p, 0, T.fmin.cap));
  CK(cudaMemset(T.base.p, 0, T.base.cap * 4));
  CK(cudaMemcpy(T.row_ptr.p, row_ptr, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice));
  if (e) {
    CK(cudaMemcpy(T.col.p, col, (size_t)e * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(T.w.p, w, (size_t)e * 4, cudaMemcpyHostToDevice));
  }
  CK(cudaMemcpy(T.free_.p, free_slots, (size_t)n * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(T.domain.p, domain, (size_t)n * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(T.owner.p, owner, (size_t)n_domains * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(T.dom_ptr.p, dom_ptr.data(), (size_t)(n_domains + 1) * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(T.dom_nodes.p, dom_nodes.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(T.tiles.p, tiles.data(), tiles.size() * sizeof(int2), cudaMemcpyHostToDevice));
  T.n = n;
  T.e = e;
  T.n_domains = n_domains;
  T.n_tiles = (int)tiles.size();
  T.wsum_max = wsum_max;
  T.generation = generation;
  T.h_domain.assign(domain, domain + n);
  T.h_degp1.resize(n);
  T.max_degp1 = 1;
  for (int i = 0; i < n; ++i) {
    T.h_degp1[i] = row_ptr[i + 1] - row_ptr[i] + 1;
    T.max_degp1 = std::max(T.max_degp1, T.h_degp1[i]);
  }
  T.refresh_ready = false;  // new sizes / pointers: re-capture the refresh chain
  T.occ = false;            // a new topology leaves occupancy mode and drops the levels
  T.n_levels = 0;
  T.lvl_nd.clear();
  T.n_classes = 0;          // ... and the node classes
  c->delta_repairs = 0;
  int rc = run_base(c, c->topo_stream, true);
  if (rc) return rc;
  T.valid = true;
  return RBGTOPO_OK;
}

int32_t rbgtopo_update_nodes(rbgtopo_ctx* c, const int32_t* free_slots, const int32_t* owner,
                             uint64_t generation) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  std::unique_lock<std::shared_mutex> lk(c->topo_mu);  // no call enqueues while we hold it ...
  Topology& T = c->topo;
  if (!T.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
  if (owner && T.occ)
    return fail(RBGTOPO_EINVAL, "domain_owner in occupancy mode: ownership comes from rbgtopo_set_exclusive_levels");
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t s = c->topo_stream;
  {  // ... and what run_staged / shard_* already enqueued (asynchronously) reads the old snapshot first
    int frc = fence_batches(c, false);
    if (frc) return frc;
  }
  const unsigned sb = c->stage_idx++ & 1u;
  CK(cudaEventSynchronize(c->stage_ev[sb]));  // the H2D copies of two updates ago have left this staging buffer
  if (free_slots) {
    CK(c->h_free[sb].reserve((size_t)T.n));
    // validate while copying (one pass over the caller's array)
    int* const dst = c->h_free[sb].p;
    int bad = -1;
    for (int i = 0; i < T.n; ++i) {
      const int f = free_slots[i];
      dst[i] = f;
      if ((unsigned)f > (unsigned)RBGTOPO_MAX_FREE && bad < 0) bad = i;
    }
    if (bad >= 0) return fail(RBGTOPO_EINVAL, "free[%d]", bad);
  }
  if (owner) {
    for (int d = 0; d < T.n_domains; ++d)
      if (owner[d] < -1) return fail(RBGTOPO_EINVAL, "domain_owner[%d]", d);
    CK(c->h_owner[sb].reserve((size_t)T.n_domains));
    memcpy(c->h_owner[sb].p, owner, (size_t)T.n_domains * 4);
  }
  if (free_slots) CK(cudaMemcpyAsync(T.free_.p, c->h_free[sb].p, (size_t)T.n * 4, cudaMemcpyHostToDevice, s));
  if (owner) CK(cudaMemcpyAsync(T.owner.p, c->h_owner[sb].p, (size_t)T.n_domains * 4, cudaMemcpyHostToDevice, s));
  CK(cudaEventRecord(c->stage_ev[sb], s));
  T.generation = generation;
  // asynchronous: the refresh (prep, base SpMV, order sort) overlaps the caller's next host
  // work; every batch stream waits on topo_ready before reading the snapshot
  return run_base(c, s, false);
}

namespace {
__global__ void k_delta_scatter(int* __restrict__ free_w, const int* __restrict__ changed, int n_changed) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_changed) free_w[changed[2 * i]] = changed[2 * i + 1];
}
}  // namespace

// Capacity of a few nodes changed (a pod was bound / deleted; the caller cadence is the reconcile
// events of rolebasedgroup_controller.go:1347-1430): incremental refresh of base and of the background
// order (kernels.cuh) instead of the full SpMV + sort.  Falls back to the full refresh when the closed
// neighbourhoods of the changed nodes hold more than DELTA_MAX_AFFECTED nodes, or with world > 1.
int32_t rbgtopo_update_nodes_delta(rbgtopo_ctx* c, int32_t n_changed, const int32_t* nodes, const int32_t* free_slots,
                                   uint64_t generation) {
  if (!c || n_changed < 0 || (n_changed && (!nodes || !free_slots))) return fail(RBGTOPO_EINVAL, "null argument");
  NvtxRange nv("rbgtopo:update_nodes_delta");
  std::unique_lock<std::shared_mutex> lk(c->topo_mu);
  Topology& T = c->topo;
  if (!T.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
  CK(cudaSetDevice(c->cfg.device));
  T.generation = generation;
  if (n_changed == 0) return RBGTOPO_OK;
  // validate + deduplicate (the last value of a node wins, as a sequence of single updates would)
  std::vector<std::pair<int32_t, int32_t>> ch((size_t)n_changed);
  for (int i = 0; i < n_changed; ++i) {
    if (nodes[i] < 0 || nodes[i] >= T.n) return fail(RBGTOPO_EINVAL, "nodes[%d] = %d", i, nodes[i]);
    if (free_slots[i] < 0 || free_slots[i] > RBGTOPO_MAX_FREE) return fail(RBGTOPO_EINVAL, "free[%d]", i);
    ch[i] = {nodes[i], i};
  }
  std::sort(ch.begin(), ch.end());
  long long est = 0;
  size_t m = 0;
  for (size_t i = 0; i < ch.size(); ++i) {
    if (i + 1 < ch.size() && ch[i + 1].first == ch[i].first) continue;  // a later entry of the same node follows
    ch[m++] = {ch[i].first, free_slots[ch[i].second]};
    est += T.h_degp1[ch[i].first];
  }
  ch.resize(m);
  cudaStream_t s = c->topo_stream;
  {
    int frc = fence_batches(c, false);  // batches already enqueued read the old snapshot first
    if (frc) return frc;
  }
  const unsigned sb = c->stage_idx++ & 1u;
  CK(cudaEventSynchronize(c->stage_ev[sb]));
  CK(c->h_free[sb].reserve(2 * m));
  for (size_t i = 0; i < m; ++i) {
    c->h_free[sb].p[2 * i] = ch[i].first;
    c->h_free[sb].p[2 * i + 1] = ch[i].second;
  }
  CK(T.d_changed.reserve(2 * m));
  CK(cudaMemcpyAsync(T.d_changed.p, c->h_free[sb].p, 2 * m * 4, cudaMemcpyHostToDevice, s));
  CK(cudaEventRecord(c->stage_ev[sb], s));
  const bool incremental = c->cfg.world == 1 && T.pos_valid && est <= DELTA_MAX_AFFECTED && getenv("RBGTOPO_NO_DELTA") == nullptr;
  if (!incremental) {  // scatter the new capacities, then the full refresh
    k_delta_scatter<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(T.free_.p, T.d_changed.p, (int)m);
    CK(cudaGetLastError());
    return run_base(c, s, false);
  }
  const bool tev = timing_events(c);
  if (tev) CK(cudaEventRecord(c->ev_base_a, s));
  CK(cudaMemsetAsync(T.aff.p, 0, 4, s));
  const TopoDev td = topo_dev(c);
  k_delta_apply<<<(unsigned)((m * 32 + 255) / 256), 256, 0, s>>>(td, T.free_.p, T.fmin.p, T.base.p, T.d_changed.p, (int)m, T.flag.p, T.aff.p);
  CK(cudaEventRecord(c->base_ready, s));  // what the dense-matrix kernel reads is up to date
  k_delta_sort<<<1, 1024, 0, s>>>(T.base.p, T.pos.p, T.flag.p, T.aff.p, T.new_keys.p, T.old_pos.p);
  const int n = c->slab_hi - c->slab_lo;  // == T.n (world == 1)
  k_delta_merge<<<(n + 255) / 256, 256, 0, s>>>(T.order.p, n, T.aff.p, T.new_keys.p, T.old_pos.p, T.order_alt.p, T.pos.p);
  CK(cudaMemcpyAsync(T.order.p, T.order_alt.p, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));  // the refresh graph holds T.order.p
  if (tev) CK(cudaEventRecord(c->ev_base_b, s));
  CK(cudaEventRecord(c->topo_ready, s));
  c->base_timing_pending = tev;
  c->delta_repairs += 1;
  CK(cudaGetLastError());
  std::lock_guard<std::mutex> g(c->stat_mu);
  c->launches += 3;
  return RBGTOPO_OK;
}

// Occupancy mode (DESIGN.md §3.9): the node partitions of the exclusive levels and the pods that carry the exclusive
// label; k_level_owner derives every level's owner vector on the refresh stream.  Installing partitions waits for the
// batches in flight (the buffers may move, as with set_topology); an occupancy-only refresh is ordered behind them like
// update_nodes and reuses its staging double buffer.  Neither touches base or the background order.
int32_t rbgtopo_set_exclusive_levels(rbgtopo_ctx* c, int32_t n_levels, const int32_t* level_domain,
                                     const int32_t* level_n_domains, int32_t n_occ, const int32_t* occ,
                                     uint64_t generation) {
  if (!c || n_occ < 0 || (n_occ > 0 && !occ) || (level_domain && n_levels > 0 && !level_n_domains))
    return fail(RBGTOPO_EINVAL, "null argument");
  if (n_levels < 0 || n_levels > RBGTOPO_MAX_EXCL_LEVELS - 1)
    return fail(RBGTOPO_EINVAL, "n_levels = %d (0 .. %d)", n_levels, RBGTOPO_MAX_EXCL_LEVELS - 1);
  std::unique_lock<std::shared_mutex> lk(c->topo_mu);
  Topology& T = c->topo;
  if (!T.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
  const int n = T.n;
  const bool install = level_domain != nullptr || !T.occ;
  if (!level_domain && n_levels != (T.occ ? T.n_levels : 0))
    return fail(RBGTOPO_EINVAL, "level_domain is NULL: n_levels = %d must equal the installed %d", n_levels, T.occ ? T.n_levels : 0);
  std::vector<int> doff((size_t)n_levels + 2, 0);
  doff[1] = T.n_domains;
  if (install) {
    for (int L = 1; L <= n_levels; ++L) {
      const int nd = level_n_domains[L - 1];
      if (nd < 1) return fail(RBGTOPO_EINVAL, "level_n_domains[%d] = %d", L - 1, nd);
      const int32_t* dl = level_domain + (size_t)(L - 1) * n;
      for (int i = 0; i < n; ++i)
        if (dl[i] < 0 || dl[i] >= nd) return fail(RBGTOPO_EINVAL, "level_domain[%d][%d] = %d outside [0, %d)", L - 1, i, dl[i], nd);
      if ((long long)doff[L] + nd > 0x3FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "domains of all levels exceed 2^30");
      doff[L + 1] = doff[L] + nd;
    }
  }
  for (int r = 0; r < n_occ; ++r) {
    const int32_t* o = occ + 3 * (size_t)r;
    if (o[0] < 0 || o[0] >= n || o[1] < 0 || o[2] < 0 || o[2] > n_levels)
      return fail(RBGTOPO_EINVAL, "occ[%d] = (%d, %d, %d): node in [0, %d), gid >= 0, level in [0, %d]", r, o[0], o[1], o[2], n, n_levels);
  }
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t s = c->topo_stream;
  const int ls = level_stride(n);
  const int n_lv = n_levels + 1;
  if (install) {
    int frc = fence_batches(c, true);
    if (frc) return frc;
    CK(cudaStreamSynchronize(s));
    CK(T.lvl_domain.reserve((size_t)n_lv * ls));
    CK(T.lvl_owner.reserve((size_t)n_lv * ls));
    CK(T.lvl_doff.reserve((size_t)n_lv + 1));
    CK(T.lvl_tab.reserve(2 * (size_t)doff[n_lv]));
    // on the refresh stream, ahead of k_level_owner (the host arrays are pageable: synchronised below before they go)
    CK(cudaMemsetAsync(T.lvl_domain.p, 0, T.lvl_domain.cap * 4, s));
    CK(cudaMemsetAsync(T.lvl_owner.p, 0xFF, T.lvl_owner.cap * 4, s));  // -1, also in the padding the int4 loads reach
    CK(cudaMemcpyAsync(T.lvl_domain.p, T.domain.p, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
    for (int L = 1; L <= n_levels; ++L)
      CK(cudaMemcpyAsync(T.lvl_domain.p + (size_t)L * ls, level_domain + (size_t)(L - 1) * n, (size_t)n * 4,
                         cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(T.lvl_doff.p, doff.data(), (size_t)n_lv * 4 + 4, cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));  // the caller's level_domain and the local doff may go once the call returns
    T.n_levels = n_levels;
    T.h_lvl_domain.assign(level_domain, level_domain + (size_t)n_levels * n);
    T.lvl_total_d = doff[n_lv];
    c->lvl_epoch += 1;
    T.lvl_nd.resize(n_lv);
    for (int L = 0; L < n_lv; ++L) T.lvl_nd[L] = doff[L + 1] - doff[L];
    T.occ = true;
  } else {
    int frc = fence_batches(c, false);  // batches already enqueued read the old owners first
    if (frc) return frc;
  }
  if (n_occ > 0) {
    const unsigned sb = c->stage_idx++ & 1u;
    CK(cudaEventSynchronize(c->stage_ev[sb]));
    CK(c->h_occ[sb].reserve(3 * (size_t)n_occ));
    memcpy(c->h_occ[sb].p, occ, 3 * (size_t)n_occ * 4);
    if (T.occ_rec.cap < 3 * (size_t)n_occ) {
      CK(cudaStreamSynchronize(s));  // an earlier derivation may still read the old records
      CK(T.occ_rec.reserve(3 * (size_t)n_occ));
    }
    CK(cudaMemcpyAsync(T.occ_rec.p, c->h_occ[sb].p, 3 * (size_t)n_occ * 4, cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(c->stage_ev[sb], s));
  }
  const int td = T.lvl_total_d;
  const int th = 256;
  auto grid = [&](long long work) { return (unsigned)std::max(1LL, std::min((work + th - 1) / th, (long long)c->sm_count * 8)); };
  k_level_owner<<<grid(2LL * td), th, 0, s>>>(0, n, n_lv, T.lvl_domain.p, T.lvl_doff.p, td, T.lvl_tab.p, T.occ_rec.p, n_occ, T.lvl_owner.p);
  if (n_occ > 0)
    k_level_owner<<<grid(n_occ), th, 0, s>>>(1, n, n_lv, T.lvl_domain.p, T.lvl_doff.p, td, T.lvl_tab.p, T.occ_rec.p, n_occ, T.lvl_owner.p);
  k_level_owner<<<grid(n), th, 0, s>>>(2, n, n_lv, T.lvl_domain.p, T.lvl_doff.p, td, T.lvl_tab.p, T.occ_rec.p, n_occ, T.lvl_owner.p);
  CK(cudaGetLastError());
  // the owners are node attributes of both the dense-matrix kernels and selection
  CK(cudaEventRecord(c->base_ready, s));
  CK(cudaEventRecord(c->topo_ready, s));
  T.generation = generation;
  std::lock_guard<std::mutex> g(c->stat_mu);
  c->launches += n_occ > 0 ? 3 : 2;
  return RBGTOPO_OK;
}

// Node classes (DESIGN.md §3.19), ordered like rbgtopo_update_nodes: the copy goes on the refresh stream behind the
// batches already enqueued (they read the classes they started with) and in front of base_ready / topo_ready, which
// every later call waits for.  Only a buffer that has to grow waits for the batches in flight.
int32_t rbgtopo_set_node_classes(rbgtopo_ctx* c, int32_t n_classes, const int32_t* node_class, uint64_t generation) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  std::unique_lock<std::shared_mutex> lk(c->topo_mu);
  Topology& T = c->topo;
  if (!T.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
  if (n_classes > RBGTOPO_MAX_NODE_CLASSES)
    return fail(RBGTOPO_ELIMIT, "%d node classes (at most %d)", n_classes, RBGTOPO_MAX_NODE_CLASSES);
  if (n_classes < 1 || !node_class) return fail(RBGTOPO_EINVAL, "n_classes = %d, node_class %p", n_classes, (const void*)node_class);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t s = c->topo_stream;
  const size_t need = (size_t)round_up(T.n, 16) + 64;
  if (T.cls.cap < need) {
    int frc = fence_batches(c, true);
    if (frc) return frc;
    CK(cudaStreamSynchronize(s));
    CK(T.cls.reserve(need));
    CK(cudaMemsetAsync(T.cls.p, 0, T.cls.cap, s));
  } else {
    int frc = fence_batches(c, false);
    if (frc) return frc;
  }
  const unsigned sb = c->stage_idx++ & 1u;
  CK(cudaEventSynchronize(c->stage_ev[sb]));
  CK(c->h_cls[sb].reserve((size_t)T.n));
  unsigned char* const dst = c->h_cls[sb].p;
  for (int i = 0; i < T.n; ++i) {
    const int k = node_class[i];
    if (k < 0 || k >= n_classes) return fail(RBGTOPO_EINVAL, "node_class[%d] = %d outside [0, %d)", i, k, n_classes);
    dst[i] = (unsigned char)k;
  }
  CK(cudaMemcpyAsync(T.cls.p, dst, (size_t)T.n, cudaMemcpyHostToDevice, s));
  CK(cudaEventRecord(c->stage_ev[sb], s));
  CK(cudaEventRecord(c->base_ready, s));
  CK(cudaEventRecord(c->topo_ready, s));
  T.n_classes = n_classes;
  T.generation = generation;
  return RBGTOPO_OK;
}

int32_t rbgtopo_score_assign(rbgtopo_ctx* c, const int32_t* blob, int64_t words, int32_t* assign,
                             int32_t* status, int32_t* domain) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");

  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  CK(cudaSetDevice(c->cfg.device));
  Batch* b = nullptr;
  int rc = acquire_batch(c, &b);
  if (rc) return rc;
  rc = stage_into(c, b, blob, words);
  if (!rc) rc = run_batch(c, b, 1);
  if (!rc) rc = fetch_batch(c, b, assign, status, domain);
  if (rc) cudaStreamSynchronize(stream_of(c, b));
  release_batch(c, b);
  return rc;
}

// ---- whole groups: level/wave loop on the host side of the ABI -------------
namespace {
const int32_t* group_rec(const int32_t* gb, int g) { return gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS; }

// The GROUPS blob header and its group table: every group record lies inside the blob.
bool groups_blob_ok(const int32_t* gb, int64_t words) {
  return words >= RBGTOPO_HDR_WORDS && gb[0] == RBGTOPO_GROUPS_MAGIC && gb[1] == RBGTOPO_ABI_VERSION && gb[3] == words &&
         gb[2] >= 0 && (int64_t)RBGTOPO_HDR_WORDS + (int64_t)gb[2] * RBGTOPO_GROUP_WORDS <= words;
}
// The same checks, reported.
int check_groups_blob(const int32_t* gb, int64_t words) {
  if (words < RBGTOPO_HDR_WORDS || gb[0] != RBGTOPO_GROUPS_MAGIC || gb[1] != RBGTOPO_ABI_VERSION || gb[3] != words)
    return fail(RBGTOPO_EINVAL, "bad groups blob header");
  if (gb[2] < 0 || (int64_t)RBGTOPO_HDR_WORDS + (int64_t)gb[2] * RBGTOPO_GROUP_WORDS > words)
    return fail(RBGTOPO_EINVAL, "group table exceeds blob");
  return RBGTOPO_OK;
}

// Per group of a GROUPS blob: its first role in a role_pods table (r0) and its first pod in assign (pod0); index
// n_groups holds the totals.  rp: the (S, C) table of place_groups_lw (§3.11), or nullptr (one pod per replica).
struct GroupOffsets {
  std::vector<int> r0;
  std::vector<int64_t> pod0;
  GroupOffsets(const int32_t* gb, const int32_t* rp) : r0((size_t)gb[2] + 1, 0), pod0((size_t)gb[2] + 1, 0) {
    for (int g = 0; g < gb[2]; ++g) {
      const int32_t* rec = group_rec(gb, g);
      r0[g + 1] = r0[g] + rec[3];
      pod0[g + 1] = pod0[g];
      for (int i = 0; i < rec[3]; ++i) pod0[g + 1] += (int64_t)gb[rec[4] + 4 * i + 1] * (rp ? rp[2 * (r0[g] + i)] : 1);
    }
  }
  const int32_t* grp(const int32_t* rp, int g) const { return rp ? rp + 2LL * r0[g] : nullptr; }  // group g's (S, C)
};

// One wave of a group: (role, first replica, replicas) per role row.  <= RBGTOPO_MAX_STEP_ROLES entries, no heap.
struct PlanWave {
  int n = 0;
  int role[RBGTOPO_MAX_STEP_ROLES], first[RBGTOPO_MAX_STEP_ROLES], count[RBGTOPO_MAX_STEP_ROLES];
  void push(int r, int f, int c) { role[n] = r; first[n] = f; count[n] = c; ++n; }
  int size() const { return n; }
};
struct WaveCursor {  // a group's next replica: replica `taken` of role `role`; role == q once every replica is in a wave
  int role = 0, taken = 0;
  void settle(const int32_t* roles, int q) {
    while (role < q && roles[4 * role + 1] - taken <= 0) { ++role; taken = 0; }
  }
};

// The wave rule of the host loops, the plan paths and plugin.py: a wave is the next replicas of the roles of one level,
// in role order, at most RBGTOPO_MAX_STEP_ROLES role rows and RBGTOPO_MAX_STEP_REPLICAS pods, a replica's S pods never
// split.  rp: the group's (S, C) per role (§3.11), nullptr = one pod per replica.  Fills w, moves cur past it and
// returns its role rows (0: no replica left).
inline int next_wave(const int32_t* roles, int q, const int32_t* rp, WaveCursor& cur, PlanWave& w) {
  w.n = 0;
  cur.settle(roles, q);
  if (cur.role >= q) return 0;
  const int level = roles[4 * cur.role];
  int n = 0;
  while (cur.role < q && roles[4 * cur.role] == level && w.n < RBGTOPO_MAX_STEP_ROLES) {
    const int left = roles[4 * cur.role + 1] - cur.taken;
    if (left <= 0) { ++cur.role; cur.taken = 0; continue; }
    const int S = rp ? rp[2 * cur.role] : 1;
    const int take = std::min(left, (RBGTOPO_MAX_STEP_REPLICAS - n) / S);
    if (take == 0) break;
    w.push(cur.role, cur.taken, take);
    n += take * S;
    cur.taken += take;
    if (cur.taken == roles[4 * cur.role + 1]) { ++cur.role; cur.taken = 0; }
  }
  cur.settle(roles, q);
  return w.n;
}

// Static wave structure of a group: calls f(index, wave) per wave, returns the count.
extern "C++" {
template <class F>
inline int walk_waves(const int32_t* roles, int q, const int32_t* rp, F&& f) {
  WaveCursor cur;
  PlanWave w;
  int nw = 0;
  while (next_wave(roles, q, rp, cur, w) > 0) f(nw++, w);
  return nw;
}
}  // extern "C++"
int gen_waves(const int32_t* roles, int q, PlanWave* out) {  // out == nullptr: count only
  return walk_waves(roles, q, nullptr, [out](int i, const PlanWave& w) { if (out) out[i] = w; });
}

// One group while a host-driven loop places its waves (run_waves) or rank_committed replays them.  Counts are in pods:
// S pods per replica from rp (place_groups_lw), one without it.
struct HostRun {
  const int32_t* rec = nullptr;
  const int32_t* roles = nullptr;  // q x (level, pending, demand, role_flags)
  const int32_t* pair = nullptr;   // q x q
  const int32_t* rp = nullptr;     // (S, C) per role, or nullptr
  int g = 0, q = 0, fixed_domain = -1, status = RBGTOPO_PLACED_ALL;
  bool failed = false;
  int64_t pod0 = 0, pods = 0;                   // the group's pods in assign
  int ord0[RBGTOPO_MAX_GROUP_ROLES] = {0};      // first pod of every role inside the group's range
  int unplaced[RBGTOPO_MAX_GROUP_ROLES] = {0};  // pods
  WaveCursor cur;
  PlanWave w;                         // the wave in flight
  std::vector<int32_t> anchors;       // (node, role, count)*
  std::vector<int32_t> consumed;      // rp == nullptr: (node, amount)*, one per placed replica
  std::map<int, int> taken;           // rp != nullptr: node -> amount (committed: earlier groups' claims included)
  std::vector<int32_t> owner_claims;  // committed at level 0, exclusive group: (node, claim gid)* of claimed domains, by node
  HostRun() = default;
  HostRun(const int32_t* gb, int g, const int32_t* grp, int64_t first_pod)
      : rec(group_rec(gb, g)), roles(gb + rec[4]), pair(gb + rec[5]), rp(grp), g(g), q(rec[3]), fixed_domain(rec[2]),
        pod0(first_pod) {
    for (int i = 0; i < q; ++i) {
      ord0[i] = (int)pods;
      unplaced[i] = roles[4 * i + 1] * S(i);
      pods += unplaced[i];
    }
    anchors.assign(gb + rec[7], gb + rec[7] + 3LL * rec[6]);
    cur.settle(roles, q);
  }
  int S(int ri) const { return rp ? rp[2 * ri] : 1; }
  bool done() const { return failed || cur.role >= q; }
  // The consumed records of the group's next step: without rp one per placed replica; with rp one per node, sorted (what
  // k_lw_assign relies on).  Only a committed round whose group is re-run later can see claims summing past free[n]
  // (stale claims of earlier groups), so clamping them to RBGTOPO_MAX_FREE changes no kept result.
  void step_consumed(std::vector<int32_t>& out) const {
    if (!rp) {
      out.assign(consumed.begin(), consumed.end());
      return;
    }
    out.clear();
    for (const auto& [node, amount] : taken) { out.push_back(node); out.push_back(std::min(amount, RBGTOPO_MAX_FREE)); }
  }
  // A pod of role ri placed on node: an anchor (node, ri, 1) of the later waves, and the demand it consumes.
  void place(int ri, int node) {
    anchors.push_back(node); anchors.push_back(ri); anchors.push_back(1);
    if (rp) {
      taken[node] += roles[4 * ri + 2];
    } else {
      consumed.push_back(node); consumed.push_back(roles[4 * ri + 2]);
    }
    unplaced[ri] -= 1;
  }
  // The group's results once its waves are placed: a failed gang places nothing.
  void results(int32_t* assign, int32_t* status_out, int32_t* domain_out) const {
    if (failed) {
      for (int64_t k = pod0; k < pod0 + pods; ++k) assign[k] = -1;
      if (status_out) status_out[g] = RBGTOPO_GANG_FAILED;
      if (domain_out) domain_out[g] = -1;
    } else {
      if (status_out) status_out[g] = status;
      if (domain_out) domain_out[g] = (rec[1] & RBGTOPO_STEP_EXCLUSIVE) ? fixed_domain : -1;
    }
  }
};

// A step blob built on the host: the step records in `tab`, their sections in `data` with offsets from the table's
// end until build() lays out the blob.
struct StepBlob {
  std::vector<int32_t> tab, data, blob;
  int ns = 0, racc = 0, rowacc = 0;
  // One step of wave w of group r: role counts in pods, `need` over r.unplaced, r.anchors; role flags keep the
  // role-exclusive bit when role_excl; n_consumed (node, amount) records from `consumed`.
  void add(const HostRun& r, const PlanWave& w, int32_t flags, int32_t dom, int32_t level, bool role_excl,
           const int32_t* consumed, int n_consumed) {
    int32_t st[RBGTOPO_STEP_WORDS] = {0};
    st[0] = r.rec[0];
    st[1] = flags;
    st[2] = dom;
    st[3] = w.n;
    while (data.size() & 3) data.push_back(0);  // role records are read as 16-byte vectors
    st[4] = (int32_t)data.size();
    int n = 0;
    for (int p = 0; p < w.n; ++p) {
      const int ri = w.role[p], pods = w.count[p] * r.S(ri);
      int need = 0;
      for (int j = 0; j < r.q; ++j)
        if (r.pair[ri * r.q + j] > 0) need += r.unplaced[j];
      data.push_back(pods);
      data.push_back(r.roles[4 * ri + 2]);
      data.push_back(std::min(need, RBGTOPO_NEED_CAP));
      data.push_back(role_excl ? r.roles[4 * ri + 3] & RBGTOPO_ROLE_EXCLUSIVE : 0);
      n += pods;
    }
    st[5] = r.q;
    st[6] = (int32_t)data.size();
    for (int p = 0; p < w.n; ++p) data.insert(data.end(), r.pair + w.role[p] * r.q, r.pair + (w.role[p] + 1) * r.q);
    st[7] = (int32_t)(r.anchors.size() / 3);
    st[8] = (int32_t)data.size();
    data.insert(data.end(), r.anchors.begin(), r.anchors.end());
    st[9] = n_consumed;
    st[10] = (int32_t)data.size();
    data.insert(data.end(), consumed, consumed + 2 * (size_t)n_consumed);
    st[11] = n;
    st[12] = racc;
    st[13] = rowacc;
    st[14] = level;
    tab.insert(tab.end(), st, st + RBGTOPO_STEP_WORDS);
    ++ns;
    racc += n;
    rowacc += w.n;
  }
  // header | step records | sections
  const std::vector<int32_t>& build() {
    const int32_t base = RBGTOPO_HDR_WORDS + ns * RBGTOPO_STEP_WORDS;  // a multiple of 4: role records stay aligned
    blob.assign((size_t)base, 0);
    for (int i = 0; i < ns; ++i) {
      int32_t* st = blob.data() + RBGTOPO_HDR_WORDS + (size_t)i * RBGTOPO_STEP_WORDS;
      memcpy(st, tab.data() + (size_t)i * RBGTOPO_STEP_WORDS, RBGTOPO_STEP_WORDS * 4);
      for (int k : {4, 6, 8, 10}) st[k] += base;
    }
    blob.insert(blob.end(), data.begin(), data.end());
    blob[0] = RBGTOPO_BLOB_MAGIC;
    blob[1] = RBGTOPO_ABI_VERSION;
    blob[2] = ns;
    blob[3] = (int32_t)blob.size();
    blob[4] = racc;
    blob[5] = rowacc;
    return blob;
  }
  void clear() {
    tab.clear();
    data.clear();
    ns = racc = rowacc = 0;
  }
};

// (wave, role) rows of group g (grp: as next_wave's rp): what a ranked host-driven loop may keep for it.
size_t group_role_rows(const int32_t* gb, int g, const int32_t* grp) {
  const int32_t* rec = group_rec(gb, g);
  size_t n = 0;
  walk_waves(gb + rec[4], rec[3], grp, [&](int, const PlanWave& w) { n += (size_t)w.n; });
  return n;
}
// The ranked host-driven loops: the matrix is overwritten by every wave, so the wave's `rows` dense rows go to
// b->kept at row *used first (cap rows reserved by reserve_kept).  The ranking runs once the placements are final.
int reserve_kept(rbgtopo_ctx* c, Batch* b, size_t cap) {
  const cudaError_t e = b->kept.reserve(std::max<size_t>(1, cap) * (size_t)c->slab_stride);
  return e == cudaSuccess ? RBGTOPO_OK : fail(RBGTOPO_ECUDA, "rows of a ranked placement: %s", cudaGetErrorString(e));
}
int keep_wave_rows(rbgtopo_ctx* c, Batch* b, int rows, size_t cap, size_t* used) {
  const size_t stride = (size_t)c->slab_stride;
  const cudaError_t e = *used + rows <= cap ? cudaMemcpyAsync(b->kept.p + *used * stride, b->matrix.p, (size_t)rows * stride * 4,
                                                              cudaMemcpyDeviceToDevice, stream_of(c, b))
                                            : cudaErrorInvalidValue;
  if (e != cudaSuccess) return fail(RBGTOPO_ECUDA, "keeping the dense rows of a wave: %s", cudaGetErrorString(e));
  *used += (size_t)rows;
  return RBGTOPO_OK;
}

// ---- ranked placement (rbgtopo_place_groups_ranked, DESIGN.md §3.10)
struct RankReq {  // the ranked outputs of one call, indexed like assign
  int n_alt;
  float* score;
  int32_t* alt_node;
  float* alt_score;
  AltExchange* x = nullptr;  // the sharded form (§3.17): the jobs' slab lists go here; the merge writes the outputs
};
struct AltRow {  // one role row of one wave: where its dense row is, and its replicas [rep0, rep0 + nrep) in assign order
  int row, group, role, rep0, nrep;
};
// The level-0 owner claims of a committed leader-worker batch (§3.15), built on the host from its final claims in the
// layout commit_owner<false> reads: dhead[d] = a group that reported domain d (-1 = none), dclaim[g] = {gid of group g,
// next group that reported the same domain}.
struct HostClaims {
  std::vector<int32_t> dhead;
  std::vector<int2> dclaim;
};
int run_alternates(rbgtopo_ctx* c, Batch* b, const float* rows, const std::vector<AltRow>& list, const int32_t* gb,
                   const int32_t* rp, const int32_t* assign, const int32_t* status, const int32_t* domain,
                   const RankReq& rk, const CommitDev* cm = nullptr, bool cm_levels = false,
                   const HostClaims* hc = nullptr);
void alt_clear(const RankReq& rk, int64_t first, int64_t count);

rbgtopo_timing add_timing(const rbgtopo_timing& a, const rbgtopo_timing& b) {
  rbgtopo_timing t = a;
  t.h2d_ms += b.h2d_ms;
  t.score_ms += b.score_ms;
  t.select_ms += b.select_ms;
  t.d2h_ms += b.d2h_ms;
  t.total_ms += b.total_ms;
  t.launches += b.launches;
  t.h2d_words += b.h2d_words;
  t.scores += b.scores;
  t.algo_bytes += b.algo_bytes;
  return t;
}

struct KeptRows {  // a ranked host-driven loop: the (wave, role) rows that placed a pod, in b->kept (cap rows reserved)
  std::vector<AltRow> list;
  size_t cap = 0, used = 0;
};
struct WaveBufs {  // run_waves' host buffers, reused by every wave of a call, across its rounds too
  StepBlob sb;
  std::vector<int32_t> w_assign, w_status, w_domain, cons;
  std::vector<int> active;
};

// The host-driven wave loop of place_groups_slow and place_groups_lw: per wave, the next wave of every run of
// runs[lo, end) not yet done becomes one step of a blob, which is staged; launch(active) enqueues the wave's kernels
// (active: the indices of those runs, in step order), the results come back and every placed pod feeds the later waves
// of its run.  Once every run is done their results are written.  total sums each wave's timing; keep != nullptr: each
// wave's dense rows go to b->kept.
extern "C++" {
template <class Launch>
int run_waves(rbgtopo_ctx* c, Batch* b, std::vector<HostRun>& runs, int lo, int32_t* assign, int32_t* status,
              int32_t* domain, KeptRows* keep, rbgtopo_timing& total, WaveBufs& wb, Launch&& launch) {
  auto& [sb, w_assign, w_status, w_domain, cons, active] = wb;
  while (true) {
    active.clear();
    for (int i = lo; i < (int)runs.size(); ++i)
      if (!runs[i].done()) active.push_back(i);
    if (active.empty()) break;
    sb.clear();
    for (int i : active) {
      HostRun& r = runs[i];
      next_wave(r.roles, r.q, r.rp, r.cur, r.w);
      r.step_consumed(cons);
      sb.add(r, r.w, r.rec[1] & (RBGTOPO_STEP_EXCLUSIVE | RBGTOPO_STEP_GANG),  // as build_plan / k_expand_plan
             (r.rec[1] & RBGTOPO_STEP_EXCLUSIVE) ? r.fixed_domain : -1, r.rec[10], true, cons.data(),
             (int)(cons.size() / 2));
    }
    const std::vector<int32_t>& blob = sb.build();
    w_assign.resize(sb.racc);
    w_status.resize(sb.ns);
    w_domain.resize(sb.ns);
    const size_t slot0 = keep ? keep->used : 0;  // this wave's rows in b->kept, in matrix order
    int rc = stage_into(c, b, blob.data(), (int64_t)blob.size());
    if (!rc) rc = launch(active);
    if (!rc) rc = fetch_batch(c, b, w_assign.data(), w_status.data(), w_domain.data());
    if (!rc && keep) rc = keep_wave_rows(c, b, sb.rowacc, keep->cap, &keep->used);
    if (rc) return rc;
    {
      std::lock_guard<std::mutex> g(c->stat_mu);
      total = add_timing(total, c->last);
    }
    int off = 0, row = 0;  // row: the role's dense row in this wave's matrix
    for (int i = 0; i < sb.ns; ++i) {
      HostRun& r = runs[active[i]];
      bool any = false;
      for (int p = 0; p < r.w.n; ++p, ++row) {
        const int ri = r.w.role[p], pods = r.w.count[p] * r.S(ri);
        const int64_t first = r.pod0 + r.ord0[ri] + (int64_t)r.w.first[p] * r.S(ri);
        bool placed = false;
        for (int k = 0; k < pods; ++k, ++off) {
          const int node = w_assign[off];
          assign[first + k] = node;
          if (node < 0) continue;
          any = placed = true;
          r.place(ri, node);
        }
        if (keep && placed) keep->list.push_back(AltRow{(int)slot0 + row, r.g, ri, (int)first, pods});
      }
      if ((r.rec[1] & RBGTOPO_STEP_EXCLUSIVE) && w_domain[i] >= 0 && any) r.fixed_domain = w_domain[i];
      r.status = std::max(r.status, w_status[i]);
      if ((r.rec[1] & RBGTOPO_STEP_GANG) && w_status[i] != RBGTOPO_PLACED_ALL) r.failed = true;
    }
  }
  for (int i = lo; i < (int)runs.size(); ++i) runs[i].results(assign, status, domain);
  return RBGTOPO_OK;
}
}  // extern "C++"

// The end of a host-driven loop on b, which it releases: after a failure the batch's stream is drained; otherwise total
// becomes the call's timing and, with keep, the kept rows of every run are ranked now that the placements are final.
int finish_waves(rbgtopo_ctx* c, Batch* b, int rc, rbgtopo_timing total, const std::vector<HostRun>& runs,
                 const KeptRows* keep, const int32_t* gb, const int32_t* rp, const int32_t* assign,
                 const int32_t* status, const int32_t* domain, const RankReq* rk) {
  if (!rc) {
    std::lock_guard<std::mutex> g(c->stat_mu);
    total.base_ms = c->topo.base_ms;
    c->last = total;
  } else {
    cudaStreamSynchronize(stream_of(c, b));
  }
  if (!rc && keep) {
    for (const HostRun& r : runs) alt_clear(*rk, r.pod0, r.pods);
    rc = run_alternates(c, b, b->kept.p, keep->list, gb, rp, assign, status, domain, *rk);
    if (rc) cudaStreamSynchronize(stream_of(c, b));
  }
  release_batch(c, b);
  return rc;
}
}  // namespace

// The host-driven wave loop: one batched launch pair per wave, placements fed back
// through the host.  Exact for every case; used for the groups the device-resident
// plan cannot finish (`only` != null: just those groups) and as its reference.
// rk != nullptr: the ranked form; each wave's rows are kept, and ranked once the placements are final.
static int32_t place_groups_slow(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t* assign,
                                 int32_t* status, int32_t* domain, const std::vector<char>* only,
                                 const RankReq* rk = nullptr) {
  if (const int hrc = check_groups_blob(gb, words)) return hrc;
  const int ng = gb[2];
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  if (!c->topo.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
  if (rk && (size_t)((c->topo.n + 31) / 32) * 4 > kFastSmemMax)  // the snapshot may have changed since the direct pass
    return fail(RBGTOPO_ELIMIT, "ranked placement: %d nodes exceed the room bitmap", c->topo.n);
  CK(cudaSetDevice(c->cfg.device));
  auto in = [&](long long off, long long cnt) { return off >= 0 && cnt >= 0 && off + cnt <= words; };
  long long pacc = 0;
  for (int g = 0; g < ng; ++g) {
    const int32_t* rec = group_rec(gb, g);
    const int q = rec[3];
    if (q < 1 || q > RBGTOPO_MAX_GROUP_ROLES) return fail(RBGTOPO_ELIMIT, "group %d: %d roles", g, q);
    if (!in(rec[4], 4LL * q) || !in(rec[5], (long long)q * q) || !in(rec[7], 3LL * rec[6]))
      return fail(RBGTOPO_EINVAL, "group %d: section out of bounds", g);
    const int32_t* roles = gb + rec[4];
    long long pend = 0;
    for (int i = 0; i < q; ++i) {
      if (roles[4 * i + 1] < 0 || (i && roles[4 * i] < roles[4 * (i - 1)]))
        return fail(RBGTOPO_EINVAL, "group %d role %d: pending < 0 or levels not ascending", g, i);
      pend += roles[4 * i + 1];
    }
    if (rec[8] != pacc || rec[9] != pend) return fail(RBGTOPO_EINVAL, "group %d: bad assign_off/n_pending", g);
    pacc += pend;
  }
  if (gb[4] != pacc) return fail(RBGTOPO_EINVAL, "total pending mismatch");
  std::vector<HostRun> runs;  // the groups placed here; the others keep their results
  KeptRows kept;              // rk: the role rows of the groups placed here
  for (int g = 0; g < ng; ++g) {
    if (only && !(*only)[g]) continue;
    const HostRun& r = runs.emplace_back(gb, g, nullptr, group_rec(gb, g)[8]);
    for (int64_t k = r.pod0; k < r.pod0 + r.pods; ++k) assign[k] = -1;
    if (rk) kept.cap += group_role_rows(gb, g, nullptr);
  }

  Batch* b = nullptr;
  int rc = acquire_batch(c, &b);
  if (rc) return rc;
  if (rk) rc = reserve_kept(c, b, kept.cap);
  rbgtopo_timing total{};
  WaveBufs wb;
  if (!rc)
    rc = run_waves(c, b, runs, 0, assign, status, domain, rk ? &kept : nullptr, total, wb,
                   [&](const std::vector<int>&) { return run_batch(c, b, 1); });
  return finish_waves(c, b, rc, total, runs, rk ? &kept : nullptr, gb, nullptr, assign, status, domain, rk);
}

// ---- device-resident multi-wave plan ------------------------------------------
// All waves of all groups as ONE step blob, wave-major.  The wave structure is
// static (it depends only on levels and pending counts), so every step's records
// can be laid out up front: its anchor list = the group's scheduled pods + one
// record per replica of the earlier waves (filled in on the device by the wave
// that places it), its consumed list likewise, `need` predicted under the
// assumption that earlier replicas get placed.  Groups for which that assumption
// fails (non-gang groups with an unplaced replica) are re-run through the
// host-driven loop afterwards (place_groups_slow) — rare, and exact either way.
namespace {

// ---- ranked placement (DESIGN.md §3.10): the role rows to rank and the kernel launch

// Replicas (pods) [first, first + count) start with no score and no alternates (what an unplaced or gang-failed one
// keeps).
void alt_clear(const RankReq& rk, int64_t first, int64_t count) {
  if (rk.x) return;  // the merge clears every replica
  for (int64_t k = 0; k < count; ++k) {
    const int64_t r = first + k;
    rk.score[r] = -INFINITY;
    for (int i = 0; i < rk.n_alt; ++i) {
      rk.alt_node[r * rk.n_alt + i] = -1;
      rk.alt_score[r * rk.n_alt + i] = -INFINITY;
    }
  }
}

// The per-replica lists o (1 + 2 * n_alt words per compact replica, as k_alternates writes them) into rk at idx.
void alt_scatter(const RankReq& rk, const int* o, const int* idx, size_t n) {
  const int F = rk.n_alt;
  for (size_t e = 0; e < n; ++e) {
    const int* v = o + e * (1 + 2 * F);
    const int64_t r = idx[e];
    memcpy(&rk.score[r], v, 4);
    if (F > 0) {
      memcpy(rk.alt_node + r * F, v + 1, (size_t)F * 4);
      memcpy(rk.alt_score + r * F, v + 1 + F, (size_t)F * 4);
    }
  }
}

// Role rows of group g on the direct and the staged plan paths, whose dense role rows start at `row` (step_drow,
// kernels.cuh): one per (wave, role) with a placed replica.  Returns the group's role rows.
int plan_alt_rows(const int32_t* gb, int g, const int32_t* assign, int row, std::vector<AltRow>* out) {
  const int32_t* rec = group_rec(gb, g);
  const int32_t* roles = gb + rec[4];
  int ord0[RBGTOPO_MAX_GROUP_ROLES];
  for (int k = 0, acc = 0; k < rec[3]; ++k) { ord0[k] = acc; acc += roles[4 * k + 1]; }
  const int row0 = row;
  walk_waves(roles, rec[3], nullptr, [&](int, const PlanWave& w) {
    for (int p = 0; p < w.n; ++p, ++row) {
      const int rep0 = rec[8] + ord0[w.role[p]] + w.first[p];
      bool placed = false;
      for (int k = 0; k < w.count[p]; ++k) placed |= assign[rep0 + k] >= 0;
      if (placed && out) out->push_back(AltRow{row, g, w.role[p], rep0, w.count[p]});
    }
  });
  return row - row0;
}

// k_alternates over `list` (rows in `rows`, slab_stride floats apart) on the batch's stream, results scattered into
// rk; synchronises.  Gang-failed groups are skipped.  The caller cleared the outputs of the groups in `list`.
// rp: the (S, C) table of place_groups_lw (§3.12), whose `list` entries and assign indices count pods, or nullptr (one
// pod per replica, no co-location).  used_g sums the demand of every placed pod of the group.  A role with C >= 0
// makes one job per co-location domain D_r its row's placed replicas chose; its unplaced replicas make none.
// cm != nullptr: the rows of a committed batch (§3.14, and §3.15 with rp): every job's room is counted after the whole
// batch (one list `used` of every group's placements), and participating jobs test the owner the batch left on a node
// (k_alternates_commit<cm_levels>, cm->g = n_groups; k_alternates_commit_coloc when a job has a co-location domain).
// hc != nullptr: cm's dhead / dclaim are hc's lists, uploaded with the jobs.
int run_alternates(rbgtopo_ctx* c, Batch* b, const float* rows, const std::vector<AltRow>& list, const int32_t* gb,
                   const int32_t* rp, const int32_t* assign, const int32_t* status, const int32_t* domain,
                   const RankReq& rk, const CommitDev* cm, bool cm_levels, const HostClaims* hc) {
  const int F = rk.n_alt;
  const int ng = gb[2];
  const GroupOffsets off(gb, rp);
  const Topology& T = c->topo;
  std::vector<AltJob> jobs;
  std::vector<int2> used, tmp;
  std::vector<int> own, idx, doms;  // own / idx: node and assign index of every compact replica
  std::vector<int> gids;            // cm: the gid of every job
  std::map<int, int2> placed;  // group -> (first, count) of its aggregated placements in `used`
  bool coloc = false;
  if (cm) {  // (node, amount) per node the whole batch took
    for (int g = 0; g < ng; ++g) {
      if (status[g] == RBGTOPO_GANG_FAILED) continue;
      const int32_t* rec = group_rec(gb, g);
      const int32_t* grp = off.grp(rp, g);
      int64_t i = off.pod0[g];
      for (int q = 0; q < rec[3]; ++q)
        for (int64_t k = 0; k < (int64_t)gb[rec[4] + 4 * q + 1] * (grp ? grp[2 * q] : 1); ++k, ++i)
          if (assign[i] >= 0) tmp.push_back(make_int2(assign[i], gb[rec[4] + 4 * q + 2]));
    }
    std::sort(tmp.begin(), tmp.end(), [](int2 a, int2 b2) { return a.x < b2.x; });
    for (const int2& u : tmp) {
      if (!used.empty() && used.back().x == u.x) used.back().y += u.y;
      else used.push_back(u);
    }
  }
  for (const AltRow& r : list) {
    if (status[r.group] == RBGTOPO_GANG_FAILED) continue;
    const int32_t* rec = group_rec(gb, r.group);
    const int32_t* roles = gb + rec[4];
    const int32_t* grp = off.grp(rp, r.group);
    auto it = cm ? placed.emplace(r.group, make_int2(0, (int)used.size())).first : placed.find(r.group);
    if (it == placed.end()) {  // (node, amount) per node the group's pods of this call took
      tmp.clear();
      int64_t i = off.pod0[r.group];
      for (int q = 0; q < rec[3]; ++q)
        for (int64_t k = 0; k < (int64_t)roles[4 * q + 1] * (grp ? grp[2 * q] : 1); ++k, ++i)
          if (assign[i] >= 0) tmp.push_back(make_int2(assign[i], roles[4 * q + 2]));
      std::sort(tmp.begin(), tmp.end(), [](int2 a, int2 b2) { return a.x < b2.x; });
      const int first = (int)used.size();
      for (const int2& u : tmp) {
        if ((int)used.size() > first && used.back().x == u.x) used.back().y += u.y;
        else used.push_back(u);
      }
      it = placed.emplace(r.group, make_int2(first, (int)used.size() - first)).first;
    }
    const bool part = (rec[1] & RBGTOPO_STEP_EXCLUSIVE) && (roles[4 * r.role + 3] & RBGTOPO_ROLE_EXCLUSIVE);
    const int S = grp ? grp[2 * r.role] : 1, C = grp ? grp[2 * r.role + 1] : -1;
    AltJob j{};
    j.row = r.row;
    j.demand = roles[4 * r.role + 2];
    j.dom = part ? (domain[r.group] >= 0 ? domain[r.group] : -2) : ALT_DOM_ANY;
    j.used0 = it->second.x;
    j.nused = it->second.y;
    j.level = rec[10];
    j.cdom = ALT_DOM_ANY;
    auto add = [&](int p, int cnt) {
      for (int k = 0; k < cnt; ++k) { own.push_back(assign[p + k]); idx.push_back(p + k); }
    };
    if (C < 0) {
      j.rep0 = (int)own.size();
      add(r.rep0, r.nrep);
      j.nrep = (int)own.size() - j.rep0;
      jobs.push_back(j);
      if (cm) gids.push_back(rec[0]);
      continue;
    }
    // D_r = dom_C of the replica's nodes (all S pods lie in it), in the order of first appearance
    const int* dc = C == 0 ? T.h_domain.data() : T.h_lvl_domain.data() + (size_t)(C - 1) * T.n;
    doms.clear();
    for (int p = r.rep0; p < r.rep0 + r.nrep; p += S)
      if (assign[p] >= 0 && std::find(doms.begin(), doms.end(), dc[assign[p]]) == doms.end()) doms.push_back(dc[assign[p]]);
    for (int d : doms) {
      j.cdom = d;
      j.clevel = C;
      j.rep0 = (int)own.size();
      for (int p = r.rep0; p < r.rep0 + r.nrep; p += S)
        if (assign[p] >= 0 && dc[assign[p]] == d) add(p, S);
      j.nrep = (int)own.size() - j.rep0;
      jobs.push_back(j);
      if (cm) gids.push_back(rec[0]);
      coloc = true;
    }
  }
  if (jobs.empty()) return RBGTOPO_OK;
  if (rk.x && rk.x->bounds.empty())
    for (int g = 0; g <= c->cfg.world; ++g) rk.x->bounds.push_back(slab_bound(T.n, c->cfg.world, g));
  const size_t smem = (size_t)((c->topo.n + 31) / 32) * 4;
  if (smem > kFastSmemMax) return fail(RBGTOPO_ELIMIT, "ranked placement: %d nodes exceed the room bitmap", c->topo.n);
  static_assert(sizeof(AltJob) % 4 == 0, "jobs are staged as words");
  const size_t w_jobs = jobs.size() * (sizeof(AltJob) / 4), w_used = used.size() * 2, w_own = own.size();
  // hc: dhead, then dclaim 8-byte aligned, after the gids
  const size_t o_dhead = w_jobs + w_used + w_own + gids.size();
  const size_t o_dclaim = hc ? (o_dhead + hc->dhead.size() + 1) & ~(size_t)1 : o_dhead;
  const size_t w_in = hc ? o_dclaim + 2 * hc->dclaim.size() : o_dhead;
  // rk.x: the slab lists (8-byte aligned) and the replicas' slab scores instead of the replicas' lists
  const size_t o_out = rk.x ? (w_in + 1) & ~(size_t)1 : w_in;
  const size_t w_out = rk.x ? jobs.size() * 2 * ALT_LIST + own.size() : own.size() * (size_t)(1 + 2 * F);
  cudaStream_t s = stream_of(c, b);
  CK(b->alt.reserve(o_out + w_out));
  CK(b->h_alt.reserve(o_out + w_out));
  int* h = b->h_alt.p;
  memcpy(h, jobs.data(), w_jobs * 4);
  memcpy(h + w_jobs, used.data(), w_used * 4);
  memcpy(h + w_jobs + w_used, own.data(), w_own * 4);
  memcpy(h + w_jobs + w_used + w_own, gids.data(), gids.size() * 4);
  if (hc) {
    memcpy(h + o_dhead, hc->dhead.data(), hc->dhead.size() * 4);
    memcpy(h + o_dclaim, hc->dclaim.data(), hc->dclaim.size() * 8);
  }
  int* d = b->alt.p;
  CK(cudaMemcpyAsync(d, h, w_in * 4, cudaMemcpyHostToDevice, s));
  CommitDev cmd = cm ? *cm : CommitDev{};
  if (hc) {
    cmd.dhead = d + o_dhead;
    cmd.dclaim = reinterpret_cast<const int2*>(d + o_dclaim);
  }
  if (rk.x)
    (coloc ? (cm ? (cm_levels ? k_alternates_slab_coloc<true, true> : k_alternates_slab_coloc<true, false>)
                 : k_alternates_slab_coloc<false, false>)
           : cm ? (cm_levels ? k_alternates_slab<true, true> : k_alternates_slab<true, false>)
                : k_alternates_slab<false, false>)
        <<<(unsigned)jobs.size(), ALT_THREADS, (size_t)((c->slab_hi - c->slab_lo + 31) / 32) * 4, s>>>(
        topo_dev(c), rows, reinterpret_cast<const AltJob*>(d), reinterpret_cast<const int2*>(d + w_jobs),
        d + w_jobs + w_used, d + o_out, cmd, d + w_jobs + w_used + w_own);
  else if (cm && coloc)
    (cm_levels ? k_alternates_commit_coloc_lv : k_alternates_commit_coloc)<<<(unsigned)jobs.size(), ALT_THREADS, smem, s>>>(
        topo_dev(c), rows, reinterpret_cast<const AltJob*>(d), reinterpret_cast<const int2*>(d + w_jobs),
        d + w_jobs + w_used, F, d + w_in, cmd, d + w_jobs + w_used + w_own);
  else if (cm)
    (cm_levels ? k_alternates_commit<true> : k_alternates_commit<false>)<<<(unsigned)jobs.size(), ALT_THREADS, smem, s>>>(
        topo_dev(c), rows, reinterpret_cast<const AltJob*>(d), reinterpret_cast<const int2*>(d + w_jobs),
        d + w_jobs + w_used, F, d + w_in, cmd, d + w_jobs + w_used + w_own);
  else
    (coloc ? k_alternates<true> : k_alternates<false>)<<<(unsigned)jobs.size(), ALT_THREADS, smem, s>>>(
        topo_dev(c), rows, reinterpret_cast<const AltJob*>(d), reinterpret_cast<const int2*>(d + w_jobs),
        d + w_jobs + w_used, F, d + w_in);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(h + o_out, d + o_out, w_out * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  const int* o = h + o_out;
  if (rk.x) {  // append the jobs, at the next global job index
    AltExchange& x = *rk.x;
    const int rep0 = (int)x.own.size();
    for (const AltJob& j : jobs) x.job.push_back(make_int2(rep0 + j.rep0, j.nrep));
    x.own.insert(x.own.end(), own.begin(), own.end());
    x.idx.insert(x.idx.end(), idx.begin(), idx.end());
    const auto* k = reinterpret_cast<const unsigned long long*>(o);
    x.keys.insert(x.keys.end(), k, k + jobs.size() * ALT_LIST);
    const auto* rs = reinterpret_cast<const float*>(o + jobs.size() * 2 * ALT_LIST);
    x.rscore.insert(x.rscore.end(), rs, rs + own.size());
    return RBGTOPO_OK;
  }
  alt_scatter(rk, o, idx.data(), idx.size());
  return RBGTOPO_OK;
}

// Ranking after a plan pass (direct or staged path; dense role rows in group order): every group the pass finished.
// The dirty ones are ranked by the host-driven loop that re-runs them.
int rank_plan(rbgtopo_ctx* c, Batch* b, const int32_t* gb, const int32_t* assign, const int32_t* status,
              const int32_t* domain, const std::vector<char>& dirty, const RankReq& rk) {
  std::vector<AltRow> list;
  for (int g = 0, row = 0; g < gb[2]; ++g) {
    if (!dirty[g]) alt_clear(rk, group_rec(gb, g)[8], group_rec(gb, g)[9]);
    row += plan_alt_rows(gb, g, assign, row, dirty[g] ? nullptr : &list);
  }
  return run_alternates(c, b, b->matrix.p, list, gb, nullptr, assign, status, domain, rk);
}

// Builds the plan IN PLACE in b->h_in (pinned); *plan_words = its size.  The GROUPS blob is
// fully validated here (ranges of every user-provided value), so staging may trust the plan.
int build_plan(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int64_t* plan_words, Batch* b) {
  if (const int hrc = check_groups_blob(gb, words)) return hrc;
  const int ng = gb[2];
  auto in = [&](long long off, long long cnt) { return off >= 0 && cnt >= 0 && off + cnt <= words; };
  static const bool prof = getenv("RBGTOPO_PROFILE_HOST") != nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto us = [](auto a, auto b2) { return (long)std::chrono::duration_cast<std::chrono::microseconds>(b2 - a).count(); };
  const auto p0 = now();
  // flat wave table (thread-local scratch keeps its capacity across calls)
  static thread_local std::vector<PlanWave> wv;
  static thread_local std::vector<int> wv_off, step_flat;
  wv_off.assign((size_t)ng + 1, 0);
  b->grp_flags.resize(ng);
  b->grp_fixed.resize(ng);
  b->grp_assign_off.resize(ng);
  b->grp_pending.resize(ng);
#define GROUP_FAIL(code, ...) return report ? fail(code, __VA_ARGS__) : (int)(code)
  int* const g_pend = b->grp_pending.data();
  int* const g_nw = wv_off.data() + 1;  // per-group wave count first, prefix-summed below
  const int n_nodes = c->topo.n, n_domains = c->topo.n_domains;
  auto check_group = [&](int g, bool report) -> int {
    const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS;
    const int q = rec[3];
    if (q < 1 || q > RBGTOPO_MAX_GROUP_ROLES) GROUP_FAIL(RBGTOPO_ELIMIT, "group %d: %d roles", g, q);
    if (!in(rec[4], 4LL * q) || !in(rec[5], (long long)q * q) || !in(rec[7], 3LL * rec[6]))
      GROUP_FAIL(RBGTOPO_EINVAL, "group %d: section out of bounds", g);
    const int32_t* roles = gb + rec[4];
    long long pend = 0;
    for (int i = 0; i < q; ++i) {
      if (roles[4 * i + 1] < 0 || (i && roles[4 * i] < roles[4 * (i - 1)]))
        GROUP_FAIL(RBGTOPO_EINVAL, "group %d role %d: pending < 0 or levels not ascending", g, i);
      if (roles[4 * i + 2] < 0 || roles[4 * i + 2] > RBGTOPO_MAX_FREE)
        GROUP_FAIL(RBGTOPO_EINVAL, "group %d role %d: demand", g, i);
      pend += roles[4 * i + 1];
    }
    if (pend > 0x3FFFFFFFLL) GROUP_FAIL(RBGTOPO_ELIMIT, "group %d: pending replicas", g);
    if (rec[0] < 0 || rec[2] < -1 || (rec[10] == 0 && rec[2] >= n_domains)) GROUP_FAIL(RBGTOPO_EINVAL, "group %d: gid / fixed_domain", g);
    if (const int lc = level_code(rec[10], installed_levels(c), places_levels(c))) GROUP_FAIL(lc, "group %d: exclusive level %d", g, rec[10]);
    if (rec[2] >= level_domains(c->topo, rec[10])) GROUP_FAIL(RBGTOPO_EINVAL, "group %d: fixed_domain %d (level %d)", g, rec[2], rec[10]);
    if (rec[1] & ~(RBGTOPO_STEP_EXCLUSIVE | RBGTOPO_STEP_GANG)) GROUP_FAIL(RBGTOPO_EINVAL, "group %d: unknown flags 0x%x", g, rec[1]);
    for (int i = 0; i < q; ++i)
      if (roles[4 * i + 3] & ~RBGTOPO_ROLE_EXCLUSIVE) GROUP_FAIL(RBGTOPO_EINVAL, "group %d role %d: unknown role flags", g, i);
    for (int i = 0; i < q * q; ++i)
      if (gb[rec[5] + i] < 0 || gb[rec[5] + i] > kMaxExactTerm) GROUP_FAIL(RBGTOPO_EINVAL, "group %d: pair weight out of [0, 2^24]", g);
    for (int a = 0; a < rec[6]; ++a) {
      const int32_t* an = gb + rec[7] + 3 * a;
      if (an[0] < 0 || an[0] >= n_nodes || an[1] < 0 || an[1] >= q || an[2] < 0 || an[2] > kMaxExactTerm)
        GROUP_FAIL(RBGTOPO_EINVAL, "group %d anchor %d out of range", g, a);
    }
    g_pend[g] = (int)pend;
    g_nw[g] = gen_waves(roles, q, nullptr);
    return RBGTOPO_OK;
  };
#undef GROUP_FAIL
  int first_bad = ng;
#pragma omp parallel for schedule(static) num_threads(kHostThreads) reduction(min : first_bad) if (ng >= 64 && kHostThreads > 1)
  for (int g = 0; g < ng; ++g)
    if (check_group(g, false) != RBGTOPO_OK) first_bad = std::min(first_bad, g);
  if (first_bad < ng) return check_group(first_bad, true);
  size_t W = 0;
  long long pacc = 0;
  for (int g = 0; g < ng; ++g) {  // prefixes
    const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS;
    if (rec[8] != pacc || rec[9] != g_pend[g]) return fail(RBGTOPO_EINVAL, "group %d: bad assign_off/n_pending", g);
    b->grp_flags[g] = rec[1];
    b->grp_fixed[g] = rec[2];
    b->grp_assign_off[g] = (int)pacc;
    pacc += g_pend[g];
    if (pacc > 0x7FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "pending replicas exceed 2^31");
    W = std::max(W, (size_t)g_nw[g]);
    wv_off[g + 1] = wv_off[g] + g_nw[g];
  }
  if (gb[4] != pacc) return fail(RBGTOPO_EINVAL, "total pending mismatch");
  wv.resize((size_t)wv_off[ng]);
  {
    PlanWave* const wout = wv.data();
    const int* const wo = wv_off.data();
#pragma omp parallel for schedule(static) num_threads(kHostThreads) if (ng >= 64 && kHostThreads > 1)
    for (int g = 0; g < ng; ++g) {
      const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS;
      gen_waves(gb + rec[4], rec[3], wout + wo[g]);
    }
  }
  const auto p1 = now();

  // step numbering (wave-major) fused with pass 1 (step order): section sizes -> offsets,
  // replica / role-row prefixes
  const int ns = wv_off[ng];
  step_flat.resize((size_t)ns);
  static thread_local std::vector<int> sec_off, rep_off, row_off, i0_of;
  sec_off.resize((size_t)ns + 1);
  rep_off.resize((size_t)ns + 1);
  row_off.resize((size_t)ns + 1);
  i0_of.assign(ng, 0);
  b->wave_begin.assign(1, 0);
  b->wave_maxp.clear();
  b->step_group.resize((size_t)ns);
  {
    const PlanWave* const wvp0 = wv.data();
    const int* const wo = wv_off.data();
    int* const stf0 = step_flat.data();
    int* const sg = b->step_group.data();
    int* const so = sec_off.data();
    int* const ro = rep_off.data();
    int* const wo2 = row_off.data();
    int* const i0p = i0_of.data();
    long long off = (long long)RBGTOPO_HDR_WORDS + (long long)ns * RBGTOPO_STEP_WORDS;  // multiple of 4
    int s = 0;
    ro[0] = 0;
    wo2[0] = 0;
    for (size_t w = 0; w < W; ++w) {
      int mp = 1;
      for (int g = 0; g < ng; ++g) {
        if (w >= (size_t)(wo[g + 1] - wo[g])) continue;
        const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS;
        const PlanWave& pw = wvp0[wo[g] + w];
        stf0[wo[g] + w] = s;
        sg[s] = g;
        mp = std::max(mp, pw.size());
        int n = 0;
        for (int k = 0; k < pw.size(); ++k) n += pw.count[k];
        const int i0 = i0p[g];
        long long sz = 4LL * pw.size() + (long long)pw.size() * rec[3] + 3LL * (rec[6] + i0) + 2LL * i0;
        sz = (sz + 3) & ~3LL;  // keeps every role section 16-byte aligned
        so[s] = (int)std::min<long long>(off, 0x7FFFFFF0LL);
        off += sz;
        ro[s + 1] = ro[s] + n;
        wo2[s + 1] = wo2[s] + pw.size();
        i0p[g] = i0 + n;
        ++s;
      }
      b->wave_begin.push_back(s);
      b->wave_maxp.push_back(mp);
    }
    if (off > 0x7FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "plan blob exceeds 2^31 words");
    so[ns] = (int)off;
  }
  const auto p2 = now();
  const auto p3 = now();
  {
    const size_t total = (size_t)sec_off[ns] + (size_t)ns + 1 + 64;  // + poff
    CK(b->h_in.reserve(total));  // no clear: pass 2 writes every word of the plan
  }
  int32_t* const out = b->h_in.p;
  const auto p4 = now();
  // pass 2 (group order): fill every step of a group while walking its waves once.  Groups
  // write disjoint regions, so the loop is spread over a few host threads (OpenMP keeps its
  // pool between calls).  thread_local scratch is reached through plain pointers: a worker
  // thread would otherwise see its own (empty) instance.
  const PlanWave* const wvp = wv.data();
  const int* const wvo = wv_off.data();
  const int* const stf = step_flat.data();
  const int* const seco = sec_off.data();
  const int* const repo = rep_off.data();
  const int* const rowo = row_off.data();
  auto nwaves2 = [wvo](int g) { return (size_t)(wvo[g + 1] - wvo[g]); };
  auto wave2 = [wvp, wvo](int g, size_t w) -> const PlanWave& { return wvp[wvo[g] + w]; };
  auto step2 = [stf, wvo](int g, size_t w) { return stf[wvo[g] + w]; };
#pragma omp parallel for schedule(static) num_threads(kHostThreads) if (ng >= 64 && kHostThreads > 1)
  for (int g = 0; g < ng; ++g) {
    const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS;
    const int q = rec[3], na = rec[6];
    const int32_t* roles = gb + rec[4];
    const int32_t* pair = gb + rec[5];
    int placed_before[RBGTOPO_MAX_GROUP_ROLES] = {0};
    int i0 = 0;
    for (size_t w = 0; w < nwaves2(g); ++w) {
      const PlanWave& pw = wave2(g, w);
      const int P = pw.size();
      const int s = step2(g, w);
      int32_t* st = out + RBGTOPO_HDR_WORDS + (size_t)s * RBGTOPO_STEP_WORDS;
      int32_t* p = out + seco[s];
      st[0] = rec[0];
      st[1] = (rec[1] & (RBGTOPO_STEP_EXCLUSIVE | RBGTOPO_STEP_GANG)) | rec[10] << STEP_LEVEL_SHIFT;
      st[2] = (rec[1] & RBGTOPO_STEP_EXCLUSIVE) ? rec[2] : -1;
      st[3] = P;
      st[4] = (int32_t)(p - out);
      int n = 0;
      for (int k = 0; k < P; ++k) {
        const int ri = pw.role[k];
        int need = 0;
        for (int j = 0; j < q; ++j)
          if (pair[ri * q + j] > 0) need += roles[4 * j + 1] - placed_before[j];
        *p++ = pw.count[k];
        *p++ = roles[4 * ri + 2];
        *p++ = std::min(need, RBGTOPO_NEED_CAP);
        *p++ = (roles[4 * ri + 3] & 0xFF) | (ri << 8);
        n += pw.count[k];
      }
      st[5] = q;
      st[6] = (int32_t)(p - out);
      for (int k = 0; k < P; ++k) {
        memcpy(p, pair + pw.role[k] * q, (size_t)q * 4);
        p += q;
      }
      st[7] = na + i0;
      st[8] = (int32_t)(p - out);
      memcpy(p, gb + rec[7], (size_t)na * 12);
      p += 3 * na;
      for (size_t w2 = 0; w2 < w; ++w2)  // one record per replica of the earlier waves, filled on the device
        for (int k = 0; k < wave2(g, w2).size(); ++k)
          for (int r = 0; r < wave2(g, w2).count[k]; ++r) {
            *p++ = 0;
            *p++ = wave2(g, w2).role[k];
            *p++ = 1;  // counted by the exactness bound; the device writes 0 for unplaced replicas
          }
      st[9] = i0;
      st[10] = (int32_t)(p - out);  // consumed records (and the pad) are zero until the device fills them
      for (int32_t* const end = out + seco[s + 1]; p < end;) *p++ = 0;
      st[11] = n;
      st[12] = rec[8] + i0;  // dense row / assign index of the wave's first replica: GROUP order (a group's waves are consecutive)
      st[13] = rowo[s];
      st[14] = (w + 1 < nwaves2(g)) ? step2(g, w + 1) : 0;
      st[15] = i0;
      for (int k = 0; k < P; ++k) placed_before[pw.role[k]] += pw.count[k];
      i0 += n;
    }
  }
  const int racc = rep_off[ns], rowacc = row_off[ns];
  out[0] = RBGTOPO_BLOB_MAGIC;
  out[1] = RBGTOPO_ABI_VERSION;
  out[2] = ns;
  out[3] = sec_off[ns];
  out[4] = racc;
  out[5] = rowacc;
  out[6] = out[7] = 0;
  *plan_words = sec_off[ns];
  if (prof)
    fprintf(stderr, "[rbgtopo plan] validate+waves %ld us, numbering %ld us, offsets %ld us, clear %ld us, fill %ld us\n",
            us(p0, p1), us(p1, p2), us(p2, p3), us(p3, p4), us(p4, now()));
  return RBGTOPO_OK;
}

// Device-expanded plan: validates the GROUPS blob, computes the per-step GEOMETRY on the host
// (numbering, section offsets, prefixes, patch capacities, exactness bound, emit work split),
// uploads GROUPS blob + geometry and lets k_expand_plan (plan.cuh) write the step blob in HBM.
// Equivalent to build_plan + stage_into, without the step blob ever existing on the host.
// Caller holds topo_mu shared.
// [g_lo, g_hi): the groups of this batch (place_groups pipelines two halves of a large fleet);
// pacc0 = pending replicas of the groups before g_lo; dev_groups = device copy of the GROUPS blob
// uploaded by an earlier batch of the same call (then only the geometry is uploaded), or nullptr.
// What the plan geometry needs to know about the snapshot (host side only).
struct TopoHost {
  int n = 0, n_domains = 0;
  int n_levels = -1;  // exclusive levels installed (occupancy mode, 0 outside it); -1: unknown (the describe calls)
  bool place_levels = false;      // levels >= 1 are placed (level_code)
  const int* level_nd = nullptr;  // [n_levels + 1] domain counts of the installed levels, or nullptr (describe calls)
  const int* degp1 = nullptr;  // [n] deg + 1, or nullptr = all 1
  int max_degp1 = 1;
  long long wsum_max = 0;
  long long row_w = RBGTOPO_SELF_W, amax_limit = 0;  // the §3.4 bound: exact while amax * row_w < 2^24, i.e. amax < amax_limit
  void set_wsum(long long w) {
    wsum_max = w;
    row_w = w + RBGTOPO_SELF_W;
    amax_limit = ((1LL << 24) + row_w - 1) / row_w;
  }
};
// The snapshot's; levels >= 1 are placed when place_levels.
TopoHost topo_host(const rbgtopo_ctx* c, bool place_levels) {
  const Topology& T = c->topo;
  TopoHost th;
  th.n = T.n;
  th.n_domains = T.n_domains;
  th.n_levels = installed_levels(c);
  th.place_levels = place_levels;
  th.level_nd = T.lvl_nd.empty() ? nullptr : T.lvl_nd.data();
  th.degp1 = T.h_degp1.data();
  th.max_degp1 = T.max_degp1;
  th.set_wsum(T.wsum_max);
  return th;
}
// The arguments of the describe calls (exclusive levels unknown).
int topo_host_args(int32_t n_nodes, int32_t n_domains, const int32_t* deg_plus1, int64_t wsum_max, TopoHost* th) {
  th->n = n_nodes;
  th->n_domains = n_domains;
  th->degp1 = deg_plus1;
  th->max_degp1 = 1;
  if (deg_plus1)
    for (int i = 0; i < n_nodes; ++i) {
      if (deg_plus1[i] < 1) return fail(RBGTOPO_EINVAL, "deg_plus1[%d]", i);
      th->max_degp1 = std::max(th->max_degp1, deg_plus1[i]);
    }
  th->set_wsum(wsum_max);
  return RBGTOPO_OK;
}
// Fleets are made of a few role templates (an RBGSet fans ONE RoleBasedGroup out into N, rolebasedgroupset_controller.go:69-207):
// what the plan geometry derives from a group's role table and pair matrix alone — validity, pending replicas, the
// wave structure, per-wave sizes and the shape part of the exactness bound — is computed once per run of identical
// shapes (per host thread) and re-used; only the anchor-dependent terms are per group.  Shapes with more than
// kShapeWaves waves are not cached.
constexpr int kShapeWaves = 16;
struct ShapeCache {
  bool valid = false;
  int q = 0, nw = 0, rr = 0;  // rr: role rows of all waves
  long long pend = 0;
  int32_t roles[4 * RBGTOPO_MAX_GROUP_ROLES];
  int32_t pair[RBGTOPO_MAX_GROUP_ROLES * RBGTOPO_MAX_GROUP_ROLES];
  // per wave (size_group)
  bool sized = false;
  int P[kShapeWaves], n[kShapeWaves], i0[kShapeWaves];
  int role[kShapeWaves][RBGTOPO_MAX_STEP_ROLES];
  long long bound[kShapeWaves][RBGTOPO_MAX_STEP_ROLES];  // sum_j pair[ri][j] * placed[j] + min(need, cap) * F (saturated)
  bool match(const int32_t* r, const int32_t* p, int qq) const {
    return valid && qq == q && memcmp(r, roles, (size_t)16 * qq) == 0 && memcmp(p, pair, (size_t)4 * qq * qq) == 0;
  }
  void set(const int32_t* r, const int32_t* p, int qq) {
    q = qq;
    memcpy(roles, r, (size_t)16 * qq);
    memcpy(pair, p, (size_t)4 * qq * qq);
    valid = true;
    sized = false;
  }
};

// A few shapes per thread (fleets interleave a handful of templates), round-robin replacement.
struct ShapeCaches {
  static constexpr int kWays = 4;
  ShapeCache way[kWays];
  int next = 0;
  ShapeCache* find(const int32_t* r, const int32_t* p, int q) {
    for (int i = 0; i < kWays; ++i)
      if (way[i].match(r, p, q)) return &way[i];
    return nullptr;
  }
  ShapeCache* victim() {
    ShapeCache* v = &way[next];
    next = (next + 1) % kWays;
    return v;
  }
};

// staging layout of one plan: GROUPS blob | pad | (group, wave, group's first dense role row) per step | geometry (8 ints
// per step) | poff
struct PlanLayout {
  size_t sgw_off = 0, aux_off = 0, tail_off = 0, tail_words = 0, src_words = 0;
  long long plan_words = 0, racc = 0, rowacc = 0;  // rowacc: role rows = dense rows
  int ns = 0;
};
// Called by plan_geometry once the step numbering exists (ns, racc = replicas of the batch, the
// (group, wave) table in the staging buffer): plan_stage uploads the first part and starts the device on
// the row tables / the dense matrix while the host goes on with section sizes and prefixes.
using PlanMidHook = std::function<int(const PlanLayout&)>;

// Pure host part of plan_stage (no CUDA call when b->h_in is pageable): validates the groups of
// [g_lo, g_hi), fills the batch's wave tables, b->m and the staging buffer b->h_in.
int plan_geometry(const TopoHost& T, int lc, Batch* b, const int32_t* gb, int64_t words, int g_lo, int g_hi,
                  long long pacc0, bool with_blob, PlanLayout* L, const PlanMidHook& mid = nullptr) {
  b->perm_n = 0;
  if (const int hrc = check_groups_blob(gb, words)) return hrc;
  const int ng_all = gb[2];
  if (g_hi < 0) g_hi = ng_all;
  if (g_lo < 0 || g_lo > g_hi || g_hi > ng_all) return fail(RBGTOPO_EINVAL, "internal: group range");
  const int ng = g_hi - g_lo;  // below, g is the index inside the range; blob records are g_lo + g
  b->g_lo = g_lo;
  if (words > 0x3FFFFFFFLL) return fail(RBGTOPO_ELIMIT, "groups blob too large");
  auto in = [&](long long off, long long cnt) { return off >= 0 && cnt >= 0 && off + cnt <= words; };
  static const bool prof = getenv("RBGTOPO_PROFILE_HOST") != nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto us = [](auto t0, auto t1) { return (long)std::chrono::duration_cast<std::chrono::microseconds>(t1 - t0).count(); };
  const auto p0 = now();
  static thread_local std::vector<int> wv_off, g_pc, g_first, ctr, g_rr;
  wv_off.assign((size_t)ng + 1, 0);
  g_pc.resize((size_t)ng);
  g_rr.resize((size_t)ng);
  g_first.resize((size_t)ng);
  b->grp_flags.resize(ng);
  b->grp_fixed.resize(ng);
  b->grp_assign_off.resize(ng);
  b->grp_pending.resize(ng);
  int* const g_pend = b->grp_pending.data();
  int* const g_nw = wv_off.data() + 1;  // per-group wave count first, prefix-summed below
  int* const g_pcp = g_pc.data();
  const int n_nodes = T.n, n_domains = T.n_domains;
  const int* const degp1 = T.degp1;
  int* const g_rrp = g_rr.data();
#define GROUP_FAIL(code, ...) return report ? fail(code, __VA_ARGS__) : (int)(code)
  // everything about group g that does not depend on the groups before it
  auto check_group = [&](int g, bool report) -> int {
    const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)(g_lo + g) * RBGTOPO_GROUP_WORDS;
    const int q = rec[3];
    if (q < 1 || q > RBGTOPO_MAX_GROUP_ROLES) GROUP_FAIL(RBGTOPO_ELIMIT, "group %d: %d roles", g, q);
    if (!in(rec[4], 4LL * q) || !in(rec[5], (long long)q * q) || !in(rec[7], 3LL * rec[6]))
      GROUP_FAIL(RBGTOPO_EINVAL, "group %d: section out of bounds", g);
    const int32_t* roles = gb + rec[4];
    static thread_local ShapeCaches sc_chk;  // the last shapes this thread validated
    long long pend = 0;
    int nw_g = 0, rr_g = 0;
    const ShapeCache* hit = report ? nullptr : sc_chk.find(roles, gb + rec[5], q);
    if (hit) {  // same role table and pair matrix as an earlier group: valid, known
      pend = hit->pend;
      nw_g = hit->nw;
      rr_g = hit->rr;
    } else {
      for (int i = 0; i < q; ++i) {
        if (roles[4 * i + 1] < 0 || (i && roles[4 * i] < roles[4 * (i - 1)]))
          GROUP_FAIL(RBGTOPO_EINVAL, "group %d role %d: pending < 0 or levels not ascending", g, i);
        if (roles[4 * i + 2] < 0 || roles[4 * i + 2] > RBGTOPO_MAX_FREE)
          GROUP_FAIL(RBGTOPO_EINVAL, "group %d role %d: demand", g, i);
        pend += roles[4 * i + 1];
      }
      if (pend > 0x3FFFFFFFLL) GROUP_FAIL(RBGTOPO_ELIMIT, "group %d: pending replicas", g);
      for (int i = 0; i < q; ++i)
        if (roles[4 * i + 3] & ~RBGTOPO_ROLE_EXCLUSIVE) GROUP_FAIL(RBGTOPO_EINVAL, "group %d role %d: unknown role flags", g, i);
      for (int i = 0; i < q * q; ++i)
        if (gb[rec[5] + i] < 0 || gb[rec[5] + i] > kMaxExactTerm) GROUP_FAIL(RBGTOPO_EINVAL, "group %d: pair weight out of [0, 2^24]", g);
      nw_g = walk_waves(roles, q, nullptr, [&](int, const PlanWave& w) { rr_g += w.n; });
      ShapeCache* v = sc_chk.victim();
      v->set(roles, gb + rec[5], q);
      v->pend = pend;
      v->nw = nw_g;
      v->rr = rr_g;
    }
    if (rec[0] < 0 || rec[2] < -1 || (rec[10] == 0 && rec[2] >= n_domains)) GROUP_FAIL(RBGTOPO_EINVAL, "group %d: gid / fixed_domain", g);
    if (const int lc = level_code(rec[10], T.n_levels, T.place_levels))
      GROUP_FAIL(lc, "group %d: exclusive level %d (%d installed%s)", g, rec[10], std::max(0, T.n_levels),
                 T.place_levels ? "" : "; placement at level 0 only");
    if (rec[10] > 0 && T.level_nd && rec[2] >= T.level_nd[rec[10]])
      GROUP_FAIL(RBGTOPO_EINVAL, "group %d: fixed_domain %d outside the %d domains of level %d", g, rec[2], T.level_nd[rec[10]], rec[10]);
    if (rec[1] & ~(RBGTOPO_STEP_EXCLUSIVE | RBGTOPO_STEP_GANG)) GROUP_FAIL(RBGTOPO_EINVAL, "group %d: unknown flags 0x%x", g, rec[1]);
    long long pc = 0;  // closed neighbourhoods of the scheduled pods
    for (int a = 0; a < rec[6]; ++a) {
      const int32_t* an = gb + rec[7] + 3 * a;
      if (an[0] < 0 || an[0] >= n_nodes || an[1] < 0 || an[1] >= q || an[2] < 0 || an[2] > kMaxExactTerm)
        GROUP_FAIL(RBGTOPO_EINVAL, "group %d anchor %d out of range", g, a);
      pc += degp1 ? degp1[an[0]] : 1;
    }
    if (pc > 0x3FFFFFFFLL) GROUP_FAIL(RBGTOPO_ELIMIT, "group %d: patch list exceeds 2^30 entries", g);
    g_pend[g] = (int)pend;
    g_pcp[g] = (int)pc;
    g_nw[g] = nw_g;
    g_rrp[g] = rr_g;
    return RBGTOPO_OK;
  };
  int first_bad = ng;
#pragma omp parallel for schedule(static) num_threads(kHostThreads) reduction(min : first_bad) if (ng >= kHostParallelMinGroups && kHostThreads > 1)
  for (int g = 0; g < ng; ++g)
    if (check_group(g, false) != RBGTOPO_OK) first_bad = std::min(first_bad, g);
  if (first_bad < ng) return check_group(first_bad, true);

  const auto p1 = now();
  // prefixes over groups, wave sizes, step numbering (wave-major)
  BatchMeta& m = b->m;
  m = BatchMeta{};
  int W = 0;
  long long pacc = pacc0, rracc = 0;
  for (int g = 0; g < ng; ++g) {
    const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)(g_lo + g) * RBGTOPO_GROUP_WORDS;
    if (rec[8] != pacc || rec[9] != g_pend[g]) return fail(RBGTOPO_EINVAL, "group %d: bad assign_off/n_pending", g);
    b->grp_flags[g] = rec[1];
    b->grp_fixed[g] = rec[2];
    b->grp_assign_off[g] = (int)pacc;
    pacc += g_pend[g];
    if (pacc > 0x3FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "pending replicas exceed 2^30");
    const int rr_g = g_rr[g];
    g_rr[g] = (int)rracc;  // now: the group's first dense role row in this batch
    rracc += rr_g;
    if ((rec[1] & RBGTOPO_STEP_EXCLUSIVE) && rec[2] < 0 && g_nw[g] > 0) m.any_excl_unknown = true;
    if (g_nw[g] > 0) m.max_q = std::max(m.max_q, rec[3]);
    if (g_nw[g] > 0 && rec[10] != 0) m.any_level = true;
    W = std::max(W, g_nw[g]);
    wv_off[g + 1] = wv_off[g] + g_nw[g];
    if (wv_off[g + 1] > 0x03FFFFFF) return fail(RBGTOPO_ELIMIT, "plan has more than 2^26 steps");
  }
  if (g_hi == ng_all && gb[4] != pacc) return fail(RBGTOPO_EINVAL, "total pending mismatch");
  const int ns = wv_off[ng];
  const int* const wvo = wv_off.data();  // g_nw[] now holds prefixes: wave count of g = wvo[g + 1] - wvo[g]
  b->wave_begin.assign((size_t)W + 1, 0);
  b->wave_maxp.assign((size_t)W, 1);
  for (int g = 0; g < ng; ++g)  // [k] = groups with exactly k waves (k >= 1)
    if (wvo[g + 1] > wvo[g]) b->wave_begin[wvo[g + 1] - wvo[g]] += 1;
  {
    // steps in wave w = groups with > w waves = sum_{k > w} exact[k]
    int more = 0;
    std::vector<int>& wb = b->wave_begin;
    static thread_local std::vector<int> cnt;
    cnt.assign((size_t)W + 1, 0);
    for (int k = W; k >= 1; --k) { more += wb[k]; cnt[k - 1] = more; }
    wb[0] = 0;
    for (int w = 0; w < W; ++w) wb[w + 1] = wb[w] + cnt[w];
  }
  // staging layout: GROUPS blob | pad | (group, wave, first dense role row of the group) per step | geometry (8 ints per
  // step) | poff
  const size_t sgw_off = with_blob ? (((size_t)words + 3) & ~(size_t)3) : 0;  // without: the blob is already on the device
  const size_t aux_off = sgw_off + (((size_t)3 * ns + 3) & ~(size_t)3);
  const size_t tail_off = aux_off + (size_t)ns * PLAN_AUX_WORDS;
  // tail: poff[ns + 1], then the launch order of k_plan_group (one entry per group with pending replicas)
  const int n0_groups = (int)(W > 0 ? b->wave_begin[1] : 0);
  const size_t tail_words = (size_t)ns + 1 + (size_t)n0_groups;
  const size_t src_words = tail_off + tail_words;
  if (src_words > 0x7FFFFFF0ULL) return fail(RBGTOPO_ELIMIT, "plan staging exceeds 2^31 words");
  if (b->prestaged_h && src_words > b->h_in.cap) CK(cudaDeviceSynchronize());  // the pre-validation upload reads the buffer about to be replaced
  CK(b->h_in.reserve(src_words));
  int32_t* const hin = b->h_in.p;
  int32_t* const aux = hin + aux_off;
  int32_t* const sgw = hin + sgw_off;
  b->step_group.resize((size_t)ns);
  {
    ctr.assign((size_t)W, 0);
    int* const sg = b->step_group.data();
    const int* const wb = b->wave_begin.data();
    for (int g = 0; g < ng; ++g) {
      int prev = -1;
      for (int w = 0; w < wvo[g + 1] - wvo[g]; ++w) {
        const int s = wb[w] + ctr[w]++;
        if (w == 0) g_first[g] = s;
        sg[s] = g;
        sgw[3 * (size_t)s] = g_lo + g;
        sgw[3 * (size_t)s + 1] = w;
        sgw[3 * (size_t)s + 2] = g_rr[g];
        aux[(size_t)s * PLAN_AUX_WORDS + 0] = g_lo + g;
        aux[(size_t)s * PLAN_AUX_WORDS + 1] = w;
        aux[(size_t)s * PLAN_AUX_WORDS + 6] = 0;
        if (prev >= 0) aux[(size_t)prev * PLAN_AUX_WORDS + 6] = s;  // next step of the group
        prev = s;
      }
    }
  }
  if (with_blob) {  // the caller's blob into the pinned staging (the hook uploads it) — unless plan_stage did both already
    if (b->prestaged_h != hin || b->prestaged_hcap != b->h_in.cap) {
      b->prestaged_h = nullptr;
      memcpy(hin, gb, (size_t)words * 4);
    }
    for (size_t i = (size_t)words; i < sgw_off; ++i) hin[i] = 0;
  }
  for (size_t i = sgw_off + 3 * (size_t)ns; i < aux_off; ++i) hin[i] = 0;
  L->sgw_off = sgw_off;
  L->aux_off = aux_off;
  L->tail_off = tail_off;
  L->tail_words = tail_words;
  L->src_words = src_words;
  L->racc = pacc - pacc0;
  L->rowacc = rracc;
  L->ns = ns;
  if (mid) {
    const int mrc = mid(*L);
    if (mrc) return mrc;
  }
  const auto p2 = now();
  // per-step sizes, patch capacity, exactness bound (per group, all its waves)
  const long long row_w = T.row_w, amax_limit = T.amax_limit;
  const int max_degp1 = T.max_degp1;
  const int* const first_of = g_first.data();
  auto size_group = [&](int g, bool report) -> int {
    const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)(g_lo + g) * RBGTOPO_GROUP_WORDS;
    const int q = rec[3], na = rec[6];
    const int32_t* roles = gb + rec[4];
    const int32_t* pair = gb + rec[5];
    long long anch_w[RBGTOPO_MAX_GROUP_ROLES];  // sum over scheduled pods of pair[ri][role]·count
    const long long sat = 1LL << 40;  // far above any admissible bound, far below overflow
    for (int ri = 0; ri < q; ++ri) {
      long long acc = 0;
      for (int a = 0; a < na && acc < sat; ++a) acc += (long long)pair[ri * q + gb[rec[7] + 3 * a + 1]] * gb[rec[7] + 3 * a + 2];
      anch_w[ri] = std::min(acc, sat);
    }
    // one step of the group: the exactness bound (anchor term of THIS group + the shape's term), sizes, capacity
    int s = -1, rc = RBGTOPO_OK;
    auto step_of = [&](int w, int P, int n, int i0, const int* role_of, const long long* bound) {
      s = (w == 0) ? first_of[g] : aux[(size_t)s * PLAN_AUX_WORDS + 6];  // follow the `next` links from the group's first step
      for (int k = 0; k < P; ++k) {
        const long long amax = std::min(anch_w[role_of[k]] + bound[k], sat);
        if (amax >= amax_limit) {
          rc = report ? fail(RBGTOPO_EINEXACT, "group %d wave %d role %d: max score bound >= 2^24 (anchor weight %lld x row weight %lld)", g, w, role_of[k], amax, row_w)
                      : (int)RBGTOPO_EINEXACT;
          return;
        }
      }
      long long sz = 4LL * P + (long long)P * q + 3LL * (na + i0) + 2LL * i0;
      sz = (sz + 3) & ~3LL;  // keeps every role section 16-byte aligned
      const long long pc = (long long)i0 + g_pcp[g] + (long long)i0 * max_degp1;
      if (sz > 0x3FFFFFFFLL || pc > 0x3FFFFFFFLL) {
        rc = report ? fail(RBGTOPO_ELIMIT, "group %d wave %d: step too large", g, w) : (int)RBGTOPO_ELIMIT;
        return;
      }
      int32_t* a = aux + (size_t)s * PLAN_AUX_WORDS;
      a[2] = (int)sz;  // -> sec_off
      a[3] = (int)pc;  // -> sec_end (after the prefix pass took the capacity)
      a[4] = n;        // -> rep_off
      a[5] = P;        // -> row_off
      a[7] = i0;
    };
    static thread_local ShapeCaches sc_szs;  // the last shapes this thread sized
    if (const ShapeCache* hit = report ? nullptr : sc_szs.find(roles, pair, q)) {
      if (hit->sized) {
        for (int w = 0; w < hit->nw && !rc; ++w) step_of(w, hit->P[w], hit->n[w], hit->i0[w], hit->role[w], hit->bound[w]);
        return rc;
      }
    }
    ShapeCache& sc_sz = *sc_szs.victim();
    sc_sz.set(roles, pair, q);
    bool cacheable = true;
    int placed[RBGTOPO_MAX_GROUP_ROLES] = {0};
    int i0 = 0;
    const int nw = walk_waves(roles, q, nullptr, [&](int w, const PlanWave& pw) {
      if (rc) return;
      const int P = pw.size();
      int n = 0;
      long long bound[RBGTOPO_MAX_STEP_ROLES];
      for (int k = 0; k < P; ++k) {
        const int ri = pw.role[k];
        int need = 0;
        long long bnd = 0;
        for (int j = 0; j < q; ++j) {
          if (pair[ri * q + j] > 0) need = (int)std::min<long long>((long long)need + roles[4 * j + 1] - placed[j], 1 << 30);
          bnd = std::min(bnd + (long long)pair[ri * q + j] * placed[j], sat);  // each term < 2^24 * 2^30
        }
        bound[k] = bnd + (long long)std::min(need, RBGTOPO_NEED_CAP) * RBGTOPO_F_CAP;
        n += pw.count[k];
      }
      step_of(w, P, n, i0, pw.role, bound);
      if (w < kShapeWaves) {
        sc_sz.P[w] = P;
        sc_sz.n[w] = n;
        sc_sz.i0[w] = i0;
        for (int k = 0; k < P; ++k) { sc_sz.role[w][k] = pw.role[k]; sc_sz.bound[w][k] = bound[k]; }
      } else {
        cacheable = false;
      }
      for (int k = 0; k < P; ++k) placed[pw.role[k]] += pw.count[k];
      i0 += n;
    });
    sc_sz.nw = nw;
    sc_sz.sized = cacheable && rc == RBGTOPO_OK && !report;
    return rc;
  };
  first_bad = ng;
#pragma omp parallel for schedule(static) num_threads(kHostThreads) reduction(min : first_bad) if (ng >= kHostParallelMinGroups && kHostThreads > 1)
  for (int g = 0; g < ng; ++g)
    if (size_group(g, false) != RBGTOPO_OK) first_bad = std::min(first_bad, g);
  if (first_bad < ng) return size_group(first_bad, true);

  const auto p3 = now();
  // prefixes over steps
  int32_t* const poff = hin + tail_off;
  b->step_row.resize((size_t)ns + 1);
  long long off = (long long)RBGTOPO_HDR_WORDS + (long long)ns * RBGTOPO_STEP_WORDS;  // multiple of 4
  long long racc = 0, rowacc = 0;
  poff[0] = 0;
  {
    int w = 0;
    for (int s = 0; s < ns; ++s) {
      while (s >= b->wave_begin[w + 1]) ++w;
      int32_t* a = aux + (size_t)s * PLAN_AUX_WORDS;
      const int sz = a[2], pc = a[3], n = a[4], P = a[5];
      if (off + sz > 0x7FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "plan blob exceeds 2^31 words");
      if (m.patch_cap + pc > 0x7FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "patch lists exceed 2^31 entries");
      a[2] = (int)off;
      off += sz;
      a[3] = (int)off;
      // dense-matrix row / assign index of the step's first replica: GROUP order (the group's offset in the
      // batch + the replicas of its earlier waves), so results need no reordering and the rows of a step
      // are known without any prefix over steps
      a[4] = b->grp_assign_off[b->step_group[s]] - (int)pacc0 + a[7];
      a[5] = (int)rowacc;
      b->step_row[s] = (int)rowacc;
      racc += n;
      rowacc += P;
      m.patch_cap += pc;
      m.max_cap = std::max(m.max_cap, pc);
      poff[s + 1] = (int)m.patch_cap;
      m.max_p = std::max(m.max_p, P);
      m.max_k = std::max(m.max_k, n);
      b->wave_maxp[w] = std::max(b->wave_maxp[w], P);
    }
    b->step_row[ns] = (int)rowacc;
  }
  // Launch order of k_plan_group: when the grid fits in one round (8 CTAs per SM on cfg3 and cfg4 — group_smem_bytes;
  // rbgtopo_plan_occupancy reports it) its CTAs all start at once and each stays on the SM it started on for the whole
  // kernel; in group order a fleet whose heavy groups recur with a period that divides the SM count (the bench fleet: every 4th group has
  // 3 scheduled pods, 132 = 4 * 33) piles the heavy groups onto the same SMs and the slowest SM sets the kernel
  // time.  Groups are dealt in descending order of their expected table size
  // (neighbourhoods of the scheduled pods + of the replicas to place): every SM gets one group of every weight stratum.
  {
    int32_t* const perm = poff + ns + 1;
    const int nb = 1024;
    static thread_local std::vector<int> bucket, wkey;
    bucket.assign(nb + 1, 0);
    wkey.resize((size_t)n0_groups);
    long long wmax = 1;
    for (int s0 = 0; s0 < n0_groups; ++s0) {
      const int g = b->step_group[s0];
      const long long w = (long long)g_pcp[g] + (long long)g_pend[g] * max_degp1;
      wmax = std::max(wmax, w);
    }
    for (int s0 = 0; s0 < n0_groups; ++s0) {
      const int g = b->step_group[s0];
      const long long w = (long long)g_pcp[g] + (long long)g_pend[g] * max_degp1;
      const int k = (nb - 1) - (int)(w * (nb - 1) / wmax);  // heaviest first
      wkey[s0] = k;
      bucket[k + 1] += 1;
    }
    for (int k = 0; k < nb; ++k) bucket[k + 1] += bucket[k];
    for (int s0 = 0; s0 < n0_groups; ++s0) perm[bucket[wkey[s0]]++] = s0;  // stable: equal weights keep group order
    b->perm_n = n0_groups;
  }
  const long long plan_words = off;
  if (emit_items(ns, lc) > 0x7FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "steps x chunks exceed 2^31 work items");
  m.poff.assign(poff, poff + ns + 1);
  const auto p4 = now();
  m.n_steps = ns;
  m.total_r = (int)racc;
  m.total_p = (int)rowacc;
  m.words = plan_words;
  m.h2d_words = (long long)src_words;
  b->aux_off = (long long)aux_off;
  L->aux_off = aux_off;
  L->tail_off = tail_off;
  L->tail_words = tail_words;
  L->src_words = src_words;
  L->plan_words = plan_words;
  L->racc = racc;
  L->rowacc = rowacc;
  L->ns = ns;
  if (prof)
    fprintf(stderr, "[rbgtopo plan] check %ld us, numbering %ld us, sizes %ld us, prefixes %ld us, copy %ld us\n",
            us(p0, p1), us(p1, p2), us(p2, p3), us(p3, p4), us(p4, now()));
  return RBGTOPO_OK;
}

// early_emit: also launch the dense-matrix kernel of the FIRST pass from inside the staging (host-buffer
// entry point: one pass follows at once); run_batch then skips that launch.
int plan_stage(rbgtopo_ctx* c, Batch* b, const int32_t* gb, int64_t words, bool early_emit = false, int g_lo = 0, int g_hi = -1,
               long long pacc0 = 0, const int* dev_groups = nullptr, cudaEvent_t dev_groups_ready = nullptr) {
  NvtxRange nv("rbgtopo:plan_stage");
  if (!c->topo.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
  const TopoHost th = topo_host(c, places_levels(c));
  PlanLayout L;
  cudaStream_t s = stream_of(c, b);
  // Runs inside plan_geometry as soon as the step numbering exists: first upload (GROUPS blob + the
  // (group, wave, row) table), row tables on the device and — for the host-buffer entry point — the dense
  // matrix launch itself, which then overlaps the host's section sizes / prefixes / second upload.
  auto mid = [&](const PlanLayout& P) -> int {
    CK(b->gsrc.reserve(P.src_words));
    CK(b->matrix.reserve((size_t)std::max<long long>(1, P.rowacc) * c->slab_stride));
    CK(b->rtab.reserve((size_t)std::max<long long>(1, P.rowacc)));
    CK(b->drow.reserve((size_t)std::max(1, P.ns)));
    CK(b->rowmap.reserve((size_t)std::max<long long>(1, P.racc)));
    b->any_excl = false;
    for (int gf : b->grp_flags) b->any_excl |= (gf & RBGTOPO_STEP_EXCLUSIVE) != 0;
    b->epoch = c->topo_epoch;
    b->lvl_epoch = c->lvl_epoch;
    b->tev = timing_events(c);
    if (b->tev) CK(cudaEventRecord(b->ev[0], s));  // staging touches the batch's own buffers only: no wait for a pending snapshot refresh
    const bool pre = b->prestaged_h && b->prestaged_h == b->h_in.p && b->prestaged_hcap == b->h_in.cap &&
                     b->prestaged_d == b->gsrc.p && b->prestaged_dcap == b->gsrc.cap;  // both buffers stayed put
    // blob (unless an earlier batch, or the pre-validation upload, brought it) + (group, wave) table
    const size_t lo = dev_groups ? P.sgw_off : (pre ? (size_t)words : 0), hi = P.aux_off;
    if (hi > lo) CK(cudaMemcpyAsync(b->gsrc.p + lo, b->h_in.p + lo, (hi - lo) * 4, cudaMemcpyHostToDevice, s));
    if (dev_groups && dev_groups_ready) CK(cudaStreamWaitEvent(s, dev_groups_ready, 0));
    if (P.ns > 0) {
      k_plan_etab<<<(P.ns + PLAN_WARPS - 1) / PLAN_WARPS, 32 * PLAN_WARPS, 0, s>>>(dev_groups ? dev_groups : b->gsrc.p, b->gsrc.p + P.sgw_off, P.ns,
                                                                                 (int)pacc0, b->drow.p, b->rtab.p, b->rowmap.p);
      CK(cudaGetLastError());
      b->pend_launches += 1;
      CK(cudaEventRecord(b->ev[2], s));  // GROUPS blob + row tables are on the device: the second half of the staging may follow on stream2
      if (early_emit) {  // pass 0 of run_batch starts here
        int erc = b->tev ? ensure_pass_events(b, b->passes + 1) : RBGTOPO_OK;
        if (erc) return erc;
        CK(cudaStreamWaitEvent(s, c->base_ready, 0));  // base / free / node_owner of a pending refresh
        if (b->tev) CK(cudaEventRecord(b->it_ev[3 * b->passes], s));
        erc = launch_emit_plan(c, b, s, P.rowacc);
        if (erc) return erc;
        if (b->tev) CK(cudaEventRecord(b->it_ev[3 * b->passes + 1], s));
        CK(cudaGetLastError());
        b->early_emit = true;
      }
    }
    return RBGTOPO_OK;
  };
  b->early_emit = false;
  // The upload of the GROUPS blob does not wait for its validation: its PCIe time hides under the host's check + numbering
  b->prestaged_h = nullptr;
  b->prestaged_d = nullptr;
  if (early_emit && !dev_groups && g_lo == 0 && words >= RBGTOPO_HDR_WORDS && !b->h_in.pageable && (size_t)words <= b->h_in.cap &&
      (size_t)words <= b->gsrc.cap) {
    memcpy(b->h_in.p, gb, (size_t)words * 4);
    CK(cudaMemcpyAsync(b->gsrc.p, b->h_in.p, (size_t)words * 4, cudaMemcpyHostToDevice, s));
    b->prestaged_h = b->h_in.p;
    b->prestaged_d = b->gsrc.p;
    b->prestaged_hcap = b->h_in.cap;
    b->prestaged_dcap = b->gsrc.cap;
  }
  int rc = plan_geometry(th, c->lc, b, gb, words, g_lo, g_hi, pacc0, dev_groups == nullptr, &L, mid);
  b->prestaged_h = nullptr;
  b->prestaged_d = nullptr;
  if (rc) return rc;
  BatchMeta& m = b->m;
  const long long slab = c->slab_hi - c->slab_lo;
  m.scores = L.racc * slab;
  m.algo_bytes = 4LL * L.rowacc * slab + 4LL * L.plan_words + 8LL * slab;  // as validate_blob
  const size_t aux_off = L.aux_off, tail_off = L.tail_off, tail_words = L.tail_words, src_words = L.src_words;
  const long long plan_words = L.plan_words, racc = L.racc, rowacc = L.rowacc;
  const int ns = L.ns;
  int32_t* const hin = b->h_in.p;
  CK(b->blob.reserve((size_t)plan_words + tail_words));
  rc = reserve_batch_buffers(c, b);
  if (rc) return rc;
  // second half of the staging: geometry + poff up, plan expanded.  With an early emit in flight on s it goes to
  // stream2 (it needs only the first upload), so the plan is ready when the dense-matrix kernel ends instead of
  // 20+ us later; s joins before anything reads the plan.
  cudaStream_t s_exp = (b->early_emit && ns > 0) ? b->stream2 : s;
  if (s_exp != s) CK(cudaStreamWaitEvent(s_exp, b->ev[2], 0));
  CK(cudaMemcpyAsync(b->gsrc.p + aux_off, hin + aux_off, (src_words - aux_off) * 4, cudaMemcpyHostToDevice, s_exp));  // geometry + poff
  {
    const long long warps = (long long)ns + ((long long)tail_words + 1 + 31) / 32;  // a warp per step + tail words
    k_expand_plan<<<(unsigned)((warps + PLAN_WARPS - 1) / PLAN_WARPS), 32 * PLAN_WARPS, 0, s_exp>>>(dev_groups ? dev_groups : b->gsrc.p, b->gsrc.p, b->blob.p, ns, (int)plan_words,
                                                                   (int)aux_off, (int)tail_off, (int)tail_words,
                                                                   (int)racc, (int)rowacc);
    CK(cudaGetLastError());
  }
  if (s_exp != s) {
    CK(cudaEventRecord(b->ev[3], s_exp));
    CK(cudaStreamWaitEvent(s, b->ev[3], 0));
  }
  if (b->tev) CK(cudaEventRecord(b->ev[1], s));  // h2d_ms = uploads + row tables + expansion (+ the early emit when there is one)
  b->pend_launches += 1;
  b->staged = true;
  b->ran = false;
  return RBGTOPO_OK;
}

// RBGTOPO_VERIFY_PLAN self-check: the plan k_expand_plan wrote (and the geometry plan_stage
// computed) must equal, word for word, what the host builder + validator produce.
int verify_plan(rbgtopo_ctx* c, Batch* b, const int32_t* gb, int64_t words) {
  cudaStream_t s = stream_of(c, b);
  const BatchMeta& m = b->m;
  const size_t dev_words = (size_t)m.words + (size_t)m.n_steps + 1;
  std::vector<int32_t> got(dev_words);
  CK(cudaStreamSynchronize(s));
  CK(cudaMemcpy(got.data(), b->blob.p, dev_words * 4, cudaMemcpyDeviceToHost));
  Batch ref;  // never staged: only its host vectors and pinned buffer are used
  int64_t plan_words = 0;
  int rc = build_plan(c, gb, words, &plan_words, &ref);
  if (rc) return rc;
  rc = validate_blob(c, ref.h_in.p, plan_words, &ref.m, true);
  if (rc) return rc;
  if (plan_words != m.words) return fail(RBGTOPO_ECUDA, "verify_plan: %lld plan words, host builder %lld", m.words, (long long)plan_words);
  for (int64_t i = 0; i < plan_words; ++i)
    if (got[i] != ref.h_in.p[i])
      return fail(RBGTOPO_ECUDA, "verify_plan: word %lld differs: device %d, host %d", (long long)i, got[i], ref.h_in.p[i]);
  if (ref.m.poff != m.poff) return fail(RBGTOPO_ECUDA, "verify_plan: poff differs");
  for (size_t i = 0; i < m.poff.size(); ++i)
    if (got[plan_words + i] != m.poff[i]) return fail(RBGTOPO_ECUDA, "verify_plan: device poff[%zu]", i);
  if (ref.m.n_steps != m.n_steps || ref.m.total_r != m.total_r || ref.m.total_p != m.total_p || ref.m.max_p != m.max_p ||
      ref.m.max_k != m.max_k || ref.m.max_q != m.max_q || ref.m.patch_cap != m.patch_cap || ref.m.max_cap != m.max_cap ||
      ref.m.any_excl_unknown != m.any_excl_unknown || ref.m.scores != m.scores || ref.m.algo_bytes != m.algo_bytes)
    return fail(RBGTOPO_ECUDA, "verify_plan: batch meta differs");
  if (ref.wave_begin != b->wave_begin || ref.wave_maxp != b->wave_maxp || ref.step_group != b->step_group)
    return fail(RBGTOPO_ECUDA, "verify_plan: wave tables differ");
  if (b->perm_n > 0) {  // the launch order of k_plan_group must be a permutation of the first wave's steps
    std::vector<int32_t> perm((size_t)b->perm_n);
    CK(cudaMemcpy(perm.data(), b->blob.p + dev_words, perm.size() * 4, cudaMemcpyDeviceToHost));
    std::vector<char> seen((size_t)b->perm_n, 0);
    for (int32_t v : perm) {
      if (v < 0 || v >= b->perm_n || seen[v]) return fail(RBGTOPO_ECUDA, "verify_plan: launch order is not a permutation (entry %d)", v);
      seen[v] = 1;
    }
  }
  // the dense-row tables k_plan_etab derived from the GROUPS blob must say what the expanded plan says: the first
  // dense role row of every step (a group's role rows consecutive, waves in order, groups in order), the row table
  // entry of every role row, the row of every replica
  const int ns = m.n_steps, nrows = m.total_p;
  std::vector<int32_t> drow((size_t)ns), rowmap((size_t)m.total_r);
  std::vector<int2> rtab((size_t)nrows);
  if (ns) CK(cudaMemcpy(drow.data(), b->drow.p, drow.size() * 4, cudaMemcpyDeviceToHost));
  if (m.total_r) CK(cudaMemcpy(rowmap.data(), b->rowmap.p, rowmap.size() * 4, cudaMemcpyDeviceToHost));
  if (nrows) CK(cudaMemcpy(rtab.data(), b->rtab.p, rtab.size() * sizeof(int2), cudaMemcpyDeviceToHost));
  std::vector<int> grow((size_t)b->grp_flags.size() + 1, 0);  // role rows per group, then the prefix
  for (int st = 0; st < ns; ++st) grow[(size_t)ref.step_group[st] + 1] += ref.h_in.p[RBGTOPO_HDR_WORDS + (size_t)st * RBGTOPO_STEP_WORDS + 3];
  for (size_t g = 1; g < grow.size(); ++g) grow[g] += grow[g - 1];
  std::vector<char> seen((size_t)nrows, 0);
  for (int st = 0; st < ns; ++st) {  // steps are wave-major: a group's steps come in wave order
    const int32_t* h = ref.h_in.p + RBGTOPO_HDR_WORDS + (size_t)st * RBGTOPO_STEP_WORDS;
    const int row0 = grow[ref.step_group[st]];
    grow[ref.step_group[st]] += h[3];
    if (drow[st] != row0) return fail(RBGTOPO_ECUDA, "verify_plan: step %d starts at dense row %d, expected %d", st, drow[st], row0);
    for (int p2 = 0, rep = h[12]; p2 < h[3]; ++p2) {
      const int32_t* r = ref.h_in.p + h[4] + 4 * p2;
      const bool rexcl = (h[1] & RBGTOPO_STEP_EXCLUSIVE) && (r[3] & RBGTOPO_ROLE_EXCLUSIVE);
      const int row = row0 + p2;
      if (row < 0 || row >= nrows || seen[row] || rtab[row].x != emit_pack_row(r[1], r[2], rexcl, step_level(h[1])) || rtab[row].y != h[0])
        return fail(RBGTOPO_ECUDA, "verify_plan: row table entry %d (step %d role %d) differs from the plan", row, st, p2);
      seen[row] = 1;
      for (int k = 0; k < r[0]; ++k, ++rep)
        if (rowmap[rep] != row) return fail(RBGTOPO_ECUDA, "verify_plan: replica %d maps to dense row %d, expected %d", rep, rowmap[rep], row);
    }
  }
  for (int r = 0; r < nrows; ++r)
    if (!seen[r]) return fail(RBGTOPO_ECUDA, "verify_plan: dense row %d belongs to no step", r);
  return RBGTOPO_OK;
}

// Step-order results of a plan batch (already in b->h_out) -> group order.  Returns
// the groups the plan could not finish exactly (dirty) in *dirty.
void plan_results(const Batch* b, int32_t* assign, int32_t* status, int32_t* domain, std::vector<char>* dirty) {
  const BatchMeta& m = b->m;
  const int32_t* a = b->h_out.p;
  const int32_t* st = a + m.total_r;
  const int32_t* dm = st + m.n_steps;
  const int ng = (int)b->grp_flags.size();
  // the device wrote assign[] in group order already (rep_off of a step = group offset + earlier waves)
  if (assign && ng > 0 && m.total_r > 0) memcpy(assign + b->grp_assign_off[0], a, (size_t)m.total_r * 4);
  std::vector<int> gstat(ng, 0), gdom(ng, -1);
  for (int g = 0; g < ng; ++g)  // an exclusive group confirms the domain it already occupies (as the host loop)
    if (b->grp_flags[g] & RBGTOPO_STEP_EXCLUSIVE) gdom[g] = b->grp_fixed[g];
  for (int s = 0; s < m.n_steps; ++s) {
    const int g = b->step_group[s];
    gstat[g] = std::max(gstat[g], st[s]);
    if (dm[s] >= 0) gdom[g] = dm[s];
  }
  const int g0 = b->g_lo;  // status / domain / dirty are indexed by the group's position in the GROUPS blob
  if ((int)dirty->size() < g0 + ng) dirty->resize((size_t)g0 + ng, 0);
  for (int g = 0; g < ng; ++g) {
    (*dirty)[g0 + g] = 0;
    const bool gang = (b->grp_flags[g] & RBGTOPO_STEP_GANG) != 0;
    if (gstat[g] == RBGTOPO_GANG_FAILED || (gang && gstat[g] != RBGTOPO_PLACED_ALL)) {
      if (assign)
        for (int k = 0; k < b->grp_pending[g]; ++k) assign[b->grp_assign_off[g] + k] = -1;
      gstat[g] = RBGTOPO_GANG_FAILED;
      gdom[g] = -1;
    } else if (gstat[g] == RBGTOPO_PLACED_PART) {
      (*dirty)[g0 + g] = 1;  // `need` of the later waves was predicted with every replica placed
    }
    if (status) status[g0 + g] = gstat[g];
    if (domain) domain[g0 + g] = (b->grp_flags[g] & RBGTOPO_STEP_EXCLUSIVE) ? gdom[g] : -1;
  }
}
}  // namespace

namespace {
// ---- rbgtopo_place_groups, direct path -------------------------------------------------------------------------------
// No expanded plan and nothing per step on the host: the GROUPS blob goes up as it came (the upload is enqueued before
// it is validated: bytes only), the host validates every group, checks the exactness bound and collects a handful of
// maxima (per-shape caches: a fleet repeats a few templates), k_group_rtab derives the row table, k_emit_rows writes the
// dense matrix and k_plan_group<true> — a programmatic dependent of it — replays each group's waves from its role
// table.  8 CUDA calls per call instead of ~20, and less than half the host time (DESIGN.md §4.4).
// Used with the default kernels (any world: selection is replicated); *handled = false -> the caller takes the staged
// path (plan_stage).
const bool kNoDirect = getenv("RBGTOPO_NO_DIRECT") != nullptr;

struct GroupFacts {
  int pend = 0, nw = 0, rr = 0, max_p = 1, max_k = 1, i0_last = 0;  // rr: role rows = dense rows
  long long pcp = 0;  // closed neighbourhoods of the scheduled pods
};
// per-shape part of the facts (thread-local, 4 ways): valid shapes only
struct ShapeFacts {
  bool valid = false;
  int q = 0, nw = 0, rr = 0, max_p = 1, max_k = 1, i0_last = 0;
  long long pend = 0;
  int32_t roles[4 * RBGTOPO_MAX_GROUP_ROLES];
  int32_t pair[RBGTOPO_MAX_GROUP_ROLES * RBGTOPO_MAX_GROUP_ROLES];
  long long role_bound[RBGTOPO_MAX_GROUP_ROLES];  // max over the waves a role appears in of sum_j pair*placed + min(need, cap)*F
  bool match(const int32_t* r, const int32_t* p, int qq) const {
    return valid && qq == q && memcmp(r, roles, (size_t)16 * qq) == 0 && memcmp(p, pair, (size_t)4 * qq * qq) == 0;
  }
};

// Everything about group g that the direct path needs; the checks are those of plan_geometry's check_group /
// size_group (same messages), the exactness bound is taken per role over its worst wave.
// phase 1: the group record, role table and pair matrix (what the row table and the dense matrix depend on);
// phase 2: the scheduled pods (ranges, neighbourhood sizes) and the exactness bound; phase 3 = both.
// role_bound: the per-role wave bound of another wave rule (place_groups_lw: pods, §3.11) instead of the replica waves'.
int group_facts(const TopoHost& T, const int32_t* gb, int64_t words, int g, bool report, GroupFacts* out, int phase = 3,
                const long long* role_bound = nullptr) {
  auto in = [&](long long off, long long cnt) { return off >= 0 && cnt >= 0 && off + cnt <= words; };
  const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS;
  const int q = rec[3];
  if (q < 1 || q > RBGTOPO_MAX_GROUP_ROLES) GROUP_FAIL(RBGTOPO_ELIMIT, "group %d: %d roles", g, q);
  if (!in(rec[4], 4LL * q) || !in(rec[5], (long long)q * q) || !in(rec[7], 3LL * rec[6]))
    GROUP_FAIL(RBGTOPO_EINVAL, "group %d: section out of bounds", g);
  const int32_t* roles = gb + rec[4];
  const int32_t* pair = gb + rec[5];
  static thread_local ShapeFacts ways[4];
  static thread_local int next_way = 0;
  const ShapeFacts* sf = nullptr;
  if (!report)
    for (const ShapeFacts& w : ways)
      if (w.match(roles, pair, q)) { sf = &w; break; }
  const long long sat = 1LL << 40;
  if (!sf) {
    long long pend = 0;
    for (int i = 0; i < q; ++i) {
      if (roles[4 * i + 1] < 0 || (i && roles[4 * i] < roles[4 * (i - 1)]))
        GROUP_FAIL(RBGTOPO_EINVAL, "group %d role %d: pending < 0 or levels not ascending", g, i);
      if (roles[4 * i + 2] < 0 || roles[4 * i + 2] > RBGTOPO_MAX_FREE)
        GROUP_FAIL(RBGTOPO_EINVAL, "group %d role %d: demand", g, i);
      pend += roles[4 * i + 1];
    }
    if (pend > 0x3FFFFFFFLL) GROUP_FAIL(RBGTOPO_ELIMIT, "group %d: pending replicas", g);
    for (int i = 0; i < q; ++i)
      if (roles[4 * i + 3] & ~RBGTOPO_ROLE_EXCLUSIVE) GROUP_FAIL(RBGTOPO_EINVAL, "group %d role %d: unknown role flags", g, i);
    for (int i = 0; i < q * q; ++i)
      if (pair[i] < 0 || pair[i] > kMaxExactTerm) GROUP_FAIL(RBGTOPO_EINVAL, "group %d: pair weight out of [0, 2^24]", g);
    ShapeFacts& w = ways[next_way];
    next_way = (next_way + 1) % 4;
    w.valid = false;
    w.q = q;
    memcpy(w.roles, roles, (size_t)16 * q);
    memcpy(w.pair, pair, (size_t)4 * q * q);
    w.pend = pend;
    w.max_p = 1;
    w.max_k = 1;
    w.i0_last = 0;
    w.rr = 0;
    for (int i = 0; i < q; ++i) w.role_bound[i] = 0;
    int placed[RBGTOPO_MAX_GROUP_ROLES] = {0};
    int i0 = 0;
    w.nw = walk_waves(roles, q, nullptr, [&](int, const PlanWave& pw) {
      const int P = pw.size();
      int n = 0;
      for (int k = 0; k < P; ++k) {
        const int ri = pw.role[k];
        int need = 0;
        long long bnd = 0;
        for (int j = 0; j < q; ++j) {
          if (pair[ri * q + j] > 0) need = (int)std::min<long long>((long long)need + roles[4 * j + 1] - placed[j], 1 << 30);
          bnd = std::min(bnd + (long long)pair[ri * q + j] * placed[j], sat);
        }
        w.role_bound[ri] = std::max(w.role_bound[ri], bnd + (long long)std::min(need, RBGTOPO_NEED_CAP) * RBGTOPO_F_CAP);
        n += pw.count[k];
      }
      w.max_p = std::max(w.max_p, P);
      w.max_k = std::max(w.max_k, n);
      w.i0_last = i0;
      w.rr += P;
      for (int k = 0; k < P; ++k) placed[pw.role[k]] += pw.count[k];
      i0 += n;
    });
    w.valid = !report;
    sf = &w;
  }
  if (phase & 1) {
    if (rec[0] < 0 || rec[2] < -1 || (rec[10] == 0 && rec[2] >= T.n_domains)) GROUP_FAIL(RBGTOPO_EINVAL, "group %d: gid / fixed_domain", g);
    if (const int lc = level_code(rec[10], T.n_levels, T.place_levels))
      GROUP_FAIL(lc, "group %d: exclusive level %d (%d installed%s)", g, rec[10], std::max(0, T.n_levels),
                 T.place_levels ? "" : "; placement at level 0 only");
    if (rec[10] > 0 && T.level_nd && rec[2] >= T.level_nd[rec[10]])
      GROUP_FAIL(RBGTOPO_EINVAL, "group %d: fixed_domain %d outside the %d domains of level %d", g, rec[2], T.level_nd[rec[10]], rec[10]);
    if (rec[1] & ~(RBGTOPO_STEP_EXCLUSIVE | RBGTOPO_STEP_GANG)) GROUP_FAIL(RBGTOPO_EINVAL, "group %d: unknown flags 0x%x", g, rec[1]);
    out->pend = (int)sf->pend;
    out->nw = sf->nw;
    out->rr = sf->rr;
    out->max_p = sf->max_p;
    out->max_k = sf->max_k;
    out->i0_last = sf->i0_last;
  }
  if (!(phase & 2)) return RBGTOPO_OK;
  long long pc = 0;
  long long anch_w[RBGTOPO_MAX_GROUP_ROLES] = {0};
  const int na = rec[6];
  for (int a = 0; a < na; ++a) {
    const int32_t* an = gb + rec[7] + 3 * a;
    if (an[0] < 0 || an[0] >= T.n || an[1] < 0 || an[1] >= q || an[2] < 0 || an[2] > kMaxExactTerm)
      GROUP_FAIL(RBGTOPO_EINVAL, "group %d anchor %d out of range", g, a);
    pc += T.degp1 ? T.degp1[an[0]] : 1;
    for (int ri = 0; ri < q; ++ri) anch_w[ri] = std::min(anch_w[ri] + (long long)pair[ri * q + an[1]] * an[2], sat);
  }
  if (pc > 0x3FFFFFFFLL) GROUP_FAIL(RBGTOPO_ELIMIT, "group %d: patch list exceeds 2^30 entries", g);
  if (sf->nw > 0)
    for (int ri = 0; ri < q; ++ri) {
      if (roles[4 * ri + 1] <= 0) continue;  // a role without pending replicas has no row
      const long long amax = std::min(anch_w[ri] + (role_bound ? role_bound : sf->role_bound)[ri], sat);
      if (amax >= T.amax_limit)
        GROUP_FAIL(RBGTOPO_EINEXACT, "group %d role %d: max score bound >= 2^24 (anchor weight %lld x row weight %lld)", g, ri, amax, T.row_w);
    }
  out->pcp = pc;
  return RBGTOPO_OK;
}

// What the direct path derives on the host, in two passes (pure host code: rbgtopo_place_describe runs it without a device).
struct DirectGeom {
  long long total_r = 0, rrows = 0, max_cap = 0;  // replicas, dense role rows
  int n0 = 0, max_q = 1, max_p = 1, nth = 128, HT = 64, CAP = 32;
  size_t smem = 0;
  bool any_excl = false;
};
// pass 1: group records, role tables, pair matrices (per-shape caches), the prefix of the assignment offsets, and the
// launch order of k_plan_group (perm[0 .. n0): groups with pending replicas, heaviest expected table first — the
// weight is the number of closed neighbourhoods the table will hold: scheduled pods + replicas to place)
int direct_pass1(const TopoHost& th, const int32_t* gb, int64_t words, int ng, std::vector<GroupFacts>& facts, int32_t* perm,
                 DirectGeom* G) {
  facts.resize((size_t)ng);
  int first_bad = ng;
#pragma omp parallel for schedule(static) num_threads(kHostThreads) reduction(min : first_bad) if (ng >= kHostParallelMinGroups && kHostThreads > 1)
  for (int g = 0; g < ng; ++g)
    if (group_facts(th, gb, words, g, false, &facts[g], 1) != RBGTOPO_OK) first_bad = std::min(first_bad, g);
  if (first_bad < ng) return group_facts(th, gb, words, first_bad, true, &facts[first_bad], 1);
  long long pacc = 0, wmax = 1;
  for (int g = 0; g < ng; ++g) {
    const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS;
    const GroupFacts& f = facts[g];
    if (rec[8] != pacc || rec[9] != f.pend) return fail(RBGTOPO_EINVAL, "group %d: bad assign_off/n_pending", g);
    pacc += f.pend;
    if (pacc > 0x3FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "pending replicas exceed 2^30");
    G->rrows += f.rr;
    if (f.nw > 0) {
      G->n0 += 1;
      G->max_q = std::max(G->max_q, rec[3]);
      G->max_p = std::max(G->max_p, f.max_p);
      G->any_excl |= (rec[1] & RBGTOPO_STEP_EXCLUSIVE) != 0;
      wmax = std::max(wmax, (long long)f.pend + std::max(0, rec[6]));
    }
  }
  if (gb[4] != pacc) return fail(RBGTOPO_EINVAL, "total pending mismatch");
  G->total_r = pacc;
  const int nb = 1024;
  static thread_local std::vector<int> bucket, wkey;
  bucket.assign(nb + 1, 0);
  wkey.resize((size_t)ng);
  for (int g = 0; g < ng; ++g) {
    if (facts[g].nw <= 0) continue;
    const long long w = (long long)facts[g].pend + std::max(0, gb[RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS + 6]);
    wkey[g] = (nb - 1) - (int)(w * (nb - 1) / wmax);
    bucket[wkey[g] + 1] += 1;
  }
  for (int k = 0; k < nb; ++k) bucket[k + 1] += bucket[k];
  for (int g = 0; g < ng; ++g)
    if (facts[g].nw > 0) perm[bucket[wkey[g]]++] = g;  // stable: equal weights keep group order
  return RBGTOPO_OK;
}
// pass 2: scheduled pods (ranges, neighbourhood sizes), the exactness bound, the table capacity and with it the launch
// geometry of k_plan_group (as plan_group_cfg)
int direct_pass2(const TopoHost& th, const int32_t* gb, int64_t words, int ng, std::vector<GroupFacts>& facts, DirectGeom* G) {
  int first_bad = ng;
#pragma omp parallel for schedule(static) num_threads(kHostThreads) reduction(min : first_bad) if (ng >= kHostParallelMinGroups && kHostThreads > 1)
  for (int g = 0; g < ng; ++g)
    if (group_facts(th, gb, words, g, false, &facts[g], 2) != RBGTOPO_OK) first_bad = std::min(first_bad, g);
  if (first_bad < ng) return group_facts(th, gb, words, first_bad, true, &facts[first_bad], 2);
  for (int g = 0; g < ng; ++g)
    if (facts[g].nw > 0)
      G->max_cap = std::max(G->max_cap, (long long)facts[g].i0_last + facts[g].pcp + (long long)facts[g].i0_last * th.max_degp1);  // the last wave's table
  G->nth = std::max(128, 32 * G->max_p);
  G->CAP = std::max(32, round_up((int)std::min<long long>(G->max_cap, 0x3FFFFFFF), 32));
  G->HT = 64;
  while (G->HT <= G->CAP && G->HT < (1 << 20)) G->HT <<= 1;
  G->smem = group_smem_bytes(G->max_q, G->nth / 32, G->HT, G->CAP);
  return RBGTOPO_OK;
}

// Dense role rows of the direct path from the GROUPS blob on the device (it may not be validated yet: the kernels
// range-check what they read and bound every row by n_rows): role rows per group, their saturating exclusive scan =
// the first dense role row of every group (b->drow, step_drow), then the row table.  alloc = false: launches nothing
// unless the buffers of an earlier call are large enough (*launched says whether it did).
int launch_group_rows(Batch* b, int words, int ng, int n_rows, cudaStream_t s, bool alloc, bool* launched) {
  *launched = false;
  size_t tmp_bytes = 0;
  CK(cub::DeviceScan::ExclusiveScan(nullptr, tmp_bytes, b->rrcnt.p, b->drow.p, SatAdd{n_rows}, 0, ng, s));
  if (alloc) {
    CK(b->rtab.reserve((size_t)std::max(1, n_rows)));
    CK(b->drow.reserve((size_t)ng));
    CK(b->rrcnt.reserve((size_t)ng));
    CK(b->scan_tmp.reserve(std::max<size_t>(1, tmp_bytes)));
  } else if ((size_t)n_rows > b->rtab.cap || (size_t)ng > b->drow.cap || (size_t)ng > b->rrcnt.cap || tmp_bytes > b->scan_tmp.cap) {
    return RBGTOPO_OK;
  }
  k_group_rrcount<<<(ng + RRCOUNT_THREADS - 1) / RRCOUNT_THREADS, RRCOUNT_THREADS, 0, s>>>(b->gsrc.p, words, ng, n_rows, b->rrcnt.p);
  CK(cub::DeviceScan::ExclusiveScan(b->scan_tmp.p, tmp_bytes, b->rrcnt.p, b->drow.p, SatAdd{n_rows}, 0, ng, s));
  k_group_rtab<<<(ng + RTAB_WARPS - 1) / RTAB_WARPS, 32 * RTAB_WARPS, 0, s>>>(b->gsrc.p, words, ng, n_rows, b->drow.p, b->rtab.p);
  CK(cudaGetLastError());
  *launched = true;
  return RBGTOPO_OK;
}

int place_groups_direct(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t* assign, int32_t* status, int32_t* domain,
                        std::vector<char>* dirty, bool* handled, const RankReq* rk = nullptr) {
  *handled = false;
  // world > 1: replicated selection (every rank places every group over all nodes; the dense matrix and its corrections
  // are limited to the rank's column slab by the kernels themselves), exactly as on the staged path
  if (kNoDirect || !kSerialPlan || kVerifyPlan || kPerWavePlan) return RBGTOPO_OK;
  if (!groups_blob_ok(gb, words) || words > 0x3FFFFFFFLL) return RBGTOPO_OK;  // the staged path reports what is wrong
  const int ng = gb[2];
  if (ng < 1 || ng >= kSplitMinGroups) return RBGTOPO_OK;
  NvtxRange nv("rbgtopo:place_groups_direct");
  static const bool prof = kProfileHost;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto us = [](auto a, auto b2) { return std::chrono::duration<double, std::micro>(b2 - a).count(); };
  const auto t0 = now();
  Batch* b = nullptr;
  int rc = acquire_batch(c, &b);
  if (rc) return rc;
  cudaStream_t s = stream_of(c, b);
  auto done = [&](int r) {
    if (r || !*handled) cudaStreamSynchronize(s);  // the early upload may still read the staging buffer the staged path re-uses
    release_batch(c, b);
    return r;
  };
  // staging layout: GROUPS blob | pad | launch order (<= ng ints)
  const size_t perm_off = ((size_t)words + 3) & ~(size_t)3;
  const size_t src_words = perm_off + (size_t)ng;
  bool rtab_early = false;
  rc = [&]() -> int {
    CK(b->h_in.reserve(src_words));
    CK(b->gsrc.reserve(src_words));
    b->tev = false;
    b->perm_n = 0;
    memcpy(b->h_in.p, gb, (size_t)words * 4);
    CK(cudaMemcpyAsync(b->gsrc.p, b->h_in.p, (size_t)words * 4, cudaMemcpyHostToDevice, s));  // before validation: bytes only
    // ... and the dense role rows and the row table behind it, from the not yet validated blob, when the buffers of an
    // earlier call are large enough: they are ready by the time pass 1 is through.  The row bound is gb[4], the
    // replicas the blob claims: a group has at most as many role rows as replicas, so it bounds the rows of a valid
    // blob, and the buffers are sized by it below so that the next call of the same fleet launches here again.
    if (gb[4] > 0) return launch_group_rows(b, (int)words, ng, gb[4], s, false, &rtab_early);
    return RBGTOPO_OK;
  }();
  if (rc) return done(rc);
  const auto t1 = now();

  // ---- pass 1: group records, role tables, pair matrices (per-shape caches) — all the row table and the dense
  // matrix depend on; the launch order of k_plan_group from (scheduled pods + pending replicas) per group
  const TopoHost th = topo_host(c, places_levels(c));
  static thread_local std::vector<GroupFacts> facts;
  DirectGeom G;
  rc = direct_pass1(th, gb, words, ng, facts, b->h_in.p + perm_off, &G);
  if (rc) return done(rc);
  const long long total_r = G.total_r, rrows = G.rrows;
  const int n0 = G.n0, max_q = G.max_q;
  const bool any_excl = G.any_excl;
  const long long segs = ((rrows + kEmitRowsBlock - 1) / kEmitRowsBlock) * c->lc;
  if (segs > 0x7FFFFFF0LL) return done(RBGTOPO_OK);
  const auto t2 = now();

  // ---- device, first half: launch order up, row table, dense matrix (it runs under pass 2)
  const size_t out_n = (size_t)total_r + 2 * (size_t)ng;
  rc = [&]() -> int {
    CK(b->matrix.reserve((size_t)std::max<long long>(1, rrows) * c->slab_stride));
    CK(b->out.reserve(out_n + 4));
    CK(b->h_out.reserve(out_n + 4));
    b->epoch = c->topo_epoch;
    b->lvl_epoch = c->lvl_epoch;
    if (n0 > 0) {
      CK(cudaMemcpyAsync(b->gsrc.p + perm_off, b->h_in.p + perm_off, (size_t)n0 * 4, cudaMemcpyHostToDevice, s));
      if (!rtab_early) {  // the same bound as the early launch (pass 1 found gb[4] == total_r >= rrows)
        bool launched = false;
        const int grc = launch_group_rows(b, (int)words, ng, (int)total_r, s, true, &launched);
        if (grc) return grc;
      }
      CK(cudaStreamWaitEvent(s, c->base_ready, 0));  // a pending snapshot refresh: base / free ...
      CK(cudaStreamWaitEvent(s, c->topo_ready, 0));  // ... and the background order, both in front of the dense-matrix kernel
      b->any_excl = any_excl;
      const int erc = launch_emit_plan(c, b, s, rrows);
      if (erc) return erc;
    }
    return RBGTOPO_OK;
  }();
  if (rc) return done(rc);
  const auto t2b = now();

  // ---- pass 2: scheduled pods (ranges, neighbourhood sizes), exactness bound, table capacity
  rc = direct_pass2(th, gb, words, ng, facts, &G);
  if (rc) return done(rc);
  const int nth = G.nth, HT = G.HT, CAP = G.CAP;
  const size_t smem = G.smem;
  // what does not fit a CTA's shared memory takes the staged path (*handled stays false; the dense matrix was emitted in vain)
  if (G.max_cap > 0x3FFFFFFFLL || smem > kFastSmemMax) return done(RBGTOPO_OK);
  const auto t2c = now();

  // ---- device, second half: selection as a programmatic dependent of the dense-matrix kernel, results
  rc = [&]() -> int {
    if (n0 > 0) {
      BatchDev d{};
      d.blob = b->gsrc.p;
      d.n_steps = ng;
      d.lc = c->lc;
      d.chunk = c->chunk;
      d.parts = 1;
      d.matrix = b->matrix.p;
      d.drow = b->drow.p;
      d.assign = b->out.p;
      d.status = b->out.p + total_r;
      d.domain_out = d.status + ng;
      d.dstar = d.domain_out;
      d.perm = b->gsrc.p + perm_off;
      cudaLaunchConfig_t cfg{};
      cfg.gridDim = dim3((unsigned)n0);
      cfg.blockDim = dim3((unsigned)nth);
      cfg.dynamicSmemBytes = smem;
      cfg.stream = s;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      at[0].val.programmaticStreamSerializationAllowed = 1;
      cfg.attrs = at;
      cfg.numAttrs = kNoPdl ? 0 : 1;
      int orc = note_plan_occupancy(c, true, nth, smem, n0);
      if (orc) return orc;
      CK(cudaLaunchKernelEx(&cfg, k_plan_group<true>, topo_dev(c), d, (int)max_q, HT, CAP, 0));
      CK(cudaMemcpyAsync(b->h_out.p, b->out.p, out_n * 4, cudaMemcpyDeviceToHost, s));
    }
    const auto t3 = now();
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    const auto t4 = now();
    const int32_t* a = b->h_out.p;
    if (total_r > 0) memcpy(assign, a, (size_t)total_r * 4);
    if ((int)dirty->size() < ng) dirty->resize((size_t)ng, 0);
    for (int g = 0; g < ng; ++g) {
      const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS;
      const bool excl = (rec[1] & RBGTOPO_STEP_EXCLUSIVE) != 0;
      int st = RBGTOPO_PLACED_ALL, dm = excl ? rec[2] : -1;  // nothing pending: placed, the domain it occupies confirmed
      if (facts[g].nw > 0) {
        st = a[total_r + g];
        dm = excl ? a[total_r + ng + g] : -1;
      }
      (*dirty)[g] = st == RBGTOPO_PLACED_PART;  // `need` of the later waves was predicted with every replica placed
      if (status) status[g] = st;
      if (domain) domain[g] = dm;
    }
    if (rk) {
      const int arc = rank_plan(c, b, gb, assign, status, domain, *dirty, *rk);
      if (arc) return arc;
    }
    if (prof)
      fprintf(stderr, "[rbgtopo direct] stage %.0f us, pass 1 %.0f us, enqueue 1 %.0f us, pass 2 %.0f us, enqueue 2 %.0f us, wait %.0f us, results %.0f us\n",
              us(t0, t1), us(t1, t2), us(t2, t2b), us(t2b, t2c), us(t2c, t3), us(t3, t4), us(t4, now()));
    return RBGTOPO_OK;
  }();
  if (rc) return done(rc);
  {
    const long long slab = c->slab_hi - c->slab_lo;
    rbgtopo_timing tm{};
    tm.scores = total_r * slab;
    tm.algo_bytes = 4LL * rrows * slab + 4LL * words + 8LL * slab;
    tm.launches = n0 > 0 ? 6 : 0;  // role-row count, the scan (2), row table, dense matrix, selection
    tm.h2d_words = (int32_t)((long long)words + n0);
    std::lock_guard<std::mutex> g(c->stat_mu);
    c->last = tm;
    c->last_score_ms.clear();
    c->last_select_ms.clear();
    c->calls += 1;
    c->scores_total += tm.scores;
    c->launches += tm.launches;
  }
  *handled = true;
  return done(RBGTOPO_OK);
}

// ---- rbgtopo_place_groups_committed -----------------------------------------------------------------------------------
// A committed batch (DESIGN.md §3.8) is rounds of selection only, no dense matrix: k_plan_group_commit over a suffix of
// the groups (each sees the claims of the previous round's results of the groups before it), k_commit_diff (the lowest
// group with a changed claim some later group read), k_commit_claims (the lookups of the next round), and one 4-byte
// read-back.  Groups up to that lowest group are final, the next round re-runs the groups above it: it only grows, so
// there are at most n_groups rounds, and a batch whose groups read nothing an earlier group took needs one.  The host
// validates the blob exactly as the direct path of rbgtopo_place_groups does (same codes).
int lw_validate(rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* rp, int64_t rp_words);

// The §3.4 bound at one pod per replica: lw_validate's with (S, C) = (1, -1) for every role, which takes every mix of
// unplaced earlier replicas a later wave can see (§3.10, §3.11 rule 7).  The group table is checked.
int exact_one_pod(rbgtopo_ctx* c, const int32_t* gb, int64_t words) {
  long long qsum = 0;
  for (int g = 0; g < gb[2]; ++g) {
    const int q = group_rec(gb, g)[3];
    if (q < 1 || q > RBGTOPO_MAX_GROUP_ROLES) return fail(RBGTOPO_ELIMIT, "group %d: %d roles", g, q);
    qsum += q;
  }
  std::vector<int32_t> unit(2 * (size_t)qsum);
  for (size_t i = 0; i < unit.size(); i += 2) { unit[i] = 1; unit[i + 1] = -1; }
  return lw_validate(c, gb, words, unit.data(), (int64_t)unit.size());
}

// Ranked alternates of a committed batch (DESIGN.md §3.14), once its rounds have converged: the dense row of every
// (group, wave) that placed a replica is scored again as a step batch — the snapshot's scores, `need` over the
// replicas still unplaced at that wave, the group's earlier waves as anchors — without consumed records and without
// the exclusive flag: room and owner are tested by k_alternates_commit after the whole batch, against the final claims
// in `cm`.  A batch whose rows exceed kReplayBytes is scored and ranked in chunks of steps.  status / domain not null.
// rp != nullptr: a committed leader-worker batch (§3.15): the (S, C) table of place_groups_lw, pod waves (next_wave),
// role counts, `need`, anchors and rows in pods; hc: its owner claims (HostClaims).
// admit != nullptr: the eligible committed form (§3.20), one class mask per role in blob order.  Every replayed step
// carries the masks of its role rows (MAXP per step, in staging order, uploaded per chunk into b->lw, which the rounds
// no longer need) and is scored by k_score_emit_elig: the class -inf does not depend on claims, so the replayed rows
// equal the masked rows of the final run at every entry the ranking reads.  b->h_lw is rewritten only once the
// previous chunk's copy has completed (run_alternates ends in a stream synchronise; a later chunk checks it again).
constexpr long long kReplayBytes = 1LL << 30;
int rank_committed(rbgtopo_ctx* c, Batch* b, const int32_t* gb, const int32_t* rp, const int32_t* assign,
                   const int32_t* status, const int32_t* domain, const CommitDev& cm, bool lv, const RankReq& rk,
                   int* launches, const HostClaims* hc = nullptr, const uint64_t* admit = nullptr) {
  const int ng = gb[2];
  const GroupOffsets off(gb, rp);
  alt_clear(rk, 0, off.pod0[ng]);
  cudaStream_t s = stream_of(c, b);
  CK(cudaStreamWaitEvent(s, c->base_ready, 0));  // the rows read base and free of the snapshot the rounds saw
  const int max_rows = (int)std::max<long long>(RBGTOPO_MAX_STEP_ROLES, kReplayBytes / 4 / c->slab_stride);
  StepBlob sb;
  std::vector<AltRow> list;
  std::vector<uint64_t> masks;  // admit: MAXP per staged step
  int rc = RBGTOPO_OK, chunks = 0;
  auto flush = [&]() -> int {
    if (sb.ns == 0) return RBGTOPO_OK;
    const std::vector<int32_t>& blob = sb.build();
    int r2 = stage_into(c, b, blob.data(), (int64_t)blob.size());
    if (!r2 && admit) {
      if (chunks++ > 0) CK(cudaStreamSynchronize(s));  // already drained by run_alternates: never waits in practice
      const size_t w = masks.size() * 2;
      CK(b->lw.reserve(w));
      CK(b->h_lw.reserve(w));
      memcpy(b->h_lw.p, masks.data(), w * 4);
      CK(cudaMemcpyAsync(b->lw.p, b->h_lw.p, w * 4, cudaMemcpyHostToDevice, s));
    }
    if (!r2) r2 = launch_score(c, b, s, nullptr, nullptr, nullptr, nullptr,
                               admit ? reinterpret_cast<const unsigned long long*>(b->lw.p) : nullptr);
    if (!r2) r2 = run_alternates(c, b, b->matrix.p, list, gb, rp, assign, status, domain, rk, &cm, lv, hc);
    *launches += 2;
    sb.clear();
    list.clear();
    masks.clear();
    return r2;
  };
  for (int g = 0; g < ng && !rc; ++g) {
    if (status[g] == RBGTOPO_GANG_FAILED) continue;
    HostRun r(gb, g, off.grp(rp, g), off.pod0[g]);
    const PlanWave& w = r.w;
    // one wave: pods of role ri from pod0 + ord0[ri] + first * S
    auto first = [&](int p) { return r.pod0 + r.ord0[w.role[p]] + (int64_t)w.first[p] * r.S(w.role[p]); };
    while (!rc && next_wave(r.roles, r.q, r.rp, r.cur, r.w) > 0) {
      bool any = false;
      for (int p = 0; p < w.n; ++p)
        for (int k = 0; k < w.count[p] * r.S(w.role[p]); ++k) any |= assign[first(p) + k] >= 0;
      if (any) {
        if (sb.rowacc + w.n > max_rows) rc = flush();
        if (rc) break;
        for (int p = 0; p < w.n; ++p) {
          const int pods = w.count[p] * r.S(w.role[p]);
          bool placed = false;
          for (int k = 0; k < pods; ++k) placed |= assign[first(p) + k] >= 0;
          if (placed) list.push_back(AltRow{sb.rowacc + p, g, w.role[p], (int)first(p), pods});
        }
        sb.add(r, w, 0, -1, 0, false, nullptr, 0);
        if (admit) {
          masks.resize(masks.size() + MAXP, 0);
          for (int p = 0; p < w.n; ++p) masks[masks.size() - MAXP + p] = admit[off.r0[g] + w.role[p]];
        }
      }
      for (int p = 0; p < w.n; ++p)  // the wave's placements: anchors of the later waves
        for (int k = 0; k < w.count[p] * r.S(w.role[p]); ++k) {
          const int node = assign[first(p) + k];
          if (node < 0) continue;
          r.anchors.push_back(node); r.anchors.push_back(w.role[p]); r.anchors.push_back(1);
          r.unplaced[w.role[p]] -= 1;
        }
    }
  }
  if (!rc) rc = flush();
  return rc;
}

// rk != nullptr: the ranked form (§3.14): the same rounds, then rank_committed before the batch's buffers are released.
int place_groups_committed(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t* assign, int32_t* status,
                           int32_t* domain, int32_t* rounds_out, const RankReq* rk = nullptr) {
  *rounds_out = 0;
  if (const int hrc = check_groups_blob(gb, words)) return hrc;
  const int ng = gb[2];
  if (words > 0x3FFFFFFFLL) return fail(RBGTOPO_ELIMIT, "groups blob too large");
  NvtxRange nv("rbgtopo:place_groups_committed");
  const Topology& T = c->topo;
  // levels >= 1 only on a ctx that opted into committed levels (DESIGN.md §3.9)
  const TopoHost th = topo_host(c, commits_levels(c));
  static thread_local std::vector<GroupFacts> facts;
  static thread_local std::vector<int32_t> order, run;
  order.resize((size_t)std::max(ng, 1));
  DirectGeom G;
  int rc = direct_pass1(th, gb, words, ng, facts, order.data(), &G);
  if (rc) return rc;
  rc = direct_pass2(th, gb, words, ng, facts, &G);
  if (rc) return rc;
  if (G.max_cap > 0x3FFFFFFFLL || G.smem > kFastSmemMax)
    return fail(RBGTOPO_ELIMIT, "a group's table of patched nodes (%lld entries, %zu B of shared memory) does not fit "
                                "k_plan_group: a committed batch has no per-wave fallback", G.max_cap, G.smem);
  if (rk) {  // before the first round: the ranking must not fail once the batch is placed
    if ((size_t)((T.n + 31) / 32) * 4 > kFastSmemMax)
      return fail(RBGTOPO_ELIMIT, "ranked placement: %d nodes exceed the room bitmap", T.n);
    rc = exact_one_pod(c, gb, words);  // over every wave the ranking can score
    if (rc) return rc;
  }
  run.clear();  // groups with pending replicas, ascending: a round runs a suffix of them
  for (int g = 0; g < ng; ++g)
    if (facts[g].nw > 0) run.push_back(g);
  const int n0 = (int)run.size();
  const long long total_r = G.total_r;
  // A group at a level >= 1 (validated: the ctx commits levels, and they are installed) selects the <true> kernels:
  // claims per (level, domain) over the levels of the batch's exclusive groups (lmask).
  bool lv = false;
  int lmask = 0;
  for (int g = 0; g < ng; ++g) {
    const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS;
    lv |= rec[10] > 0;
    if (rec[1] & RBGTOPO_STEP_EXCLUSIVE) lmask |= 1 << rec[10];
  }
  const size_t out_n = (size_t)total_r + 2 * (size_t)ng;
  Batch* b = nullptr;
  rc = acquire_batch(c, &b);
  if (rc) return rc;
  cudaStream_t s = stream_of(c, b);
  const bool timed = c->kernel_timing.load(std::memory_order_relaxed);
  std::vector<float> round_ms;
  int rounds = 0;
  CommitDev cm{};  // the claims lists; after the last round they hold the final claims (the ranking reads them)
  rc = [&]() -> int {
    if (n0 == 0) return RBGTOPO_OK;
    const size_t run_off = ((size_t)words + 3) & ~(size_t)3;  // staging: GROUPS blob | pad | run[n0]
    const size_t src_words = run_off + (size_t)n0;
    CK(b->h_in.reserve(src_words));
    CK(b->gsrc.reserve(src_words));
    CK(b->out.reserve(out_n + 4));
    CK(b->h_out.reserve(out_n + 4));
    // ND = domain heads: level 0's, or (lv) those of every installed level at lvl_doff[L], and as many pod heads
    const int N = T.n, ND = lv ? T.lvl_total_d : T.n_domains, NP = lv ? ND : 0, NL = lv ? __builtin_popcount(lmask) : 0;
    const size_t o_dhead = (size_t)N, o_phead = o_dhead + ND, o_reader = o_phead + NP, o_dreader = o_reader + N,
                 o_prev = o_dreader + ND, o_cmin = o_prev + out_n, n_int = o_cmin + 1;
    CK(b->cm_int.reserve(n_int));
    CK(b->cm_claim.reserve((size_t)std::max<long long>(total_r, 1)));
    CK(b->cm_dclaim.reserve((size_t)std::max(ng, 1)));
    if (lv) CK(b->cm_pclaim.reserve((size_t)std::max<long long>(total_r * NL, 1)));
    memcpy(b->h_in.p, gb, (size_t)words * 4);
    memcpy(b->h_in.p + run_off, run.data(), (size_t)n0 * 4);
    CK(cudaMemcpyAsync(b->gsrc.p, b->h_in.p, src_words * 4, cudaMemcpyHostToDevice, s));
    int* const ci = b->cm_int.p;
    int* const o_assign = b->out.p;
    int* const o_domain = b->out.p + total_r + ng;
    // nothing placed and no domain reported yet: the claims before round 0 are those of groups with nothing pending
    CK(cudaMemsetAsync(b->out.p, 0xFF, out_n * 4, s));
    CK(cudaMemsetAsync(ci + o_prev, 0xFF, out_n * 4, s));
    CK(cudaMemsetAsync(ci, 0xFF, (size_t)(N + ND + NP) * 4, s));
    cm.head = ci;
    cm.claim = b->cm_claim.p;
    cm.dhead = ci + o_dhead;
    cm.dclaim = b->cm_dclaim.p;
    cm.reader = ci + o_reader;
    cm.dreader = ci + o_dreader;
    cm.occ = T.occ;
    if (lv) {
      cm.ldom = T.lvl_domain.p;
      cm.doff = T.lvl_doff.p;
      cm.phead = ci + o_phead;
      cm.pclaim = b->cm_pclaim.p;
      cm.lstride = level_stride(N);
      cm.lmask = lmask;
    }
    const auto claims = lv ? k_commit_claims<true> : k_commit_claims<false>;
    const auto diff = lv ? k_commit_diff<true> : k_commit_diff<false>;
    const auto plan = lv ? k_plan_group_commit<true> : k_plan_group_commit<false>;
    const int claim_grid = (ng + RTAB_WARPS - 1) / RTAB_WARPS;
    claims<<<claim_grid, 32 * RTAB_WARPS, 0, s>>>(b->gsrc.p, ng, o_assign, o_domain, ci, b->cm_claim.p, ci + o_dhead,
                                                  b->cm_dclaim.p, cm);
    CK(cudaStreamWaitEvent(s, c->topo_ready, 0));  // a pending snapshot refresh: free, owners, base and the order
    BatchDev d{};
    d.blob = b->gsrc.p;
    d.n_steps = ng;
    d.lc = c->lc;
    d.chunk = c->chunk;
    d.parts = 1;
    d.assign = o_assign;
    d.status = b->out.p + total_r;
    d.domain_out = o_domain;
    d.dstar = o_domain;
    int first = 0;  // run[first ..) = the groups of the next round
    while (first < n0) {
      if (rounds >= ng) return fail(RBGTOPO_ECUDA, "internal: committed batch did not converge in %d rounds", ng);
      const int n_run = n0 - first;
      d.perm = b->gsrc.p + run_off + first;
      CK(cudaMemsetAsync(ci + o_reader, 0xFF, (size_t)(N + ND) * 4, s));  // reader and dreader: -1
      CK(cudaMemsetAsync(ci + o_cmin, 0x7F, 4, s));                        // > any group index
      if (timed) CK(cudaEventRecord(b->ev[0], s));
      plan<<<n_run, G.nth, G.smem, s>>>(topo_dev(c), d, G.max_q, G.HT, G.CAP, cm);
      CK(cudaGetLastError());
      if (timed) CK(cudaEventRecord(b->ev[1], s));
      diff<<<(n_run + RTAB_WARPS - 1) / RTAB_WARPS, 32 * RTAB_WARPS, 0, s>>>(
          b->gsrc.p, d.perm, n_run, o_assign, o_domain, ci + o_prev, ci + o_prev + total_r + ng, ci + o_reader,
          ci + o_dreader, ci + o_cmin, cm);
      CK(cudaMemsetAsync(ci, 0xFF, (size_t)(N + ND + NP) * 4, s));  // head, dhead and phead
      claims<<<claim_grid, 32 * RTAB_WARPS, 0, s>>>(b->gsrc.p, ng, o_assign, o_domain, ci, b->cm_claim.p, ci + o_dhead,
                                                    b->cm_dclaim.p, cm);
      CK(cudaMemcpyAsync(b->h_out.p + out_n, ci + o_cmin, 4, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      CK(cudaGetLastError());
      ++rounds;
      if (timed) {
        float ms = 0.0f;
        CK(cudaEventElapsedTime(&ms, b->ev[0], b->ev[1]));
        round_ms.push_back(ms);
      }
      const int cmin = b->h_out.p[out_n];
      if (cmin >= ng) break;  // no changed claim was read by a later group: every group saw its final input
      first = (int)(std::upper_bound(run.begin(), run.end(), cmin) - run.begin());
    }
    CK(cudaMemcpyAsync(b->h_out.p, b->out.p, out_n * 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return RBGTOPO_OK;
  }();
  if (rc) {
    cudaStreamSynchronize(s);
    release_batch(c, b);
    return rc;
  }
  const int32_t* a = b->h_out.p;
  if (total_r > 0) memcpy(assign, a, (size_t)total_r * 4);
  for (int g = 0; g < ng; ++g) {
    const int32_t* rec = gb + RBGTOPO_HDR_WORDS + (int64_t)g * RBGTOPO_GROUP_WORDS;
    const bool excl = (rec[1] & RBGTOPO_STEP_EXCLUSIVE) != 0;
    int st = RBGTOPO_PLACED_ALL, dm = excl ? rec[2] : -1;  // nothing pending: placed, the domain it occupies confirmed
    if (facts[g].nw > 0) {
      st = a[total_r + g];
      dm = excl ? a[total_r + ng + g] : -1;
    }
    if (status) status[g] = st;
    if (domain) domain[g] = dm;
  }
  int rank_launches = 0;
  if (rk && n0 > 0) {
    cm.g = ng;
    rc = rank_committed(c, b, gb, nullptr, assign, status, domain, cm, lv, *rk, &rank_launches);
    if (rc) {
      cudaStreamSynchronize(s);
      release_batch(c, b);
      return rc;
    }
  } else if (rk) {
    alt_clear(*rk, 0, total_r);
  }
  release_batch(c, b);
  *rounds_out = rounds;
  {
    rbgtopo_timing tm{};
    // kernels: the first claims build, then plan + diff + claims per round; ranked: score + k_alternates per chunk
    tm.launches = 3 * rounds + (n0 > 0 ? 1 : 0) + rank_launches;
    tm.h2d_words = (int32_t)std::min<long long>((long long)words + n0, INT32_MAX);
    std::lock_guard<std::mutex> g(c->stat_mu);
    c->last = tm;
    c->last_score_ms.assign(round_ms.size(), 0.0f);  // no dense matrix; one selection time per round
    c->last_select_ms = round_ms;
    c->calls += 1;
    c->launches += tm.launches;
  }
  return RBGTOPO_OK;
}

}  // namespace

namespace {
// rbgtopo_place_groups, and its ranked form when rk != nullptr (status and domain are then not null)
int32_t place_groups_impl(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t* assign, int32_t* status,
                          int32_t* domain, const RankReq* rk) {
  std::vector<char> dirty;
  {
    std::shared_lock<std::shared_mutex> lk(c->topo_mu);
    if (!c->topo.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
    if (rk && (size_t)((c->topo.n + 31) / 32) * 4 > kFastSmemMax)  // before placing: the ranking must not fail afterwards
      return fail(RBGTOPO_ELIMIT, "ranked placement: %d nodes exceed the room bitmap", c->topo.n);
    // before placing: a group the host loop re-runs must not meet the §3.4 bound in a later wave (§3.10).  Only
    // RBGTOPO_EINEXACT is returned here: a malformed blob gets the code the placement itself gives it.
    if (rk && groups_blob_ok(gb, words) && exact_one_pod(c, gb, words) == RBGTOPO_EINEXACT) return RBGTOPO_EINEXACT;
    CK(cudaSetDevice(c->cfg.device));
    static const bool prof = getenv("RBGTOPO_PROFILE_HOST") != nullptr;
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto us = [](auto a, auto b2) { return std::chrono::duration<double, std::micro>(b2 - a).count(); };
    // Optional (RBGTOPO_SPLIT_MIN_GROUPS): two pipelined halves (groups are independent, spec §3.7) —
    // the host computes the geometry of the second half while the device expands, scores and places
    // the first, and unpacks the first half's results while the second runs.  The GROUPS blob is
    // uploaded once.
    const int ng_all = words >= RBGTOPO_HDR_WORDS ? gb[2] : 0;
    const bool split = ng_all >= kSplitMinGroups && !kVerifyPlan && !rk;
    // the direct path (no expanded plan, nothing per step on the host) when it applies
    bool handled = false;
    const int drc = place_groups_direct(c, gb, words, assign, status, domain, &dirty, &handled, rk);
    if (drc) return drc;
    Batch* b = nullptr;
    int rc = handled ? RBGTOPO_OK : acquire_batch(c, &b);
    if (rc) return rc;
    static const bool no_early = getenv("RBGTOPO_NO_EARLY_EMIT") != nullptr;  // A/B switch
    if (handled) {
      // results and dirty groups are in place: the host loop for the latter follows below, outside the lock
    } else if (!split) {
      auto t0 = now();
      rc = plan_stage(c, b, gb, words, kSerialPlan && !no_early);  // early emit: the dense matrix starts while the host finishes the geometry
      auto t1 = now();
      if (!rc && kVerifyPlan) rc = verify_plan(c, b, gb, words);
      auto t2 = now();
      if (!rc) rc = run_batch(c, b, 1);
      auto t3 = now();
      if (!rc) rc = fetch_batch(c, b, nullptr, nullptr, nullptr);
      auto t4 = now();
      if (!rc) plan_results(b, assign, status, domain, &dirty);
      if (!rc && rk) rc = rank_plan(c, b, gb, assign, status, domain, dirty, *rk);
      if (prof)
        fprintf(stderr, "[rbgtopo host] plan+stage %.0f us, verify %.0f us, enqueue %.0f us, wait+fetch %.0f us, results %.0f us\n",
                us(t0, t1), us(t1, t2), us(t2, t3), us(t3, t4), us(t4, now()));
      if (rc) cudaStreamSynchronize(stream_of(c, b));
      release_batch(c, b);
      if (rc) return rc;
    } else {
      Batch* b2 = nullptr;
      rc = acquire_batch(c, &b2);
      if (rc) {
        release_batch(c, b);
        return rc;
      }
      const int mid = ng_all / 2;
      auto t0 = now();
      rc = plan_stage(c, b, gb, words, kSerialPlan && !no_early, 0, mid);
      if (!rc) rc = run_batch(c, b, 1);
      if (!rc) rc = enqueue_d2h(c, b);
      auto t1 = now();
      if (!rc) rc = plan_stage(c, b2, gb, words, kSerialPlan && !no_early, mid, ng_all, b->m.total_r, b->gsrc.p, b->ev[2]);  // ev[2]: the blob is up
      if (!rc) rc = run_batch(c, b2, 1);
      if (!rc) rc = enqueue_d2h(c, b2);
      auto t2 = now();
      rbgtopo_timing first{};
      if (!rc) rc = fetch_batch(c, b, nullptr, nullptr, nullptr);
      auto t3 = now();
      if (!rc) {
        std::lock_guard<std::mutex> g(c->stat_mu);
        first = c->last;
      }
      if (!rc) plan_results(b, assign, status, domain, &dirty);
      auto t4 = now();
      if (!rc) rc = fetch_batch(c, b2, nullptr, nullptr, nullptr);
      auto t5 = now();
      if (!rc) plan_results(b2, assign, status, domain, &dirty);
      if (!rc) {
        std::lock_guard<std::mutex> g(c->stat_mu);
        c->last = add_timing(first, c->last);
      }
      if (prof)
        fprintf(stderr, "[rbgtopo host] half 1 plan+enqueue %.0f us, half 2 plan+enqueue %.0f us, wait 1 %.0f us, results 1 %.0f us, "
                        "wait 2 %.0f us, results 2 %.0f us\n",
                us(t0, t1), us(t1, t2), us(t2, t3), us(t3, t4), us(t4, t5), us(t5, now()));
      if (rc) {
        cudaStreamSynchronize(stream_of(c, b));
        cudaStreamSynchronize(stream_of(c, b2));
      }
      release_batch(c, b2);
      release_batch(c, b);
      if (rc) return rc;
    }
  }
  bool any = false;
  for (char d : dirty) any |= d != 0;
  if (!any) return RBGTOPO_OK;
  return place_groups_slow(c, gb, words, assign, status, domain, &dirty, rk);
}
}  // namespace

// ---- leader-worker replicas (rbgtopo_place_groups_lw, DESIGN.md §3.11)
namespace {
// Validation: the checks and messages of rbgtopo_place_groups (group_facts phase 1, offsets), the role_pods table, then
// group_facts phase 2 (scheduled pods, exactness bound) with the bound taken over the pod waves.
int lw_validate(rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* rp, int64_t rp_words) {
  if (const int hrc = check_groups_blob(gb, words)) return hrc;
  const int ng = gb[2];
  const TopoHost th = topo_host(c, places_levels(c));
  GroupFacts f;
  for (int g = 0; g < ng; ++g) {
    int rc = group_facts(th, gb, words, g, true, &f, 1);
    if (rc) return rc;
  }
  long long pacc = 0, qsum = 0;
  for (int g = 0; g < ng; ++g) {
    const int32_t* rec = group_rec(gb, g);
    long long pend = 0;
    for (int i = 0; i < rec[3]; ++i) pend += gb[rec[4] + 4 * i + 1];
    if (rec[8] != pacc || rec[9] != pend) return fail(RBGTOPO_EINVAL, "group %d: bad assign_off/n_pending", g);
    pacc += pend;
    if (pacc > 0x3FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "pending replicas exceed 2^30");
    qsum += rec[3];
  }
  if (gb[4] != pacc) return fail(RBGTOPO_EINVAL, "total pending mismatch");
  if (!rp || rp_words != 2 * qsum)
    return fail(RBGTOPO_EINVAL, "role_pods: %lld words for %lld roles (2 per role)", (long long)rp_words, qsum);
  const int nl = installed_levels(c);
  long long pods = 0;
  const long long sat = 1LL << 40;
  for (int g = 0, r0 = 0; g < ng; ++g) {
    const int32_t* rec = group_rec(gb, g);
    const int q = rec[3];
    const int32_t* roles = gb + rec[4];
    const int32_t* pair = gb + rec[5];
    const int32_t* grp = rp + 2LL * r0;
    r0 += q;
    for (int i = 0; i < q; ++i) {
      if (grp[2 * i] < 1 || grp[2 * i] > RBGTOPO_MAX_STEP_REPLICAS)
        return fail(RBGTOPO_EINVAL, "group %d role %d: %d pods per replica (1 .. %d)", g, i, grp[2 * i], RBGTOPO_MAX_STEP_REPLICAS);
      if (grp[2 * i + 1] < -1 || grp[2 * i + 1] > nl)
        return fail(RBGTOPO_EINVAL, "group %d role %d: co-location level %d (-1 .. %d installed)", g, i, grp[2 * i + 1], nl);
      pods += (long long)roles[4 * i + 1] * grp[2 * i];
    }
    if (pods > 0x3FFFFFF0LL) return fail(RBGTOPO_ELIMIT, "pending pods exceed 2^30");
    // The exactness bound of §3.4 per role over the pod waves: the largest need·F_CAP + sum_j pair·(pods of j placed
    // before the wave) any wave of the call can stage.  A gang group stops at its first wave with an unplaced replica,
    // so every earlier pod is placed.  Any other group may reach a wave with pods of earlier waves unplaced: each one
    // raises need by 1 (up to the cap) and lowers the anchor weight by its pair weight, so the bound takes the worst
    // such mix — the per-wave validation can then never find an inexact step in the middle of a call.
    const bool gang = (rec[1] & RBGTOPO_STEP_GANG) != 0;
    long long bound[RBGTOPO_MAX_GROUP_ROLES] = {0}, placed[RBGTOPO_MAX_GROUP_ROLES] = {0};
    walk_waves(roles, q, grp, [&](int, const PlanWave& w) {
      for (int k = 0; k < w.n; ++k) {
        const int ri = w.role[k];
        long long need = 0, bnd = 0;
        for (int j = 0; j < q; ++j) {
          if (pair[ri * q + j] > 0) need += (long long)roles[4 * j + 1] * grp[2 * j] - placed[j];
          bnd = std::min(bnd + (long long)pair[ri * q + j] * placed[j], sat);
        }
        bnd += std::min<long long>(need, RBGTOPO_NEED_CAP) * RBGTOPO_F_CAP;
        long long left[RBGTOPO_MAX_GROUP_ROLES];  // earlier pods that may still be unplaced, per role
        for (int j = 0; j < q; ++j) left[j] = gang ? 0 : placed[j];
        for (long long room = RBGTOPO_NEED_CAP - std::min<long long>(need, RBGTOPO_NEED_CAP); room > 0;) {
          int best = -1;  // the smallest pair weight in (0, F_CAP) gains the most per unplaced pod
          for (int j = 0; j < q; ++j)
            if (left[j] > 0 && pair[ri * q + j] > 0 && pair[ri * q + j] < RBGTOPO_F_CAP &&
                (best < 0 || pair[ri * q + j] < pair[ri * q + best]))
              best = j;
          if (best < 0) break;
          const long long u = std::min(room, left[best]);
          bnd += u * (RBGTOPO_F_CAP - pair[ri * q + best]);
          room -= u;
          left[best] = 0;
        }
        bound[ri] = std::max(bound[ri], bnd);
      }
      for (int k = 0; k < w.n; ++k) placed[w.role[k]] += (long long)w.count[k] * grp[2 * w.role[k]];
    });
    int rc = group_facts(th, gb, words, g, true, &f, 2, bound);
    if (rc) return rc;
  }
  return RBGTOPO_OK;
}

// One CTA per step up to the CTAs that fit the device at once; with a co-location level in the wave, no more CTAs
// than kLwScratchBytes of level-C domain scratch (12 bytes per domain) allow.
constexpr size_t kLwScratchBytes = 64u << 20;

// What a group of a committed leader-worker batch takes from the groups after it (§3.13): (node, demand) of its placed
// pods, aggregated by node, and the exclusive domain it reports (-1 = none) at its level.  At levels (§3.16) also the
// nodes of its placed participating pods (sorted), which later groups keyed at other levels read.  A gang-failed group
// takes nothing.
struct LwClaims {
  std::vector<std::pair<int, int>> cap;
  std::vector<int> pods;
  int dom = -1, gid = -1;
  bool operator==(const LwClaims& o) const { return cap == o.cap && pods == o.pods && dom == o.dom && gid == o.gid; }
};

// The claim lists of a committed leader-worker batch at levels (§3.16), in the layout commit_owner<true> reads, built
// from every group's claims: a reporting group h links into dhead[doff[L_h] + D] (dclaim[h] = {gid, next}), each
// placed participating pod into phead[doff[L] + dom_L(node)] for every level L != L_h of lmask (pclaim = {group, gid,
// next, 0}).  Only the heads a list starts at are written (k_set_heads): `heads` maps a slot of cm_int (phead after
// the lvl_total_d dhead slots) to its first entry, and holds -1 for the slots the previous lists used.  What a round
// uploads grows with the groups and the placed pods, not with the size of the claimed domains.
struct LwLists {
  std::vector<int2> dclaim;
  std::vector<int4> pclaim;
  std::map<int, int> heads;
  void build(const Topology& T, const int32_t* gb, const std::vector<LwClaims>& claims, int lmask) {
    for (auto& kv : heads) kv.second = -1;
    const int ng = (int)claims.size();
    dclaim.assign((size_t)std::max(ng, 1), make_int2(-1, -1));
    pclaim.clear();
    int doff[RBGTOPO_MAX_EXCL_LEVELS + 1] = {0};
    for (int L = 0; L < T.n_levels + 1 && L < RBGTOPO_MAX_EXCL_LEVELS; ++L) doff[L + 1] = doff[L] + level_domains(T, L);
    auto head = [&](int slot) -> int& { return heads.emplace(slot, -1).first->second; };
    for (int g = 0; g < ng; ++g) {
      const LwClaims& cl = claims[g];
      const int lh = group_rec(gb, g)[10];
      if (cl.dom >= 0) {
        int& h = head(doff[lh] + cl.dom);
        dclaim[g] = make_int2(cl.gid, h);
        h = g;
      }
      for (const int node : cl.pods)
        for (int m = lmask; m; m &= m - 1) {
          const int L = __builtin_ctz(m);
          if (L == lh) continue;
          const int d = L == 0 ? T.h_domain[node] : T.h_lvl_domain[(size_t)(L - 1) * T.n + node];
          int& h = head(T.lvl_total_d + doff[L] + d);
          pclaim.push_back(make_int4(g, cl.gid, h, 0));
          h = (int)pclaim.size() - 1;
        }
    }
  }
};

// The committed rounds of a leader-worker batch (§3.13): every group's claims as the latest round left them, and what a
// round hands the groups it re-runs.  Capacity claims seed a run's `taken`.  Owner claims are, in a batch at level 0,
// the (node, claim gid) records of every node of a claimed domain, per step in the wave's side table; in a batch with a
// group at a level >= 1 (§3.16), the claim lists of commit_owner<true> (LwLists) over the levels of the batch's
// exclusive groups (lmask), read through cm.
struct LwRounds {
  const Topology& T;
  const int32_t* gb;
  int ng, lmask = 0;
  bool at_lv = false;
  std::vector<LwClaims> claims;
  std::vector<int> dom_ptr, dom_nodes;  // level 0: the nodes of every level-0 domain
  std::vector<std::pair<int, int>> oc;  // level 0: a run's owner claims as (node, gid) while seed sorts them
  LwLists lists;
  CommitDev cm{};  // at levels: the lists' heads live in cm_int (dhead | phead, all -1 at the start of the call)
  int lo = 0, n_rounds = 0;  // the round's first group, rounds run
  int list_launches = 0;
  long long list_words = 0;
  size_t sec_at = 0, rec_at = 0;  // the wave's claim section in the side table; at level 0 its records, 8-byte aligned
  LwRounds(const Topology& topo, const int32_t* groups) : T(topo), gb(groups), ng(groups[2]), claims((size_t)groups[2]) {}
  int init(const rbgtopo_ctx* c) {
    for (int g = 0; g < ng; ++g) {
      const int32_t* rec = group_rec(gb, g);
      if (rec[10] > 0 && !(c->cfg.flags & RBGTOPO_CFG_LW_COMMIT_LEVELS))
        return fail(RBGTOPO_ELIMIT, "committed leader-worker batch: group %d is exclusive at level %d; only level 0 is "
                                    "committed without RBGTOPO_CFG_LW_COMMIT_LEVELS", g, rec[10]);
      at_lv |= rec[10] > 0;
      if (rec[1] & RBGTOPO_STEP_EXCLUSIVE) lmask |= 1 << rec[10];
    }
    if (at_lv) return RBGTOPO_OK;
    dom_ptr.assign((size_t)T.n_domains + 1, 0);
    for (int n = 0; n < T.n; ++n) ++dom_ptr[T.h_domain[n] + 1];
    for (int d = 0; d < T.n_domains; ++d) dom_ptr[d + 1] += dom_ptr[d];
    dom_nodes.resize(T.n);
    std::vector<int> fill(dom_ptr.begin(), dom_ptr.end() - 1);
    for (int n = 0; n < T.n; ++n) dom_nodes[fill[T.h_domain[n]]++] = n;
    return RBGTOPO_OK;
  }
  // At levels: the dense head arrays in b->cm_int, cleared once per call.
  int start(Batch* b, cudaStream_t s) {
    if (!at_lv) return RBGTOPO_OK;
    CK(b->cm_int.reserve(2 * (size_t)T.lvl_total_d));
    CK(cudaMemsetAsync(b->cm_int.p, 0xFF, 2 * (size_t)T.lvl_total_d * 4, s));
    cm.dhead = b->cm_int.p;
    cm.phead = b->cm_int.p + T.lvl_total_d;
    cm.ldom = T.lvl_domain.p;
    cm.doff = T.lvl_doff.p;
    cm.lstride = level_stride(T.n);
    cm.lmask = lmask;
    cm.occ = true;  // levels >= 1 exist in occupancy mode only
    return RBGTOPO_OK;
  }
  // At levels: the lists of the current claims, with the heads that changed written by k_set_heads.
  int upload(Batch* b, cudaStream_t s) {
    lists.build(T, gb, claims, lmask);
    std::vector<int2> set;
    for (const auto& [slot, first] : lists.heads) set.push_back(make_int2(slot, first));
    for (auto it = lists.heads.begin(); it != lists.heads.end();)  // slots back at -1 need no reset next time
      it = it->second < 0 ? lists.heads.erase(it) : std::next(it);
    const size_t o_d = 2 * set.size(), o_p = (o_d + 2 * lists.dclaim.size() + 3) & ~(size_t)3;  // int4-aligned
    const size_t w = o_p + 4 * lists.pclaim.size();
    CK(b->lwc.reserve(w + 4));
    CK(b->h_lwc.reserve(w + 4));
    memcpy(b->h_lwc.p, set.data(), set.size() * 8);
    memcpy(b->h_lwc.p + o_d, lists.dclaim.data(), lists.dclaim.size() * 8);
    memcpy(b->h_lwc.p + o_p, lists.pclaim.data(), lists.pclaim.size() * 16);
    CK(cudaMemcpyAsync(b->lwc.p, b->h_lwc.p, w * 4, cudaMemcpyHostToDevice, s));
    if (!set.empty()) {
      k_set_heads<<<(unsigned)std::min<size_t>((set.size() + 255) / 256, 1024), 256, 0, s>>>(
          b->cm_int.p, reinterpret_cast<const int2*>(b->lwc.p), (int)set.size());
      CK(cudaGetLastError());
      ++list_launches;
    }
    cm.dclaim = reinterpret_cast<const int2*>(b->lwc.p + o_d);
    cm.pclaim = reinterpret_cast<int4*>(b->lwc.p + o_p);
    list_words += (long long)w;
    return RBGTOPO_OK;
  }
  // The start of a round: every run of [lo, ng) starts from the claims of the groups before it.
  int seed(std::vector<HostRun>& runs, Batch* b, cudaStream_t s) {
    if (at_lv)
      if (const int rc = upload(b, s)) return rc;
    std::map<int, int> cap, own;  // node -> capacity taken; level-0 domain -> gid of its last reporter
    for (int g = 0; g < ng; ++g) {
      if (g >= lo) {
        HostRun& r = runs[g];
        r.taken = cap;
        if (!at_lv && (r.rec[1] & RBGTOPO_STEP_EXCLUSIVE)) {
          oc.clear();
          for (const auto& [d, gid] : own)
            for (int k = dom_ptr[d]; k < dom_ptr[d + 1]; ++k) oc.emplace_back(dom_nodes[k], gid);
          std::sort(oc.begin(), oc.end());
          for (const auto& [n, gid] : oc) { r.owner_claims.push_back(n); r.owner_claims.push_back(gid); }
        }
      }
      for (const auto& [n, a] : claims[g].cap) cap[n] += a;
      if (claims[g].dom >= 0) own[claims[g].dom] = claims[g].gid;
    }
    return RBGTOPO_OK;
  }
  // The claim section of a wave's side table (active: the steps' groups): at levels the group index of every step; at
  // level 0 per step the offsets of its owner claims, then the (node, gid) records.
  void add_side(const std::vector<HostRun>& runs, const std::vector<int>& active, std::vector<int32_t>& side) {
    sec_at = side.size();
    if (at_lv) {
      side.insert(side.end(), active.begin(), active.end());
      return;
    }
    int acc = 0;
    side.push_back(0);
    for (int i : active) side.push_back(acc += (int)runs[i].owner_claims.size() / 2);
    if (side.size() & 1) side.push_back(0);
    rec_at = side.size();
    for (int i : active) side.insert(side.end(), runs[i].owner_claims.begin(), runs[i].owner_claims.end());
  }
  // The wave's dense rows, with the owner claims of the earlier groups (lw: the side table on the device; admit: its
  // mask section in the eligible form, §3.20).
  int score(rbgtopo_ctx* c, Batch* b, cudaStream_t s, const int* lw, const unsigned long long* admit) const {
    return at_lv ? launch_score(c, b, s, nullptr, nullptr, lw + sec_at, &cm, admit)
                 : launch_score(c, b, s, lw + sec_at, reinterpret_cast<const int2*>(lw + rec_at), nullptr, nullptr, admit);
  }
  // The end of a round: the new claims of the groups it ran.  c = the lowest group whose claims changed; groups <= c
  // saw their final input.  Returns whether another round is needed; it starts at c + 1.
  bool settle(const std::vector<HostRun>& runs, const int32_t* assign) {
    ++n_rounds;
    int cmin = -1;
    for (int g = lo; g < ng; ++g) {
      const HostRun& r = runs[g];
      LwClaims nc;
      if (!r.failed) {
        std::map<int, int> cap;
        for (int i = 0; i < r.q; ++i)
          for (long long k = 0; k < (long long)r.roles[4 * i + 1] * r.rp[2 * i]; ++k)
            if (const int node = assign[r.pod0 + r.ord0[i] + k]; node >= 0) cap[node] += r.roles[4 * i + 2];
        nc.cap.assign(cap.begin(), cap.end());
        if ((r.rec[1] & RBGTOPO_STEP_EXCLUSIVE) && r.fixed_domain >= 0) {
          nc.dom = r.fixed_domain;
          nc.gid = r.rec[0];
        }
        if (at_lv && (r.rec[1] & RBGTOPO_STEP_EXCLUSIVE)) {  // the placed pods of its participating roles
          for (int i = 0; i < r.q; ++i)
            if (r.roles[4 * i + 3] & RBGTOPO_ROLE_EXCLUSIVE)
              for (long long k = 0; k < (long long)r.roles[4 * i + 1] * r.rp[2 * i]; ++k)
                if (const int node = assign[r.pod0 + r.ord0[i] + k]; node >= 0) nc.pods.push_back(node);
          std::sort(nc.pods.begin(), nc.pods.end());
          if (!nc.pods.empty()) nc.gid = r.rec[0];
        }
      }
      if (cmin < 0 && !(nc == claims[g])) cmin = g;
      claims[g] = std::move(nc);
    }
    if (cmin < 0 || cmin + 1 >= ng) return false;
    lo = cmin + 1;
    return true;
  }
  // The end of the rounds, which ended with rc.  rk: the committed ranked form (§3.15), rank_committed against every
  // group's final claims, the lists of commit_owner<true> at levels, and at level 0 the owner lists of
  // commit_owner<false> (HostClaims), which are LwLists' dhead / dclaim.  What the claim lists took (k_set_heads
  // launches, uploaded words) counts toward a call that succeeds.
  // admit: the class masks of the eligible form (§3.20), which the replay applies to its rows.
  int finish(rbgtopo_ctx* c, Batch* b, int rc, const int32_t* rp, const int32_t* assign, const int32_t* status,
             const int32_t* domain, const RankReq* rk, rbgtopo_timing& total, const uint64_t* admit) {
    int rank_launches = 0;
    if (!rc && rk) {
      HostClaims hc;
      if (at_lv) {
        rc = upload(b, stream_of(c, b));
      } else {
        lists.build(T, gb, claims, lmask);
        hc.dhead.assign((size_t)T.n_domains, -1);
        for (const auto& [d, first] : lists.heads) hc.dhead[d] = first;
        hc.dclaim = std::move(lists.dclaim);
        cm.occ = T.occ;
      }
      cm.g = ng;
      if (!rc)
        rc = rank_committed(c, b, gb, rp, assign, status, domain, cm, at_lv, *rk, &rank_launches, at_lv ? nullptr : &hc,
                            admit);
    }
    std::lock_guard<std::mutex> g(c->stat_mu);
    total.launches += rank_launches;
    c->launches += rank_launches;
    if (rc) return rc;
    total.launches += list_launches;
    total.h2d_words += (int32_t)std::min<long long>(list_words, INT32_MAX);
    c->launches += list_launches;
    return RBGTOPO_OK;
  }
};

// rk != nullptr: the ranked form (§3.12).  The matrix is overwritten by every wave, so each wave's rows are copied
// out before the next wave scores (one copy per wave); once the placements are final one k_alternates launch ranks
// the rows of every (wave, role) that placed a pod.
// rounds != nullptr: the committed form (§3.13, LwRounds).  A round runs the wave loop for groups [lo, ng); group g
// sees the claims of groups < g as the previous round left them (final below lo).  c = the lowest group whose claims
// changed: groups <= c saw their final input, the next round starts at c + 1, and a round that changes nothing ends
// the call.
// Both: the committed ranked form (§3.15).  The rounds keep no rows (a re-run would keep its rows again); once they
// converge, rank_committed replays the rows of every group's final run and ranks them after the whole batch.
// admit != nullptr: the eligible form (§3.19), n_admit class masks, one per role in blob order; every wave's rows are
// written by k_score_emit_elig with the masks of its role rows, carried after the (S, C) section of the side table.
int place_groups_lw(rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* rp, int64_t rp_words,
                    int32_t* assign, int32_t* status, int32_t* domain, const RankReq* rk = nullptr,
                    int32_t* rounds = nullptr, const uint64_t* admit = nullptr, int64_t n_admit = 0) {
  int rc = lw_validate(c, gb, words, rp, rp_words);
  if (rc) return rc;
  const Topology& T = c->topo;
  const int ng = gb[2];
  if (admit) {
    if (T.n_classes < 1) return fail(RBGTOPO_EINVAL, "eligible placement: no node classes installed (rbgtopo_set_node_classes)");
    if (n_admit != rp_words / 2)
      return fail(RBGTOPO_EINVAL, "role_admit: %lld masks for %lld roles", (long long)n_admit, (long long)(rp_words / 2));
  }
  std::optional<LwRounds> cr;  // the committed rounds
  if (rounds && (rc = cr.emplace(T, gb).init(c))) return rc;
  const size_t smem = (size_t)((T.n + 31) / 32) * 4;
  if (smem > kFastSmemMax) return fail(RBGTOPO_ELIMIT, "leader-worker placement: %d nodes exceed the room bitmap", T.n);
  const GroupOffsets off(gb, rp);
  std::vector<HostRun> runs(ng);
  auto init_run = [&](int g) {
    runs[g] = HostRun(gb, g, off.grp(rp, g), off.pod0[g]);
    for (int64_t k = off.pod0[g]; k < off.pod0[g + 1]; ++k) assign[k] = -1;
  };
  const bool keep = rk && !rounds;
  // world > 1 (RBGTOPO_CFG_LW_SHARDS or a sharded ranked form, §3.18): k_lw_assign_repl evaluates the rows from the
  // snapshot; the slab rows are emitted only where a ranking reads them (kept per wave; a committed ranking replays them)
  const bool repl = c->cfg.world > 1, emit = !repl || keep;
  KeptRows kept;
  for (int g = 0; g < ng; ++g) {
    init_run(g);
    if (keep) kept.cap += group_role_rows(gb, g, off.grp(rp, g));
  }
  LwLevels lv{};
  for (int L = 0; L <= installed_levels(c); ++L) lv.nd[L] = level_domains(T, L);

  Batch* b = nullptr;
  rc = acquire_batch(c, &b);
  if (rc) return rc;
  cudaStream_t s = stream_of(c, b);
  if (keep) rc = reserve_kept(c, b, kept.cap);
  if (!rc && cr) rc = cr->start(b, s);
  std::vector<int32_t> side;  // per wave: the (S, C) of every role row of every step, then the claim section
  auto launch = [&](const std::vector<int>& active) -> int {
    const int ns = (int)active.size();
    side.assign((size_t)ns * MAXP, 0);
    int dmax = 0;
    for (int i = 0; i < ns; ++i) {
      const HostRun& r = runs[active[i]];
      for (int p = 0; p < r.w.n; ++p) {
        const int ri = r.w.role[p], C = r.rp[2 * ri + 1];
        side[(size_t)i * MAXP + p] = lw_pack_role(r.S(ri), C);
        if (C >= 0) dmax = std::max(dmax, lv.nd[C]);
      }
    }
    if (cr) cr->add_side(runs, active, side);
    // admit: MAXP masks per step, read as u64.  The (S, C) section is even (MAXP is); the claim section at levels is
    // one int per step, so an odd step count is padded to an even word here.
    static_assert(MAXP % 2 == 0, "the (S, C) section ends 8-byte aligned");
    if (admit && (side.size() & 1)) side.push_back(0);
    const size_t admit_at = side.size();
    if (admit) {
      side.resize(admit_at + (size_t)ns * MAXP * 2, 0);
      for (int i = 0; i < ns; ++i) {
        const HostRun& r = runs[active[i]];
        for (int p = 0; p < r.w.n; ++p)
          memcpy(side.data() + admit_at + 2 * ((size_t)i * MAXP + p), &admit[off.r0[r.g] + r.w.role[p]], 8);
      }
    }
    // grid: every step resident at once if the device holds them, the level-C scratch bounded by kLwScratchBytes
    const auto repl_k = !cr ? k_lw_assign_repl<LW_REPL>
                        : cr->at_lv ? k_lw_assign_repl<LW_REPL_CLAIMS_LV> : k_lw_assign_repl<LW_REPL_CLAIMS>;
    int per_sm = 0;
    if (repl) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, repl_k, LW_THREADS, smem));
    else CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_lw_assign, LW_THREADS, smem));
    long long grid = std::min<long long>(ns, (long long)std::max(1, per_sm) * c->sm_count);
    if (dmax > 0) grid = std::min<long long>(grid, std::max<long long>(1, kLwScratchBytes / (12LL * dmax)));
    CK(b->lw.reserve(side.size()));
    CK(b->h_lw.reserve(side.size()));
    CK(b->lw_best.reserve((size_t)grid * dmax + 1));
    CK(b->lw_cap.reserve((size_t)grid * dmax + 1));
    memcpy(b->h_lw.p, side.data(), side.size() * 4);
    CK(cudaMemcpyAsync(b->lw.p, b->h_lw.p, side.size() * 4, cudaMemcpyHostToDevice, s));
    CK(cudaStreamWaitEvent(s, c->base_ready, 0));  // a pending snapshot refresh
    CK(cudaStreamWaitEvent(s, c->topo_ready, 0));
    const auto* adm = admit ? reinterpret_cast<const unsigned long long*>(b->lw.p + admit_at) : nullptr;
    if (emit)
      if (const int r2 = cr ? cr->score(c, b, s, b->lw.p, adm)
                            : launch_score(c, b, s, nullptr, nullptr, nullptr, nullptr, adm))
        return r2;
    if (!repl) {
      k_lw_assign<<<(unsigned)grid, LW_THREADS, smem, s>>>(topo_dev(c), batch_dev(c, b), b->lw.p, b->lw_best.p,
                                                           b->lw_cap.p, dmax, lv);
    } else {  // the patch tables: one record of 2 + max_p words per patched node of a step
      const int w = 2 + b->m.max_p;
      CK(b->corr.reserve((size_t)b->m.patch_cap * w + 1));
      BatchDev d = batch_dev(c, b);
      d.corr = b->corr.p;
      d.corr_w = w;
      const int* co = cr ? b->lw.p + cr->sec_at : nullptr;
      const int2* cl = cr && !cr->at_lv ? reinterpret_cast<const int2*>(b->lw.p + cr->rec_at) : nullptr;
      repl_k<<<(unsigned)grid, LW_THREADS, smem, s>>>(topo_dev(c), d, b->lw.p, b->lw_best.p, b->lw_cap.p, dmax, lv, co,
                                                      cl, T.occ, cr ? cr->cm : CommitDev{});
    }
    CK(cudaGetLastError());
    const int launched = emit ? 2 : 1;
    b->pend_launches += launched;
    b->ran = true;
    std::lock_guard<std::mutex> g(c->stat_mu);
    c->launches += launched;
    return RBGTOPO_OK;
  };
  rbgtopo_timing total{};
  WaveBufs wb;
  while (!rc) {  // the rounds; one when not committed
    if (cr && (rc = cr->seed(runs, b, s))) break;
    rc = run_waves(c, b, runs, cr ? cr->lo : 0, assign, status, domain, keep ? &kept : nullptr, total, wb, launch);
    if (rc || !cr || !cr->settle(runs, assign)) break;
    for (int g = cr->lo; g < ng; ++g) init_run(g);
  }
  if (cr) {
    *rounds = cr->n_rounds;
    rc = cr->finish(c, b, rc, rp, assign, status, domain, rk, total, admit);
  }
  if (!rc) harvest_base_ms(c);
  // The waves record no pass events, so their pass times are 0, unless the pooled batch still holds those of a staged
  // pass released without a fetch; those are not this call's.
  total.score_ms = total.select_ms = 0.f;
  return finish_waves(c, b, rc, total, runs, keep ? &kept : nullptr, gb, rp, assign, status, domain, rk);
}

// The entry checks of every rbgtopo_place_groups* function, in this order: rounds = 0, null arguments, n_alt, world
// == 1 (a leader-worker form without ranking also at world > 1 on a ctx with RBGTOPO_CFG_LW_SHARDS, §3.18), lock /
// topology / device, own status and domain for a ranked form given NULL; then the placement of `form`.
// rbgtopo_place_groups and its ranked form take the lock inside place_groups_impl, which releases it before the
// host-driven re-run.  kPlaceShard (with kPlaceRanked, x != nullptr): the local half of §3.17, valid at any world; the
// slab lists go to x and the outputs score / alt_node / alt_score are the merge's.
enum PlaceForm { kPlaceReplicas = 0, kPlaceCommitted = 1, kPlaceLw = 2, kPlaceRanked = 4, kPlaceShard = 8 };
// admit: the class masks of the eligible forms (§3.19, kPlaceLw only), n_admit of them.
int32_t place_entry(int form, rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* rp, int64_t rp_words,
                    int32_t n_alt, int32_t* assign, int32_t* status, int32_t* domain, int32_t* rounds, float* score,
                    int32_t* alt_node, float* alt_score, AltExchange* x = nullptr, const uint64_t* admit = nullptr,
                    int64_t n_admit = 0) {
  const bool committed = form & kPlaceCommitted, lw = form & kPlaceLw, ranked = form & kPlaceRanked;
  const bool shard = form & kPlaceShard;
  if (rounds) *rounds = 0;
  if (!c || !gb || !assign || (lw && !rp) ||
      (ranked && !shard && (!score || (n_alt > 0 && (!alt_node || !alt_score)))))
    return fail(RBGTOPO_EINVAL, "null argument");
  if (ranked && (n_alt < 0 || n_alt > RBGTOPO_MAX_ALTERNATES))
    return fail(RBGTOPO_EINVAL, "n_alt %d outside [0, %d]", n_alt, RBGTOPO_MAX_ALTERNATES);
  if ((ranked || lw) && !shard && c->cfg.world > 1 && !(lw && !ranked && lw_shards(c)))
    return fail(RBGTOPO_ELIMIT, "%s needs world == 1: a rank holds only its slab of every dense row",
                !lw ? "ranked placement" : committed ? "committed leader-worker placement" : "leader-worker placement");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu, std::defer_lock);  // one snapshot for the rounds and the ranking
  if (committed || lw) {
    lk.lock();
    if (!c->topo.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
    CK(cudaSetDevice(c->cfg.device));
  }
  std::vector<int32_t> own_status, own_domain;  // status / domain may be NULL: the ranking still needs them
  if (ranked) {
    const int64_t ng = words >= RBGTOPO_HDR_WORDS ? std::max<int64_t>(0, std::min<int64_t>(gb[2], words / RBGTOPO_GROUP_WORDS)) : 0;
    if (!status) { own_status.resize((size_t)ng + 1); status = own_status.data(); }
    if (!domain) { own_domain.resize((size_t)ng + 1); domain = own_domain.data(); }
  }
  const RankReq rk{n_alt, score, alt_node, alt_score, shard ? x : nullptr};
  const RankReq* rkp = ranked ? &rk : nullptr;
  if (!lw && !committed) return place_groups_impl(c, gb, words, assign, status, domain, rkp);
  int32_t r = 0;
  const int rc = lw ? place_groups_lw(c, gb, words, rp, rp_words, assign, status, domain, rkp, committed ? &r : nullptr,
                                     admit, n_admit)
                    : place_groups_committed(c, gb, words, assign, status, domain, &r, rkp);
  if (rounds) *rounds = r;
  return rc;
}
}  // namespace

int32_t rbgtopo_place_groups(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t* assign,
                             int32_t* status, int32_t* domain) {
  return place_entry(kPlaceReplicas, c, gb, words, nullptr, 0, 0, assign, status, domain, nullptr, nullptr, nullptr,
                     nullptr);
}

int32_t rbgtopo_place_groups_ranked(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t n_alt, int32_t* assign,
                                    int32_t* status, int32_t* domain, float* score, int32_t* alt_node, float* alt_score) {
  return place_entry(kPlaceRanked, c, gb, words, nullptr, 0, n_alt, assign, status, domain, nullptr, score, alt_node,
                     alt_score);
}

int32_t rbgtopo_place_groups_committed(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t* assign,
                                       int32_t* status, int32_t* domain, int32_t* rounds) {
  return place_entry(kPlaceCommitted, c, gb, words, nullptr, 0, 0, assign, status, domain, rounds, nullptr, nullptr,
                     nullptr);
}

int32_t rbgtopo_place_groups_committed_ranked(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t n_alt,
                                              int32_t* assign, int32_t* status, int32_t* domain, int32_t* rounds,
                                              float* score, int32_t* alt_node, float* alt_score) {
  return place_entry(kPlaceCommitted | kPlaceRanked, c, gb, words, nullptr, 0, n_alt, assign, status, domain, rounds,
                     score, alt_node, alt_score);
}

int32_t rbgtopo_place_groups_lw(rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* role_pods,
                                int64_t role_pods_words, int32_t* assign, int32_t* status, int32_t* domain) {
  return place_entry(kPlaceLw, c, gb, words, role_pods, role_pods_words, 0, assign, status, domain, nullptr, nullptr,
                     nullptr, nullptr);
}

int32_t rbgtopo_place_groups_lw_ranked(rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* role_pods,
                                       int64_t role_pods_words, int32_t n_alt, int32_t* assign, int32_t* status,
                                       int32_t* domain, float* score, int32_t* alt_node, float* alt_score) {
  return place_entry(kPlaceLw | kPlaceRanked, c, gb, words, role_pods, role_pods_words, n_alt, assign, status, domain,
                     nullptr, score, alt_node, alt_score);
}

int32_t rbgtopo_place_groups_lw_committed(rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* role_pods,
                                          int64_t role_pods_words, int32_t* assign, int32_t* status, int32_t* domain,
                                          int32_t* rounds) {
  return place_entry(kPlaceLw | kPlaceCommitted, c, gb, words, role_pods, role_pods_words, 0, assign, status, domain,
                     rounds, nullptr, nullptr, nullptr);
}

int32_t rbgtopo_place_groups_lw_committed_ranked(rbgtopo_ctx* c, const int32_t* gb, int64_t words,
                                                 const int32_t* role_pods, int64_t role_pods_words, int32_t n_alt,
                                                 int32_t* assign, int32_t* status, int32_t* domain, int32_t* rounds,
                                                 float* score, int32_t* alt_node, float* alt_score) {
  return place_entry(kPlaceLw | kPlaceCommitted | kPlaceRanked, c, gb, words, role_pods, role_pods_words, n_alt, assign,
                     status, domain, rounds, score, alt_node, alt_score);
}

// ---- node eligibility (DESIGN.md §3.19) -------------------------------------------------------------------------------
namespace {
// The eligible forms: the leader-worker loop with class masks.  role_pods == NULL stands for (S, C) = (1, -1) for every
// role, which places replicas exactly as rbgtopo_place_groups[_ranked] does.  world > 1 is refused before anything runs.
// committed (§3.20): the committed leader-worker rounds with the same masks; rounds as rbgtopo_place_groups_lw_committed.
int32_t eligible_entry(bool committed, bool ranked, rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* rp,
                       int64_t rp_words, const uint64_t* admit, int64_t n_admit, int32_t n_alt, int32_t* assign,
                       int32_t* status, int32_t* domain, int32_t* rounds, float* score, int32_t* alt_node,
                       float* alt_score) {
  if (rounds) *rounds = 0;
  if (!c || !gb || !assign || !admit) return fail(RBGTOPO_EINVAL, "null argument");
  if (c->cfg.world > 1)
    return fail(RBGTOPO_ELIMIT, "eligible placement needs world == 1: a rank holds only its slab of every dense row");
  std::vector<int32_t> own_rp;
  if (!rp) {
    if (const int hrc = check_groups_blob(gb, words)) return hrc;
    own_rp.reserve(2);  // non-null data() for a blob without groups
    for (int g = 0; g < gb[2]; ++g)  // a q outside [1, MAXQ] fails validation before the table is read
      for (int i = 0, q = std::clamp(group_rec(gb, g)[3], 0, MAXQ); i < q; ++i) {
        own_rp.push_back(1);
        own_rp.push_back(-1);
      }
    rp = own_rp.data();
    rp_words = (int64_t)own_rp.size();
  }
  return place_entry(kPlaceLw | (committed ? kPlaceCommitted : 0) | (ranked ? kPlaceRanked : 0), c, gb, words, rp,
                     rp_words, n_alt, assign, status, domain, rounds, score, alt_node, alt_score, nullptr, admit,
                     n_admit);
}
}  // namespace

int32_t rbgtopo_place_groups_eligible(rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* role_pods,
                                      int64_t role_pods_words, const uint64_t* role_admit, int64_t n_role_admit,
                                      int32_t* assign, int32_t* status, int32_t* domain) {
  return eligible_entry(false, false, c, gb, words, role_pods, role_pods_words, role_admit, n_role_admit, 0, assign,
                        status, domain, nullptr, nullptr, nullptr, nullptr);
}

int32_t rbgtopo_place_groups_eligible_ranked(rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* role_pods,
                                             int64_t role_pods_words, const uint64_t* role_admit, int64_t n_role_admit,
                                             int32_t n_alt, int32_t* assign, int32_t* status, int32_t* domain,
                                             float* score, int32_t* alt_node, float* alt_score) {
  return eligible_entry(false, true, c, gb, words, role_pods, role_pods_words, role_admit, n_role_admit, n_alt, assign,
                        status, domain, nullptr, score, alt_node, alt_score);
}

int32_t rbgtopo_place_groups_eligible_committed(rbgtopo_ctx* c, const int32_t* gb, int64_t words,
                                                const int32_t* role_pods, int64_t role_pods_words,
                                                const uint64_t* role_admit, int64_t n_role_admit, int32_t* assign,
                                                int32_t* status, int32_t* domain, int32_t* rounds) {
  return eligible_entry(true, false, c, gb, words, role_pods, role_pods_words, role_admit, n_role_admit, 0, assign,
                        status, domain, rounds, nullptr, nullptr, nullptr);
}

int32_t rbgtopo_place_groups_eligible_committed_ranked(rbgtopo_ctx* c, const int32_t* gb, int64_t words,
                                                       const int32_t* role_pods, int64_t role_pods_words,
                                                       const uint64_t* role_admit, int64_t n_role_admit, int32_t n_alt,
                                                       int32_t* assign, int32_t* status, int32_t* domain,
                                                       int32_t* rounds, float* score, int32_t* alt_node,
                                                       float* alt_score) {
  return eligible_entry(true, true, c, gb, words, role_pods, role_pods_words, role_admit, n_role_admit, n_alt, assign,
                        status, domain, rounds, score, alt_node, alt_score);
}

// ---- ranked alternates on node-axis shards (DESIGN.md §3.17) ---------------------------------------------------------
namespace {
// The local half: a handle of its own from the pool, the placement of `form` with the slab lists collected in its
// AltExchange, then the exchange buffer and the merge's tables uploaded.  Nothing is left behind when the placement
// fails; once it has placed, only the device can fail.
// rp: the (S, C) table of a leader-worker form (§3.18), whose jobs and compact replicas count pods.
int32_t shard_ranked_local(int form, rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* rp,
                           int64_t rp_words, int32_t n_alt, int32_t* assign, int32_t* status, int32_t* domain,
                           int32_t* rounds, int32_t* xhandle, void** keys_dev, int64_t* keys_bytes) {
  if (rounds) *rounds = 0;
  if (!c || !xhandle || !keys_dev || !keys_bytes) return fail(RBGTOPO_EINVAL, "null argument");
  Batch* xb = nullptr;
  int rc = acquire_batch(c, &xb);
  if (rc) return rc;
  AltExchange& x = xb->x;
  x.reset(n_alt);
  rc = place_entry(form | kPlaceRanked | kPlaceShard, c, gb, words, rp, rp_words, n_alt, assign, status, domain,
                   rounds, nullptr, nullptr, nullptr, &x);
  if (rc) {
    release_batch(c, xb);
    return rc;
  }
  rc = [&]() -> int {
    CK(cudaSetDevice(c->cfg.device));
    x.total_r = rp ? GroupOffsets(gb, rp).pod0[gb[2]] : gb[4];
    const size_t J = x.job.size(), R = x.own.size(), W = x.bounds.size();
    x.bytes = (int64_t)std::max<size_t>(8, (J * ALT_LIST * 8 + R * 4 + 7) & ~(size_t)7);
    // pinned: the exchange buffer | the merge's tables (job, own, bounds), then the merge's outputs; device: the
    // tables | the outputs.  Everything the merge needs is allocated here.
    const size_t xw = (size_t)x.bytes / 4, tw = 2 * J + R + W, ow = R * (size_t)(1 + 2 * n_alt);
    CK(x.buf.reserve((size_t)x.bytes / 8));
    CK(xb->h_alt.reserve(std::max(xw + tw, ow)));
    CK(xb->alt.reserve(tw + ow + 1));
    int* h = xb->h_alt.p;
    memset(h, 0, (size_t)x.bytes);
    memcpy(h, x.keys.data(), J * ALT_LIST * 8);
    memcpy(h + 2 * J * ALT_LIST, x.rscore.data(), R * 4);
    memcpy(h + xw, x.job.data(), J * 8);
    memcpy(h + xw + 2 * J, x.own.data(), R * 4);
    memcpy(h + xw + 2 * J + R, x.bounds.data(), W * 4);
    cudaStream_t s = stream_of(c, xb);
    CK(cudaMemcpyAsync(x.buf.p, h, (size_t)x.bytes, cudaMemcpyHostToDevice, s));
    if (tw) CK(cudaMemcpyAsync(xb->alt.p, h + xw, tw * 4, cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));
    return RBGTOPO_OK;
  }();
  if (rc) {
    cudaStreamSynchronize(stream_of(c, xb));
    release_batch(c, xb);
    return rc;
  }
  {
    std::lock_guard<std::mutex> g(c->pool_mu);
    xb->xchg = true;
  }
  *xhandle = handle_of(c, xb);
  *keys_dev = x.buf.p;
  *keys_bytes = x.bytes;
  return RBGTOPO_OK;
}
}  // namespace

int32_t rbgtopo_shard_place_groups_ranked(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t n_alt,
                                          int32_t* assign, int32_t* status, int32_t* domain, int32_t* xhandle,
                                          void** keys_dev, int64_t* keys_bytes) {
  return shard_ranked_local(kPlaceReplicas, c, gb, words, nullptr, 0, n_alt, assign, status, domain, nullptr, xhandle,
                            keys_dev, keys_bytes);
}

int32_t rbgtopo_shard_place_groups_committed_ranked(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t n_alt,
                                                    int32_t* assign, int32_t* status, int32_t* domain, int32_t* rounds,
                                                    int32_t* xhandle, void** keys_dev, int64_t* keys_bytes) {
  return shard_ranked_local(kPlaceCommitted, c, gb, words, nullptr, 0, n_alt, assign, status, domain, rounds, xhandle,
                            keys_dev, keys_bytes);
}

int32_t rbgtopo_shard_place_groups_lw_ranked(rbgtopo_ctx* c, const int32_t* gb, int64_t words, const int32_t* role_pods,
                                             int64_t role_pods_words, int32_t n_alt, int32_t* assign, int32_t* status,
                                             int32_t* domain, int32_t* xhandle, void** keys_dev, int64_t* keys_bytes) {
  return shard_ranked_local(kPlaceLw, c, gb, words, role_pods, role_pods_words, n_alt, assign, status, domain, nullptr,
                            xhandle, keys_dev, keys_bytes);
}

int32_t rbgtopo_shard_place_groups_lw_committed_ranked(rbgtopo_ctx* c, const int32_t* gb, int64_t words,
                                                       const int32_t* role_pods, int64_t role_pods_words, int32_t n_alt,
                                                       int32_t* assign, int32_t* status, int32_t* domain,
                                                       int32_t* rounds, int32_t* xhandle, void** keys_dev,
                                                       int64_t* keys_bytes) {
  return shard_ranked_local(kPlaceLw | kPlaceCommitted, c, gb, words, role_pods, role_pods_words, n_alt, assign, status,
                            domain, rounds, xhandle, keys_dev, keys_bytes);
}

int32_t rbgtopo_shard_alternates_merge(rbgtopo_ctx* c, int32_t xhandle, const void* keys_all_dev, float* score,
                                       int32_t* alt_node, float* alt_score) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* xb = nullptr;
  {
    std::lock_guard<std::mutex> g(c->pool_mu);
    if (xhandle >= 0 && xhandle < (int)c->batches.size() && c->batches[xhandle]->in_use && c->batches[xhandle]->xchg)
      xb = c->batches[xhandle].get();
  }
  if (!xb) return fail(RBGTOPO_EINVAL, "handle %d is not an exchange of a sharded ranked placement", xhandle);
  const AltExchange& x = xb->x;
  const int F = x.n_alt;
  if (!keys_all_dev || !score || (F > 0 && (!alt_node || !alt_score))) return fail(RBGTOPO_EINVAL, "null argument");
  const RankReq rk{F, score, alt_node, alt_score};
  alt_clear(rk, 0, x.total_r);
  int rc = [&]() -> int {
    const size_t J = x.job.size(), R = x.own.size();
    if (J == 0) return RBGTOPO_OK;
    CK(cudaSetDevice(c->cfg.device));
    cudaStream_t s = stream_of(c, xb);
    const int W = (int)x.bounds.size() - 1;
    int* d = xb->alt.p;
    const size_t o_out = 2 * J + R + x.bounds.size();
    const unsigned grid = (unsigned)((J + ALT_MERGE_WARPS - 1) / ALT_MERGE_WARPS);
    k_alternates_merge<<<grid, 32 * ALT_MERGE_WARPS, 0, s>>>(
        static_cast<const unsigned long long*>(keys_all_dev), x.bytes / 8, W, (int)J, reinterpret_cast<const int2*>(d),
        d + 2 * J, d + 2 * J + R, F, d + o_out);
    CK(cudaGetLastError());
    int* h = xb->h_alt.p;  // the staged exchange buffer is no longer needed (the local call reserved ow here)
    const size_t ow = R * (size_t)(1 + 2 * F);
    CK(cudaMemcpyAsync(h, d + o_out, ow * 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    alt_scatter(rk, h, x.idx.data(), R);
    {
      std::lock_guard<std::mutex> g(c->stat_mu);
      c->launches += 1;
    }
    return RBGTOPO_OK;
  }();
  if (rc) cudaStreamSynchronize(stream_of(c, xb));
  release_batch(c, xb);
  return rc;
}

int32_t rbgtopo_plan_describe(const int32_t* gb, int64_t words, int32_t n_nodes, int32_t n_domains,
                              const int32_t* deg_plus1, int64_t wsum_max, int32_t* out_steps, int64_t out_cap_steps,
                              int32_t* n_steps, int32_t* n_waves, int64_t* plan_words) {
  if (!gb || !n_steps) return fail(RBGTOPO_EINVAL, "null argument");
  if (n_nodes < 1 || n_domains < 1 || wsum_max < 0) return fail(RBGTOPO_EINVAL, "n_nodes / n_domains / wsum_max");
  TopoHost th;
  if (const int trc = topo_host_args(n_nodes, n_domains, deg_plus1, wsum_max, &th)) return trc;
  static thread_local std::unique_ptr<Batch> scratch;  // host vectors + a pageable staging buffer only
  if (!scratch) {
    scratch = std::make_unique<Batch>();
    scratch->h_in.pageable = true;
  }
  PlanLayout L;
  const int lc = (n_nodes + 2047) / 2048;
  int rc = plan_geometry(th, lc, scratch.get(), gb, words, 0, -1, 0, false, &L);
  if (rc) return rc;
  *n_steps = L.ns;
  if (n_waves) *n_waves = (int)scratch->wave_begin.size() - 1;
  if (plan_words) *plan_words = L.plan_words;
  if (out_steps && out_cap_steps > 0)
    memcpy(out_steps, scratch->h_in.p + L.aux_off,
           (size_t)std::min<int64_t>(out_cap_steps, L.ns) * RBGTOPO_PLAN_STEP_WORDS * 4);
  return RBGTOPO_OK;
}

int32_t rbgtopo_place_describe(const int32_t* gb, int64_t words, int32_t n_nodes, int32_t n_domains, const int32_t* deg_plus1,
                               int64_t wsum_max, int32_t* order, int64_t order_cap, int32_t* geom) {
  if (!gb || !geom) return fail(RBGTOPO_EINVAL, "null argument");
  if (n_nodes < 1 || n_domains < 1 || wsum_max < 0) return fail(RBGTOPO_EINVAL, "n_nodes / n_domains / wsum_max");
  if (words > 0x3FFFFFFFLL) return fail(RBGTOPO_EINVAL, "bad groups blob header");
  if (const int hrc = check_groups_blob(gb, words)) return hrc;
  const int ng = gb[2];
  TopoHost th;
  if (const int trc = topo_host_args(n_nodes, n_domains, deg_plus1, wsum_max, &th)) return trc;
  static thread_local std::vector<GroupFacts> facts;
  static thread_local std::vector<int32_t> perm;
  perm.assign((size_t)std::max(1, ng), 0);
  DirectGeom G;
  int rc = direct_pass1(th, gb, words, ng, facts, perm.data(), &G);
  if (!rc) rc = direct_pass2(th, gb, words, ng, facts, &G);
  if (rc) return rc;
  geom[0] = (int32_t)G.total_r;
  geom[1] = G.n0;
  geom[2] = G.max_q;
  geom[3] = G.max_p;
  geom[4] = (int32_t)std::min<long long>(G.max_cap, 0x7FFFFFFF);
  geom[5] = G.nth;
  geom[6] = G.HT;
  geom[7] = G.CAP;
  if (order && order_cap > 0) memcpy(order, perm.data(), (size_t)std::min<int64_t>(order_cap, G.n0) * 4);
  return RBGTOPO_OK;
}

int32_t rbgtopo_stage_groups(rbgtopo_ctx* c, const int32_t* gb, int64_t words, int32_t* handle) {
  if (!c || !gb || !handle) return fail(RBGTOPO_EINVAL, "null argument");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  if (!c->topo.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
  CK(cudaSetDevice(c->cfg.device));
  Batch* b = nullptr;
  int rc = acquire_batch(c, &b);
  if (rc) return rc;
  rc = plan_stage(c, b, gb, words);
  if (!rc && kVerifyPlan) rc = verify_plan(c, b, gb, words);
  if (rc) {
    cudaStreamSynchronize(stream_of(c, b));  // the first upload / row tables may be in flight
    release_batch(c, b);
    return rc;
  }
  CK(cudaStreamSynchronize(stream_of(c, b)));
  *handle = handle_of(c, b);
  return RBGTOPO_OK;
}

int32_t rbgtopo_stage(rbgtopo_ctx* c, const int32_t* blob, int64_t words, int32_t* handle) {
  if (!c || !handle) return fail(RBGTOPO_EINVAL, "null argument");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  CK(cudaSetDevice(c->cfg.device));
  Batch* b = nullptr;
  int rc = acquire_batch(c, &b);
  if (rc) return rc;
  rc = stage_into(c, b, blob, words);
  if (rc) {
    release_batch(c, b);
    return rc;
  }
  CK(cudaStreamSynchronize(stream_of(c, b)));
  *handle = handle_of(c, b);
  return RBGTOPO_OK;
}

int32_t rbgtopo_run_staged(rbgtopo_ctx* c, int32_t handle, int32_t iters) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");

  if (iters < 1 || iters > 4096) return fail(RBGTOPO_EINVAL, "iters");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* b = batch_of(c, handle);
  if (!b) return fail(RBGTOPO_EINVAL, "bad or stale handle %d", handle);
  CK(cudaSetDevice(c->cfg.device));
  return run_batch(c, b, iters);
}

int32_t rbgtopo_run_staged_chain(rbgtopo_ctx* c, const int32_t* handles, int32_t n_handles, int32_t passes) {
  if (!c || !handles) return fail(RBGTOPO_EINVAL, "null argument");
  if (n_handles < 1 || n_handles > 64 || passes < 1 || passes > 65536) return fail(RBGTOPO_EINVAL, "n_handles / passes");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* bs[64];
  for (int i = 0; i < n_handles; ++i) {
    bs[i] = batch_of(c, handles[i]);
    if (!bs[i]) return fail(RBGTOPO_EINVAL, "bad or stale handle %d", handles[i]);
    for (int j = 0; j < i; ++j)
      if (bs[j] == bs[i]) return fail(RBGTOPO_EINVAL, "handle %d listed twice: the batches of a chain must be distinct", handles[i]);
  }
  CK(cudaSetDevice(c->cfg.device));
  return run_chain(c, bs, n_handles, passes);
}

int32_t rbgtopo_fetch(rbgtopo_ctx* c, int32_t handle, int32_t* assign, int32_t* status, int32_t* domain) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* b = batch_of(c, handle);
  if (!b || !b->ran) return fail(RBGTOPO_EINVAL, "handle %d has no results (or is stale: the topology changed)", handle);
  CK(cudaSetDevice(c->cfg.device));
  if (b->wave_begin.empty()) return fetch_batch(c, b, assign, status, domain);
  int rc = fetch_batch(c, b, nullptr, nullptr, nullptr);
  if (rc) return rc;
  std::vector<char> dirty;  // plan batches report in group order; unfinished groups keep status 1
  plan_results(b, assign, status, domain, &dirty);
  return RBGTOPO_OK;
}

int32_t rbgtopo_release(rbgtopo_ctx* c, int32_t handle) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* b = batch_of(c, handle, true);
  if (!b) return fail(RBGTOPO_EINVAL, "bad or stale handle %d", handle);
  cudaSetDevice(c->cfg.device);
  cudaStreamSynchronize(stream_of(c, b));
  release_batch(c, b);
  return RBGTOPO_OK;
}

int32_t rbgtopo_read_scores(rbgtopo_ctx* c, int32_t handle, int32_t row, float* out, int32_t out_len) {
  if (!c || !out) return fail(RBGTOPO_EINVAL, "null argument");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* b = batch_of(c, handle);
  if (!b || !b->ran) return fail(RBGTOPO_EINVAL, "handle %d has no results (or is stale: the topology changed)", handle);
  const int slab = c->slab_hi - c->slab_lo;
  if (row < 0 || row >= b->m.total_r || out_len < slab) return fail(RBGTOPO_EINVAL, "row/out_len");
  CK(cudaSetDevice(c->cfg.device));
  CK(cudaStreamSynchronize(stream_of(c, b)));
  int drow = 0;  // replicas of a role in a wave share one stored row (step_drow, kernels.cuh)
  if (b->wave_begin.empty()) drow = b->m.rowmap[row];
  else CK(cudaMemcpy(&drow, b->rowmap.p + row, 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(out, b->matrix.p + (size_t)drow * c->slab_stride, (size_t)slab * 4, cudaMemcpyDeviceToHost));
  return RBGTOPO_OK;
}

int32_t rbgtopo_read_topk(rbgtopo_ctx* c, int32_t handle, int32_t rolerow, uint64_t* out, int32_t k) {
  if (!c || !out) return fail(RBGTOPO_EINVAL, "null argument");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* b = batch_of(c, handle);
  if (!b || !b->ran) return fail(RBGTOPO_EINVAL, "handle %d has no results (or is stale: the topology changed)", handle);
  if (rolerow < 0 || rolerow >= b->m.total_p || k < 1 || k > KS) return fail(RBGTOPO_EINVAL, "rolerow/k");
  CK(cudaSetDevice(c->cfg.device));
  CK(cudaStreamSynchronize(stream_of(c, b)));
  CK(cudaMemcpy(out, b->merged.p + (size_t)rolerow * KS, (size_t)k * 8, cudaMemcpyDeviceToHost));
  return RBGTOPO_OK;
}

// The device buffer as it is: nothing is recomputed or re-sorted, so a stale or wrong vector shows.
int32_t rbgtopo_read_snapshot(rbgtopo_ctx* c, int32_t what, void* out, int64_t out_bytes, int64_t* n_out) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  const Topology& T = c->topo;
  if (!T.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
  const void* src = nullptr;
  long long n = 0;
  size_t elem = 8;
  switch (what) {
    case RBGTOPO_SNAP_BASE: src = T.base.p; n = T.n; elem = 4; break;
    case RBGTOPO_SNAP_ORDER: src = T.order.p; n = c->slab_hi - c->slab_lo; break;
    case RBGTOPO_SNAP_ORDER_ALL: src = c->cfg.world > 1 ? T.order_all.p : T.order.p; n = T.n; break;
    case RBGTOPO_SNAP_POS:
      if (c->cfg.world != 1) return fail(RBGTOPO_EINVAL, "pos exists with world == 1 only");
      src = T.pos.p; n = T.n; elem = 4;
      break;
    case RBGTOPO_SNAP_DELTA_REPAIRS: n = 1; break;
    case RBGTOPO_SNAP_LEVEL_OWNER: n = T.occ ? (long long)(T.n_levels + 1) * T.n : 0; elem = 4; break;
    default: return fail(RBGTOPO_EINVAL, "what = %d", what);
  }
  if (n_out) *n_out = n;
  if (n == 0) return RBGTOPO_OK;
  if (!out || out_bytes < n * (long long)elem) return fail(RBGTOPO_EINVAL, "out_bytes %lld < %lld", (long long)out_bytes, n * (long long)elem);
  if (what == RBGTOPO_SNAP_DELTA_REPAIRS) {
    const int64_t v = c->delta_repairs;
    memcpy(out, &v, sizeof v);
    return RBGTOPO_OK;
  }
  CK(cudaSetDevice(c->cfg.device));
  CK(cudaEventSynchronize(c->topo_ready));
  if (what == RBGTOPO_SNAP_LEVEL_OWNER) {  // rows of level_stride(n) on the device, packed rows of n here
    CK(cudaMemcpy2D(out, (size_t)T.n * 4, T.lvl_owner.p, (size_t)level_stride(T.n) * 4, (size_t)T.n * 4, T.n_levels + 1,
                    cudaMemcpyDeviceToHost));
    return RBGTOPO_OK;
  }
  if (n) CK(cudaMemcpy(out, src, (size_t)n * elem, cudaMemcpyDeviceToHost));
  return RBGTOPO_OK;
}

// ---- node-axis sharding --------------------------------------------------
int32_t rbgtopo_slab(rbgtopo_ctx* c, int32_t* lo, int32_t* hi) {
  if (!c || !lo || !hi) return fail(RBGTOPO_EINVAL, "null argument");
  if (!c->topo.valid) return fail(RBGTOPO_ENOTOPO, "set_topology has not been called");
  *lo = c->slab_lo;
  *hi = c->slab_hi;
  return RBGTOPO_OK;
}

// ---- wave-ranged sharded pipeline.  A step batch (rbgtopo_stage) is one wave; a plan
// (rbgtopo_stage_groups) has W waves: wave 0's score call also enqueues the ONE
// k_score_emit launch that writes the background rows of every wave on this rank's slab.
namespace {
struct WaveRange { int s0, s1, rr0, rr1, maxp; };
int wave_range(rbgtopo_ctx* c, Batch* b, int wave, WaveRange* w) {
  const BatchMeta& m = b->m;
  if (b->wave_begin.empty()) {
    if (wave != 0) return fail(RBGTOPO_EINVAL, "wave %d of a single-wave batch", wave);
    *w = WaveRange{0, m.n_steps, 0, m.total_p, m.max_p};
    return RBGTOPO_OK;
  }
  if (wave < 0 || wave + 1 >= (int)b->wave_begin.size()) return fail(RBGTOPO_EINVAL, "wave %d", wave);
  w->s0 = b->wave_begin[wave];
  w->s1 = b->wave_begin[wave + 1];
  w->maxp = b->wave_maxp[wave];
  w->rr0 = b->step_row[w->s0];
  w->rr1 = b->step_row[w->s1];
  (void)c;
  return RBGTOPO_OK;
}
void wave_table(Batch* b, const WaveRange& w, int* CAP, int* HT) {
  int mc = 0;
  for (int s = w.s0; s < w.s1; ++s) mc = std::max(mc, b->m.poff[s + 1] - b->m.poff[s]);
  *CAP = std::max(32, round_up(mc, 32));
  *HT = 64;
  while (2 * *HT < 3 * *CAP && *HT < (1 << 20)) *HT <<= 1;
}
}  // namespace

int32_t rbgtopo_shard_waves(rbgtopo_ctx* c, int32_t handle, int32_t* n_waves) {
  if (!c || !n_waves) return fail(RBGTOPO_EINVAL, "null argument");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* b = batch_of(c, handle);
  if (!b) return fail(RBGTOPO_EINVAL, "bad or stale handle %d", handle);
  *n_waves = b->wave_begin.empty() ? 1 : (int)b->wave_begin.size() - 1;
  return RBGTOPO_OK;
}

int32_t rbgtopo_shard_wave_score(rbgtopo_ctx* c, int32_t handle, int32_t wave, void** keys_dev, int64_t* keys_bytes) {
  if (!c || !keys_dev || !keys_bytes) return fail(RBGTOPO_EINVAL, "null argument");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* b = batch_of(c, handle);
  if (!b) return fail(RBGTOPO_EINVAL, "bad or stale handle %d", handle);
  WaveRange w;
  int rc = wave_range(c, b, wave, &w);
  if (rc) return rc;
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t s = stream_of(c, b);
  int launches = 0;
  const bool plan = !b->wave_begin.empty();
  BatchDev d = batch_dev(c, b);
  if (wave == 0) {
    CK(cudaStreamWaitEvent(s, c->topo_ready, 0));
    const bool timed = b->passes < kMaxTimedPasses;
    const int e0 = 3 * b->passes;
    if (timed) {
      int rc0 = ensure_pass_events(b, b->passes + 1);
      if (rc0) return rc0;
      CK(cudaEventRecord(b->it_ev[e0], s));
    }
    rc = launch_score(c, b, s);  // step batch: its rows + corrections; plan: background of every wave
    if (rc) return rc;
    ++launches;
    if (timed) CK(cudaEventRecord(b->it_ev[e0 + 1], s));
    b->shard_timed = timed;
  }
  const int n = w.s1 - w.s0;
  if (n > 0) {
    int CAP, HT;
    wave_table(b, w, &CAP, &HT);
    const int nth = std::max(128, 32 * w.maxp);
    if (fast_smem_bytes(nth / 32, HT, CAP) <= kFastSmemMax) {
      (b->m.any_level ? k_shard_select<true> : k_shard_select<false>)<<<n, nth, fast_smem_bytes(nth / 32, HT, CAP), s>>>(topo_dev(c), d, w.s0, 0, plan ? SEL_CORRECT : 0, HT, CAP, P2PDev{}, 0, 0, 0ull, nullptr);
    } else {
      if (plan) return fail(RBGTOPO_ELIMIT, "plan step with more than %d patched nodes on the sharded path", CAP);
      k_select<<<n, 32 * w.maxp, select_smem_bytes(w.maxp), s>>>(topo_dev(c), d, 0);
    }
    ++launches;
  }
  CK(cudaGetLastError());
  *keys_dev = b->lists.p + (size_t)w.rr0 * KS;
  *keys_bytes = (int64_t)std::max(1, w.rr1 - w.rr0) * KS * 8;
  b->pend_launches += launches;
  std::lock_guard<std::mutex> g(c->stat_mu);
  c->launches += launches;
  return RBGTOPO_OK;
}

int32_t rbgtopo_shard_wave_merge(rbgtopo_ctx* c, int32_t handle, int32_t wave, const void* keys_all,
                                 int32_t* need_pass2, void** keys2_dev, int64_t* keys2_bytes) {
  if (!c || !keys_all || !need_pass2 || !keys2_dev || !keys2_bytes) return fail(RBGTOPO_EINVAL, "null argument");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* b = batch_of(c, handle);
  if (!b) return fail(RBGTOPO_EINVAL, "bad or stale handle %d", handle);
  WaveRange w;
  int rc = wave_range(c, b, wave, &w);
  if (rc) return rc;
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t s = stream_of(c, b);
  BatchDev d = batch_dev(c, b);
  const long long rows = std::max(1, w.rr1 - w.rr0);
  d.parts = c->cfg.world;
  d.part_stride = rows * KS;
  d.lists_all = static_cast<const unsigned long long*>(keys_all) - (long long)w.rr0 * KS;  // indexed by global role row
  int launches = 0;
  const int n = w.s1 - w.s0;
  // an exclusive group's D* can also appear in a later wave (first placed replica), so plans
  // take the second pass whenever the GROUP is exclusive and the step has no fixed domain yet;
  // that is only known on the device -> conservatively: any exclusive step in the wave
  bool excl_unknown = b->m.any_excl_unknown;
  if (!b->wave_begin.empty()) {
    excl_unknown = false;
    for (int s2 = w.s0; s2 < w.s1 && !excl_unknown; ++s2)
      excl_unknown = (b->grp_flags[b->step_group[s2]] & RBGTOPO_STEP_EXCLUSIVE) != 0;
  }
  if (n > 0) {
    k_merge<<<(n + SEL_WARPS - 1) / SEL_WARPS, SEL_THREADS, 0, s>>>(topo_dev(c), d, w.s0, n, P2PWait{});
    ++launches;
    if (excl_unknown) {
      int CAP, HT;
      wave_table(b, w, &CAP, &HT);
      const int nth = std::max(128, 32 * w.maxp);
      if (fast_smem_bytes(nth / 32, HT, CAP) <= kFastSmemMax)
        (b->m.any_level ? k_shard_select<true> : k_shard_select<false>)<<<n, nth, fast_smem_bytes(nth / 32, HT, CAP), s>>>(topo_dev(c), d, w.s0, 1, 0, HT, CAP, P2PDev{}, 0, 0, 0ull, nullptr);
      else
        k_select<<<n, 32 * w.maxp, select_smem_bytes(w.maxp), s>>>(topo_dev(c), d, 1);
      ++launches;
    }
  }
  CK(cudaGetLastError());
  *need_pass2 = excl_unknown ? 1 : 0;
  *keys2_dev = b->excl.p + (size_t)w.rr0 * KS;
  *keys2_bytes = (int64_t)rows * KS * 8;
  b->pend_launches += launches;
  std::lock_guard<std::mutex> g(c->stat_mu);
  c->launches += launches;
  return RBGTOPO_OK;
}

int32_t rbgtopo_shard_wave_assign(rbgtopo_ctx* c, int32_t handle, int32_t wave, const void* keys2_all) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  Batch* b = batch_of(c, handle);
  if (!b) return fail(RBGTOPO_EINVAL, "bad or stale handle %d", handle);
  WaveRange w;
  int rc = wave_range(c, b, wave, &w);
  if (rc) return rc;
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t s = stream_of(c, b);
  BatchDev d = batch_dev(c, b);
  d.parts = c->cfg.world;
  const long long rows = std::max(1, w.rr1 - w.rr0);
  if (keys2_all) {
    d.excl_all = static_cast<const unsigned long long*>(keys2_all) - (long long)w.rr0 * KS;
    d.excl_part_stride = rows * KS;
  } else {
    d.parts = 1;  // no second pass: k_greedy never reads excl_all for steps with a fixed / no domain
  }
  int launches = 0;
  const int n = w.s1 - w.s0;
  const bool plan = !b->wave_begin.empty();
  if (n > 0) {
    k_greedy<<<(n + SEL_WARPS - 1) / SEL_WARPS, SEL_THREADS, 0, s>>>(topo_dev(c), d, w.s0, n, plan ? 1 : 0, P2PWait{});
    ++launches;
  }
  const bool last = !plan || wave + 2 == (int)b->wave_begin.size();
  if (last) {
    if (b->shard_timed) {
      CK(cudaEventRecord(b->it_ev[3 * b->passes + 2], s));
      b->passes += 1;
      b->shard_timed = false;
    }
    b->untimed_or_timed_passes += 1;
    b->ran = true;
  }
  CK(cudaGetLastError());
  b->pend_launches += launches;
  std::lock_guard<std::mutex> g(c->stat_mu);
  c->launches += launches;
  return RBGTOPO_OK;
}

// single-wave forms (step batches)
int32_t rbgtopo_shard_score(rbgtopo_ctx* c, int32_t handle, void** keys_dev, int64_t* keys_bytes) {
  return rbgtopo_shard_wave_score(c, handle, 0, keys_dev, keys_bytes);
}
int32_t rbgtopo_shard_merge(rbgtopo_ctx* c, int32_t handle, const void* keys_all, int32_t* need_pass2,
                            void** keys2_dev, int64_t* keys2_bytes) {
  return rbgtopo_shard_wave_merge(c, handle, 0, keys_all, need_pass2, keys2_dev, keys2_bytes);
}
int32_t rbgtopo_shard_assign(rbgtopo_ctx* c, int32_t handle, const void* keys2_all) {
  return rbgtopo_shard_wave_assign(c, handle, 0, keys2_all);
}

// ---- all-gather over NVLink peer memory, inside the library (p2p.cuh) ------------------------
int32_t rbgtopo_p2p_export(rbgtopo_ctx* c, int32_t rows_cap, void* handle_out, int32_t handle_len, void** local_ptr) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  if (c->cfg.world > P2P_MAX_WORLD) return fail(RBGTOPO_ELIMIT, "world %d > %d", c->cfg.world, P2P_MAX_WORLD);
  if (rows_cap <= 0) rows_cap = 16384;
  if (handle_out && handle_len < (int32_t)sizeof(cudaIpcMemHandle_t)) return fail(RBGTOPO_EINVAL, "handle buffer < %zu bytes", sizeof(cudaIpcMemHandle_t));
  std::unique_lock<std::shared_mutex> lk(c->topo_mu);
  CK(cudaSetDevice(c->cfg.device));
  const int W = c->cfg.world;
  const size_t data = (size_t)2 * W * rows_cap * KS;
  const size_t total = data + (size_t)2 * W * P2P_FLAG_STRIDE + 64;
  CK(c->xbuf.reserve(total));
  CK(cudaMemset(c->xbuf.p, 0, c->xbuf.cap * 8));
  CK(c->p2p_ctr.reserve(4));
  CK(cudaMemset(c->p2p_ctr.p, 0, c->p2p_ctr.cap * 4));
  CK(cudaDeviceSynchronize());
  c->p2p_rows_cap = rows_cap;
  c->p2p = P2PDev{};
  c->p2p.world = W;
  c->p2p.rank = c->cfg.rank;
  c->p2p.slot_stride = (long long)rows_cap * KS;
  c->p2p.flags_off = (long long)data;
  c->p2p.peer[c->cfg.rank] = c->xbuf.p;
  c->p2p_ready = false;
  c->p2p_seq = 0;
  if (handle_out) {
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, c->xbuf.p));
    memcpy(handle_out, &h, sizeof h);
  }
  if (local_ptr) *local_ptr = c->xbuf.p;
  return RBGTOPO_OK;
}

int32_t rbgtopo_p2p_import(rbgtopo_ctx* c, const void* handles_all, void* const* peer_ptrs) {
  if (!c || (!handles_all && !peer_ptrs)) return fail(RBGTOPO_EINVAL, "null argument");
  std::unique_lock<std::shared_mutex> lk(c->topo_mu);
  if (!c->xbuf.p) return fail(RBGTOPO_EINVAL, "rbgtopo_p2p_export has not been called");
  CK(cudaSetDevice(c->cfg.device));
  const int W = c->cfg.world;
  for (int g = 0; g < W; ++g) {
    if (g == c->cfg.rank) continue;
    if (peer_ptrs) {  // peers inside this process (several contexts of one process): plain device pointers
      if (!peer_ptrs[g]) return fail(RBGTOPO_EINVAL, "peer pointer %d is null", g);
      c->p2p.peer[g] = static_cast<unsigned long long*>(peer_ptrs[g]);
    } else {          // one process per GPU: map the peer's buffer (enables peer access over NVLink)
      cudaIpcMemHandle_t h;
      memcpy(&h, static_cast<const char*>(handles_all) + (size_t)g * sizeof h, sizeof h);
      void* q = nullptr;
      CK(cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess));
      c->p2p_opened.push_back(q);
      c->p2p.peer[g] = static_cast<unsigned long long*>(q);
    }
  }
  c->p2p_ready = true;
  return RBGTOPO_OK;
}

// The sharded pipeline of a staged batch / plan with the exchanges done by the library itself:
// per wave k_shard_select (+ fused push) -> k_merge (waits first) [-> restricted reselect (+ push)] ->
// k_greedy (waits for it), all enqueued on the call's stream; no NCCL, no host synchronisation.  SPMD: every rank calls it
// with the same staged batch.
int32_t rbgtopo_run_staged_p2p(rbgtopo_ctx* c, int32_t handle, int32_t iters) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  if (iters < 1 || iters > 4096) return fail(RBGTOPO_EINVAL, "iters");
  std::shared_lock<std::shared_mutex> lk(c->topo_mu);
  if (c->cfg.world > 1 && !c->p2p_ready) return fail(RBGTOPO_EINVAL, "rbgtopo_p2p_import has not been called");
  Batch* b = batch_of(c, handle);
  if (!b) return fail(RBGTOPO_EINVAL, "bad or stale handle %d", handle);
  if (c->cfg.world == 1) return run_batch(c, b, iters);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t s = stream_of(c, b);
  const bool plan = !b->wave_begin.empty();
  const int n_waves = plan ? (int)b->wave_begin.size() - 1 : 1;
  std::lock_guard<std::mutex> seq_guard(c->pool_mu);  // one exchange sequence at a time per ctx (the seq counter is SPMD state)
  CK(cudaStreamWaitEvent(s, c->topo_ready, 0));
  // ... and one on the device: this pass starts after the ctx's previous pass ended, whichever stream that used.  Every
  // return below records the end, an RBGTOPO_ELIMIT after some waves were enqueued included
  CK(cudaStreamWaitEvent(s, c->p2p_done, 0));
  struct RecordDone {
    cudaEvent_t e;
    cudaStream_t s;
    ~RecordDone() { cudaEventRecord(e, s); }
  } record_done{c->p2p_done, s};
  int launches = 0;
  for (int it = 0; it < iters; ++it) {
    c->p2p_bytes_last = 0;
    const bool timed = b->passes < kMaxTimedPasses;
    const int e0 = 3 * b->passes;
    if (timed) {
      int rc0 = ensure_pass_events(b, b->passes + 1);
      if (rc0) return rc0;
      CK(cudaEventRecord(b->it_ev[e0], s));
    }
    int rc = launch_score(c, b, s);
    if (rc) return rc;
    ++launches;
    if (timed) CK(cudaEventRecord(b->it_ev[e0 + 1], s));
    for (int wv = 0; wv < n_waves; ++wv) {
      WaveRange w;
      rc = wave_range(c, b, wv, &w);
      if (rc) return rc;
      const int n = w.s1 - w.s0;
      if (n <= 0) continue;
      BatchDev d = batch_dev(c, b);
      int CAP, HT;
      wave_table(b, w, &CAP, &HT);
      const int nth = std::max(128, 32 * w.maxp);
      if (fast_smem_bytes(nth / 32, HT, CAP) > kFastSmemMax)
        return fail(RBGTOPO_ELIMIT, "a step's patched set exceeds shared memory on the sharded path");
      const long long rows = std::max(1, w.rr1 - w.rr0);
      if (rows > c->p2p_rows_cap)
        return fail(RBGTOPO_ELIMIT, "%lld role rows in one wave exceed the exchange buffer (%d)", rows, c->p2p_rows_cap);
      static const long long timeout_cycles =
          (getenv("RBGTOPO_P2P_TIMEOUT_MS") ? std::max(1, atoi(getenv("RBGTOPO_P2P_TIMEOUT_MS"))) : 2000) * 2000000LL;  // ~2 GHz
      const int W = c->cfg.world;
      auto phase = [&](unsigned long long* seq, int* parity, P2PWait* pw) {  // next exchange phase of the SPMD sequence
        *seq = ++c->p2p_seq;
        *parity = (int)(*seq & 1ull);
        pw->flags = c->xbuf.p + c->p2p.flags_off + (long long)*parity * W * P2P_FLAG_STRIDE;
        pw->seq = *seq;
        pw->timeout_cycles = timeout_cycles;
        pw->err = c->p2p_ctr.p + 1;
        pw->world = W;
        c->p2p_bytes_last += rows * KS * 8 * (W - 1);
      };
      unsigned long long seq;
      int parity;
      P2PWait pw{};
      phase(&seq, &parity, &pw);
      // select + fused push (peer stores of every list, release flags by the last CTA)
      (b->m.any_level ? k_shard_select<true> : k_shard_select<false>)<<<n, nth, fast_smem_bytes(nth / 32, HT, CAP), s>>>(topo_dev(c), d, w.s0, 0, plan ? SEL_CORRECT : 0, HT, CAP,
                                                                       c->p2p, w.rr0, parity, seq, c->p2p_ctr.p);
      d.parts = W;
      d.part_stride = c->p2p.slot_stride;
      d.lists_all = c->xbuf.p + (long long)parity * W * c->p2p.slot_stride - (long long)w.rr0 * KS;
      k_merge<<<(n + SEL_WARPS - 1) / SEL_WARPS, SEL_THREADS, 0, s>>>(topo_dev(c), d, w.s0, n, pw);  // waits (acquire) first
      launches += 2;
      bool excl_unknown = b->m.any_excl_unknown;
      if (plan) {
        excl_unknown = false;
        for (int s2 = w.s0; s2 < w.s1 && !excl_unknown; ++s2)
          excl_unknown = (b->grp_flags[b->step_group[s2]] & RBGTOPO_STEP_EXCLUSIVE) != 0;
      }
      P2PWait pw2{};
      if (excl_unknown) {
        phase(&seq, &parity, &pw2);
        (b->m.any_level ? k_shard_select<true> : k_shard_select<false>)<<<n, nth, fast_smem_bytes(nth / 32, HT, CAP), s>>>(topo_dev(c), d, w.s0, 1, 0, HT, CAP, c->p2p, w.rr0, parity, seq,
                                                                         c->p2p_ctr.p);
        d.excl_all = c->xbuf.p + (long long)parity * W * c->p2p.slot_stride - (long long)w.rr0 * KS;
        d.excl_part_stride = c->p2p.slot_stride;
        ++launches;
      } else {
        d.parts = 1;  // k_greedy never reads excl_all for steps with a fixed / no domain
      }
      k_greedy<<<(n + SEL_WARPS - 1) / SEL_WARPS, SEL_THREADS, 0, s>>>(topo_dev(c), d, w.s0, n, plan ? 1 : 0, pw2);
      ++launches;
    }
    if (timed) {
      CK(cudaEventRecord(b->it_ev[e0 + 2], s));
      b->passes += 1;
    }
    b->untimed_or_timed_passes += 1;
  }
  CK(cudaGetLastError());
  b->ran = true;
  b->pend_launches += launches;
  std::lock_guard<std::mutex> g(c->stat_mu);
  c->launches += launches;
  return RBGTOPO_OK;
}

int32_t rbgtopo_p2p_stats(rbgtopo_ctx* c, int64_t* peer_bytes_last_pass, int32_t* timed_out) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  if (peer_bytes_last_pass) *peer_bytes_last_pass = c->p2p_bytes_last;
  if (timed_out) {
    *timed_out = 0;
    if (c->p2p_ctr.p) {
      CK(cudaSetDevice(c->cfg.device));
      int v = 0;
      CK(cudaMemcpy(&v, c->p2p_ctr.p + 1, 4, cudaMemcpyDeviceToHost));
      *timed_out = v;
    }
  }
  return RBGTOPO_OK;
}

int32_t rbgtopo_set_kernel_timing(rbgtopo_ctx* c, int32_t on) {
  if (!c) return RBGTOPO_EINVAL;
  c->kernel_timing.store(on != 0, std::memory_order_relaxed);
  return RBGTOPO_OK;
}

// Joins the outgoing streams into the incoming ones without blocking the host: everything enqueued before the switch
// (a pass, a staging, a D2H) is ordered before everything enqueued after it, whichever streams the two sides use.  The
// batch streams are non-blocking, so nothing else orders them against an external stream.  The pending waits make the
// incoming streams busy, so fence_batches orders a later refresh behind the outgoing work as well.  topo_mu held
// exclusively: nothing is enqueued meanwhile, and fence_ev / ev[6] / ev[7] are not recorded elsewhere (fence_batches
// holds it too).
int32_t rbgtopo_set_stream(rbgtopo_ctx* c, void* stream) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  std::unique_lock<std::shared_mutex> lk(c->topo_mu);
  cudaStream_t in = static_cast<cudaStream_t>(stream);
  {
    CK(cudaSetDevice(c->cfg.device));
    std::lock_guard<std::mutex> g(c->pool_mu);
    if (c->use_ext_stream) {
      if (in != c->ext_stream) {
        CK(cudaEventRecord(c->fence_ev, c->ext_stream));
        if (in) {
          CK(cudaStreamWaitEvent(in, c->fence_ev, 0));
        } else {
          for (auto& b : c->batches) {  // a batch acquired later starts on its own streams too
            CK(cudaStreamWaitEvent(b->stream, c->fence_ev, 0));
            CK(cudaStreamWaitEvent(b->stream2, c->fence_ev, 0));
          }
        }
      }
    } else if (in) {
      for (auto& b : c->batches) {
        CK(cudaEventRecord(b->ev[6], b->stream));
        CK(cudaStreamWaitEvent(in, b->ev[6], 0));
        CK(cudaEventRecord(b->ev[7], b->stream2));
        CK(cudaStreamWaitEvent(in, b->ev[7], 0));
      }
    }
  }
  c->ext_stream = in;
  c->use_ext_stream = in != nullptr;
  return RBGTOPO_OK;
}

int32_t rbgtopo_last_timing(rbgtopo_ctx* c, rbgtopo_timing* out) {
  if (!c || !out) return fail(RBGTOPO_EINVAL, "null argument");
  std::lock_guard<std::mutex> g(c->stat_mu);
  *out = c->last;
  out->base_ms = c->topo.base_ms;
  return RBGTOPO_OK;
}

int32_t rbgtopo_last_pass_times(rbgtopo_ctx* c, float* score_ms, float* select_ms, int32_t cap, int32_t* n_passes) {
  if (!c || !n_passes || cap < 0) return fail(RBGTOPO_EINVAL, "null argument");
  std::lock_guard<std::mutex> g(c->stat_mu);
  const int n = (int)std::min(c->last_score_ms.size(), c->last_select_ms.size());
  *n_passes = n;
  for (int i = 0; i < std::min(n, cap); ++i) {
    if (score_ms) score_ms[i] = c->last_score_ms[i];
    if (select_ms) select_ms[i] = c->last_select_ms[i];
  }
  return RBGTOPO_OK;
}

int32_t rbgtopo_stats(rbgtopo_ctx* c, uint64_t* generation, int64_t* calls, int64_t* scores_total,
                      int64_t* kernel_launches) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  std::lock_guard<std::mutex> g(c->stat_mu);
  if (generation) *generation = c->topo.generation;
  if (calls) *calls = c->calls;
  if (scores_total) *scores_total = c->scores_total;
  if (kernel_launches) *kernel_launches = c->launches;
  return RBGTOPO_OK;
}

int32_t rbgtopo_plan_occupancy(rbgtopo_ctx* c, int32_t* ctas, int32_t* ctas_per_sm, int32_t* rounds) {
  if (!c) return fail(RBGTOPO_EINVAL, "null ctx");
  std::lock_guard<std::mutex> g(c->stat_mu);
  const long long slots = (long long)c->plan_ctas_per_sm * c->sm_count;
  if (ctas) *ctas = c->plan_ctas;
  if (ctas_per_sm) *ctas_per_sm = c->plan_ctas_per_sm;
  if (rounds) *rounds = slots > 0 ? (int32_t)((c->plan_ctas + slots - 1) / slots) : 0;
  return RBGTOPO_OK;
}

}  // extern "C"
