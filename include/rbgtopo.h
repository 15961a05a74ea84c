/*
 * rbgtopo.h — C ABI of the H100-native topology-aware placement engine for
 * sgl-project/rbg RoleBasedGroups.
 *
 * This is the drop-in boundary (DESIGN.md §2). The reference has NO FFI for
 * this path (SURVEY.md §0/§8b): its plugin boundary is the Go interface
 * scheduler.PodGroupManager (pkg/scheduler/podgroup_manager.go:64-78), selected
 * by --scheduler-name (cmd/rbgs/main.go:148-152) through NewPodGroupManager
 * (pkg/scheduler/podgroup_manager.go:82-92).  A third PodGroupManager
 * implementation ("b200-topo", INTEGRATION.md) binds the entry points below
 * through cgo.  Every entry point cites the reference symbol whose output it
 * consumes or whose call site it plugs into.
 *
 * Rules of the ABI
 *   - plain C: int32_t/int64_t/uint64_t/float pointers + sizes, no C++ types,
 *     no torch types, no exceptions across the boundary, never abort().
 *   - every function returns an int32 status: 0 = RBGTOPO_OK, <0 = error; the
 *     text is available from rbgtopo_last_error().
 *   - the caller owns every buffer it passes; nothing is retained after return
 *     (cgo pointer rules).  The opaque rbgtopo_ctx owns all device memory,
 *     streams and staging buffers.
 *   - thread-safe: up to --max-concurrent-reconciles goroutines (default 10,
 *     cmd/rbgs/main.go:140-143) may call into one ctx concurrently; calls take
 *     a slot (stream + pinned staging + device scratch) from an internal pool.
 *   - there is NO CPU fallback: without a CUDA device rbgtopo_create fails
 *     with RBGTOPO_ENODEVICE.  (The Go shim then degrades to "no placement
 *     hint", the controller's behaviour today.)
 *
 * The batch wire format ("blob") is one contiguous int32 array so that a Go
 * []int32 can be handed over with a single unsafe.Pointer and DMA'd to the GPU
 * unmodified; the kernels index it directly.  Layout in the BLOB section.
 */
#ifndef RBGTOPO_H_
#define RBGTOPO_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RBGTOPO_ABI_VERSION 1

/* ---- status codes ------------------------------------------------------ */
#define RBGTOPO_OK          0
#define RBGTOPO_EINVAL     -1  /* malformed argument / blob                     */
#define RBGTOPO_ENODEVICE  -2  /* no CUDA device / wrong arch (needs sm_90)      */
#define RBGTOPO_ECUDA      -3  /* CUDA runtime error (text in last_error)       */
#define RBGTOPO_EINEXACT   -4  /* input violates the fp32 exactness contract     */
#define RBGTOPO_ENOTOPO    -5  /* score/assign called before set_topology        */
#define RBGTOPO_ELIMIT     -6  /* a documented limit (roles/step, K, N) exceeded */
#define RBGTOPO_ENOMEM     -7

/* ---- spec constants (DESIGN.md §3, frozen) ----------------------------- */
#define RBGTOPO_F_CAP            8     /* A.2: min(free[m], F)                  */
#define RBGTOPO_SELF_W           8000  /* A.3: self term = 8 x NVLink weight    */
#define RBGTOPO_NEED_CAP         16    /* A.2: need_rho is clamped by the host   */
#define RBGTOPO_MAX_STEP_ROLES   8     /* role rows scored per step             */
#define RBGTOPO_MAX_STEP_REPLICAS 32   /* = KMAX; bigger levels go in waves     */
#define RBGTOPO_MAX_GROUP_ROLES  16    /* pair-matrix columns (Q)               */
#define RBGTOPO_MAX_FREE         32767 /* free[n], consumed amounts             */
#define RBGTOPO_MAX_EDGE_W       65535

/* step flags */
#define RBGTOPO_STEP_EXCLUSIVE   1  /* group-exclusive-topology set:
                                       api/workloads/constants/annotation.go:25,
                                       pkg/reconciler/pod_reconciler.go:125-137 */
#define RBGTOPO_STEP_GANG        2  /* group-gang-scheduling == "true":
                                       api/workloads/constants/annotation.go:37 */
/* role flags */
#define RBGTOPO_ROLE_EXCLUSIVE   1  /* role takes part in exclusive topology; 0 =
                                       role-disable-exclusive opt-out
                                       (annotation.go:29,60; pod_reconciler.go:127) */

/* per-step result status */
#define RBGTOPO_PLACED_ALL   0
#define RBGTOPO_PLACED_PART  1  /* some replicas have no feasible node (-1)     */
#define RBGTOPO_GANG_FAILED  2  /* gang step: nothing placed, all -1            */

/* ---- BLOB: one batch of placement steps -------------------------------- *
 * A "step" is one wave of one dependency level of one RoleBasedGroup: the
 * roles of that level (pkg/dependency/dependency.go:129-205 order) with their
 * pending replica counts (rolebasedgroup_controller.go:509-518 override by the
 * coordination target, scaler.go:141-169), at most RBGTOPO_MAX_STEP_REPLICAS
 * replicas.  All int32 words, little endian:
 *
 *   word 0  magic 0x54474252 ("RBGT")      word 1  RBGTOPO_ABI_VERSION
 *   word 2  n_steps                        word 3  total words in the blob
 *   word 4  total replicas  (sum of R)     word 5  total role rows (sum of P)
 *   word 6,7 reserved (0)
 *   then n_steps step records of RBGTOPO_STEP_WORDS words:
 *     +0 gid            group id (>=0), compared with domain_owner[]
 *     +1 flags          RBGTOPO_STEP_*
 *     +2 fixed_domain   -1, or the domain the group already occupies
 *     +3 n_roles  P     1..RBGTOPO_MAX_STEP_ROLES
 *     +4 role_off       word offset of P role records (4 words each:
 *                       count, demand, need, role_flags); MUST be a multiple
 *                       of 4 (the kernels read a record as one 16-byte vector)
 *     +5 q              number of group roles = pair-matrix columns (0..16)
 *     +6 pair_off       word offset of pair[P][q] (row-major int32)
 *     +7 n_anchors      pods of this group already placed (sparse anchor[q][n])
 *     +8 anchor_off     word offset of n_anchors records (node, role q, count)
 *     +9 n_consumed     nodes whose capacity this group already took in this
 *                       reconcile and that free[] does not reflect yet
 *     +10 consumed_off  word offset of n_consumed records (node, amount)
 *     +11 n_replicas R  = sum of role counts, 1..RBGTOPO_MAX_STEP_REPLICAS
 *     +12 replica_off   prefix sum of R over earlier steps (row of the dense
 *                       matrix and index into assign[])
 *     +13 rolerow_off   prefix sum of P over earlier steps
 *     +14 exclusive level (0; see rbgtopo_set_exclusive_levels)
 *     +15 reserved (0)
 *   then the variable sections the offsets point at.
 * Replica order inside a step: role records in the given order (the host
 * passes them lexicographically, dependency.go:133-137), ordinal ascending
 * (stateful_instance_set_utils.go:74-76).
 * ------------------------------------------------------------------------ */
#define RBGTOPO_BLOB_MAGIC   0x54474252
#define RBGTOPO_HDR_WORDS    8
#define RBGTOPO_STEP_WORDS   16
#define RBGTOPO_ROLE_WORDS   4
#define RBGTOPO_ANCHOR_WORDS 3
#define RBGTOPO_CONS_WORDS   2

typedef struct rbgtopo_ctx rbgtopo_ctx;

typedef struct rbgtopo_config {
  int32_t device;        /* CUDA device ordinal                                */
  int32_t rank;          /* node-axis shard of this process, 0..world-1        */
  int32_t world;         /* number of node-axis shards (GPUs), >= 1            */
  int32_t slots;         /* concurrent in-flight calls, 0 = default (4)        */
  int32_t emit_matrix;   /* reserved: the dense (replica x node) matrix is
                            always materialised                                */
  int32_t chunk_nodes;   /* nodes per CTA work item, 0 = default (2048)        */
  int32_t flags;         /* RBGTOPO_CFG_*; unknown bits: RBGTOPO_EINVAL        */
  int32_t reserved;      /* 0                                                  */
} rbgtopo_config;

/* config flags */
#define RBGTOPO_CFG_LEVEL_PLACEMENT 1  /* place groups / steps at exclusive levels >= 1
                                          (rbgtopo_set_exclusive_levels); without it a
                                          level >= 1 answers RBGTOPO_ELIMIT */
#define RBGTOPO_CFG_COMMIT_LEVELS 2    /* rbgtopo_place_groups_committed also places groups
                                          at levels >= 1 (claims across levels); valid only
                                          with RBGTOPO_CFG_LEVEL_PLACEMENT, alone EINVAL */

/* Per-call device timing, milliseconds from CUDA events on the call's stream. */
typedef struct rbgtopo_timing {
  float h2d_ms, base_ms, score_ms, select_ms, d2h_ms, total_ms;
  int32_t launches;      /* kernels launched by the call                       */
  int32_t h2d_words;     /* int32 words uploaded for the batch (blob + offsets)    */
  int64_t scores;        /* (replica x node) scores produced by the call       */
  int64_t algo_bytes;    /* algorithmic bytes of the score kernel, DESIGN §5   */
} rbgtopo_timing;

/* ---- lifecycle ---------------------------------------------------------- */
/* Plug-in construction: called from the b200-topo case added to
 * NewPodGroupManager (pkg/scheduler/podgroup_manager.go:82-92). */
int32_t rbgtopo_create(const rbgtopo_config* cfg, rbgtopo_ctx** out);
int32_t rbgtopo_destroy(rbgtopo_ctx* ctx);
int32_t rbgtopo_abi_version(void);
/* Copies the calling thread's last error text for ctx (ctx may be NULL for
 * create failures); returns the text length. */
int32_t rbgtopo_last_error(rbgtopo_ctx* ctx, char* buf, int32_t len);

/* ---- cluster snapshot (new input; the reference has no node informer,
 *      SURVEY.md §8f rank 1).  Called when the Node cache changes. ---------- */
/* CSR must be symmetric (undirected topology), col_idx strictly ascending per
 * row, no self loops; edge_w in [0, RBGTOPO_MAX_EDGE_W]; free in
 * [0, RBGTOPO_MAX_FREE]; domain in [0, n_domains); domain_owner[d] = -1 or gid.
 * `generation` is echoed by rbgtopo_stats; the device-resident CSR is the cache
 * keyed by it (SURVEY.md §5 checkpoint row). */
int32_t rbgtopo_set_topology(rbgtopo_ctx* ctx, int32_t n_nodes, int64_t n_edges,
                             const int32_t* row_ptr, const int32_t* col_idx,
                             const int32_t* edge_w, const int32_t* free_slots,
                             const int32_t* domain, int32_t n_domains,
                             const int32_t* domain_owner, uint64_t generation);
/* Capacity / ownership refresh between reconciles (scheduled-pod counts change:
 * rolebasedgroup_controller.go:1057-1080).  Either pointer may be NULL. */
int32_t rbgtopo_update_nodes(rbgtopo_ctx* ctx, const int32_t* free_slots,
                             const int32_t* domain_owner, uint64_t generation);

/* Incremental form (SURVEY.md §8f rank 3): the free capacity of n_changed nodes changed (a pod was
 * bound / deleted — the reconcile events of rolebasedgroup_controller.go:1347-1430).  The library
 * updates base = W * min(free, F) on the closed neighbourhoods of those nodes only (exact integer
 * deltas: bit-identical to a full recomputation) and repairs the background order by taking the
 * affected entries out and merging them back, instead of the full SpMV + sort of
 * rbgtopo_update_nodes.  Duplicate nodes: the last value wins.  Falls back to the full refresh when
 * the neighbourhoods hold more than 2 048 nodes together (e.g. 10 % churn) or with world > 1. */
int32_t rbgtopo_update_nodes_delta(rbgtopo_ctx* ctx, int32_t n_changed, const int32_t* nodes,
                                   const int32_t* free_slots, uint64_t generation);

/* Exclusive topology at the key each group names (DESIGN.md §3.9).  The annotation
 * rbg.workloads.x-k8s.io/group-exclusive-topology names a topology key
 * (api/workloads/constants/annotation.go:23-25) and pod_reconciler.go:126-137,172-231 turns it into two
 * required terms on that key: pod affinity group-unique-hash In {own key} and pod anti-affinity
 * group-unique-hash Exists, NotIn {own key}.  The snapshot holds up to RBGTOPO_MAX_EXCL_LEVELS node
 * partitions ("levels"): level 0 is set_topology's domain[], levels 1..n_levels come from here, each with
 * its own domain count.  Ownership is then derived from the pods that carry the exclusive label:
 * occ[n_occ][3] = (node, gid, level) says "a pod of exclusive group gid, whose key is `level`, is bound on
 * node".  With a = b -> a, -1 (+) x = x and anything else -> -2 (blocked for every group):
 *   present_L[d] = (+) of the gids of ALL records on nodes of domain d of level L,
 *   keyed_L[d]   = (+) of the gids of the records OF LEVEL L on nodes of domain d of level L,
 *   owner_L[n]   = present_L[dom_L(n)] (+) keyed_0[dom_0(n)] (+) ... (+) keyed_K[dom_K(n)],
 * which restates both terms, including the symmetric enforcement of an existing pod's anti-affinity.
 * A participating role of an exclusive group g at level L may not use node n when owner_L[n] is not -1 or g.
 *
 * The first call after set_topology enters OCCUPANCY MODE: from then on every level's owner vector, level 0
 * included, is derived from the records (domain_owner of set_topology no longer counts, and
 * rbgtopo_update_nodes with domain_owner != NULL returns RBGTOPO_EINVAL); set_topology leaves the mode and
 * drops the levels.  With level-0 records only, owner_0 equals owner[domain[n]] of the domain-owner map the
 * records imply, and every result equals that of a ctx given that map.
 *   level_domain [n_levels][n_nodes] (level-major; domain of every node at levels 1..n_levels) and
 *   level_n_domains[n_levels]: installs the partitions (the call then waits for in-flight batches, like
 *   set_topology); level_domain == NULL keeps the installed ones (n_levels must match them; 0 before any
 *   were installed) and refreshes the occupancy only, ordered behind in-flight batches like update_nodes.
 *   Neither form recomputes base or the background order: ownership does not enter them.
 * Limits: n_levels <= RBGTOPO_MAX_EXCL_LEVELS - 1; record node in [0, n), gid >= 0, level in [0, n_levels].
 * Placement: groups and steps at level 0 (word +10 of a GROUPS record, word +14 of a step record = 0) are
 * placed against owner_0 on every entry point.  A level above n_levels (or any level >= 1 without installed
 * levels) returns RBGTOPO_EINVAL.  A level L in [1, n_levels] is placed only by a ctx created with
 * RBGTOPO_CFG_LEVEL_PLACEMENT; without the flag it returns RBGTOPO_ELIMIT, so that hosts built against a
 * level-0-only library keep withholding such hints.  With the flag the rules of level 0 apply with every
 * level-0 quantity replaced by level L's: a participating role may not use n when owner_L[n] is not -1 or
 * gid (dense rows and selection), D* = dom_L of the best feasible node of the first participating role and
 * the participating roles select inside dom_L = D*, fixed_domain and the reported domain are level-L domain
 * ids (fixed_domain >= level_n_domains[L - 1]: RBGTOPO_EINVAL).  Opted-out roles and non-exclusive groups
 * are unaffected.  Level-0 groups give the same results with and without the flag.  Every entry point
 * places at levels >= 1; rbgtopo_place_groups_committed does so only on a ctx created with
 * RBGTOPO_CFG_COMMIT_LEVELS as well (flags = 3), where the claims of earlier groups cross levels (see there),
 * and returns RBGTOPO_ELIMIT without it.  The describe calls accept any level >= 0.  Installing
 * partitions makes every staged handle with a step at a level >= 1 stale (run / fetch return RBGTOPO_EINVAL; release
 * still works): its level ids and fixed domains belong to the partitions it was validated against. */
#define RBGTOPO_MAX_EXCL_LEVELS 8
int32_t rbgtopo_set_exclusive_levels(rbgtopo_ctx* ctx, int32_t n_levels, const int32_t* level_domain,
                                     const int32_t* level_n_domains, int32_t n_occ, const int32_t* occ,
                                     uint64_t generation);

/* ---- the hot path ------------------------------------------------------- */
/* Score + select + greedy-assign one batch of steps (host buffers in, host
 * buffers out; H2D/D2H inside).  Plugs in between step 5 and step 7 of
 * Reconcile (rolebasedgroup_controller.go:193-207), i.e. from
 * ReconcilePodGroup (podgroup_manager.go:67-73).
 *   blob / blob_words  : the batch (layout above)
 *   assign[total R]    : node per replica in replica order, -1 = unplaced
 *   status[n_steps]    : RBGTOPO_PLACED_* per step
 *   domain[n_steps]    : exclusive domain chosen / confirmed, -1 if none
 * With world > 1 every rank calls it with the same blob: each scores its column
 * slab of the matrix and computes the identical assignment (replicated selection,
 * DESIGN.md §7). */
int32_t rbgtopo_score_assign(rbgtopo_ctx* ctx, const int32_t* blob,
                             int64_t blob_words, int32_t* assign,
                             int32_t* status, int32_t* domain);

/* ---- GROUPS blob: whole RoleBasedGroups, all dependency levels ------------ *
 * rbgtopo_place_groups runs the level/wave loop of the plugin on the host side
 * of the ABI (C++): for every group it forms the steps wave by wave — roles in
 * the given order (the caller passes them sorted by (level, name), i.e. the
 * output of rbgtopo_dependency_levels / dependency.go:129-205), a new wave at
 * every level change and whenever RBGTOPO_MAX_STEP_REPLICAS / _ROLES would be
 * exceeded — feeds the placements of wave w back as anchors / consumed
 * capacity / fixed exclusive domain of wave w+1 (levels see earlier levels:
 * rolebasedgroup_controller.go:448-476), and applies gang all-or-nothing over
 * the whole group (k8s-scheduler-plugin/manager.go:131).  On the device the
 * GROUPS blob itself is the plan: it is uploaded while the host still validates it,
 * one small launch derives the row table of the dense matrix from it, one launch
 * writes the dense rows of every wave, and one launch — a programmatic dependent
 * of the former — replays every group's waves from its role table in one CTA
 * (the direct path, DESIGN.md §4.4).  Groups whose table of patched nodes does not
 * fit a CTA's shared memory, RBGTOPO_VERIFY_PLAN and the opt-in pipelines take
 * the staged path instead: the blob is expanded into one step blob in HBM
 * (rbgtopo_stage_groups below) with the dense-matrix launch started from inside the
 * staging.  Same results, same error codes either way.
 * The dense rows of a plan are in GROUP order: row i is the
 * i-th pending replica of the blob (assign[] order).  With world > 1 every rank calls it with
 * the same blob and gets the same result (replicated selection, DESIGN.md §7).  need_rho of a wave is
 * min(RBGTOPO_NEED_CAP, still-unplaced replicas of the roles q with
 * pair[rho][q] > 0), DESIGN.md §3.2.
 *   word 0 magic 0x47474252 ("RBGG")  1 version  2 n_groups  3 total words
 *   word 4 total pending replicas     5..7 reserved
 *   n_groups records of RBGTOPO_GROUP_WORDS words:
 *     +0 gid  +1 flags (RBGTOPO_STEP_*)  +2 fixed_domain (-1 = none yet)
 *     +3 q = number of roles  +4 role_off (q records of 4 words:
 *        level, pending replicas, demand, role_flags)
 *     +5 pair_off (pair[q][q])  +6 n_anchors  +7 anchor_off (node, role, count)
 *     +8 assign_off (prefix sum of pending over earlier groups)
 *     +9 n_pending (sum of the roles' pending)  +10 exclusive level (0; see
 *        rbgtopo_set_exclusive_levels)  +11 reserved
 * Output: assign[total pending] in (group, role order, ordinal) order,
 * status[n_groups] (RBGTOPO_PLACED_*), domain[n_groups]. */
#define RBGTOPO_GROUPS_MAGIC 0x47474252
#define RBGTOPO_GROUP_WORDS  12
int32_t rbgtopo_place_groups(rbgtopo_ctx* ctx, const int32_t* groups,
                             int64_t groups_words, int32_t* assign,
                             int32_t* status, int32_t* domain);

/* Committed batch (DESIGN.md §3.8).  Same GROUPS blob, same outputs, same validation and error codes
 * as rbgtopo_place_groups, but the groups are placed IN BLOB ORDER, each seeing what the groups before
 * it took: every replica an earlier group placed consumes (node, demand) — a failed gang consumes
 * nothing — and every exclusive domain an earlier group reports (status != RBGTOPO_GANG_FAILED) counts
 * as owned by that group's gid (the last such group's, when several report it).  Scores, base and the
 * background order stay those of the snapshot.  So the hints of one call never ask a node for more
 * than free[n], and two exclusive groups with different gids never get the same domain unless the
 * caller fixed it (fixed_domain) for the later of the two.  Group 0 gets exactly what
 * rbgtopo_place_groups gives it.  The call holds the snapshot shared for all its rounds (one host
 * synchronisation each), so a long committed batch delays set_topology / update_nodes on the ctx.
 * Use it for batches of concurrent reconciles whose hints must hold together; rbgtopo_place_groups
 * keeps snapshot semantics (§3.7).  No dense matrix is computed; selection runs in rounds (at most
 * n_groups, one when no group reads a node or domain an earlier group took), *rounds (may be NULL) =
 * selection rounds run.  Valid for any world: every rank returns the identical result.  Gids need not
 * be distinct.  A group whose table of patched nodes does not fit k_plan_group's shared memory makes
 * the call return RBGTOPO_ELIMIT (there is no per-wave fallback for committed batches).
 * Levels (rbgtopo_set_exclusive_levels): a group at an exclusive level >= 1 is placed only by a ctx created
 * with RBGTOPO_CFG_LEVEL_PLACEMENT | RBGTOPO_CFG_COMMIT_LEVELS; with RBGTOPO_CFG_LEVEL_PLACEMENT alone it
 * returns RBGTOPO_ELIMIT, so hosts built against the level-0 contract keep withholding those hints.  Levels,
 * fixed domains and error codes are checked as by rbgtopo_place_groups.  A participating role of exclusive
 * group g at level L_g may not use node n when owner_{L_g}[n] (+) K (+) P is not -1 or gid_g, where
 *   K = (+) over the levels L of the batch's exclusive groups of the gid of the LAST earlier exclusive group
 *       at level L (status != RBGTOPO_GANG_FAILED) that reports dom_L(n) (an earlier group's anti-affinity on
 *       its own key, which kube-scheduler enforces symmetrically), and
 *   P = (+) of gid_h over every replica this call placed for a participating role of an earlier exclusive
 *       group h at a level L_h != L_g on a node m with dom_{L_g}(m) = dom_{L_g}(n) (g's own anti-affinity).
 * For a batch whose groups are all at level 0 this is the rule above: same results, same rounds. */
int32_t rbgtopo_place_groups_committed(rbgtopo_ctx* ctx, const int32_t* groups, int64_t groups_words,
                                       int32_t* assign, int32_t* status, int32_t* domain, int32_t* rounds);

/* Ranked placement (DESIGN.md §3.10).  rbgtopo_place_groups — same GROUPS blob, same validation and
 * error codes, bit-identical assign / status / domain on every path — plus, per pending replica r (in
 * assign order): score[r] = its dense-row score at assign[r], and alt_node[r * n_alt + i] /
 * alt_score[r * n_alt + i], i < n_alt, the next-best nodes of its row in descending key order (score
 * descending, node ascending) that still have room for one more replica of its role once the group's
 * own placements of this call are taken off free[], and, for a participating role of an exclusive
 * group, lie in the group's reported domain (a domain of the group's exclusive level: dom_L[n] = domain[g]).
 * Never the replica's own node.  The row of a replica is
 * the one of its wave that produced the final assignment (groups re-run by the host-driven loop
 * included).  Unfilled slots: node -1, score -inf; an unplaced replica and every replica of a
 * gang-failed group get score -inf and no alternates.  n_alt in [0, RBGTOPO_MAX_ALTERNATES], else
 * RBGTOPO_EINVAL; alt_node / alt_score may be NULL when n_alt == 0.
 * Documented limit: a ctx with world > 1 holds only its slab of every dense row, so the call returns
 * RBGTOPO_ELIMIT there.  An RBGTOPO_SPLIT_MIN_GROUPS split does not apply to this call. */
#define RBGTOPO_MAX_ALTERNATES 8
int32_t rbgtopo_place_groups_ranked(rbgtopo_ctx* ctx, const int32_t* groups, int64_t groups_words,
                                    int32_t n_alt, int32_t* assign, int32_t* status, int32_t* domain,
                                    float* score, int32_t* alt_node, float* alt_score);

/* rbgtopo_place_groups pipeline, staged: the groups are compiled into a
 * device-resident multi-wave plan (one step blob, wave-major, expanded on the
 * device), so rbgtopo_run_staged runs ONE score launch for the dense rows of every
 * wave plus one launch that walks every group's waves (or one launch per wave when
 * a group's table does not fit shared memory) with no host round trip; valid for
 * any world.  rbgtopo_fetch then
 * returns group-order results like place_groups (groups the plan could not finish
 * exactly — non-gang groups with an unplaced replica — keep status 1; place_groups
 * itself re-runs those through the host-driven loop). */
int32_t rbgtopo_stage_groups(rbgtopo_ctx* ctx, const int32_t* groups,
                             int64_t groups_words, int32_t* handle);

/* Same computation with the batch kept resident in HBM (bench `value` leg,
 * CUDA-graph replay): stage once, run many times, fetch results on demand. */
int32_t rbgtopo_stage(rbgtopo_ctx* ctx, const int32_t* blob, int64_t blob_words,
                      int32_t* handle);
/* run_staged only ENQUEUES `iters` passes on the call's stream (asynchronous);
 * rbgtopo_fetch synchronises, copies the results of the last pass (any output
 * pointer may be NULL) and harvests the timing of every pass since the
 * previous fetch (rbgtopo_last_timing: score_ms = average dense-matrix kernel (k_emit_rows for plans, k_score_emit for step batches)
 * duration from CUDA events recorded around each launch).  Valid for any world
 * (replicated selection); the shard calls below are the all-gather alternative. */
int32_t rbgtopo_run_staged(rbgtopo_ctx* ctx, int32_t handle, int32_t iters);

/* Pipeline of staged GROUPS batches (rbgtopo_stage_groups): enqueues `passes` passes, pass k over handles[k %
 * n_handles] — the reconcile loop of a controller that re-places several independent batches round robin
 * (rolebasedgroupset_controller.go:69-207 fans one RBGSet out into such batches).  The batches share nothing but the
 * snapshot, so the dense-matrix kernel of pass k + 1 is chained behind the selection kernel of pass k as a programmatic
 * dependent and fills the SMs while the slowest groups of pass k are still being placed.  Results as with
 * rbgtopo_run_staged: rbgtopo_fetch per handle.  The handles must be distinct; with one handle, kernel timing on, or
 * batches on different streams the passes run one after the other. */
int32_t rbgtopo_run_staged_chain(rbgtopo_ctx* ctx, const int32_t* handles, int32_t n_handles, int32_t passes);
int32_t rbgtopo_fetch(rbgtopo_ctx* ctx, int32_t handle, int32_t* assign,
                      int32_t* status, int32_t* domain);
int32_t rbgtopo_release(rbgtopo_ctx* ctx, int32_t handle);

/* Inspection of a staged+run batch (parity tests): one dense row
 * scores[n_nodes] of replica `row` (global replica index — for a staged GROUPS plan
 * the index into assign[], i.e. group order; local slab only when world > 1: out
 * has slab length), and the merged top-K keys of one role row (role rows of a
 * plan are numbered wave-major, rbgtopo_plan_describe column 5). */
int32_t rbgtopo_read_scores(rbgtopo_ctx* ctx, int32_t handle, int32_t row,
                            float* out, int32_t out_len);
int32_t rbgtopo_read_topk(rbgtopo_ctx* ctx, int32_t handle, int32_t rolerow,
                          uint64_t* out_keys, int32_t k);

/* Diagnostics / tests: copy one per-snapshot vector of the current snapshot to the host once the refresh
 * that produced it has completed, exactly as the device holds it.  what = RBGTOPO_SNAP_BASE (float[n]),
 * RBGTOPO_SNAP_ORDER (uint64[slab], key(base, node) form), RBGTOPO_SNAP_ORDER_ALL (uint64[n]; the same
 * buffer as ORDER when world == 1), RBGTOPO_SNAP_POS (int32[n], world == 1 only),
 * RBGTOPO_SNAP_DELTA_REPAIRS (int64[1]: incremental repairs since the last set_topology).  *n_out (may be
 * NULL) receives the element count, also when out_bytes is too small; then RBGTOPO_EINVAL is returned.
 * RBGTOPO_SNAP_LEVEL_OWNER (int32[(n_levels + 1) * n], level-major): the owner vectors of occupancy mode
 * (rbgtopo_set_exclusive_levels), 0 elements outside it. */
#define RBGTOPO_SNAP_BASE          0
#define RBGTOPO_SNAP_ORDER         1
#define RBGTOPO_SNAP_ORDER_ALL     2
#define RBGTOPO_SNAP_POS           3
#define RBGTOPO_SNAP_DELTA_REPAIRS 4
#define RBGTOPO_SNAP_LEVEL_OWNER   5
int32_t rbgtopo_read_snapshot(rbgtopo_ctx* ctx, int32_t what, void* out, int64_t out_bytes, int64_t* n_out);

/* ---- node-axis sharding over `world` GPUs (SURVEY.md §8e) --------------- *
 * rank g scores columns [slab_lo, slab_hi) and selects a local top-K; the
 * caller all-gathers the key lists (NCCL, one collective per pass) and every
 * rank runs the identical merge + greedy.
 *   shard_score : run score+select for the local slab of a staged batch;
 *                 (keys_dev, keys_bytes) = device buffer to all-gather.
 *   shard_merge : keys_all_dev = world x keys_bytes gathered buffer.  Returns
 *                 *need_pass2 = 1 when some exclusive step has to reselect
 *                 inside its chosen domain; then (keys2_dev, keys2_bytes) is
 *                 the second (small) buffer to all-gather.
 *   shard_assign: final merge + greedy (keys2_all_dev may be NULL when
 *                 need_pass2 was 0); results via rbgtopo_fetch. */
/* Wave-ranged forms.  A staged step batch has 1 wave; a staged GROUPS plan
 * (rbgtopo_stage_groups, also valid with world > 1) has W = rbgtopo_shard_waves
 * waves that must be run in order 0..W-1, each as score -> all-gather -> merge
 * [-> all-gather -> ] assign.  Wave 0's score call also enqueues the single
 * dense-matrix launch (k_emit_rows) for the rows of every wave on this rank's slab; the
 * placements are chained into later waves on every rank identically. */
int32_t rbgtopo_shard_waves(rbgtopo_ctx* ctx, int32_t handle, int32_t* n_waves);
int32_t rbgtopo_shard_wave_score(rbgtopo_ctx* ctx, int32_t handle, int32_t wave,
                                 void** keys_dev, int64_t* keys_bytes);
int32_t rbgtopo_shard_wave_merge(rbgtopo_ctx* ctx, int32_t handle, int32_t wave,
                                 const void* keys_all_dev, int32_t* need_pass2,
                                 void** keys2_dev, int64_t* keys2_bytes);
int32_t rbgtopo_shard_wave_assign(rbgtopo_ctx* ctx, int32_t handle, int32_t wave,
                                  const void* keys2_all_dev);
/* single-wave forms (wave 0 of a step batch) */
int32_t rbgtopo_shard_score(rbgtopo_ctx* ctx, int32_t handle, void** keys_dev,
                            int64_t* keys_bytes);
int32_t rbgtopo_shard_merge(rbgtopo_ctx* ctx, int32_t handle,
                            const void* keys_all_dev, int32_t* need_pass2,
                            void** keys2_dev, int64_t* keys2_bytes);
int32_t rbgtopo_shard_assign(rbgtopo_ctx* ctx, int32_t handle,
                             const void* keys2_all_dev);
int32_t rbgtopo_slab(rbgtopo_ctx* ctx, int32_t* lo, int32_t* hi);

/* ---- the same all-gather done by the library itself over NVLink peer memory (no NCCL call and no
 * host round trip on the step path; DESIGN.md §7).  Setup once per ctx, SPMD:
 *   rbgtopo_p2p_export : allocates this rank's exchange buffer (rows_cap role rows per wave and
 *                        source rank, 0 = 16 384) and returns its cudaIpcMemHandle (64 bytes) and /
 *                        or its device pointer (contexts of ONE process exchange the pointer);
 *   (caller all-gathers the handles — any transport: torch.distributed, MPI, the shim's gRPC)
 *   rbgtopo_p2p_import : maps the peers' buffers (handles_all = world x 64 bytes, rank-major) or
 *                        takes their pointers (peer_ptrs[world]); exactly one of the two.
 * rbgtopo_run_staged_p2p then enqueues, per pass and wave: k_shard_select -> k_p2p_push (peer stores
 * of the lists into every rank's buffer + a release flag) -> k_p2p_wait (acquire, bounded spin) ->
 * k_merge [-> restricted reselect -> push -> wait] -> k_greedy.  Every rank must make the same calls
 * in the same order.  Results via rbgtopo_fetch; rbgtopo_p2p_stats reports the bytes this rank
 * stored into peer memory during the last pass and whether a wait timed out (a peer never arrived:
 * the results of that pass are invalid). */
int32_t rbgtopo_p2p_export(rbgtopo_ctx* ctx, int32_t rows_cap, void* handle_out,
                           int32_t handle_len, void** local_ptr);
int32_t rbgtopo_p2p_import(rbgtopo_ctx* ctx, const void* handles_all, void* const* peer_ptrs);
int32_t rbgtopo_run_staged_p2p(rbgtopo_ctx* ctx, int32_t handle, int32_t iters);
int32_t rbgtopo_p2p_stats(rbgtopo_ctx* ctx, int64_t* peer_bytes_last_pass, int32_t* timed_out);

/* Use an external CUDA stream (e.g. the one the caller's NCCL runs on) for
 * every call on this ctx; NULL restores the internal per-slot streams (pass
 * cudaStreamLegacy, (void*)0x1, to select the legacy default stream). */
int32_t rbgtopo_set_stream(rbgtopo_ctx* ctx, void* cuda_stream);

/* Per-kernel CUDA events inside a pass.  Off (default): a pass is timed as a whole and the selection
 * kernel of a plan is launched as a programmatic dependent of the dense-matrix kernel (its CTAs become
 * resident while the last dense-matrix CTAs drain).  On: an event is recorded between the two kernels —
 * rbgtopo_last_timing / rbgtopo_last_pass_times then report each kernel, and the two kernels serialise
 * (what bench.py's roofline leg measures).  With timing off the passes of the resident entry points
 * (rbgtopo_run_staged) record no events at all (an event record between two kernels costs microseconds of
 * stream time): rbgtopo_last_timing then reports the staging and the D2H only.  Initial value: environment
 * RBGTOPO_KERNEL_TIMING. */
int32_t rbgtopo_set_kernel_timing(rbgtopo_ctx* ctx, int32_t on);

/* ---- stats (SURVEY.md §5 metrics row) ----------------------------------- */
int32_t rbgtopo_last_timing(rbgtopo_ctx* ctx, rbgtopo_timing* out);
/* Per-pass CUDA-event durations (ms) of the dense-matrix kernel (k_emit_rows for plans, k_score_emit for step batches) and of the
 * selection / assignment kernel(s), for every timed pass the last rbgtopo_fetch harvested
 * (bench.py prints their min / median so that a reported average can be checked).  At most `cap`
 * entries are written; *n_passes is the number available. */
int32_t rbgtopo_last_pass_times(rbgtopo_ctx* ctx, float* score_ms, float* select_ms,
                                int32_t cap, int32_t* n_passes);
int32_t rbgtopo_stats(rbgtopo_ctx* ctx, uint64_t* generation, int64_t* calls,
                      int64_t* scores_total, int64_t* kernel_launches);
/* Occupancy of the last launch of the selection kernel that walks every group's waves (k_plan_group): its CTAs
 * (groups with pending replicas), how many of them one SM holds at once with the launch's shared memory
 * (cudaOccupancyMaxActiveBlocksPerMultiprocessor) and the resulting rounds, ceil(ctas / (ctas_per_sm x SMs)).
 * Its launch order deals the heavy groups across the SMs assuming one round.  All 0 before the first launch.
 * Any output pointer may be NULL. */
int32_t rbgtopo_plan_occupancy(rbgtopo_ctx* ctx, int32_t* ctas, int32_t* ctas_per_sm, int32_t* rounds);

/* ======================================================================== *
 * Host-side plugin arithmetic (reference-pinned, SURVEY.md §8a a7-a15).
 * In production the Go shim calls the controller's own Go functions; these
 * C mirrors exist so that a C/C++/Python host above the ABI builds the same
 * steps the Go host would.  All follow the cited Go code exactly.
 * ======================================================================== */

/* RoleBasedGroup.GetGroupSize, api/workloads/v1alpha2/helper.go:50-65.
 * lws_size[i] <= 0 means "not a leader-worker role or size unset". */
int32_t rbgtopo_group_size(int32_t n_roles, const int32_t* replicas,
                           const int32_t* lws_size);

/* dependencyOrder, pkg/dependency/dependency.go:129-205.  Roles are given in
 * any order by name; dep_off[n_roles+1]/dep_idx index into the same role list.
 * Writes level_of[n_roles] and order[n_roles] (role indices sorted by (level,
 * name)); returns the number of levels, or RBGTOPO_EINVAL on a cycle. */
int32_t rbgtopo_dependency_levels(int32_t n_roles, const char* const* names,
                                  const int32_t* dep_off, const int32_t* dep_idx,
                                  int32_t* level_of, int32_t* order);

/* parsePercentage, pkg/coordination/coordinationscaling/scaler.go:253-270. */
int32_t rbgtopo_parse_percentage(const char* s, double* out);

/* CoordinationScaler.CalculateTargetReplicas, scaler.go:70-172 (+ progression
 * gate :192-242).  progression: 0 = unset (the Go switch then gates nothing),
 * 1 = OrderScheduled, 2 = OrderReady. */
int32_t rbgtopo_calculate_target_replicas(double max_skew, int32_t progression,
                                          int32_t n_roles,
                                          const int32_t* desired,
                                          const int32_t* current,
                                          const int32_t* scheduled,
                                          const int32_t* ready,
                                          int32_t* target);

/* GetScaledValueFromIntOrPercent,
 * vendor/k8s.io/apimachinery/pkg/util/intstr/intstr.go:181-197. */
int32_t rbgtopo_scaled_value(int32_t is_percent, int32_t value, int32_t total,
                             int32_t round_up);

/* calculateCoordinationUpdatedReplicasBound,
 * rolebasedgroup_controller.go:1328-1345. */
int32_t rbgtopo_updated_replicas_bound(int32_t max_skew_percent,
                                       int32_t ref_updated, int32_t ref_desired,
                                       int32_t request_desired, int32_t* lower,
                                       int32_t* upper);

/* calculateNextRollingTarget, rolebasedgroup_controller.go:1223-1263 (with
 * getFastestAndSlowestRole :1265-1282; ties beyond the reference's comparator
 * are broken by role index).  rolling_target[n_roles] out. Returns 0, or 1 when
 * the reference returns nil (fewer than two roles). */
int32_t rbgtopo_next_rolling_target(int32_t max_skew_percent, int32_t n_roles,
                                    const int32_t* desired,
                                    const int32_t* updated,
                                    const int32_t* ready,
                                    int32_t* rolling_target);

/* CalculatePartitionReplicas, pkg/utils/utils.go:139-162.  has_partition = 0: nil partition;
 * is_percent: the partition is the string "<value>%"; replicas < 0 = nil replicas pointer. */
int32_t rbgtopo_partition_replicas(int32_t has_partition, int32_t is_percent, int32_t value,
                                   int32_t replicas, int32_t* out);

/* ParseIntStrAsNonZero, pkg/utils/utils.go:177-185. */
int32_t rbgtopo_intstr_non_zero(int32_t is_percent, int32_t value, int32_t replicas,
                                int32_t* out);

/* mergeStrategyRollingUpdate, rolebasedgroup_controller.go:1284-1314, for one role present in
 * both maps.  Strategy = 6 ints: maxUnavailable (has, is_percent, value), partition (has,
 * is_percent, value).  out = the merged strategy. */
int32_t rbgtopo_merge_rolling_update(const int32_t* strategy_a, const int32_t* strategy_b,
                                     int32_t* out);

/* GetWorkloadName, api/workloads/v1alpha2/helper.go:68-81 ("{rbg}-{role}", 63 bytes, trailing '-'
 * trimmed); out_len >= 64; returns the length. */
int32_t rbgtopo_workload_name(const char* rbg_name, const char* role_name, char* out,
                              int32_t out_len);

/* GenGroupUniqueKey, helper.go:135-144: hex SHA-1 of "namespace/name" — the value of the
 * group-unique-hash label the exclusive-topology affinity terms match on
 * (pkg/reconciler/pod_reconciler.go:172-231); out_len >= 41; returns 40. */
int32_t rbgtopo_group_unique_key(const char* ns, const char* name, char* out, int32_t out_len);

/* InheritPodGroupAnnotations, pkg/scheduler/common/annotation_inheritance.go:23-43, per key:
 * 1 when the PodGroup inherits the annotation (the key starts with one of the prefixes). */
int32_t rbgtopo_inherits_annotation(const char* key, int32_t n_prefixes,
                                    const char* const* prefixes);

/* ---- host-only inspection of the multi-wave plan (no GPU needed) ----------- *
 * The step geometry rbgtopo_place_groups / rbgtopo_stage_groups derive from a
 * GROUPS blob — which wave every pending replica is placed in, how the waves of
 * all groups are laid out wave-major — computed by the very code path those
 * calls use, without touching a device (unit tests, capacity planning).
 *   deg_plus1[n_nodes] = CSR degree + 1 per node (NULL: 1 everywhere), wsum_max =
 *   largest row sum of edge weights (0: none): they only enter the patch-list
 *   capacities and the exactness bound (RBGTOPO_EINEXACT).
 * out_steps receives RBGTOPO_PLAN_STEP_WORDS ints per step, steps in wave-major
 * order: group index, wave of the group, section offset, section end (words of
 * the step blob), first replica row (= the group's assign_off + the replicas of
 * its earlier waves: dense rows and assign[] are in GROUP order), first role row
 * (wave-major prefix), next step of the group (0 = last), replicas of the group
 * placed by its earlier waves.  At most
 * out_cap_steps steps are written; *n_steps / *n_waves / *plan_words report the
 * totals. */
#define RBGTOPO_PLAN_STEP_WORDS 8
int32_t rbgtopo_plan_describe(const int32_t* groups, int64_t groups_words,
                              int32_t n_nodes, int32_t n_domains,
                              const int32_t* deg_plus1, int64_t wsum_max,
                              int32_t* out_steps, int64_t out_cap_steps,
                              int32_t* n_steps, int32_t* n_waves,
                              int64_t* plan_words);

/* What the DIRECT path of rbgtopo_place_groups derives on the host (the code path the call uses, without a device):
 * both validation passes — a malformed blob returns the code rbgtopo_place_groups returns — and
 *   geom[0] pending replicas (dense rows)   [1] groups with pending replicas (= CTAs of the selection kernel)
 *   geom[2] / [3] largest role count of a group / of a wave
 *   geom[4] largest table capacity (closed neighbourhoods of the scheduled pods and of the replicas placed before the last
 *           wave, + those replicas)   [5] threads per CTA   [6] / [7] hash-table and dense-view sizes of the selection kernel
 * order[0 .. geom[1]) = the groups in the launch order of the selection kernel: descending (pending replicas + scheduled
 * pods), ties in group order — while the grid fits in one round (rbgtopo_plan_occupancy) every CTA starts at once and
 * stays on its SM for the whole kernel, so the order decides which groups share an SM.  deg_plus1 / wsum_max as for rbgtopo_plan_describe. */
int32_t rbgtopo_place_describe(const int32_t* groups, int64_t groups_words, int32_t n_nodes, int32_t n_domains,
                               const int32_t* deg_plus1, int64_t wsum_max, int32_t* order, int64_t order_cap, int32_t* geom);

#ifdef __cplusplus
}
#endif
#endif /* RBGTOPO_H_ */
