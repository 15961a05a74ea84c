/*
 * cabi_eligible_committed.c — calls rbgtopo_place_groups_eligible_committed[_ranked] the way the cgo shim does
 * (go/pkg/scheduler/b200topo/cgo_bridge.go, rbgtopo_go_place_groups_eligible_committed[_ranked]): plain C arrays and
 * sizes, the call and the error fetch in one helper on one OS thread.  TEST INFRASTRUCTURE (the companion of
 * tests/cabi_eligible.c).
 *
 *   cabi_eligible_committed host   no device needed: bad arguments come back as codes with their text, rounds = 0
 *   cabi_eligible_committed gpu    the fleet of cabi_eligible.c as one committed batch: with full masks the outputs
 *                                  equal rbgtopo_place_groups_lw_committed[_ranked]'s, rounds included; with masks of
 *                                  2, 2 and 4 of 4 classes every pod and alternate lies on an admitted node and no
 *                                  node receives more than its capacity; then 10 OS threads make both calls on one
 *                                  ctx while another re-installs the same classes and capacities: every output equals
 *                                  the sequential one; the error codes, each followed by a call that works
 * Prints "CABI_ELIGIBLE_COMMITTED_OK <mode>" and exits 0 on success.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/rbgtopo.h"

#define CHECK(cond, ...) do { if (!(cond)) { fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); \
  fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); exit(1); } } while (0)

/* the cgo preamble helpers: call + error text on the same OS thread */
static int32_t go_place_groups_eligible_committed(rbgtopo_ctx* ctx, const int32_t* groups, int64_t words,
                                                  const int32_t* rp, int64_t rp_words, const uint64_t* admit,
                                                  int64_t n_admit, int32_t* assign, int32_t* status, int32_t* domain,
                                                  int32_t* rounds, char* err, int errlen) {
  int32_t rc = rbgtopo_place_groups_eligible_committed(ctx, groups, words, rp, rp_words, admit, n_admit, assign, status,
                                                       domain, rounds);
  if (rc != RBGTOPO_OK) rbgtopo_last_error(ctx, err, errlen); else err[0] = 0;
  return rc;
}
static int32_t go_place_groups_eligible_committed_ranked(rbgtopo_ctx* ctx, const int32_t* groups, int64_t words,
                                                         const int32_t* rp, int64_t rp_words, const uint64_t* admit,
                                                         int64_t n_admit, int32_t n_alt, int32_t* assign,
                                                         int32_t* status, int32_t* domain, int32_t* rounds,
                                                         float* score, int32_t* alt_node, float* alt_score, char* err,
                                                         int errlen) {
  int32_t rc = rbgtopo_place_groups_eligible_committed_ranked(ctx, groups, words, rp, rp_words, admit, n_admit, n_alt,
                                                              assign, status, domain, rounds, score, alt_node,
                                                              alt_score);
  if (rc != RBGTOPO_OK) rbgtopo_last_error(ctx, err, errlen); else err[0] = 0;
  return rc;
}

static int run_host(void) {
  char err[256];
  int32_t rounds = 77;
  int32_t rc = go_place_groups_eligible_committed(NULL, NULL, 0, NULL, 0, NULL, 0, NULL, NULL, NULL, &rounds, err,
                                                  sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strlen(err) > 0 && rounds == 0, "committed, null ctx: %d '%s' %d", rc, err, rounds);
  rounds = 77;
  rc = go_place_groups_eligible_committed_ranked(NULL, NULL, 0, NULL, 0, NULL, 0, 2, NULL, NULL, NULL, &rounds, NULL,
                                                 NULL, NULL, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strlen(err) > 0 && rounds == 0, "ranked, null ctx: %d '%s' %d", rc, err, rounds);
  printf("CABI_ELIGIBLE_COMMITTED_OK host\n");
  return 0;
}

#define NN 4096
#define NG 48
#define PG 15 /* pods per group: a 1 x 1, b 3 x 2 (co-located at level 0), c 2 x 4 */
#define NP (NG * PG)
#define NALT 4
#define NCLS 4
static const uint64_t kMask[3] = {0x3, 0x6, 0xF}; /* roles a, b, c */
static const int32_t kDemand[3] = {1, 1, 1};

typedef struct {
  rbgtopo_ctx* ctx;
  const int32_t *blob, *rp;
  int64_t words;
  const uint64_t* admit;
  const int32_t *want_assign, *want_status, *want_domain, *want_alt;
  int32_t want_rounds;
  const float* want_score;
  int bad;
} job_t;

static void* worker(void* arg) {
  job_t* j = (job_t*)arg;
  int32_t assign[NP], status[NG], domain[NG], alt[NP * NALT], rounds;
  float score[NP], alt_score[NP * NALT];
  char err[256];
  for (int it = 0; it < 3; ++it) {
    int32_t rc = go_place_groups_eligible_committed_ranked(j->ctx, j->blob, j->words, j->rp, 6 * NG, j->admit, 3 * NG,
                                                           NALT, assign, status, domain, &rounds, score, alt, alt_score,
                                                           err, sizeof err);
    if (rc != RBGTOPO_OK || rounds != j->want_rounds || memcmp(assign, j->want_assign, sizeof assign) != 0 ||
        memcmp(status, j->want_status, sizeof status) != 0 || memcmp(domain, j->want_domain, sizeof domain) != 0 ||
        memcmp(alt, j->want_alt, sizeof alt) != 0 || memcmp(score, j->want_score, sizeof score) != 0)
      j->bad++;
    rc = go_place_groups_eligible_committed(j->ctx, j->blob, j->words, j->rp, 6 * NG, j->admit, 3 * NG, assign, status,
                                            domain, &rounds, err, sizeof err);
    if (rc != RBGTOPO_OK || rounds != j->want_rounds || memcmp(assign, j->want_assign, sizeof assign) != 0 ||
        memcmp(status, j->want_status, sizeof status) != 0 || memcmp(domain, j->want_domain, sizeof domain) != 0)
      j->bad++;
  }
  return NULL;
}

typedef struct {
  rbgtopo_ctx* ctx;
  const int32_t *cls, *free_slots;
  int bad;
} refresh_t;

/* the same classes and capacities again and again: a refresh that changes nothing, interleaved with the placements */
static void* refresher(void* arg) {
  refresh_t* r = (refresh_t*)arg;
  for (int it = 0; it < 20; ++it) {
    if (rbgtopo_set_node_classes(r->ctx, NCLS, r->cls, 2 + it) != RBGTOPO_OK) r->bad++;
    if (rbgtopo_update_nodes(r->ctx, r->free_slots, NULL, 2 + it) != RBGTOPO_OK) r->bad++;
  }
  return NULL;
}

static int run_gpu(void) {
  rbgtopo_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.world = 1;
  rbgtopo_ctx* ctx = NULL;
  char err[256];
  int32_t rc = rbgtopo_create(&cfg, &ctx);
  if (rc != RBGTOPO_OK) {
    rbgtopo_last_error(NULL, err, sizeof err);
    CHECK(0, "rbgtopo_create: %d %s", rc, err);
  }
  /* topology: NVLink cliques of 8 (weight 1000) + a ring across domains (weight 10), symmetric, sorted rows */
  static int32_t row_ptr[NN + 1], col[NN * 9], w[NN * 9], free_slots[NN], domain_of[NN], owner[NN / 8];
  int64_t e = 0;
  for (int i = 0; i < NN; ++i) {
    row_ptr[i] = (int32_t)e;
    int nb[9], nw[9], k = 0;
    for (int o = 0; o < 8; ++o) {
      int p = (i / 8) * 8 + o;
      if (p != i) { nb[k] = p; nw[k++] = 1000; }
    }
    nb[k] = (i + 8) % NN; nw[k++] = 10;
    nb[k] = (i + NN - 8) % NN; nw[k++] = 10;
    for (int a = 0; a < k; ++a)   /* insertion sort by column */
      for (int b = a + 1; b < k; ++b)
        if (nb[b] < nb[a]) { int t = nb[a]; nb[a] = nb[b]; nb[b] = t; t = nw[a]; nw[a] = nw[b]; nw[b] = t; }
    for (int a = 0; a < k; ++a) { col[e] = nb[a]; w[e] = nw[a]; ++e; }
    free_slots[i] = (int32_t)((i * 2654435761u >> 7) % 9);
    domain_of[i] = i / 8;
  }
  row_ptr[NN] = (int32_t)e;
  for (int d = 0; d < NN / 8; ++d) owner[d] = -1;
  rc = rbgtopo_set_topology(ctx, NN, e, row_ptr, col, w, free_slots, domain_of, NN / 8, owner, 1);
  if (rc != RBGTOPO_OK) { rbgtopo_last_error(ctx, err, sizeof err); CHECK(0, "set_topology: %s", err); }

  /* GROUPS blob: NG groups, roles (level, pending, demand, flags): a(0,1,1) | b(1,3,1), c(1,2,1); pair = all ones;
   * every 4th group gang, every 3rd exclusive, gids shared in pairs; one scheduled pod each */
  const int q = 3, per = 4 * q + q * q + 3;
  const int words = RBGTOPO_HDR_WORDS + NG * RBGTOPO_GROUP_WORDS + NG * per;
  int32_t* blob = (int32_t*)calloc((size_t)words, sizeof(int32_t));
  blob[0] = RBGTOPO_GROUPS_MAGIC; blob[1] = RBGTOPO_ABI_VERSION; blob[2] = NG; blob[3] = words; blob[4] = NG * 6;
  int off = RBGTOPO_HDR_WORDS + NG * RBGTOPO_GROUP_WORDS;
  for (int g = 0; g < NG; ++g) {
    int32_t* rec = blob + RBGTOPO_HDR_WORDS + g * RBGTOPO_GROUP_WORDS;
    rec[0] = g / 2;
    rec[1] = ((g % 4 == 0) ? RBGTOPO_STEP_GANG : 0) | ((g % 3 == 0) ? RBGTOPO_STEP_EXCLUSIVE : 0);
    rec[2] = -1; rec[3] = q;
    rec[4] = off;
    const int32_t roles[12] = {0, 1, kDemand[0], RBGTOPO_ROLE_EXCLUSIVE, 1, 3, kDemand[1], RBGTOPO_ROLE_EXCLUSIVE,
                               1, 2, kDemand[2], RBGTOPO_ROLE_EXCLUSIVE};
    memcpy(blob + off, roles, sizeof roles); off += 12;
    rec[5] = off;
    for (int i = 0; i < q * q; ++i) blob[off++] = 1;
    rec[6] = 1; rec[7] = off;
    blob[off++] = (g * 83) % NN; blob[off++] = 0; blob[off++] = 1;
    rec[8] = g * 6; rec[9] = 6;
  }
  CHECK(off == words, "blob size");
  int32_t rp[6 * NG];
  for (int g = 0; g < NG; ++g) {
    const int32_t t[6] = {1, -1, 2, 0, 4, -1};
    memcpy(rp + 6 * g, t, sizeof t);
  }

  static int32_t cls[NN];
  for (int i = 0; i < NN; ++i) cls[i] = i % NCLS;
  uint64_t admit[3 * NG], full[3 * NG];
  for (int g = 0; g < NG; ++g)
    for (int r = 0; r < 3; ++r) { admit[3 * g + r] = kMask[r]; full[3 * g + r] = ~0ull; }

  static int32_t a1[NP], a2[NP], alt1[NP * NALT], alt2[NP * NALT];
  static float sc1[NP], sc2[NP], as1[NP * NALT], as2[NP * NALT];
  int32_t s1[NG], s2[NG], d1[NG], d2[NG], r1 = 77, r2 = 77;
  /* no classes installed yet: refused, nothing placed, rounds 0 */
  rc = go_place_groups_eligible_committed(ctx, blob, words, rp, 6 * NG, admit, 3 * NG, a1, s1, d1, &r1, err,
                                          sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strstr(err, "classes") && r1 == 0, "no classes installed: %d '%s'", rc, err);
  rc = rbgtopo_set_node_classes(ctx, NCLS, cls, 1);
  CHECK(rc == RBGTOPO_OK, "set_node_classes: %d", rc);

  /* full masks: rbgtopo_place_groups_lw_committed_ranked bit for bit, rounds included */
  rc = go_place_groups_eligible_committed_ranked(ctx, blob, words, rp, 6 * NG, full, 3 * NG, NALT, a1, s1, d1, &r1,
                                                 sc1, alt1, as1, err, sizeof err);
  CHECK(rc == RBGTOPO_OK, "full masks: %d %s", rc, err);
  rc = rbgtopo_place_groups_lw_committed_ranked(ctx, blob, words, rp, 6 * NG, NALT, a2, s2, d2, &r2, sc2, alt2, as2);
  CHECK(rc == RBGTOPO_OK && r1 == r2 && memcmp(a1, a2, sizeof a1) == 0 && memcmp(s1, s2, sizeof s1) == 0 &&
        memcmp(d1, d2, sizeof d1) == 0 && memcmp(sc1, sc2, sizeof sc1) == 0 && memcmp(alt1, alt2, sizeof alt1) == 0 &&
        memcmp(as1, as2, sizeof as1) == 0, "full masks differ from rbgtopo_place_groups_lw_committed_ranked");

  /* restricting masks: sequential twice, the unranked call equal, every pod and alternate admitted, no node over */
  rc = go_place_groups_eligible_committed_ranked(ctx, blob, words, rp, 6 * NG, admit, 3 * NG, NALT, a1, s1, d1, &r1,
                                                 sc1, alt1, as1, err, sizeof err);
  CHECK(rc == RBGTOPO_OK && r1 >= 1 && r1 <= NG, "ranked: %d %s (rounds %d)", rc, err, r1);
  rc = go_place_groups_eligible_committed_ranked(ctx, blob, words, rp, 6 * NG, admit, 3 * NG, NALT, a2, s2, d2, &r2,
                                                 sc2, alt2, as2, err, sizeof err);
  CHECK(rc == RBGTOPO_OK && r1 == r2 && memcmp(a1, a2, sizeof a1) == 0 && memcmp(alt1, alt2, sizeof alt1) == 0 &&
        memcmp(sc1, sc2, sizeof sc1) == 0, "the sequential repeat differs");
  rc = go_place_groups_eligible_committed(ctx, blob, words, rp, 6 * NG, admit, 3 * NG, a2, s2, d2, &r2, err, sizeof err);
  CHECK(rc == RBGTOPO_OK && r1 == r2 && memcmp(a2, a1, sizeof a1) == 0 && memcmp(s2, s1, sizeof s1) == 0 &&
        memcmp(d2, d1, sizeof d1) == 0, "the unranked call differs");
  static int32_t used[NN];
  int placed = 0, alts = 0;
  for (int i = 0; i < NP; ++i) {
    const int k = i % PG, role = k < 1 ? 0 : k < 7 ? 1 : 2;
    if (a1[i] < 0) continue;
    ++placed;
    used[a1[i]] += kDemand[role];
    CHECK((kMask[role] >> cls[a1[i]]) & 1, "pod %d of role %d on node %d of class %d", i, role, a1[i], cls[a1[i]]);
    for (int m = 0; m < NALT; ++m) {
      const int32_t n = alt1[i * NALT + m];
      if (n < 0) continue;
      ++alts;
      CHECK((kMask[role] >> cls[n]) & 1, "pod %d: alternate %d of class %d", i, n, cls[n]);
    }
  }
  for (int i = 0; i < NN; ++i) CHECK(used[i] <= free_slots[i], "node %d: %d of %d", i, used[i], free_slots[i]);
  CHECK(placed > NP / 2 && alts > placed, "placed %d of %d, %d alternates", placed, NP, alts);

  /* argument errors: rounds 0 */
  r2 = 77;
  rc = go_place_groups_eligible_committed(ctx, blob, words, rp, 6 * NG, admit, 3 * NG - 1, a2, s2, d2, &r2, err,
                                          sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strstr(err, "role_admit") && r2 == 0, "one mask short: %d '%s'", rc, err);
  r2 = 77;
  rc = go_place_groups_eligible_committed(ctx, blob, words, rp, 6 * NG, NULL, 3 * NG, a2, s2, d2, &r2, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strlen(err) > 0 && r2 == 0, "NULL masks: %d '%s'", rc, err);
  r2 = 77;
  rc = go_place_groups_eligible_committed_ranked(ctx, blob, words, rp, 6 * NG, admit, 3 * NG,
                                                 RBGTOPO_MAX_ALTERNATES + 1, a2, s2, d2, &r2, sc2, alt2, as2, err,
                                                 sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strstr(err, "n_alt") && r2 == 0, "n_alt out of range: %d '%s'", rc, err);

  /* concurrency: 10 threads making both calls and one refresher on one ctx */
  pthread_t th[10], rt;
  job_t jobs[10];
  refresh_t ref = {ctx, cls, free_slots, 0};
  pthread_create(&rt, NULL, refresher, &ref);
  for (int t = 0; t < 10; ++t) {
    jobs[t] = (job_t){ctx, blob, rp, words, admit, a1, s1, d1, alt1, r1, sc1, 0};
    pthread_create(&th[t], NULL, worker, &jobs[t]);
  }
  int bad = 0;
  for (int t = 0; t < 10; ++t) { pthread_join(th[t], NULL); bad += jobs[t].bad; }
  pthread_join(rt, NULL);
  CHECK(ref.bad == 0, "%d refreshes failed", ref.bad);
  CHECK(bad == 0, "%d concurrent calls differ from the sequential result", bad);
  rbgtopo_destroy(ctx);
  free(blob);
  printf("CABI_ELIGIBLE_COMMITTED_OK gpu placed %d rounds %d\n", placed, r1);
  return 0;
}

int main(int argc, char** argv) {
  if (argc > 1 && strcmp(argv[1], "gpu") == 0) return run_gpu();
  return run_host();
}
