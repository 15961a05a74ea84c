/*
 * cabi_lw_committed_levels.c — rbgtopo_place_groups_lw_committed and its ranked form on a ctx created with
 * RBGTOPO_CFG_LW_COMMIT_LEVELS (flags = 7, DESIGN.md §3.16), called the way the cgo shim calls them: plain C, int32
 * arrays and sizes, the call and the error fetch in one helper on one OS thread, and ten OS threads on one ctx.
 * TEST INFRASTRUCTURE (modelled on tests/cabi_lw_committed.c).
 *
 *   cabi_lw_committed_levels host   no device needed: bad arguments and flags come back as codes with their text
 *   cabi_lw_committed_levels gpu    a synthetic 2-tier topology with two partitions installed (hostnames, racks of
 *                                   64) + a fleet of 3-role groups whose roles run 2-pod replicas, exclusive groups
 *                                   at levels 0, 1 and 2 in turn, placed as one committed batch, repeated sequentially
 *                                   and then 10 x 3 times concurrently, plain and ranked: assign, status, domain,
 *                                   rounds and alternates identical every time; no node over-committed over the batch;
 *                                   no two gids report one (level, domain)
 * Prints "CABI_LW_COMMITTED_LEVELS_OK <mode>" and exits 0 on success.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/rbgtopo.h"

#define CHECK(cond, ...) do { if (!(cond)) { fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); \
  fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); exit(1); } } while (0)

/* the cgo preamble helper: call + error text on the same OS thread */
static int32_t go_place_groups_lw_committed(rbgtopo_ctx* ctx, const int32_t* groups, int64_t words,
                                            const int32_t* role_pods, int64_t role_pods_words, int32_t* assign,
                                            int32_t* status, int32_t* domain, int32_t* rounds, char* err, int errlen) {
  int32_t rc = rbgtopo_place_groups_lw_committed(ctx, groups, words, role_pods, role_pods_words, assign, status, domain,
                                                 rounds);
  if (rc != RBGTOPO_OK) rbgtopo_last_error(ctx, err, errlen); else err[0] = 0;
  return rc;
}

static int32_t go_place_groups_lw_committed_ranked(rbgtopo_ctx* ctx, const int32_t* groups, int64_t words,
                                                   const int32_t* role_pods, int64_t role_pods_words, int32_t n_alt,
                                                   int32_t* assign, int32_t* status, int32_t* domain, int32_t* rounds,
                                                   float* score, int32_t* alt_node, float* alt_score, char* err,
                                                   int errlen) {
  int32_t rc = rbgtopo_place_groups_lw_committed_ranked(ctx, groups, words, role_pods, role_pods_words, n_alt, assign,
                                                        status, domain, rounds, score, alt_node, alt_score);
  if (rc != RBGTOPO_OK) rbgtopo_last_error(ctx, err, errlen); else err[0] = 0;
  return rc;
}

static int run_host(void) {
  char err[256];
  int32_t rounds = 7;
  int32_t rc = go_place_groups_lw_committed(NULL, NULL, 0, NULL, 0, NULL, NULL, NULL, &rounds, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strlen(err) > 0 && rounds == 0, "null ctx: %d '%s' rounds %d", rc, err, rounds);
  /* the new flag without RBGTOPO_CFG_COMMIT_LEVELS: checked before any device is looked for */
  rbgtopo_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.world = 1;
  cfg.flags = RBGTOPO_CFG_LEVEL_PLACEMENT | RBGTOPO_CFG_LW_COMMIT_LEVELS;
  rbgtopo_ctx* ctx = NULL;
  rc = rbgtopo_create(&cfg, &ctx);
  rbgtopo_last_error(NULL, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && ctx == NULL && strstr(err, "RBGTOPO_CFG_LW_COMMIT_LEVELS"), "flags 5: %d '%s'", rc, err);
  printf("CABI_LW_COMMITTED_LEVELS_OK host\n");
  return 0;
}

#define NN 4096
#define NG 48
#define PODS 9      /* per group: role a 1 x 2 pods (co-located at level 0), b 3 x 1, c 2 x 2 */
#define NP (NG * PODS)
#define NALT 3
typedef struct {
  rbgtopo_ctx* ctx;
  const int32_t* blob;
  int64_t words;
  const int32_t* rp;
  const int32_t *want_assign, *want_status, *want_domain;
  int32_t want_rounds;
  const float *want_score, *want_alt_score;
  const int32_t* want_alt;
  int bad;
} job_t;

static void* worker(void* arg) {
  job_t* j = (job_t*)arg;
  int32_t assign[NP], status[NG], domain[NG], rounds = 0, alt[NP * NALT];
  float score[NP], alt_score[NP * NALT];
  char err[256];
  for (int it = 0; it < 3; ++it) {
    int32_t rc = go_place_groups_lw_committed(j->ctx, j->blob, j->words, j->rp, 6 * NG, assign, status, domain, &rounds,
                                              err, sizeof err);
    if (rc != RBGTOPO_OK || memcmp(assign, j->want_assign, sizeof assign) != 0 ||
        memcmp(status, j->want_status, sizeof status) != 0 || memcmp(domain, j->want_domain, sizeof domain) != 0 ||
        rounds != j->want_rounds)
      j->bad++;
    rc = go_place_groups_lw_committed_ranked(j->ctx, j->blob, j->words, j->rp, 6 * NG, NALT, assign, status, domain,
                                             &rounds, score, alt, alt_score, err, sizeof err);
    if (rc != RBGTOPO_OK || memcmp(assign, j->want_assign, sizeof assign) != 0 || rounds != j->want_rounds ||
        memcmp(score, j->want_score, sizeof score) != 0 || memcmp(alt, j->want_alt, sizeof alt) != 0 ||
        memcmp(alt_score, j->want_alt_score, sizeof alt_score) != 0)
      j->bad++;
  }
  return NULL;
}

static int run_gpu(void) {
  rbgtopo_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.world = 1;
  cfg.flags = RBGTOPO_CFG_LEVEL_PLACEMENT | RBGTOPO_CFG_COMMIT_LEVELS | RBGTOPO_CFG_LW_COMMIT_LEVELS;
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
  /* levels 1 (hostnames) and 2 (racks of 64), no records */
  static int32_t level_domain[2 * NN];
  const int32_t level_nd[2] = {NN, NN / 64};
  for (int i = 0; i < NN; ++i) { level_domain[i] = i; level_domain[NN + i] = i / 64; }
  rc = rbgtopo_set_exclusive_levels(ctx, 2, level_domain, level_nd, 0, NULL, 2);
  if (rc != RBGTOPO_OK) { rbgtopo_last_error(ctx, err, sizeof err); CHECK(0, "set_exclusive_levels: %s", err); }

  /* GROUPS blob: NG groups, roles (level, pending, demand, flags): a(0,1,1) | b(1,3,1), c(1,2,1); pair = all ones;
   * every 4th group gang, every 2nd exclusive at level 0, 1, 2 in turn; one scheduled pod each */
  const int q = 3, per = 4 * q + q * q + 3;
  const int words = RBGTOPO_HDR_WORDS + NG * RBGTOPO_GROUP_WORDS + NG * per;
  int32_t* blob = (int32_t*)calloc((size_t)words, sizeof(int32_t));
  blob[0] = RBGTOPO_GROUPS_MAGIC; blob[1] = RBGTOPO_ABI_VERSION; blob[2] = NG; blob[3] = words; blob[4] = NG * 6;
  int off = RBGTOPO_HDR_WORDS + NG * RBGTOPO_GROUP_WORDS;
  for (int g = 0; g < NG; ++g) {
    int32_t* rec = blob + RBGTOPO_HDR_WORDS + g * RBGTOPO_GROUP_WORDS;
    rec[0] = g;
    rec[1] = ((g % 4 == 0) ? RBGTOPO_STEP_GANG : 0) | ((g % 2 == 0) ? RBGTOPO_STEP_EXCLUSIVE : 0);
    rec[10] = (g / 2) % 3;
    rec[2] = -1; rec[3] = q;
    rec[4] = off;
    const int32_t roles[12] = {0, 1, 1, RBGTOPO_ROLE_EXCLUSIVE, 1, 3, 1, RBGTOPO_ROLE_EXCLUSIVE, 1, 2, 1, RBGTOPO_ROLE_EXCLUSIVE};
    memcpy(blob + off, roles, sizeof roles); off += 12;
    rec[5] = off;
    for (int i = 0; i < q * q; ++i) blob[off++] = 1;
    rec[6] = 1; rec[7] = off;
    blob[off++] = (g * 83) % NN; blob[off++] = 0; blob[off++] = 1;
    rec[8] = g * 6; rec[9] = 6;  /* replicas; the pods follow from role_pods */
  }
  CHECK(off == words, "blob size");
  static int32_t rp[6 * NG];
  for (int g = 0; g < NG; ++g) {
    const int32_t sc[6] = {2, 0, 1, -1, 2, -1};
    memcpy(rp + 6 * g, sc, sizeof sc);
  }

  static int32_t a1[NP], a2[NP];
  int32_t s1[NG], s2[NG], d1[NG], d2[NG], r1 = 0, r2 = 0;
  rc = go_place_groups_lw_committed(ctx, blob, words, rp, 6 * NG, a1, s1, d1, &r1, err, sizeof err);
  CHECK(rc == RBGTOPO_OK && r1 >= 1 && r1 <= NG, "committed: %d rounds %d %s", rc, r1, err);
  rc = go_place_groups_lw_committed(ctx, blob, words, rp, 6 * NG, a2, s2, d2, &r2, err, sizeof err);
  CHECK(rc == RBGTOPO_OK, "committed again: %d %s", rc, err);
  CHECK(memcmp(a1, a2, sizeof a1) == 0 && memcmp(s1, s2, sizeof s1) == 0 && memcmp(d1, d2, sizeof d1) == 0 && r1 == r2,
        "the sequential repeat differs (rounds %d vs %d)", r1, r2);
  static int32_t alt1[NP * NALT];
  static float sc1[NP], asc1[NP * NALT];
  int32_t r3 = 0;
  rc = go_place_groups_lw_committed_ranked(ctx, blob, words, rp, 6 * NG, NALT, a2, s2, d2, &r3, sc1, alt1, asc1, err,
                                           sizeof err);
  CHECK(rc == RBGTOPO_OK && memcmp(a1, a2, sizeof a1) == 0 && r3 == r1, "ranked: %d %s", rc, err);
  /* within capacity over the whole batch; no (level, domain) reported by two gids (no group fixes one) */
  static int32_t used[NN];
  int placed = 0;
  for (int i = 0; i < NP; ++i) {
    CHECK(a1[i] >= -1 && a1[i] < NN, "assign[%d] = %d", i, a1[i]);
    if (a1[i] >= 0) { ++placed; CHECK(++used[a1[i]] <= free_slots[a1[i]], "node %d over-committed", a1[i]); }
  }
  CHECK(placed > NP / 2, "only %d of %d placed", placed, NP);
  for (int g = 0; g < NG; ++g) {  /* pods 0, 1: the co-located replica of role a; 5..8: the two replicas of c */
    const int32_t* p = a1 + g * PODS;
    CHECK((p[0] < 0) == (p[1] < 0), "group %d: replica of a split", g);
    if (p[0] >= 0) CHECK(domain_of[p[0]] == domain_of[p[1]], "group %d: replica of a in two domains", g);
    CHECK((p[5] < 0) == (p[6] < 0) && (p[7] < 0) == (p[8] < 0), "group %d: replica of c split", g);
  }
  int excl_seen = 0;
  for (int g = 0; g < NG; ++g) {
    if (d1[g] < 0) continue;
    CHECK(g % 2 == 0, "group %d is not exclusive but reports domain %d", g, d1[g]);
    ++excl_seen;
    for (int h = g % 6; h < g; h += 6) CHECK(d1[h] != d1[g], "groups %d and %d share domain %d", h, g, d1[g]);
  }
  CHECK(excl_seen > 0, "no exclusive domain reported");

  /* malformed input: a code and its message from the same thread, the ctx stays usable */
  rp[0] = 33; /* S above RBGTOPO_MAX_STEP_REPLICAS */
  rc = go_place_groups_lw_committed(ctx, blob, words, rp, 6 * NG, a2, s2, d2, &r2, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strstr(err, "pods per replica") && r2 == 0, "bad S: %d '%s'", rc, err);
  rp[0] = 2;

  pthread_t th[10];
  job_t jobs[10];
  for (int t = 0; t < 10; ++t) {
    jobs[t] = (job_t){ctx, blob, words, rp, a1, s1, d1, r1, sc1, asc1, alt1, 0};
    pthread_create(&th[t], NULL, worker, &jobs[t]);
  }
  int bad = 0;
  for (int t = 0; t < 10; ++t) { pthread_join(th[t], NULL); bad += jobs[t].bad; }
  CHECK(bad == 0, "%d concurrent calls differ from the sequential result", bad);
  rbgtopo_destroy(ctx);
  free(blob);
  printf("CABI_LW_COMMITTED_LEVELS_OK gpu rounds %d\n", r1);
  return 0;
}

int main(int argc, char** argv) {
  if (argc > 1 && strcmp(argv[1], "gpu") == 0) return run_gpu();
  return run_host();
}
