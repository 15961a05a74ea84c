/*
 * cabi_lw_committed_ranked.c — calls rbgtopo_place_groups_lw_committed_ranked exactly the way the cgo shim does
 * (go/pkg/scheduler/b200topo/cgo_bridge.go, rbgtopo_go_place_groups_lw_committed_ranked /
 * placeGroupsLWCommittedRanked): plain C, int32 / float arrays and sizes, the call and the error fetch in one helper on
 * one OS thread, and ten OS threads on one ctx.  TEST INFRASTRUCTURE (the companion of tests/cabi_lw_committed.c).
 *
 *   cabi_lw_committed_ranked host   no device needed: bad arguments come back as codes with their text
 *   cabi_lw_committed_ranked gpu    the fleet of cabi_lw_committed.c (2-pod replicas, one role co-located at level 0)
 *                                   as one ranked committed batch (4 alternates), repeated sequentially and then
 *                                   10 x 3 times concurrently: every output identical every time; assign, status,
 *                                   domain and rounds equal to rbgtopo_place_groups_lw_committed's; moving a pod to any
 *                                   of its alternates over-commits no node over the batch and keeps a co-located
 *                                   replica in its domain; n_alt = 9 and a bad role_pods table return a code and its
 *                                   text, and the ctx stays usable
 * Prints "CABI_LW_COMMITTED_RANKED_OK <mode>" and exits 0 on success.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/rbgtopo.h"

#define CHECK(cond, ...) do { if (!(cond)) { fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); \
  fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); exit(1); } } while (0)

#define NALT 4
/* the cgo preamble helper: call + error text on the same OS thread */
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
  int32_t rc = go_place_groups_lw_committed_ranked(NULL, NULL, 0, NULL, 0, 0, NULL, NULL, NULL, &rounds, NULL, NULL,
                                                   NULL, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strlen(err) > 0 && rounds == 0, "null ctx: %d '%s' rounds %d", rc, err, rounds);
  printf("CABI_LW_COMMITTED_RANKED_OK host\n");
  return 0;
}

#define NN 4096
#define NG 48
#define PODS 9      /* per group: role a 1 x 2 pods (co-located at level 0), b 3 x 1, c 2 x 2 */
#define NP (NG * PODS)
typedef struct {
  rbgtopo_ctx* ctx;
  const int32_t* blob;
  int64_t words;
  const int32_t* rp;
  const int32_t *want_assign, *want_status, *want_domain, *want_alt;
  const float *want_score, *want_alt_score;
  int32_t want_rounds;
  int bad;
} job_t;

static void* worker(void* arg) {
  job_t* j = (job_t*)arg;
  int32_t assign[NP], status[NG], domain[NG], rounds = 0, alt[NP * NALT];
  float score[NP], alt_score[NP * NALT];
  char err[256];
  for (int it = 0; it < 3; ++it) {
    int32_t rc = go_place_groups_lw_committed_ranked(j->ctx, j->blob, j->words, j->rp, 6 * NG, NALT, assign, status,
                                                     domain, &rounds, score, alt, alt_score, err, sizeof err);
    if (rc != RBGTOPO_OK || memcmp(assign, j->want_assign, sizeof assign) != 0 ||
        memcmp(status, j->want_status, sizeof status) != 0 || memcmp(domain, j->want_domain, sizeof domain) != 0 ||
        memcmp(score, j->want_score, sizeof score) != 0 || memcmp(alt, j->want_alt, sizeof alt) != 0 ||
        memcmp(alt_score, j->want_alt_score, sizeof alt_score) != 0 || rounds != j->want_rounds)
      j->bad++;
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
   * every 4th group gang, every 3rd exclusive; one scheduled pod each, near the head of the background order */
  const int q = 3, per = 4 * q + q * q + 3;
  const int words = RBGTOPO_HDR_WORDS + NG * RBGTOPO_GROUP_WORDS + NG * per;
  int32_t* blob = (int32_t*)calloc((size_t)words, sizeof(int32_t));
  blob[0] = RBGTOPO_GROUPS_MAGIC; blob[1] = RBGTOPO_ABI_VERSION; blob[2] = NG; blob[3] = words; blob[4] = NG * 6;
  int off = RBGTOPO_HDR_WORDS + NG * RBGTOPO_GROUP_WORDS;
  for (int g = 0; g < NG; ++g) {
    int32_t* rec = blob + RBGTOPO_HDR_WORDS + g * RBGTOPO_GROUP_WORDS;
    rec[0] = g;
    rec[1] = ((g % 4 == 0) ? RBGTOPO_STEP_GANG : 0) | ((g % 3 == 0) ? RBGTOPO_STEP_EXCLUSIVE : 0);
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

  static int32_t a1[NP], a2[NP], a0[NP], n1[NP * NALT], n2[NP * NALT];
  static float c1[NP], c2[NP], x1[NP * NALT], x2[NP * NALT];
  int32_t s1[NG], s2[NG], d1[NG], d2[NG], s0[NG], d0[NG], r1 = 0, r2 = 0, r0 = 0;
  rc = go_place_groups_lw_committed_ranked(ctx, blob, words, rp, 6 * NG, NALT, a1, s1, d1, &r1, c1, n1, x1, err,
                                           sizeof err);
  CHECK(rc == RBGTOPO_OK && r1 >= 1 && r1 <= NG, "committed ranked: %d rounds %d %s", rc, r1, err);
  rc = go_place_groups_lw_committed_ranked(ctx, blob, words, rp, 6 * NG, NALT, a2, s2, d2, &r2, c2, n2, x2, err,
                                           sizeof err);
  CHECK(rc == RBGTOPO_OK, "committed ranked again: %d %s", rc, err);
  CHECK(memcmp(a1, a2, sizeof a1) == 0 && memcmp(s1, s2, sizeof s1) == 0 && memcmp(d1, d2, sizeof d1) == 0 && r1 == r2 &&
        memcmp(c1, c2, sizeof c1) == 0 && memcmp(n1, n2, sizeof n1) == 0 && memcmp(x1, x2, sizeof x1) == 0,
        "the sequential repeat differs (rounds %d vs %d)", r1, r2);
  rc = rbgtopo_place_groups_lw_committed(ctx, blob, words, rp, 6 * NG, a0, s0, d0, &r0);
  CHECK(rc == RBGTOPO_OK && memcmp(a0, a1, sizeof a1) == 0 && memcmp(s0, s1, sizeof s1) == 0 &&
        memcmp(d0, d1, sizeof d1) == 0 && r0 == r1, "differs from rbgtopo_place_groups_lw_committed");
  /* within capacity over the whole batch */
  static int32_t used[NN];
  int placed = 0;
  for (int i = 0; i < NP; ++i) {
    CHECK(a1[i] >= -1 && a1[i] < NN, "assign[%d] = %d", i, a1[i]);
    if (a1[i] >= 0) { ++placed; CHECK(++used[a1[i]] <= free_slots[a1[i]], "node %d over-committed", a1[i]); }
  }
  CHECK(placed > NP / 2, "only %d of %d placed", placed, NP);
  int alts = 0;  /* every pod demands 1: an alternate of a placed pod has a free slot after the batch */
  for (int i = 0; i < NP; ++i)
    for (int k = 0; k < NALT; ++k) {
      const int32_t x = n1[i * NALT + k];
      CHECK(x >= -1 && x < NN && (x < 0 || (a1[i] >= 0 && x != a1[i] && used[x] < free_slots[x])),
            "pod %d alternate %d = %d", i, k, x);
      if (x >= 0 && i % PODS < 2) CHECK(domain_of[x] == domain_of[a1[i]], "pod %d alternate %d leaves its domain", i, x);
      alts += x >= 0;
    }
  CHECK(alts > NP, "only %d alternates", alts);

  /* malformed input: a code and its message from the same thread, the ctx stays usable */
  rc = go_place_groups_lw_committed_ranked(ctx, blob, words, rp, 6 * NG, 9, a2, s2, d2, &r2, c2, n2, x2, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strstr(err, "n_alt") && r2 == 0, "n_alt 9: %d '%s'", rc, err);
  rp[0] = 33; /* S above RBGTOPO_MAX_STEP_REPLICAS */
  rc = go_place_groups_lw_committed_ranked(ctx, blob, words, rp, 6 * NG, NALT, a2, s2, d2, &r2, c2, n2, x2, err,
                                           sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strstr(err, "pods per replica") && r2 == 0, "bad S: %d '%s'", rc, err);
  rp[0] = 2;

  pthread_t th[10];
  job_t jobs[10];
  for (int t = 0; t < 10; ++t) {
    jobs[t] = (job_t){ctx, blob, words, rp, a1, s1, d1, n1, c1, x1, r1, 0};
    pthread_create(&th[t], NULL, worker, &jobs[t]);
  }
  int bad = 0;
  for (int t = 0; t < 10; ++t) { pthread_join(th[t], NULL); bad += jobs[t].bad; }
  CHECK(bad == 0, "%d concurrent calls differ from the sequential result", bad);
  rbgtopo_destroy(ctx);
  free(blob);
  printf("CABI_LW_COMMITTED_RANKED_OK gpu rounds %d alternates %d\n", r1, alts);
  return 0;
}

int main(int argc, char** argv) {
  if (argc > 1 && strcmp(argv[1], "gpu") == 0) return run_gpu();
  return run_host();
}
