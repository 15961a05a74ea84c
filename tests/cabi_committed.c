/*
 * cabi_committed.c — calls rbgtopo_place_groups_committed exactly the way the cgo shim does
 * (go/pkg/scheduler/b200topo/cgo_bridge.go, rbgtopo_go_place_groups_committed / placeGroupsCommitted):
 * plain C, int32 arrays and sizes, the call and the error fetch in one helper on one OS thread, and ten
 * OS threads on one ctx.  TEST INFRASTRUCTURE (the companion of tests/cabi_driver.c).
 *
 *   cabi_committed host   no device needed: bad arguments come back as codes with their text
 *   cabi_committed gpu    a synthetic 2-tier topology + a fleet of 3-role groups (gang, exclusive, plain), placed
 *                         as one committed batch, repeated sequentially and then 10 x 3 times concurrently: assign,
 *                         status, domain and rounds identical every time; no node over-committed over the batch;
 *                         a malformed blob returns a code and its text, and the ctx stays usable
 * Prints "CABI_COMMITTED_OK <mode>" and exits 0 on success.
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
static int32_t go_place_groups_committed(rbgtopo_ctx* ctx, const int32_t* groups, int64_t words, int32_t* assign,
                                         int32_t* status, int32_t* domain, int32_t* rounds, char* err, int errlen) {
  int32_t rc = rbgtopo_place_groups_committed(ctx, groups, words, assign, status, domain, rounds);
  if (rc != RBGTOPO_OK) rbgtopo_last_error(ctx, err, errlen); else err[0] = 0;
  return rc;
}

static int run_host(void) {
  char err[256];
  int32_t rounds = 7;
  int32_t rc = go_place_groups_committed(NULL, NULL, 0, NULL, NULL, NULL, &rounds, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strlen(err) > 0 && rounds == 0, "null ctx: %d '%s' rounds %d", rc, err, rounds);
  printf("CABI_COMMITTED_OK host\n");
  return 0;
}

#define NN 4096
#define NG 48
#define NP (NG * 6)
typedef struct {
  rbgtopo_ctx* ctx;
  const int32_t* blob;
  int64_t words;
  const int32_t *want_assign, *want_status, *want_domain;
  int32_t want_rounds;
  int bad;
} job_t;

static void* worker(void* arg) {
  job_t* j = (job_t*)arg;
  int32_t assign[NP], status[NG], domain[NG], rounds = 0;
  char err[256];
  for (int it = 0; it < 3; ++it) {
    int32_t rc = go_place_groups_committed(j->ctx, j->blob, j->words, assign, status, domain, &rounds, err, sizeof err);
    if (rc != RBGTOPO_OK || memcmp(assign, j->want_assign, sizeof assign) != 0 ||
        memcmp(status, j->want_status, sizeof status) != 0 || memcmp(domain, j->want_domain, sizeof domain) != 0 ||
        rounds != j->want_rounds)
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
  blob[0] = RBGTOPO_GROUPS_MAGIC; blob[1] = RBGTOPO_ABI_VERSION; blob[2] = NG; blob[3] = words; blob[4] = NP;
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
    rec[8] = g * 6; rec[9] = 6;
  }
  CHECK(off == words, "blob size");

  static int32_t a1[NP], a2[NP];
  int32_t s1[NG], s2[NG], d1[NG], d2[NG], r1 = 0, r2 = 0;
  rc = go_place_groups_committed(ctx, blob, words, a1, s1, d1, &r1, err, sizeof err);
  CHECK(rc == RBGTOPO_OK && r1 >= 1 && r1 <= NG, "committed: %d rounds %d %s", rc, r1, err);
  rc = go_place_groups_committed(ctx, blob, words, a2, s2, d2, &r2, err, sizeof err);
  CHECK(rc == RBGTOPO_OK, "committed again: %d %s", rc, err);
  CHECK(memcmp(a1, a2, sizeof a1) == 0 && memcmp(s1, s2, sizeof s1) == 0 && memcmp(d1, d2, sizeof d1) == 0 && r1 == r2,
        "the sequential repeat differs (rounds %d vs %d)", r1, r2);
  /* within capacity over the whole batch; exclusive domains not shared between gids (no group fixes one) */
  static int32_t used[NN];
  int placed = 0;
  for (int i = 0; i < NP; ++i) {
    CHECK(a1[i] >= -1 && a1[i] < NN, "assign[%d] = %d", i, a1[i]);
    if (a1[i] >= 0) { ++placed; CHECK(++used[a1[i]] <= free_slots[a1[i]], "node %d over-committed", a1[i]); }
  }
  CHECK(placed > NP / 2, "only %d of %d placed", placed, NP);
  int excl_seen = 0;
  for (int g = 0; g < NG; ++g) {
    if (d1[g] < 0) continue;
    CHECK(g % 3 == 0, "group %d is not exclusive but reports domain %d", g, d1[g]);
    ++excl_seen;
    for (int h = 0; h < g; ++h) CHECK(d1[h] != d1[g], "groups %d and %d share domain %d", h, g, d1[g]);
  }
  CHECK(excl_seen > 0, "no exclusive domain reported");

  /* malformed input: a code and its message from the same thread, the ctx stays usable */
  blob[RBGTOPO_HDR_WORDS + 1] = 64; /* unknown flag bit */
  rc = go_place_groups_committed(ctx, blob, words, a2, s2, d2, &r2, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strstr(err, "flags") && r2 == 0, "unknown flags: %d '%s'", rc, err);
  blob[RBGTOPO_HDR_WORDS + 1] = RBGTOPO_STEP_GANG | RBGTOPO_STEP_EXCLUSIVE;

  pthread_t th[10];
  job_t jobs[10];
  for (int t = 0; t < 10; ++t) {
    jobs[t] = (job_t){ctx, blob, words, a1, s1, d1, r1, 0};
    pthread_create(&th[t], NULL, worker, &jobs[t]);
  }
  int bad = 0;
  for (int t = 0; t < 10; ++t) { pthread_join(th[t], NULL); bad += jobs[t].bad; }
  CHECK(bad == 0, "%d concurrent calls differ from the sequential result", bad);
  rbgtopo_destroy(ctx);
  free(blob);
  printf("CABI_COMMITTED_OK gpu rounds %d\n", r1);
  return 0;
}

int main(int argc, char** argv) {
  if (argc > 1 && strcmp(argv[1], "gpu") == 0) return run_gpu();
  return run_host();
}
