/*
 * cabi_ranked.c — calls rbgtopo_place_groups_ranked exactly the way the cgo shim does
 * (go/pkg/scheduler/b200topo/cgo_bridge.go, rbgtopo_go_place_groups_ranked / placeGroupsRanked):
 * plain C, int32 / float arrays and sizes, the call and the error fetch in one helper on one OS thread, and ten
 * OS threads on one ctx.  TEST INFRASTRUCTURE (the companion of tests/cabi_driver.c).
 *
 *   cabi_ranked host   no device needed: bad arguments come back as codes with their text
 *   cabi_ranked gpu    a synthetic 2-tier topology + a fleet of 3-role groups (gang, exclusive, plain), placed
 *                      with NALT alternates, repeated sequentially and then 10 x 3 times concurrently: every output
 *                      identical every time and assign / status / domain equal to rbgtopo_place_groups; alternates
 *                      distinct, never the replica's own node; a malformed blob returns a code and its text, and the
 *                      ctx stays usable
 * Prints "CABI_RANKED_OK <mode>" and exits 0 on success.
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
static int32_t go_place_groups_ranked(rbgtopo_ctx* ctx, const int32_t* groups, int64_t words, int32_t n_alt,
                                      int32_t* assign, int32_t* status, int32_t* domain, float* score,
                                      int32_t* alt_node, float* alt_score, char* err, int errlen) {
  int32_t rc = rbgtopo_place_groups_ranked(ctx, groups, words, n_alt, assign, status, domain, score, alt_node, alt_score);
  if (rc != RBGTOPO_OK) rbgtopo_last_error(ctx, err, errlen); else err[0] = 0;
  return rc;
}

static int run_host(void) {
  char err[256];
  int32_t rc = go_place_groups_ranked(NULL, NULL, 0, 2, NULL, NULL, NULL, NULL, NULL, NULL, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strlen(err) > 0, "null ctx: %d '%s'", rc, err);
  printf("CABI_RANKED_OK host\n");
  return 0;
}

#define NN 4096
#define NG 48
#define NP (NG * 6)
#define NALT 4
typedef struct {
  rbgtopo_ctx* ctx;
  const int32_t* blob;
  int64_t words;
  const int32_t *want_assign, *want_status, *want_domain, *want_alt;
  const float* want_score;
  int bad;
} job_t;

static void* worker(void* arg) {
  job_t* j = (job_t*)arg;
  int32_t assign[NP], status[NG], domain[NG], alt[NP * NALT];
  float score[NP], alt_score[NP * NALT];
  char err[256];
  for (int it = 0; it < 3; ++it) {
    int32_t rc = go_place_groups_ranked(j->ctx, j->blob, j->words, NALT, assign, status, domain, score, alt, alt_score,
                                        err, sizeof err);
    if (rc != RBGTOPO_OK || memcmp(assign, j->want_assign, sizeof assign) != 0 ||
        memcmp(status, j->want_status, sizeof status) != 0 || memcmp(domain, j->want_domain, sizeof domain) != 0 ||
        memcmp(alt, j->want_alt, sizeof alt) != 0 || memcmp(score, j->want_score, sizeof score) != 0)
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

  static int32_t a1[NP], a2[NP], a0[NP], alt1[NP * NALT], alt2[NP * NALT];
  static float sc1[NP], sc2[NP], as1[NP * NALT], as2[NP * NALT];
  int32_t s1[NG], s2[NG], s0[NG], d1[NG], d2[NG], d0[NG];
  rc = go_place_groups_ranked(ctx, blob, words, NALT, a1, s1, d1, sc1, alt1, as1, err, sizeof err);
  CHECK(rc == RBGTOPO_OK, "ranked: %d %s", rc, err);
  rc = go_place_groups_ranked(ctx, blob, words, NALT, a2, s2, d2, sc2, alt2, as2, err, sizeof err);
  CHECK(rc == RBGTOPO_OK, "ranked again: %d %s", rc, err);
  CHECK(memcmp(a1, a2, sizeof a1) == 0 && memcmp(s1, s2, sizeof s1) == 0 && memcmp(d1, d2, sizeof d1) == 0 &&
        memcmp(sc1, sc2, sizeof sc1) == 0 && memcmp(alt1, alt2, sizeof alt1) == 0 && memcmp(as1, as2, sizeof as1) == 0,
        "the sequential repeat differs");
  rc = rbgtopo_place_groups(ctx, blob, words, a0, s0, d0);
  CHECK(rc == RBGTOPO_OK && memcmp(a0, a1, sizeof a0) == 0 && memcmp(s0, s1, sizeof s0) == 0 &&
        memcmp(d0, d1, sizeof d0) == 0, "assign / status / domain differ from rbgtopo_place_groups");
  int placed = 0, with_alt = 0;
  for (int i = 0; i < NP; ++i) {
    CHECK(a1[i] >= -1 && a1[i] < NN, "assign[%d] = %d", i, a1[i]);
    if (a1[i] < 0) {
      CHECK(alt1[i * NALT] == -1, "unplaced replica %d has alternates", i);
      continue;
    }
    ++placed;
    for (int k = 0; k < NALT; ++k) {
      const int32_t n = alt1[i * NALT + k];
      if (n < 0) continue;
      with_alt += k == 0;
      CHECK(n < NN && n != a1[i], "replica %d: alternate %d = %d (own node %d)", i, k, n, a1[i]);
      CHECK(as1[i * NALT + k] <= (k ? as1[i * NALT + k - 1] : as1[i * NALT]), "replica %d: scores not descending", i);
      for (int m = 0; m < k; ++m) CHECK(alt1[i * NALT + m] != n, "replica %d: alternate %d repeated", i, n);
    }
  }
  CHECK(placed > NP / 2 && with_alt > placed / 2, "placed %d of %d, %d with alternates", placed, NP, with_alt);

  /* malformed input and an out-of-range n_alt: a code and its message from the same thread, the ctx stays usable */
  rc = go_place_groups_ranked(ctx, blob, words, RBGTOPO_MAX_ALTERNATES + 1, a2, s2, d2, sc2, alt2, as2, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strstr(err, "n_alt"), "n_alt out of range: %d '%s'", rc, err);
  blob[RBGTOPO_HDR_WORDS + 1] = 64; /* unknown flag bit */
  rc = go_place_groups_ranked(ctx, blob, words, NALT, a2, s2, d2, sc2, alt2, as2, err, sizeof err);
  CHECK(rc == RBGTOPO_EINVAL && strstr(err, "flags"), "unknown flags: %d '%s'", rc, err);
  blob[RBGTOPO_HDR_WORDS + 1] = RBGTOPO_STEP_GANG | RBGTOPO_STEP_EXCLUSIVE;

  pthread_t th[10];
  job_t jobs[10];
  for (int t = 0; t < 10; ++t) {
    jobs[t] = (job_t){ctx, blob, words, a1, s1, d1, alt1, sc1, 0};
    pthread_create(&th[t], NULL, worker, &jobs[t]);
  }
  int bad = 0;
  for (int t = 0; t < 10; ++t) { pthread_join(th[t], NULL); bad += jobs[t].bad; }
  CHECK(bad == 0, "%d concurrent calls differ from the sequential result", bad);
  rbgtopo_destroy(ctx);
  free(blob);
  printf("CABI_RANKED_OK gpu placed %d\n", placed);
  return 0;
}

int main(int argc, char** argv) {
  if (argc > 1 && strcmp(argv[1], "gpu") == 0) return run_gpu();
  return run_host();
}
