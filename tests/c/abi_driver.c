/* Plain-C driver of the drop-in boundary (SURVEY 8b "what calls it"): proves include/sdbgpu.h is C (not C++),
 * that a C caller links against libsdbgpu.so, and -- when an H100 is present -- runs one brute-force KNN, one graph
 * hop and one staged HNSW load through the ABI exactly as the Rust shim of INTEGRATION.md would.
 * Exit code 0 = ok; prints "NO_GPU <message>" and exits 0 when the library refuses to start without a device
 * (that refusal is the behaviour under test on CPU-only machines). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "sdbgpu.h"

#define CHECK(call)                                                        \
  do {                                                                     \
    sdb_status s_ = (call);                                                \
    if (s_ != SDB_OK) {                                                    \
      fprintf(stderr, "%s -> %d: %s\n", #call, (int)s_, sdb_last_error()); \
      return 1;                                                            \
    }                                                                      \
  } while (0)

int main(void) {
  sdb_ctx* ctx = NULL;
  sdb_status s = sdb_ctx_create(0, &ctx);
  if (s == SDB_ECUDA) {
    printf("NO_GPU %s\n", sdb_last_error());
    return 0;
  }
  if (s != SDB_OK) return 1;
  printf("%s\n", sdb_version());

  /* brute force: 4 rows in 2-D, euclidean, k = 2 around (0.9, 0) */
  {
    const float rows[8] = {0, 0, 1, 0, 0, 1, 1, 1};
    const double q[2] = {0.9, 0.0};
    uint64_t out_rows[2];
    double out_dist[2];
    uint32_t cnt = 0;
    sdb_corpus* c = NULL;
    CHECK(sdb_corpus_create(ctx, 2, SDB_F32, SDB_EUCLIDEAN, 4, &c));
    CHECK(sdb_corpus_append(c, rows, 4));
    CHECK(sdb_corpus_finalize(c));
    CHECK(sdb_knn_bruteforce(c, q, 1, 2, out_rows, out_dist, &cnt, NULL));
    if (cnt != 2 || out_rows[0] != 1 || out_rows[1] != 0) {
      fprintf(stderr, "knn: unexpected result %u [%llu %llu]\n", cnt, (unsigned long long)out_rows[0],
              (unsigned long long)out_rows[1]);
      return 1;
    }
    sdb_corpus_destroy(c);
  }
  /* graph: 0->{1,2}, 1->{2}, 2->{} ; two hops from {0} = [2] */
  {
    const uint64_t rp[4] = {0, 2, 3, 3};
    const uint32_t ci[3] = {1, 2, 2};
    const uint32_t frontier[1] = {0};
    sdb_graph* g = NULL;
    sdb_graph* hops[2];
    uint32_t* out = NULL;
    uint64_t n = 0;
    CHECK(sdb_graph_load_csr(ctx, 3, rp, ci, &g));
    hops[0] = hops[1] = g;
    CHECK(sdb_graph_expand(hops, 2, frontier, 1, 0, &out, &n));
    if (n != 1 || out[0] != 2) {
      fprintf(stderr, "graph: unexpected result\n");
      return 1;
    }
    sdb_free(out);
    sdb_graph_destroy(g);
  }
  /* staged HNSW: 3 elements on a line, one layer, raw He / Hn values */
  {
    uint8_t he[3][11], hn[3][18];
    uint64_t he_off[4], hn_off[4], ids[3] = {0, 1, 2};
    const float x[3][2] = {{0, 0}, {1, 0}, {2, 0}};
    const uint64_t nb[3][2] = {{1, 2}, {0, 2}, {1, 0}};
    const uint8_t* node_blob[1];
    const uint64_t* node_off[1];
    const uint64_t* node_ids[1];
    uint64_t n_nodes[1] = {3}, bad = 99, elems[2];
    const float q[2] = {1.9f, 0.f};
    double dist[2];
    uint32_t cnt = 0;
    sdb_hnsw* h = NULL;
    int i, j, b;
    for (i = 0; i < 3; i++) {
      he[i][0] = 1; he[i][1] = 1; he[i][2] = 2; /* revision 1, variant F32, len 2 */
      memcpy(&he[i][3], x[i], 8);
      he_off[i] = (uint64_t)i * 11;
      hn[i][0] = 0; hn[i][1] = 2; /* BE u16 count */
      for (j = 0; j < 2; j++)
        for (b = 0; b < 8; b++) hn[i][2 + 8 * j + b] = (uint8_t)(nb[i][j] >> (8 * (7 - b)));
      hn_off[i] = (uint64_t)i * 18;
    }
    he_off[3] = 33;
    hn_off[3] = 54;
    node_blob[0] = &hn[0][0];
    node_off[0] = hn_off;
    node_ids[0] = ids;
    CHECK(sdb_hnsw_load_staged(ctx, 2, SDB_EUCLIDEAN, 3, &he[0][0], he_off, ids, 3, 1, node_blob, node_off, node_ids,
                               n_nodes, 0, &h, &bad));
    CHECK(sdb_hnsw_search(h, q, 1, 2, 8, elems, dist, &cnt, NULL));
    if (bad != 0 || cnt != 2 || elems[0] != 2 || elems[1] != 1) {
      fprintf(stderr, "hnsw: unexpected result bad=%llu cnt=%u\n", (unsigned long long)bad, cnt);
      return 1;
    }
    sdb_hnsw_destroy(h);
  }
  sdb_ctx_destroy(ctx);
  printf("ABI_DRIVER_OK\n");
  return 0;
}
