/* The C ABI of libpna_sm90.so used from plain C (what a cgo / JNI / N-API binding would wrap): build the CSR of a tiny
 * graph, run the PNA aggregation (mean max min std x identity amplification attenuation), print two rows.
 *
 *   gcc -std=c99 -I include -I /usr/local/cuda/include examples/c_caller.c -o /tmp/c_caller \
 *       -L pna_b200 -l:libpna_sm90.so -L /usr/local/cuda/lib64 -lcudart -Wl,-rpath,$PWD/pna_b200 && /tmp/c_caller
 *
 * Reference being replaced: PNAConvSimple.aggregate, models/pytorch_geometric/pna.py:242-249. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <cuda_runtime_api.h>
#include "pna_b200.h"

#define CU(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)
#define PNA(x) do { if ((x) != 0) { fprintf(stderr, "%s: %s\n", #x, pna_last_error()); return 1; } } while (0)

static void* dmalloc(size_t bytes) { void* p = NULL; return cudaMalloc(&p, bytes ? bytes : 4) == cudaSuccess ? p : NULL; }

int main(int argc, char** argv) {
  enum { N = 5, E = 6, F = 4 };
  /* edges j -> i (PyG: row 0 = source j, row 1 = target i); node 4 has no in-edge */
  const int64_t src[E] = {1, 2, 3, 0, 2, 4}, dst[E] = {0, 0, 0, 1, 1, 3};
  float x[N * F];
  for (int i = 0; i < N * F; ++i) x[i] = (float)(i % 7) - 3.0f;
  if (pna_query(PNA_QUERY_ABI_VERSION) != PNA_ABI_VERSION) { fprintf(stderr, "ABI mismatch\n"); return 1; }

  const int split = pna_query(PNA_QUERY_DEFAULT_SPLIT), chunk = pna_query(PNA_QUERY_DEFAULT_CHUNK);
  pna_csr_t csr = {0};
  csr.n_nodes = N; csr.n_edges = E; csr.split_threshold = split; csr.chunk_edges = chunk;
  csr.cap_hubs = E / split + 1; csr.cap_chunks = E / chunk + csr.cap_hubs + 1; csr.n_part = 1;
  csr.rowptr = dmalloc((N + 1) * 4); csr.col = dmalloc(E * 4); csr.perm = dmalloc(E * 4);
  csr.hub_info = dmalloc(4 * csr.cap_hubs * 4); csr.chunk_items = dmalloc(2 * csr.cap_chunks * 4);
  csr.light_rowptr = dmalloc((N + csr.cap_chunks + 1) * 4); csr.light_deg = dmalloc((N + csr.cap_chunks) * 4);
  csr.light_col = dmalloc(E * 4); csr.part = dmalloc((csr.n_part + 1) * 4);
  int64_t *d_src = dmalloc(sizeof src), *d_dst = dmalloc(sizeof dst);
  float *d_x = dmalloc(sizeof x), *d_out = dmalloc(N * 12 * F * 4);
  CU(cudaMemcpy(d_src, src, sizeof src, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(d_dst, dst, sizeof dst, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(d_x, x, sizeof x, cudaMemcpyHostToDevice));
  size_t ws_bytes = 0;
  PNA(pna_csr_workspace_bytes(N, E, &ws_bytes));
  void* ws = dmalloc(ws_bytes);
  PNA(pna_csr_build(d_src, d_dst, &csr, ws, ws_bytes, NULL));          /* NULL = the default stream */

  /* avg_deg['log'] of the layer ctor (pna.py:212-219): mean of log(in_degree + 1) over the training graphs */
  const int indeg[N] = {3, 2, 0, 1, 0};
  float avg_log = 0.f;
  for (int i = 0; i < N; ++i) avg_log += logf((float)indeg[i] + 1.0f) / N;

  pna_agg_t d = {0};
  d.gathered = d_x; d.ld_gathered = F; d.rowptr = csr.rowptr; d.col = csr.col; d.out = d_out; d.ld_out = 12 * F;
  d.n_rows = N; d.n_feat = F; d.n_towers = 1; d.dtype = PNA_F32;
  d.n_aggr = 4; d.aggr_codes = PNA_AGGR_MEAN | PNA_AGGR_MAX << 4 | PNA_AGGR_MIN << 8 | PNA_AGGR_STD << 12;
  d.n_scalers = 3; d.scaler_codes = PNA_SCALE_IDENTITY | PNA_SCALE_AMPLIFICATION << 4 | PNA_SCALE_ATTENUATION << 8;
  d.avg_log = avg_log; d.avg_lin = 1.0f; d.split_threshold = split; d.chunk_edges = chunk;
  d.hub_info = csr.hub_info; d.chunk_items = csr.chunk_items; d.n_hubs = csr.n_hubs; d.n_chunks = csr.n_chunks;
  d.light_rowptr = csr.light_rowptr; d.light_deg = csr.light_deg; d.light_col = csr.light_col; d.part = csr.part;
  d.n_part = csr.n_part; d.n_view_rows = N + csr.n_chunks;
  PNA(pna_aggregate_fwd(&d, NULL));
  float out[N * 12 * F];
  CU(cudaMemcpy(out, d_out, sizeof out, cudaMemcpyDeviceToHost));
  if (argc > 1 && strcmp(argv[1], "--dump") == 0) {   /* every value, one row per line (tests/test_gpu_parity.py diffs it) */
    for (int r = 0; r < N; ++r) {
      for (int c = 0; c < 12 * F; ++c) printf("%s%.9g", c ? " " : "", out[r * 12 * F + c]);
      printf("\n");
    }
    return 0;
  }
  for (int r = 0; r < N; r += 4) {            /* row 0: three in-edges; row 4: none -> [0, 0, 0, sqrt(1e-5)] blocks */
    printf("row %d (in-degree %d):", r, indeg[r]);
    for (int c = 0; c < 4 * F; ++c) printf(" %.4f", out[r * 12 * F + c]);
    printf("  | amplified mean[0] %.4f, attenuated mean[0] %.4f\n", out[r * 12 * F + 4 * F], out[r * 12 * F + 8 * F]);
  }
  return 0;
}
