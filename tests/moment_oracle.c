/*
 * Plain-C restatement of the moment aggregators -- TEST INFRASTRUCTURE (tests/moment_oracle.py builds and loads it; never
 * used by pna_b200/).  Scalar fp32 loops compiled with -ffp-contract=off, so no FMA is formed: it states the roundings the
 * CUDA kernel reproduces.
 *
 * Central moments (dense reference models/pytorch/pna/aggregators.py:122-146) in the order the CUDA kernel uses
 * (pna_b200/csrc/pna_aggregate_moments.cuh): per destination i and feature f, over the in-edges in edge order,
 *   mu = (sum of m) / d;  delta = m - mu;  delta^k = ((delta * delta) * delta) ...;  M = (sum of delta^k) / d;
 *   r = sign(M) * powf(|M| + 1e-5, 1/k) with 1/k rounded to float;  d == 0: r = 0.
 * out[i * F + f] = r (unscaled).  m = x[src[e] * F + f].
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

int pna_oracle_moment(const float* x, int64_t n_nodes, int64_t n_feat, const int64_t* src, const int64_t* dst,
                      int64_t n_edges, int32_t k, float* out) {
  const int64_t N = n_nodes, F = n_feat;
  if (k < 3 || k > 5) return -3;
  float* sum = (float*)calloc((size_t)(N * F), sizeof(float));
  float* cs = (float*)calloc((size_t)(N * F), sizeof(float));
  int64_t* deg = (int64_t*)calloc((size_t)N, sizeof(int64_t));
  if (!sum || !cs || !deg) return -1;
  for (int64_t e = 0; e < n_edges; ++e) {
    const int64_t i = dst[e];
    if (i < 0 || i >= N) return -2;
    deg[i]++;
    for (int64_t f = 0; f < F; ++f) sum[i * F + f] = sum[i * F + f] + x[src[e] * F + f];
  }
  for (int64_t e = 0; e < n_edges; ++e) {
    const int64_t i = dst[e];
    const float d = (float)deg[i];
    for (int64_t f = 0; f < F; ++f) {
      const float delta = x[src[e] * F + f] - sum[i * F + f] / d;
      float p = delta * delta;
      for (int j = 2; j < k; ++j) p = p * delta;
      cs[i * F + f] = cs[i * F + f] + p;
    }
  }
  const float inv = k == 3 ? 1.0f / 3.0f : (k == 4 ? 0.25f : 0.2f);
  for (int64_t i = 0; i < N; ++i)
    for (int64_t f = 0; f < F; ++f) {
      float r = 0.0f;
      if (deg[i] > 0) {
        const float M = cs[i * F + f] / (float)deg[i];
        if (M != 0.0f) {
          r = powf(fabsf(M) + 1e-5f, inv);
          if (M < 0.0f) r = -r;
        } else {
          r = M;
        }
      }
      out[i * F + f] = r;
    }
  free(sum); free(cs); free(deg);
  return 0;
}
