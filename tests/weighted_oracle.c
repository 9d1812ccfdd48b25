/*
 * Plain-C restatement of the softmax / softmin / normalised_mean aggregators -- TEST INFRASTRUCTURE (tests/weighted_oracle.py
 * builds and loads it; never used by pna_b200/).  Scalar fp32 loops compiled with -ffp-contract=off, so no FMA is formed:
 * it states the roundings the CUDA kernel (pna_b200/csrc/pna_aggregate_weighted.cuh) reproduces.
 *
 * Per destination i and feature f, over the edges e with dst[e] == i in edge order, messages m = msg[e * F + f]:
 *   code 9 / 10 (softmax / softmin), sigma = +1 / -1, n = sigma * m:
 *     M = max n;  e = expf(n - M);  Z = sum e;  S = sum (e * n);  y = sigma * (S / Z)
 *   code 11 (normalised_mean):  D_k = |{e : dst[e] == k}|,  r_k = D_k ? 1 / sqrt(D_k) (correctly rounded) : 0,
 *     w = r_i * r_j with j = wsrc[e] (0 for j outside [0, n_nodes)),  y = sum (m * w)
 *   rows without edges: y = 0.  out[i * F + f] = y (unscaled).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

static float rsqrt_rn(int64_t D) { return D > 0 ? (float)(1.0 / sqrt((double)D)) : 0.0f; }

int pna_oracle_weighted(const float* msg, int64_t n_nodes, int64_t n_feat, const int64_t* dst, const int64_t* wsrc,
                        int64_t n_edges, int32_t code, float* out) {
  const int64_t N = n_nodes, F = n_feat;
  if (code < 9 || code > 11) return -3;
  float* M = (float*)malloc((size_t)(N * F) * sizeof(float));
  float* Z = (float*)calloc((size_t)(N * F), sizeof(float));
  float* S = (float*)calloc((size_t)(N * F), sizeof(float));
  int64_t* deg = (int64_t*)calloc((size_t)N, sizeof(int64_t));
  if (!M || !Z || !S || !deg) return -1;
  for (int64_t k = 0; k < N * F; ++k) M[k] = -INFINITY;
  for (int64_t e = 0; e < n_edges; ++e) {
    if (dst[e] < 0 || dst[e] >= N) return -2;
    deg[dst[e]]++;
  }
  const float sigma = code == 10 ? -1.0f : 1.0f;
  if (code == 11) {
    for (int64_t e = 0; e < n_edges; ++e) {
      const int64_t i = dst[e], j = wsrc[e];
      const float w = rsqrt_rn(deg[i]) * ((j >= 0 && j < N) ? rsqrt_rn(deg[j]) : 0.0f);
      for (int64_t f = 0; f < F; ++f) S[i * F + f] = S[i * F + f] + msg[e * F + f] * w;
    }
  } else {
    for (int64_t e = 0; e < n_edges; ++e)
      for (int64_t f = 0; f < F; ++f) M[dst[e] * F + f] = fmaxf(M[dst[e] * F + f], sigma * msg[e * F + f]);
    for (int64_t e = 0; e < n_edges; ++e) {
      const int64_t i = dst[e];
      for (int64_t f = 0; f < F; ++f) {
        const float n = sigma * msg[e * F + f];
        const float ex = expf(n - M[i * F + f]);
        Z[i * F + f] = Z[i * F + f] + ex;
        S[i * F + f] = S[i * F + f] + ex * n;
      }
    }
  }
  for (int64_t i = 0; i < N; ++i)
    for (int64_t f = 0; f < F; ++f) {
      float y = 0.0f;
      if (deg[i] > 0) y = code == 11 ? S[i * F + f] : sigma * (S[i * F + f] / Z[i * F + f]);
      out[i * F + f] = y;
    }
  free(M); free(Z); free(S); free(deg);
  return 0;
}
