/*
 * Plain-C restatement of the per-edge messages of pna_edge_msg_fwd / pna_edge_msg_bwd -- TEST INFRASTRUCTURE
 * (tests/test_edge_msg_emulated.py builds and loads it; never used by pna_b200/).  Scalar fp32 loops compiled with
 * -ffp-contract=off, so no FMA is formed: it states the roundings the CUDA kernels (pna_b200/csrc/pna_edge_mlp.cu)
 * reproduce.  All arrays row-major, TF = T * F, messages at pitch P >= F per tower.
 *
 * Forward, slot s of row i (rowptr[i] <= s < rowptr[i+1]), j = col[s], tower t, o < F:
 *   u = ((a[i][tF+o] + b[j][tF+o]) + b1[tF+o]) + C[s][tF+o]   (C == NULL: no last add)
 *   L == 1: M[s][tP+o] = u
 *   L >= 2: z_1 = u > 0 ? u : 0;  k = 2..L: acc = 0; for c in order: acc += W[k-2][t][o][c] * z_(k-1)[c];
 *           u = acc + bias[k-2][t][o];  z_k = u > 0 ? u : 0 (k < L), M[s][tP+o] = u (k == L);  act[k-2][s][tF+o] = z_(k-1)[o]
 *   M[s][tP+o] = 0 for F <= o < P
 * Backward (L >= 2): g = dM[s][tP..tP+F); k = L..2: q[c] = 0; for o in order: q[c] += W[k-2][t][o][c] * g[o];
 *           g[c] = act[k-2][s][tF+c] > 0 ? q[c] : 0;  grad_pre[k-2][s][tF+c] = g[c]
 */
#include <stdint.h>
#include <stdlib.h>

void edge_msg_fwd_ref(const int32_t* rowptr, const int32_t* col, int64_t n_rows, int64_t E, const float* a, const float* b,
                      const float* b1, const float* C, const float* W, const float* bias, int L, int T, int F, int P, float* M,
                      float* act) {
  const int TF = T * F;
  float* z = malloc(sizeof(float) * F);
  float* u = malloc(sizeof(float) * F);
  for (int64_t i = 0; i < n_rows; ++i)
    for (int64_t s = rowptr[i]; s < rowptr[i + 1]; ++s) {
      const int64_t j = col[s];
      for (int t = 0; t < T; ++t) {
        for (int o = 0; o < F; ++o) {
          float v = a[i * TF + t * F + o] + b[j * TF + t * F + o];
          v = v + b1[t * F + o];
          if (C) v = v + C[s * TF + t * F + o];
          z[o] = (L == 1 || v > 0.f) ? v : 0.f;
        }
        for (int k = 2; k <= L; ++k) {
          if (act)
            for (int o = 0; o < F; ++o) act[((int64_t)(k - 2) * E + s) * TF + t * F + o] = z[o];
          const float* Wk = W + ((int64_t)(k - 2) * T + t) * F * F;
          const float* bk = bias + ((int64_t)(k - 2) * T + t) * F;
          for (int o = 0; o < F; ++o) {
            float acc = 0.f;
            for (int c = 0; c < F; ++c) {
              const float p = Wk[o * F + c] * z[c];
              acc = acc + p;
            }
            u[o] = acc + bk[o];
          }
          for (int o = 0; o < F; ++o) z[o] = (k == L || u[o] > 0.f) ? u[o] : 0.f;
        }
        for (int o = 0; o < P; ++o) M[s * T * P + t * P + o] = o < F ? z[o] : 0.f;
      }
    }
  free(z);
  free(u);
}

void edge_msg_bwd_ref(const float* dM, int P, const float* act, const float* W, int64_t E, int L, int T, int F,
                      float* grad_pre) {
  const int TF = T * F;
  float* g = malloc(sizeof(float) * F);
  float* q = malloc(sizeof(float) * F);
  for (int64_t s = 0; s < E; ++s)
    for (int t = 0; t < T; ++t) {
      for (int o = 0; o < F; ++o) g[o] = dM[s * T * P + t * P + o];
      for (int k = L; k >= 2; --k) {
        const float* Wk = W + ((int64_t)(k - 2) * T + t) * F * F;
        for (int c = 0; c < F; ++c) q[c] = 0.f;
        for (int o = 0; o < F; ++o)
          for (int c = 0; c < F; ++c) {
            const float p = Wk[o * F + c] * g[o];
            q[c] = q[c] + p;
          }
        for (int c = 0; c < F; ++c) {
          const int64_t idx = ((int64_t)(k - 2) * E + s) * TF + t * F + c;
          g[c] = act[idx] > 0.f ? q[c] : 0.f;
          grad_pre[idx] = g[c];
        }
      }
    }
  free(g);
  free(q);
}
