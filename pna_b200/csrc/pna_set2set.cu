// Set2Set graph readout (reference models/layers.py:53-98, the readout of S2SReadout :271-289) on sm_90a, fp32.
//
// Every graph's recurrence is independent of every other graph's (only the LSTM weights are shared), so one CTA per graph
// runs all T steps in one launch with the graph's node rows in shared memory; the backward walks the steps back in one
// launch the same way (back-propagation through time).  The LSTM weights (12 D^2 floats: 12 KB at D = 16, 209 KB at D = 66)
// are copied into shared memory once per CTA when they fit next to the node rows (smem_limit below); otherwise every step
// reads them through the read-only path, from L1 / L2.  Where they live changes no sum.  Every sum has a
// fixed order that depends on the shape alone and there are no atomics, so both kernels are fixed functions of their
// inputs.  DESIGN section 9 states the scheme, the limits and the accuracy.
#include "common.cuh"

#include <math.h>

namespace pna {
namespace {

constexpr int S2S_THREADS = 256;
constexpr int S2S_WARPS = S2S_THREADS / 32;
constexpr int S2S_MAX_FEAT = 128;
constexpr int S2S_MAX_ELEMS = 16384;     // n_nodes * n_feat: the node rows (and in the backward their gradient) in smem

// Row pitch of the staged node rows: odd, so that threads walking different rows of one column hit different banks.
__host__ __device__ inline int s2s_ldx(int d) { return d | 1; }

__device__ __forceinline__ float sigmoid_f(float v) { return 1.0f / (1.0f + expf(-v)); }

// Sum (or max) over the CTA: butterfly within each warp, then the warp totals in ascending warp order.  Every thread
// gets the result.  `red` holds S2S_WARPS + 1 floats.
template <bool MAX>
__device__ __forceinline__ float block_reduce(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = MAX ? fmaxf(v, w) : v + w;
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = red[0];
    for (int w = 1; w < S2S_WARPS; ++w) a = MAX ? fmaxf(a, red[w]) : a + red[w];
    red[S2S_WARPS] = a;
  }
  __syncthreads();
  return red[S2S_WARPS];
}

// Columns of the node rows in shared memory (pitch ld).
struct RowsAt {
  const float* m;
  int ld;
  __device__ float operator()(int r, int c) const { return m[r * ld + c]; }
};

// [W_ih | W_hh] as one [4D, 3D] matrix: column c < 2D of W_ih, column 2D + k of W_hh.  In global memory (read through the
// read-only path) or staged in shared memory; the arithmetic is the same either way.
struct GateWeights {
  const float* w_ih;
  const float* w_hh;
  int d;
  bool staged;
  __device__ float operator()(int r, int c) const {
    const float* p = c < 2 * d ? w_ih + (size_t)r * 2 * d + c : w_hh + (size_t)r * d + (c - 2 * d);
    return staged ? *p : __ldg(p);
  }
};

// Copies the weights into smem (12 D^2 floats) when `stage`; returns the view the kernel reads them through.
__device__ __forceinline__ GateWeights stage_weights(const float* __restrict__ w_ih, const float* __restrict__ w_hh, int d,
                                                     bool stage, float* smem) {
  if (!stage) return GateWeights{w_ih, w_hh, d, false};
  const int n_ih = 8 * d * d, n_hh = 4 * d * d;
  for (int k = threadIdx.x; k < n_ih; k += S2S_THREADS) smem[k] = __ldg(w_ih + k);
  for (int k = threadIdx.x; k < n_hh; k += S2S_THREADS) smem[n_ih + k] = __ldg(w_hh + k);
  return GateWeights{smem, smem + n_ih, d, true};
}

// out[c] = sum_r w[r] * M(r, c), c < ncols.  P = max(1, S2S_THREADS / ncols) row partitions: partition p sums rows
// p, p + P, ... in ascending order and the P partials are added in ascending p.  Ends with a barrier.
template <class M>
__device__ __forceinline__ void col_sum(M m, const float* w, int nrows, int ncols, float* part, float* out) {
  const int tid = threadIdx.x;
  const int P = max(1, S2S_THREADS / ncols);
  if (P == 1) {
    for (int c = tid; c < ncols; c += S2S_THREADS) {
      float a = 0.0f;
      for (int r = 0; r < nrows; ++r) a = a + w[r] * m(r, c);
      out[c] = a;
    }
  } else {
    if (tid < P * ncols) {
      const int p = tid / ncols, c = tid - p * ncols;
      float a = 0.0f;
      for (int r = p; r < nrows; r += P) a = a + w[r] * m(r, c);
      part[tid] = a;
    }
    __syncthreads();
    for (int c = tid; c < ncols; c += S2S_THREADS) {
      float a = part[c];
      for (int p = 1; p < P; ++p) a = a + part[p * ncols + c];
      out[c] = a;
    }
  }
  __syncthreads();
}

// gp[j] = (sum_c [W_ih | W_hh](j, c) * [q* | q](c) + b_ih[j]) + b_hh[j] for the 4D gate rows.  One warp per row (four rows
// in flight per warp), lanes over the 3D columns in ascending strides of 32, then a butterfly.  The hidden input h is q,
// the first half of q*.
__device__ __forceinline__ void gate_matvec(const GateWeights& W, const float* __restrict__ b_ih, const float* __restrict__ b_hh,
                            const float* qs, float* gp) {
  const int d = W.d, G = 4 * d, C = 3 * d;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j0 = warp; j0 < G; j0 += 4 * S2S_WARPS) {
    const int j1 = j0 + S2S_WARPS, j2 = j0 + 2 * S2S_WARPS, j3 = j0 + 3 * S2S_WARPS;
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
    for (int c = lane; c < C; c += 32) {
      const float v = qs[c < 2 * d ? c : c - 2 * d];
      a0 = a0 + W(j0, c) * v;
      if (j1 < G) a1 = a1 + W(j1, c) * v;
      if (j2 < G) a2 = a2 + W(j2, c) * v;
      if (j3 < G) a3 = a3 + W(j3, c) * v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a0 = a0 + __shfl_xor_sync(0xffffffffu, a0, o);
      a1 = a1 + __shfl_xor_sync(0xffffffffu, a1, o);
      a2 = a2 + __shfl_xor_sync(0xffffffffu, a2, o);
      a3 = a3 + __shfl_xor_sync(0xffffffffu, a3, o);
    }
    if (lane == 0) {
      gp[j0] = (a0 + __ldg(b_ih + j0)) + __ldg(b_hh + j0);
      if (j1 < G) gp[j1] = (a1 + __ldg(b_ih + j1)) + __ldg(b_hh + j1);
      if (j2 < G) gp[j2] = (a2 + __ldg(b_ih + j2)) + __ldg(b_hh + j2);
      if (j3 < G) gp[j3] = (a3 + __ldg(b_ih + j3)) + __ldg(b_hh + j3);
    }
  }
}

__device__ __forceinline__ float dot_row(const float* xr, const float* v, int d) {
  float a = 0.0f;
  for (int k = 0; k < d; ++k) a = a + xr[k] * v[k];
  return a;
}

// Forward: one CTA per graph b.  Per step t: the LSTM cell on q*_{t-1} (thread f < D owns feature f and keeps c in a
// register), e_i = x_i . q, alpha = softmax(e) with the maximum subtracted, r = sum_i alpha_i x_i, q*_t = [q, r].
// saved (optional): per (t, b) the record [q*_t (2D) | c_t (D) | i f g o (4D) | alpha_t (N)], record (t * B + b).
__global__ void __launch_bounds__(S2S_THREADS) k_set2set_fwd(const float* __restrict__ x, int n_graphs, int n, int d, int steps,
                                                             const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                                                             bool stage, const float* __restrict__ b_ih,
                                                             const float* __restrict__ b_hh, float* __restrict__ out,
                                                             float* __restrict__ saved) {
  extern __shared__ float sm[];
  const int ldx = s2s_ldx(d);
  float* xs = sm;                       // n * ldx
  float* al = xs + (size_t)n * ldx;     // n: logits, then exp, then alpha
  float* qs = al + n;                   // 2d: q*
  float* gp = qs + 2 * d;               // 4d: gate pre-activations
  float* part = gp + 4 * d;             // S2S_THREADS partials
  float* red = part + S2S_THREADS;      // S2S_WARPS + 1
  const GateWeights W = stage_weights(w_ih, w_hh, d, stage, red + S2S_WARPS + 1);   // 12 d^2 when staged
  const int b = blockIdx.x, tid = threadIdx.x;
  const long long rec_len = 7LL * d + n;
  const float* xb = x + (size_t)b * n * d;
  for (int e = tid; e < n * d; e += S2S_THREADS) {
    const int i = e / d;
    xs[i * ldx + (e - i * d)] = xb[e];
  }
  for (int k = tid; k < 2 * d; k += S2S_THREADS) qs[k] = 0.0f;
  float c = 0.0f;
  __syncthreads();
  for (int t = 0; t < steps; ++t) {
    float* rec = saved ? saved + ((long long)t * n_graphs + b) * rec_len : nullptr;
    gate_matvec(W, b_ih, b_hh, qs, gp);
    __syncthreads();
    if (tid < d) {
      const float ig = sigmoid_f(gp[tid]), fg = sigmoid_f(gp[d + tid]), gg = tanhf(gp[2 * d + tid]), og = sigmoid_f(gp[3 * d + tid]);
      c = fg * c + ig * gg;
      qs[tid] = og * tanhf(c);
      if (rec) {
        rec[2 * d + tid] = c;
        rec[3 * d + tid] = ig;
        rec[4 * d + tid] = fg;
        rec[5 * d + tid] = gg;
        rec[6 * d + tid] = og;
      }
    }
    __syncthreads();
    float m = -INFINITY;
    for (int i = tid; i < n; i += S2S_THREADS) {
      const float e = dot_row(xs + i * ldx, qs, d);
      al[i] = e;
      m = fmaxf(m, e);
    }
    m = block_reduce<true>(m, red);
    float s = 0.0f;
    for (int i = tid; i < n; i += S2S_THREADS) {
      const float p = expf(al[i] - m);
      al[i] = p;
      s = s + p;
    }
    s = block_reduce<false>(s, red);
    for (int i = tid; i < n; i += S2S_THREADS) {
      const float a = al[i] / s;
      al[i] = a;
      if (rec) rec[7 * d + i] = a;
    }
    __syncthreads();
    col_sum(RowsAt{xs, ldx}, al, n, d, part, qs + d);
    if (rec)
      for (int k = tid; k < 2 * d; k += S2S_THREADS) rec[k] = qs[k];
  }
  for (int k = tid; k < 2 * d; k += S2S_THREADS) out[(size_t)b * 2 * d + k] = qs[k];
}

// Backward: one CTA per graph walks t = T-1 .. 0 carrying dq* (shared memory) and dc (register of thread f < D).
//   attention:  dalpha_i = x_i . dr,  de_i = alpha_i (dalpha_i - sum_j alpha_j dalpha_j)
//               dx_i += alpha_i dr + de_i q,  dq = dq*[:D] + sum_i de_i x_i
//   cell:       dG = pre-activation gate gradients (written to grad_gates[t, b, :])
//   recurrence: dq*_{t-1} = W_ih^T dG + [W_hh^T dG, 0]
// dx is summed in shared memory and written once.
__global__ void __launch_bounds__(S2S_THREADS) k_set2set_bwd(const float* __restrict__ x, int n_graphs, int n, int d, int steps,
                                                             const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                                                             bool stage, const float* __restrict__ saved,
                                                             const float* __restrict__ grad_out, float* __restrict__ grad_x,
                                                             float* __restrict__ grad_gates) {
  extern __shared__ float sm[];
  const int ldx = s2s_ldx(d);
  const bool want_dx = grad_x != nullptr;
  float* xs = sm;                                          // n * ldx
  float* dxs = xs + (size_t)n * ldx;                       // n * ldx when grad_x is wanted
  float* de = dxs + (want_dx ? (size_t)n * ldx : 0);       // n
  float* dqs = de + n;                                     // 2d: dq*
  float* qv = dqs + 2 * d;                                 // d: q_t
  float* dg = qv + d;                                      // 4d: dG
  float* tmp = dg + 4 * d;                                 // 3d
  float* part = tmp + 3 * d;                               // S2S_THREADS
  float* red = part + S2S_THREADS;                         // S2S_WARPS + 1
  const GateWeights W = stage_weights(w_ih, w_hh, d, stage, red + S2S_WARPS + 1);   // 12 d^2 when staged
  const int b = blockIdx.x, tid = threadIdx.x;
  const long long rec_len = 7LL * d + n;
  const float* xb = x + (size_t)b * n * d;
  for (int e = tid; e < n * d; e += S2S_THREADS) {
    const int i = e / d, o = i * ldx + (e - i * d);
    xs[o] = xb[e];
    if (want_dx) dxs[o] = 0.0f;
  }
  for (int k = tid; k < 2 * d; k += S2S_THREADS) dqs[k] = grad_out[(size_t)b * 2 * d + k];
  float dc = 0.0f;
  for (int t = steps - 1; t >= 0; --t) {
    const float* rec = saved + ((long long)t * n_graphs + b) * rec_len;
    const float* alpha = rec + 7 * d;
    for (int k = tid; k < d; k += S2S_THREADS) qv[k] = rec[k];
    __syncthreads();
    float s = 0.0f;
    for (int i = tid; i < n; i += S2S_THREADS) {
      const float da = dot_row(xs + i * ldx, dqs + d, d);
      de[i] = da;
      s = s + __ldg(alpha + i) * da;
    }
    s = block_reduce<false>(s, red);
    for (int i = tid; i < n; i += S2S_THREADS) de[i] = __ldg(alpha + i) * (de[i] - s);
    __syncthreads();
    if (want_dx) {
      for (int e = tid; e < n * d; e += S2S_THREADS) {
        const int i = e / d, f = e - i * d, o = i * ldx + f;
        dxs[o] = dxs[o] + (__ldg(alpha + i) * dqs[d + f] + de[i] * qv[f]);
      }
    }
    col_sum(RowsAt{xs, ldx}, de, n, d, part, tmp);
    if (tid < d) {
      const float dq = dqs[tid] + tmp[tid];
      const float ct = rec[2 * d + tid];
      const float ig = rec[3 * d + tid], fg = rec[4 * d + tid], gg = rec[5 * d + tid], og = rec[6 * d + tid];
      const float cp = t > 0 ? rec[2 * d + tid - n_graphs * rec_len] : 0.0f;
      const float tc = tanhf(ct);
      dc = dc + dq * og * (1.0f - tc * tc);
      const float dgi = dc * gg * ig * (1.0f - ig);
      const float dgf = dc * cp * fg * (1.0f - fg);
      const float dgg = dc * ig * (1.0f - gg * gg);
      const float dgo = dq * tc * og * (1.0f - og);
      dc = dc * fg;
      dg[tid] = dgi;
      dg[d + tid] = dgf;
      dg[2 * d + tid] = dgg;
      dg[3 * d + tid] = dgo;
      float* gg_out = grad_gates + ((long long)t * n_graphs + b) * 4 * d;
      gg_out[tid] = dgi;
      gg_out[d + tid] = dgf;
      gg_out[2 * d + tid] = dgg;
      gg_out[3 * d + tid] = dgo;
    }
    __syncthreads();
    if (t > 0) {                                           // q*_{-1} = 0: nothing flows out of step 0
      col_sum(W, dg, 4 * d, 3 * d, part, tmp);
      for (int k = tid; k < 2 * d; k += S2S_THREADS) dqs[k] = k < d ? tmp[k] + tmp[2 * d + k] : tmp[k];
    }
  }
  if (want_dx) {
    __syncthreads();
    float* gx = grad_x + (size_t)b * n * d;
    for (int e = tid; e < n * d; e += S2S_THREADS) {
      const int i = e / d;
      gx[e] = dxs[i * ldx + (e - i * d)];
    }
  }
}

size_t fwd_smem_bytes(int n, int d, bool stage) {
  return sizeof(float) * ((size_t)n * s2s_ldx(d) + n + 6 * d + S2S_THREADS + S2S_WARPS + 1 + (stage ? 12 * d * d : 0));
}

size_t bwd_smem_bytes(int n, int d, bool want_dx, bool stage) {
  return sizeof(float) * ((size_t)n * s2s_ldx(d) * (want_dx ? 2 : 1) + n + 10 * d + S2S_THREADS + S2S_WARPS + 1 +
                          (stage ? 12 * d * d : 0));
}

// The weights are staged in shared memory when fwd_smem_bytes / bwd_smem_bytes with them fit the device's opt-in limit
// (232448 bytes on H100).  There, at D = 66: forward N <= 76, backward N <= 36 with dx (N <= 72 without); at D = 16 every
// N the limits allow; never above D = 69.  A host query, legal while a stream is capturing.
int smem_limit(int* bytes) {
  static int limit = 0;
  if (limit == 0) {
    int dev = 0;
    PNA_CUDA_TRY(cudaGetDevice(&dev));
    PNA_CUDA_TRY(cudaDeviceGetAttribute(&limit, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  }
  *bytes = limit;
  return PNA_OK;
}

int check_sizes(const char* fn, int64_t n_graphs, int32_t n_nodes, int32_t n_feat, int32_t steps) {
  PNA_REQUIRE(n_graphs > 0 && n_nodes > 0 && n_feat > 0 && steps > 0, PNA_ERR_BAD_ARG,
              "%s: sizes must be positive (n_graphs %lld, n_nodes %d, n_feat %d, steps %d)", fn, (long long)n_graphs, n_nodes,
              n_feat, steps);
  PNA_REQUIRE(n_feat <= S2S_MAX_FEAT && (int64_t)n_nodes * n_feat <= S2S_MAX_ELEMS, PNA_ERR_UNSUPPORTED,
              "%s: n_feat %d, n_nodes %d outside n_feat <= %d, n_nodes * n_feat <= %d", fn, n_feat, n_nodes, S2S_MAX_FEAT,
              S2S_MAX_ELEMS);
  PNA_REQUIRE(n_graphs <= INT32_MAX, PNA_ERR_UNSUPPORTED, "%s: n_graphs %lld above 2^31 - 1", fn, (long long)n_graphs);
  const int64_t per_step = n_graphs * (7LL * n_feat + n_nodes);
  PNA_REQUIRE(per_step <= INT64_MAX / steps, PNA_ERR_UNSUPPORTED, "%s: saved buffer size overflows int64", fn);
  return PNA_OK;
}

template <class K>
int set_smem(K kern, size_t bytes, int* done) {
  if ((int)bytes > *done) {
    PNA_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    *done = (int)bytes;
  }
  return PNA_OK;
}

}  // namespace
}  // namespace pna

using namespace pna;

extern "C" int pna_set2set_saved_floats(int64_t n_graphs, int32_t n_nodes, int32_t n_feat, int32_t steps, int64_t* n_floats) {
  PNA_REQUIRE(n_floats, PNA_ERR_BAD_ARG, "pna_set2set_saved_floats: null pointer");
  const int st = check_sizes("pna_set2set_saved_floats", n_graphs, n_nodes, n_feat, steps);
  if (st != PNA_OK) return st;
  *n_floats = (int64_t)steps * n_graphs * (7LL * n_feat + n_nodes);
  return PNA_OK;
}

extern "C" int pna_set2set_fwd(const float* x, int64_t n_graphs, int32_t n_nodes, int32_t n_feat, int32_t steps, const float* w_ih,
                               const float* w_hh, const float* b_ih, const float* b_hh, float* out, float* saved,
                               pna_stream_t stream) {
  const int st = check_sizes("pna_set2set_fwd", n_graphs, n_nodes, n_feat, steps);
  if (st != PNA_OK) return st;
  PNA_REQUIRE(x && w_ih && w_hh && b_ih && b_hh && out, PNA_ERR_BAD_ARG, "pna_set2set_fwd: null pointer");
  int limit = 0;
  const int lst = smem_limit(&limit);
  if (lst != PNA_OK) return lst;
  const bool stage = fwd_smem_bytes(n_nodes, n_feat, true) <= (size_t)limit;
  static int smem_set = 0;
  const size_t smem = fwd_smem_bytes(n_nodes, n_feat, stage);
  const int sst = set_smem(k_set2set_fwd, smem, &smem_set);
  if (sst != PNA_OK) return sst;
  k_set2set_fwd<<<(unsigned)n_graphs, S2S_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      x, (int)n_graphs, n_nodes, n_feat, steps, w_ih, w_hh, stage, b_ih, b_hh, out, saved);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

extern "C" int pna_set2set_bwd(const float* x, int64_t n_graphs, int32_t n_nodes, int32_t n_feat, int32_t steps, const float* w_ih,
                               const float* w_hh, const float* saved, const float* grad_out, float* grad_x, float* grad_gates,
                               pna_stream_t stream) {
  const int st = check_sizes("pna_set2set_bwd", n_graphs, n_nodes, n_feat, steps);
  if (st != PNA_OK) return st;
  PNA_REQUIRE(x && w_ih && w_hh && saved && grad_out && grad_gates, PNA_ERR_BAD_ARG, "pna_set2set_bwd: null pointer");
  int limit = 0;
  const int lst = smem_limit(&limit);
  if (lst != PNA_OK) return lst;
  const bool stage = bwd_smem_bytes(n_nodes, n_feat, grad_x != nullptr, true) <= (size_t)limit;
  static int smem_set = 0;
  const size_t smem = bwd_smem_bytes(n_nodes, n_feat, grad_x != nullptr, stage);
  const int sst = set_smem(k_set2set_bwd, smem, &smem_set);
  if (sst != PNA_OK) return sst;
  k_set2set_bwd<<<(unsigned)n_graphs, S2S_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      x, (int)n_graphs, n_nodes, n_feat, steps, w_ih, w_hh, stage, saved, grad_out, grad_x, grad_gates);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}
