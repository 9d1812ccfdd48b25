// pna_edge_mlp_fwd / pna_edge_mlp_bwd: the per-edge pretrans MLP of the dense layer with pretrans_layers = L >= 2
// (reference models/layers.py:200-229: FCLayer(2F -> F, relu), L-2 x FCLayer(F -> F, relu), FCLayer(F -> F, none)),
// evaluated once per slot of a destination-sorted CSR with every intermediate in registers.
//
// The first layer splits into node-level GEMMs done by the caller: A = h W1[:, :F]^T (the destination half), Bm =
// h W1[:, F:]^T (the source half), b1.  For slot s of row i with source j = col[s], tower t, width F (all fp32):
//   u1_o = fl(fl(A[i, tF+o] + Bm[j, tF+o]) + b1[tF+o]),                  z1_o = u1_o > 0 ? u1_o : 0
//   layer k = 2..L:  acc_o = 0;  for c = 0..F-1 in order: acc_o = fl(acc_o + fl(W_k[t][o][c] * z_(k-1),c))
//                    u_k,o = fl(acc_o + b_k[t][o]);   z_k,o = u_k,o > 0 ? u_k,o : 0   (k < L)
//   M[s, tF+o] = u_L,o
// Backward, with G_L = dM[s, tF : tF+F]:
//   layer k = L..2:  q_c = 0;  for o = 0..F-1 in order: q_c = fl(q_c + fl(W_k[t][o][c] * G_k,o))
//                    G_(k-1),c = z_(k-1),c > 0 ? q_c : 0
// Every product and sum is rounded once (the library is built with -fmad=false; the host emulation with
// -ffp-contract=off), so a slot's values are a fixed function of its inputs: no atomics, no reductions across threads.
// The weight and bias gradients (G_k^T z_(k-1), sum_s G_k) and dA / dBm (sums of G_1 over the rows / the sources) are
// the caller's, as library GEMMs and the aggregation's `sum`.
//
// Layout: one thread per (slot, tower); blockIdx.y is the tower, so every weight address is warp-uniform and goes
// through the read-only path.  No shared memory, no shuffles, no barriers (tests run the kernels on the host thread by
// thread).  The width is a compile-time bucket W in {4, 8, 16, 32, 64} (fully unrolled loops keep z in registers);
// EXACT drops the width guards when F == W.
#include "common.cuh"

namespace pna {

constexpr int kMlpThreads = 128;

// row of slot s: the last i with rowptr[i] <= s (empty rows share their rowptr value with the next row)
__device__ __forceinline__ long long mlp_row_of(const int* __restrict__ rowptr, long long n_rows, long long s) {
  long long lo = 0, hi = n_rows - 1;
  while (lo < hi) {
    const long long mid = (lo + hi + 1) >> 1;
    if (__ldg(rowptr + mid) <= s) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

template <int W, bool EXACT>
__global__ void __launch_bounds__(kMlpThreads) k_edge_mlp_fwd(const int* __restrict__ rowptr, const int* __restrict__ col,
                                                              long long n_rows, long long n_edges, const float* __restrict__ a,
                                                              const float* __restrict__ b, const float* __restrict__ bias1,
                                                              const float* __restrict__ weight, const float* __restrict__ bias,
                                                              int n_layers, int F, float* __restrict__ msg,
                                                              float* __restrict__ act) {
  const long long s = (long long)blockIdx.x * kMlpThreads + threadIdx.x;
  if (s >= n_edges) return;
  const int t = blockIdx.y, T = gridDim.y;
  const int TF = T * F;
  const long long i = mlp_row_of(rowptr, n_rows, s);
  const long long j = __ldg(col + s);
  const float* ai = a + i * TF + t * F;
  const float* bj = b + j * TF + t * F;
  const float* b1 = bias1 + t * F;
  float z[W];
#pragma unroll
  for (int o = 0; o < W; ++o) {
    if (EXACT || o < F) {
      const float u = __fadd_rn(__fadd_rn(__ldg(ai + o), __ldg(bj + o)), __ldg(b1 + o));
      z[o] = u > 0.f ? u : 0.f;
    } else {
      z[o] = 0.f;
    }
  }
  const long long slot_off = s * TF + t * F;
  const long long layer_stride = n_edges * TF;
  for (int k = 2; k <= n_layers; ++k) {
    if (act) {      // z_(k-1)
      float* dst = act + (long long)(k - 2) * layer_stride + slot_off;
#pragma unroll
      for (int o = 0; o < W; ++o)
        if (EXACT || o < F) dst[o] = z[o];
    }
    const float* Wk = weight + ((long long)(k - 2) * T + t) * F * F;
    const float* bk = bias + ((long long)(k - 2) * T + t) * F;
    float u[W];
#pragma unroll
    for (int o = 0; o < W; ++o) {
      float acc = 0.f;
      if (EXACT || o < F) {
#pragma unroll
        for (int c = 0; c < W; ++c)
          if (EXACT || c < F) acc = __fadd_rn(acc, __fmul_rn(__ldg(Wk + o * F + c), z[c]));
        acc = __fadd_rn(acc, __ldg(bk + o));
      }
      u[o] = acc;
    }
    const bool last = k == n_layers;
#pragma unroll
    for (int o = 0; o < W; ++o) z[o] = (last || u[o] > 0.f) ? u[o] : 0.f;
  }
  float* m = msg + slot_off;
#pragma unroll
  for (int o = 0; o < W; ++o)
    if (EXACT || o < F) m[o] = z[o];
}

template <int W, bool EXACT>
__global__ void __launch_bounds__(kMlpThreads) k_edge_mlp_bwd(const float* __restrict__ grad_msg, const float* __restrict__ act,
                                                              const float* __restrict__ weight, long long n_edges, int n_layers,
                                                              int F, float* __restrict__ grad_pre) {
  const long long s = (long long)blockIdx.x * kMlpThreads + threadIdx.x;
  if (s >= n_edges) return;
  const int t = blockIdx.y, T = gridDim.y;
  const int TF = T * F;
  const long long slot_off = s * TF + t * F;
  const long long layer_stride = n_edges * TF;
  float g[W];
#pragma unroll
  for (int o = 0; o < W; ++o) g[o] = (EXACT || o < F) ? __ldg(grad_msg + slot_off + o) : 0.f;
  for (int k = n_layers; k >= 2; --k) {
    const float* Wk = weight + ((long long)(k - 2) * T + t) * F * F;
    float q[W];
#pragma unroll
    for (int c = 0; c < W; ++c) q[c] = 0.f;
#pragma unroll
    for (int o = 0; o < W; ++o) {
      if (EXACT || o < F) {
#pragma unroll
        for (int c = 0; c < W; ++c)
          if (EXACT || c < F) q[c] = __fadd_rn(q[c], __fmul_rn(__ldg(Wk + o * F + c), g[o]));
      }
    }
    const float* z = act + (long long)(k - 2) * layer_stride + slot_off;      // z_(k-1)
    float* dst = grad_pre + (long long)(k - 2) * layer_stride + slot_off;     // G_(k-1)
#pragma unroll
    for (int c = 0; c < W; ++c) {
      if (EXACT || c < F) {
        g[c] = __ldg(z + c) > 0.f ? q[c] : 0.f;
        dst[c] = g[c];
      }
    }
  }
}

template <int W>
static int launch_fwd(dim3 grid, const int* rowptr, const int* col, long long n_rows, long long n_edges, const float* a,
                      const float* b, const float* bias1, const float* weight, const float* bias, int n_layers, int F,
                      float* msg, float* act, cudaStream_t st) {
  if (F == W)
    k_edge_mlp_fwd<W, true><<<grid, kMlpThreads, 0, st>>>(rowptr, col, n_rows, n_edges, a, b, bias1, weight, bias, n_layers, F,
                                                            msg, act);
  else
    k_edge_mlp_fwd<W, false><<<grid, kMlpThreads, 0, st>>>(rowptr, col, n_rows, n_edges, a, b, bias1, weight, bias, n_layers, F,
                                                             msg, act);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

template <int W>
static int launch_bwd(dim3 grid, const float* grad_msg, const float* act, const float* weight, long long n_edges, int n_layers,
                      int F, float* grad_pre, cudaStream_t st) {
  if (F == W)
    k_edge_mlp_bwd<W, true><<<grid, kMlpThreads, 0, st>>>(grad_msg, act, weight, n_edges, n_layers, F, grad_pre);
  else
    k_edge_mlp_bwd<W, false><<<grid, kMlpThreads, 0, st>>>(grad_msg, act, weight, n_edges, n_layers, F, grad_pre);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

static int check_shape(const char* who, long long n_edges, int n_layers, int n_towers, int width, dim3* grid) {
  PNA_REQUIRE(n_edges >= 0, PNA_ERR_BAD_ARG, "%s: n_edges %lld < 0", who, n_edges);
  PNA_REQUIRE(n_layers >= 2, PNA_ERR_BAD_ARG, "%s: n_layers %d < 2 (one layer is affine: use the node-level GEMMs)", who,
              n_layers);
  PNA_REQUIRE(n_towers >= 1 && width >= 1, PNA_ERR_BAD_ARG, "%s: n_towers %d, width %d", who, n_towers, width);
  PNA_REQUIRE(width <= PNA_EDGE_MLP_MAX_WIDTH, PNA_ERR_UNSUPPORTED, "%s: width %d > %d", who, width, PNA_EDGE_MLP_MAX_WIDTH);
  PNA_REQUIRE(n_towers <= 65535, PNA_ERR_UNSUPPORTED, "%s: n_towers %d > 65535", who, n_towers);
  const long long gx = (n_edges + kMlpThreads - 1) / kMlpThreads;
  PNA_REQUIRE(gx <= 0x7fffffffll, PNA_ERR_UNSUPPORTED, "%s: too many edges", who);
  *grid = dim3((unsigned)gx, (unsigned)n_towers);
  return PNA_OK;
}

}  // namespace pna

using namespace pna;

extern "C" int pna_edge_mlp_fwd(const int32_t* rowptr, const int32_t* col, int64_t n_rows, int64_t n_edges, const float* a,
                                const float* b, const float* bias1, const float* weight, const float* bias, int32_t n_layers,
                                int32_t n_towers, int32_t width, float* messages, float* activations, pna_stream_t stream) {
  dim3 grid;
  const int rc = check_shape("pna_edge_mlp_fwd", n_edges, n_layers, n_towers, width, &grid);
  if (rc != PNA_OK) return rc;
  PNA_REQUIRE(n_rows >= 0 && (n_rows > 0 || n_edges == 0), PNA_ERR_BAD_ARG, "pna_edge_mlp_fwd: n_rows %lld",
              (long long)n_rows);
  if (n_edges == 0) return PNA_OK;
  PNA_REQUIRE(rowptr && col && a && b && bias1 && weight && bias && messages, PNA_ERR_BAD_ARG, "pna_edge_mlp_fwd: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long N = n_rows, E = n_edges;
  if (width <= 4) return launch_fwd<4>(grid, rowptr, col, N, E, a, b, bias1, weight, bias, n_layers, width, messages, activations, st);
  if (width <= 8) return launch_fwd<8>(grid, rowptr, col, N, E, a, b, bias1, weight, bias, n_layers, width, messages, activations, st);
  if (width <= 16) return launch_fwd<16>(grid, rowptr, col, N, E, a, b, bias1, weight, bias, n_layers, width, messages, activations, st);
  if (width <= 32) return launch_fwd<32>(grid, rowptr, col, N, E, a, b, bias1, weight, bias, n_layers, width, messages, activations, st);
  return launch_fwd<64>(grid, rowptr, col, N, E, a, b, bias1, weight, bias, n_layers, width, messages, activations, st);
}

extern "C" int pna_edge_mlp_bwd(const float* grad_messages, const float* activations, const float* weight, int64_t n_edges,
                                int32_t n_layers, int32_t n_towers, int32_t width, float* grad_pre, pna_stream_t stream) {
  dim3 grid;
  const int rc = check_shape("pna_edge_mlp_bwd", n_edges, n_layers, n_towers, width, &grid);
  if (rc != PNA_OK) return rc;
  if (n_edges == 0) return PNA_OK;
  PNA_REQUIRE(grad_messages && activations && weight && grad_pre, PNA_ERR_BAD_ARG, "pna_edge_mlp_bwd: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long E = n_edges;
  if (width <= 4) return launch_bwd<4>(grid, grad_messages, activations, weight, E, n_layers, width, grad_pre, st);
  if (width <= 8) return launch_bwd<8>(grid, grad_messages, activations, weight, E, n_layers, width, grad_pre, st);
  if (width <= 16) return launch_bwd<16>(grid, grad_messages, activations, weight, E, n_layers, width, grad_pre, st);
  if (width <= 32) return launch_bwd<32>(grid, grad_messages, activations, weight, E, n_layers, width, grad_pre, st);
  return launch_bwd<64>(grid, grad_messages, activations, weight, E, n_layers, width, grad_pre, st);
}
