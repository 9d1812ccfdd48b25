// pna_edge_mlp_fwd / pna_edge_mlp_bwd: the per-edge pretrans MLP of the dense layer with pretrans_layers = L >= 2
// (reference models/layers.py:200-229: FCLayer(2F -> F, relu), L-2 x FCLayer(F -> F, relu), FCLayer(F -> F, none)),
// evaluated once per slot of a destination-sorted CSR with every intermediate in registers.
// pna_edge_msg_fwd / pna_edge_msg_bwd: the same per-slot arithmetic for the PyG and DGL layers, with a per-slot edge term
// C (the edge-feature columns of the first layer), any L >= 1, and messages written at a per-tower pitch P >= F.
//
// The first layer splits into node-level GEMMs done by the caller: A = h W1[:, :F]^T (the destination half), Bm =
// h W1[:, F:]^T (the source half), b1, and C[s] = e[s] W1[:, 2F:]^T (edge term, optional).  For slot s of row i with
// source j = col[s], tower t, width F (all fp32):
//   u1_o = fl(fl(fl(A[i, tF+o] + Bm[j, tF+o]) + b1[tF+o]) + C[s, tF+o])   (no C: the last add is not made)
//   z1_o = u1_o > 0 ? u1_o : 0
//   layer k = 2..L:  acc_o = 0;  for c = 0..F-1 in order: acc_o = fl(acc_o + fl(W_k[t][o][c] * z_(k-1),c))
//                    u_k,o = fl(acc_o + b_k[t][o]);   z_k,o = u_k,o > 0 ? u_k,o : 0   (k < L)
//   M[s, tP+o] = u_L,o for o < F (L = 1: u1 itself), M[s, tP+o] = 0 for F <= o < P   (edge_mlp: P = F)
// Backward, with G_L = dM[s, tP : tP+F]:
//   layer k = L..2:  q_c = 0;  for o = 0..F-1 in order: q_c = fl(q_c + fl(W_k[t][o][c] * G_k,o))
//                    G_(k-1),c = z_(k-1),c > 0 ? q_c : 0
// Every product and sum is rounded once (the library is built with -fmad=false; the host emulation with
// -ffp-contract=off), so a slot's values are a fixed function of its inputs: no atomics, no reductions across threads.
// The weight and bias gradients (G_k^T z_(k-1), sum_s G_k) and dA / dBm / dC (sums of G_1 over the rows / the sources,
// G_1 itself) are the caller's, as library GEMMs and the aggregation's `sum`.
//
// Layout: one thread per (slot, tower); blockIdx.y is the tower, so every weight address is warp-uniform and goes
// through the read-only path.  No shared memory, no shuffles, no barriers (tests run the kernels on the host thread by
// thread).  For L >= 2 the width is a compile-time bucket W in {4, 8, 16, 32, 64} (fully unrolled loops keep z in
// registers); EXACT drops the width guards when F == W.  With L = 1 nothing is held across layers: k_edge_msg_fwd_affine
// loops over the width and takes any F.  The activations and G_1 .. G_(L-1) are always at pitch F.
//
// bf16 storage (pna_edge_msg_fwd_bf16 / pna_edge_msg_bwd_bf16, the layers under bf16 autocast): A, Bm, C, the messages, the
// stored activations and grad_messages are bf16; weights, biases and G_1 .. G_(L-1) stay fp32.  The same bodies, templated
// on the storage type S: a load widens to fp32 (exact), every operation after it is the fp32 kernel's, and a store of M or
// z_k rounds to nearest once.  So M_bf16 = RN(M_fp32(A, Bm, C widened)), and the backward on (dM, z_bf16) is the fp32
// backward on the widened (dM, z_bf16): its ReLU mask is `stored z > 0`.
#include "common.cuh"

namespace pna {

constexpr int kMlpThreads = 128;

// storage of a message-path operand: fp32 as it is, bf16 widened on load (exact) and rounded to nearest on store
__device__ __forceinline__ float st_ld(const float* p) { return __ldg(p); }
__device__ __forceinline__ float st_ld(const __nv_bfloat16* p) {
  return __uint_as_float(static_cast<unsigned>(__ldg(reinterpret_cast<const unsigned short*>(p))) << 16);
}
__device__ __forceinline__ void st_st(float* p, float v) { *p = v; }
__device__ __forceinline__ void st_st(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

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

// u1 of one (slot, tower) column: fl(fl(fl(A[i] + Bm[j]) + b1) + C[s]), the edge term last (none when cs is null)
template <typename S>
__device__ __forceinline__ float mlp_u1(const S* __restrict__ ai, const S* __restrict__ bj,
                                        const float* __restrict__ b1, const S* __restrict__ cs, int o) {
  float u = __fadd_rn(__fadd_rn(st_ld(ai + o), st_ld(bj + o)), __ldg(b1 + o));
  if (cs) u = __fadd_rn(u, st_ld(cs + o));
  return u;
}

// Layers 1..L (L >= 2) of one (slot, tower): z receives u_L; act (nullable) receives z_1 .. z_(L-1) at act_off
template <int W, bool EXACT, typename S>
__device__ __forceinline__ void mlp_slot_fwd(const S* __restrict__ ai, const S* __restrict__ bj,
                                             const float* __restrict__ b1, const S* __restrict__ cs,
                                             const float* __restrict__ weight, const float* __restrict__ bias, int n_layers,
                                             int T, int t, int F, S* __restrict__ act, long long act_off,
                                             long long layer_stride, float (&z)[W]) {
#pragma unroll
  for (int o = 0; o < W; ++o) {
    if (EXACT || o < F) {
      const float u = mlp_u1(ai, bj, b1, cs, o);
      z[o] = u > 0.f ? u : 0.f;
    } else {
      z[o] = 0.f;
    }
  }
  for (int k = 2; k <= n_layers; ++k) {
    if (act) {      // z_(k-1)
      S* dst = act + (long long)(k - 2) * layer_stride + act_off;
#pragma unroll
      for (int o = 0; o < W; ++o)
        if (EXACT || o < F) st_st(dst + o, z[o]);
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
}

// Backward of layers L..2 of one (slot, tower): gm is G_L (F values); grad_pre receives G_(L-1) .. G_1 at act_off
template <int W, bool EXACT, typename S>
__device__ __forceinline__ void mlp_slot_bwd(const S* __restrict__ gm, const S* __restrict__ act,
                                             const float* __restrict__ weight, int n_layers, int T, int t, int F,
                                             long long act_off, long long layer_stride, float* __restrict__ grad_pre) {
  float g[W];
#pragma unroll
  for (int o = 0; o < W; ++o) g[o] = (EXACT || o < F) ? st_ld(gm + o) : 0.f;
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
    const S* z = act + (long long)(k - 2) * layer_stride + act_off;          // z_(k-1)
    float* dst = grad_pre + (long long)(k - 2) * layer_stride + act_off;     // G_(k-1)
#pragma unroll
    for (int c = 0; c < W; ++c) {
      if (EXACT || c < F) {
        g[c] = st_ld(z + c) > 0.f ? q[c] : 0.f;
        dst[c] = g[c];
      }
    }
  }
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
  const long long slot_off = s * TF + t * F;
  float z[W];
  mlp_slot_fwd<W, EXACT, float>(a + i * TF + t * F, b + j * TF + t * F, bias1 + t * F, nullptr, weight, bias, n_layers, T, t, F,
                                act, slot_off, n_edges * TF, z);
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
  mlp_slot_bwd<W, EXACT, float>(grad_msg + slot_off, act, weight, n_layers, T, t, F, slot_off, n_edges * TF, grad_pre);
}

// pna_edge_msg_fwd, n_layers >= 2: the same per-slot body, the edge term (nullable) in u1, messages at pitch P with zero pads
template <int W, bool EXACT, typename S>
__device__ __forceinline__ void edge_msg_fwd_slot(const int* __restrict__ rowptr, const int* __restrict__ col, long long n_rows,
                                                  long long n_edges, const S* __restrict__ a, const S* __restrict__ b,
                                                  const float* __restrict__ bias1, const S* __restrict__ term,
                                                  const float* __restrict__ weight, const float* __restrict__ bias, int n_layers,
                                                  int F, int P, S* __restrict__ msg, S* __restrict__ act) {
  const long long s = (long long)blockIdx.x * kMlpThreads + threadIdx.x;
  if (s >= n_edges) return;
  const int t = blockIdx.y, T = gridDim.y;
  const int TF = T * F;
  const long long i = mlp_row_of(rowptr, n_rows, s);
  const long long j = __ldg(col + s);
  const long long slot_off = s * TF + t * F;
  float z[W];
  mlp_slot_fwd<W, EXACT, S>(a + i * TF + t * F, b + j * TF + t * F, bias1 + t * F, term ? term + slot_off : nullptr, weight,
                            bias, n_layers, T, t, F, act, slot_off, n_edges * TF, z);
  S* m = msg + s * T * P + (long long)t * P;
#pragma unroll
  for (int o = 0; o < W; ++o)
    if (EXACT || o < F) st_st(m + o, z[o]);
  for (int o = F; o < P; ++o) st_st(m + o, 0.f);
}

// pna_edge_msg_fwd, n_layers == 1: the message is u1 itself (no ReLU, nothing held across layers), any width
template <typename S>
__device__ __forceinline__ void edge_msg_fwd_affine_slot(const int* __restrict__ rowptr, const int* __restrict__ col,
                                                         long long n_rows, long long n_edges, const S* __restrict__ a,
                                                         const S* __restrict__ b, const float* __restrict__ bias1,
                                                         const S* __restrict__ term, int F, int P, S* __restrict__ msg) {
  const long long s = (long long)blockIdx.x * kMlpThreads + threadIdx.x;
  if (s >= n_edges) return;
  const int t = blockIdx.y, T = gridDim.y;
  const int TF = T * F;
  const long long i = mlp_row_of(rowptr, n_rows, s);
  const long long j = __ldg(col + s);
  const S* ai = a + i * TF + t * F;
  const S* bj = b + j * TF + t * F;
  const float* b1 = bias1 + t * F;
  const S* cs = term ? term + s * TF + t * F : nullptr;
  S* m = msg + s * T * P + (long long)t * P;
#pragma unroll 4
  for (int o = 0; o < F; ++o) st_st(m + o, mlp_u1(ai, bj, b1, cs, o));
  for (int o = F; o < P; ++o) st_st(m + o, 0.f);
}

// pna_edge_msg_bwd: the per-slot backward with G_L read at pitch P
template <int W, bool EXACT, typename S>
__device__ __forceinline__ void edge_msg_bwd_slot(const S* __restrict__ grad_msg, int P, const S* __restrict__ act,
                                                  const float* __restrict__ weight, long long n_edges, int n_layers, int F,
                                                  float* __restrict__ grad_pre) {
  const long long s = (long long)blockIdx.x * kMlpThreads + threadIdx.x;
  if (s >= n_edges) return;
  const int t = blockIdx.y, T = gridDim.y;
  const long long slot_off = s * T * F + t * F;
  mlp_slot_bwd<W, EXACT, S>(grad_msg + s * T * P + (long long)t * P, act, weight, n_layers, T, t, F, slot_off, n_edges * T * F,
                            grad_pre);
}

// the fp32 kernels (pna_edge_msg_fwd / _bwd) and the bf16-storage ones (pna_edge_msg_fwd_bf16 / _bwd_bf16)
template <int W, bool EXACT>
__global__ void __launch_bounds__(kMlpThreads) k_edge_msg_fwd(const int* __restrict__ rowptr, const int* __restrict__ col,
                                                              long long n_rows, long long n_edges, const float* __restrict__ a,
                                                              const float* __restrict__ b, const float* __restrict__ bias1,
                                                              const float* __restrict__ term, const float* __restrict__ weight,
                                                              const float* __restrict__ bias, int n_layers, int F, int P,
                                                              float* __restrict__ msg, float* __restrict__ act) {
  edge_msg_fwd_slot<W, EXACT, float>(rowptr, col, n_rows, n_edges, a, b, bias1, term, weight, bias, n_layers, F, P, msg, act);
}
template <int W, bool EXACT>
__global__ void __launch_bounds__(kMlpThreads) k_bf16_msg_fwd(const int* __restrict__ rowptr, const int* __restrict__ col,
                                                              long long n_rows, long long n_edges, const __nv_bfloat16* __restrict__ a,
                                                              const __nv_bfloat16* __restrict__ b, const float* __restrict__ bias1,
                                                              const __nv_bfloat16* __restrict__ term, const float* __restrict__ weight,
                                                              const float* __restrict__ bias, int n_layers, int F, int P,
                                                              __nv_bfloat16* __restrict__ msg, __nv_bfloat16* __restrict__ act) {
  edge_msg_fwd_slot<W, EXACT, __nv_bfloat16>(rowptr, col, n_rows, n_edges, a, b, bias1, term, weight, bias, n_layers, F, P, msg,
                                             act);
}

__global__ void __launch_bounds__(kMlpThreads) k_edge_msg_fwd_affine(const int* __restrict__ rowptr, const int* __restrict__ col,
                                                                     long long n_rows, long long n_edges,
                                                                     const float* __restrict__ a, const float* __restrict__ b,
                                                                     const float* __restrict__ bias1,
                                                                     const float* __restrict__ term, int F, int P,
                                                                     float* __restrict__ msg) {
  // edge_msg_fwd_affine_slot<float> spelled out: through the shared body ptxas allocates the pad loop's registers differently
  const long long s = (long long)blockIdx.x * kMlpThreads + threadIdx.x;
  if (s >= n_edges) return;
  const int t = blockIdx.y, T = gridDim.y;
  const int TF = T * F;
  const long long i = mlp_row_of(rowptr, n_rows, s);
  const long long j = __ldg(col + s);
  const float* ai = a + i * TF + t * F;
  const float* bj = b + j * TF + t * F;
  const float* b1 = bias1 + t * F;
  const float* cs = term ? term + s * TF + t * F : nullptr;
  float* m = msg + s * T * P + (long long)t * P;
#pragma unroll 4
  for (int o = 0; o < F; ++o) m[o] = mlp_u1(ai, bj, b1, cs, o);
  for (int o = F; o < P; ++o) m[o] = 0.f;
}
__global__ void __launch_bounds__(kMlpThreads) k_bf16_msg_fwd_affine(const int* __restrict__ rowptr, const int* __restrict__ col,
                                                                     long long n_rows, long long n_edges,
                                                                     const __nv_bfloat16* __restrict__ a,
                                                                     const __nv_bfloat16* __restrict__ b,
                                                                     const float* __restrict__ bias1,
                                                                     const __nv_bfloat16* __restrict__ term, int F, int P,
                                                                     __nv_bfloat16* __restrict__ msg) {
  edge_msg_fwd_affine_slot<__nv_bfloat16>(rowptr, col, n_rows, n_edges, a, b, bias1, term, F, P, msg);
}

template <int W, bool EXACT>
__global__ void __launch_bounds__(kMlpThreads) k_edge_msg_bwd(const float* __restrict__ grad_msg, int P,
                                                              const float* __restrict__ act, const float* __restrict__ weight,
                                                              long long n_edges, int n_layers, int F,
                                                              float* __restrict__ grad_pre) {
  edge_msg_bwd_slot<W, EXACT, float>(grad_msg, P, act, weight, n_edges, n_layers, F, grad_pre);
}
template <int W, bool EXACT>
__global__ void __launch_bounds__(kMlpThreads) k_bf16_msg_bwd(const __nv_bfloat16* __restrict__ grad_msg, int P,
                                                              const __nv_bfloat16* __restrict__ act, const float* __restrict__ weight,
                                                              long long n_edges, int n_layers, int F,
                                                              float* __restrict__ grad_pre) {
  edge_msg_bwd_slot<W, EXACT, __nv_bfloat16>(grad_msg, P, act, weight, n_edges, n_layers, F, grad_pre);
}

// kernel instances per storage type: the launchers below are written once for both
template <typename S>
struct MsgKernels;
template <>
struct MsgKernels<float> {
  template <int W, bool EXACT>
  static constexpr auto fwd() { return k_edge_msg_fwd<W, EXACT>; }
  template <int W, bool EXACT>
  static constexpr auto bwd() { return k_edge_msg_bwd<W, EXACT>; }
  static constexpr auto affine() { return k_edge_msg_fwd_affine; }
};
template <>
struct MsgKernels<__nv_bfloat16> {
  template <int W, bool EXACT>
  static constexpr auto fwd() { return k_bf16_msg_fwd<W, EXACT>; }
  template <int W, bool EXACT>
  static constexpr auto bwd() { return k_bf16_msg_bwd<W, EXACT>; }
  static constexpr auto affine() { return k_bf16_msg_fwd_affine; }
};

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

template <int W, typename S>
static int launch_msg_fwd(dim3 grid, const int* rowptr, const int* col, long long n_rows, long long n_edges, const S* a,
                          const S* b, const float* bias1, const S* term, const float* weight, const float* bias,
                          int n_layers, int F, int P, S* msg, S* act, cudaStream_t st) {
  auto kern = F == W ? MsgKernels<S>::template fwd<W, true>() : MsgKernels<S>::template fwd<W, false>();
  kern<<<grid, kMlpThreads, 0, st>>>(rowptr, col, n_rows, n_edges, a, b, bias1, term, weight, bias, n_layers, F, P, msg, act);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

template <int W, typename S>
static int launch_msg_bwd(dim3 grid, const S* grad_msg, int P, const S* act, const float* weight, long long n_edges,
                          int n_layers, int F, float* grad_pre, cudaStream_t st) {
  auto kern = F == W ? MsgKernels<S>::template bwd<W, true>() : MsgKernels<S>::template bwd<W, false>();
  kern<<<grid, kMlpThreads, 0, st>>>(grad_msg, P, act, weight, n_edges, n_layers, F, grad_pre);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

// min_layers: 2 for the edge-MLP entry points (one layer is affine), 1 for the message entry points; the register width
// limit applies from two layers on
static int check_shape(const char* who, long long n_edges, int n_layers, int min_layers, int n_towers, int width, dim3* grid) {
  PNA_REQUIRE(n_edges >= 0, PNA_ERR_BAD_ARG, "%s: n_edges %lld < 0", who, n_edges);
  PNA_REQUIRE(n_layers >= min_layers, PNA_ERR_BAD_ARG, "%s: n_layers %d < %d%s", who, n_layers, min_layers,
              min_layers == 2 ? " (one layer is affine: use the node-level GEMMs)" : "");
  PNA_REQUIRE(n_towers >= 1 && width >= 1, PNA_ERR_BAD_ARG, "%s: n_towers %d, width %d", who, n_towers, width);
  PNA_REQUIRE(n_layers < 2 || width <= PNA_EDGE_MLP_MAX_WIDTH, PNA_ERR_UNSUPPORTED, "%s: width %d > %d with %d layers", who,
              width, PNA_EDGE_MLP_MAX_WIDTH, n_layers);
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
  const int rc = check_shape("pna_edge_mlp_fwd", n_edges, n_layers, 2, n_towers, width, &grid);
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
  const int rc = check_shape("pna_edge_mlp_bwd", n_edges, n_layers, 2, n_towers, width, &grid);
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

namespace pna {

// pna_edge_msg_fwd / pna_edge_msg_fwd_bf16: S is the storage type of a, b, edge_term, messages and activations
template <typename S>
static int edge_msg_fwd(const char* who, const int32_t* rowptr, const int32_t* col, int64_t n_rows, int64_t n_edges, const S* a,
                        const S* b, const float* bias1, const S* edge_term, const float* weight, const float* bias,
                        int32_t n_layers, int32_t n_towers, int32_t width, int32_t msg_pitch, S* messages, S* activations,
                        pna_stream_t stream) {
  dim3 grid;
  const int rc = check_shape(who, n_edges, n_layers, 1, n_towers, width, &grid);
  if (rc != PNA_OK) return rc;
  PNA_REQUIRE(msg_pitch >= width, PNA_ERR_BAD_ARG, "%s: msg_pitch %d < width %d", who, msg_pitch, width);
  PNA_REQUIRE(n_rows >= 0 && (n_rows > 0 || n_edges == 0), PNA_ERR_BAD_ARG, "%s: n_rows %lld", who, (long long)n_rows);
  if (n_edges == 0) return PNA_OK;
  PNA_REQUIRE(rowptr && col && a && b && bias1 && messages && (n_layers == 1 || (weight && bias)), PNA_ERR_BAD_ARG,
              "%s: null pointer", who);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long N = n_rows, E = n_edges;
  const S* C = edge_term;
  const int P = msg_pitch;
  if (n_layers == 1) {
    auto kern = MsgKernels<S>::affine();
    kern<<<grid, kMlpThreads, 0, st>>>(rowptr, col, N, E, a, b, bias1, C, width, P, messages);
    PNA_CUDA_TRY(cudaGetLastError());
    return PNA_OK;
  }
  if (width <= 4) return launch_msg_fwd<4>(grid, rowptr, col, N, E, a, b, bias1, C, weight, bias, n_layers, width, P, messages, activations, st);
  if (width <= 8) return launch_msg_fwd<8>(grid, rowptr, col, N, E, a, b, bias1, C, weight, bias, n_layers, width, P, messages, activations, st);
  if (width <= 16) return launch_msg_fwd<16>(grid, rowptr, col, N, E, a, b, bias1, C, weight, bias, n_layers, width, P, messages, activations, st);
  if (width <= 32) return launch_msg_fwd<32>(grid, rowptr, col, N, E, a, b, bias1, C, weight, bias, n_layers, width, P, messages, activations, st);
  return launch_msg_fwd<64>(grid, rowptr, col, N, E, a, b, bias1, C, weight, bias, n_layers, width, P, messages, activations, st);
}

template <typename S>
static int edge_msg_bwd(const char* who, const S* grad_messages, int32_t msg_pitch, const S* activations, const float* weight,
                        int64_t n_edges, int32_t n_layers, int32_t n_towers, int32_t width, float* grad_pre, pna_stream_t stream) {
  dim3 grid;
  const int rc = check_shape(who, n_edges, n_layers, 2, n_towers, width, &grid);
  if (rc != PNA_OK) return rc;
  PNA_REQUIRE(msg_pitch >= width, PNA_ERR_BAD_ARG, "%s: msg_pitch %d < width %d", who, msg_pitch, width);
  if (n_edges == 0) return PNA_OK;
  PNA_REQUIRE(grad_messages && activations && weight && grad_pre, PNA_ERR_BAD_ARG, "%s: null pointer", who);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long E = n_edges;
  const int P = msg_pitch;
  if (width <= 4) return launch_msg_bwd<4>(grid, grad_messages, P, activations, weight, E, n_layers, width, grad_pre, st);
  if (width <= 8) return launch_msg_bwd<8>(grid, grad_messages, P, activations, weight, E, n_layers, width, grad_pre, st);
  if (width <= 16) return launch_msg_bwd<16>(grid, grad_messages, P, activations, weight, E, n_layers, width, grad_pre, st);
  if (width <= 32) return launch_msg_bwd<32>(grid, grad_messages, P, activations, weight, E, n_layers, width, grad_pre, st);
  return launch_msg_bwd<64>(grid, grad_messages, P, activations, weight, E, n_layers, width, grad_pre, st);
}

}  // namespace pna

extern "C" int pna_edge_msg_fwd(const int32_t* rowptr, const int32_t* col, int64_t n_rows, int64_t n_edges, const float* a,
                                const float* b, const float* bias1, const float* edge_term, const float* weight, const float* bias,
                                int32_t n_layers, int32_t n_towers, int32_t width, int32_t msg_pitch, float* messages,
                                float* activations, pna_stream_t stream) {
  return edge_msg_fwd<float>("pna_edge_msg_fwd", rowptr, col, n_rows, n_edges, a, b, bias1, edge_term, weight, bias, n_layers,
                             n_towers, width, msg_pitch, messages, activations, stream);
}

extern "C" int pna_edge_msg_bwd(const float* grad_messages, int32_t msg_pitch, const float* activations, const float* weight,
                                int64_t n_edges, int32_t n_layers, int32_t n_towers, int32_t width, float* grad_pre,
                                pna_stream_t stream) {
  return edge_msg_bwd<float>("pna_edge_msg_bwd", grad_messages, msg_pitch, activations, weight, n_edges, n_layers, n_towers, width,
                             grad_pre, stream);
}

extern "C" int pna_edge_msg_fwd_bf16(const int32_t* rowptr, const int32_t* col, int64_t n_rows, int64_t n_edges, const void* a,
                                     const void* b, const float* bias1, const void* edge_term, const float* weight, const float* bias,
                                     int32_t n_layers, int32_t n_towers, int32_t width, int32_t msg_pitch, void* messages,
                                     void* activations, pna_stream_t stream) {
  typedef __nv_bfloat16 B;
  return edge_msg_fwd<B>("pna_edge_msg_fwd_bf16", rowptr, col, n_rows, n_edges, static_cast<const B*>(a), static_cast<const B*>(b),
                         bias1, static_cast<const B*>(edge_term), weight, bias, n_layers, n_towers, width, msg_pitch,
                         static_cast<B*>(messages), static_cast<B*>(activations), stream);
}

extern "C" int pna_edge_msg_bwd_bf16(const void* grad_messages, int32_t msg_pitch, const void* activations, const float* weight,
                                     int64_t n_edges, int32_t n_layers, int32_t n_towers, int32_t width, float* grad_pre,
                                     pna_stream_t stream) {
  typedef __nv_bfloat16 B;
  return edge_msg_bwd<B>("pna_edge_msg_bwd_bf16", static_cast<const B*>(grad_messages), msg_pitch, static_cast<const B*>(activations),
                         weight, n_edges, n_layers, n_towers, width, grad_pre, stream);
}
