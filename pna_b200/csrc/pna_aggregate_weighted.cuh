// The softmax / softmin / normalised_mean aggregators (reference models/pytorch/pna/aggregators.py:87-119), forward and
// backward.  All three are weighted sums of the row's messages.
//
// For destination row i with messages m_s (row_bias added when given), d = |In(i)|, and sigma = +1 (softmax) or -1
// (softmin); n_s = sigma * m_s (exact):
//   M   = max over slots of n_s                                   (exact, order-free)
//   e_s = expf(fl(n_s - M))                                       (full-precision expf, not __expf)
//   Z   = fp32 sum of e_s in slot order,  S = fp32 sum of fl(e_s * n_s) in slot order
//   y   = sigma * __fdiv_rn(S, Z)                                 d == 0: y = 0
// This is the reference's exp(m) / sum exp(m) shifted by the row maximum: equal in exact arithmetic, finite wherever y is
// (the reference gives inf / inf = NaN above m ~ 88.7).  normalised_mean:
//   r_k = D_k ? __frsqrt_rn(D_k) : 0,  D_k = rowptr[k+1] - rowptr[k] (the same CSR; D_j = 0 for j >= n_rows),
//   w_s = fl(r_i * r_j),  j = degree_col[s] when given (messages in CSR order), else col[s],
//   y = fp32 sum of fl(m_s * w_s) in slot order.
// y is scaled by the row's scaler factors and stored in its column slot like every other aggregator.  Gradient, with
// G = sum over the list positions of this aggregator and over the scalers of  scale * grad_out  (positions, then scalers,
// in order), y' = S / Z:
//   softmax / softmin:  a = __fdiv_rn(G, Z),  g_j = fl( fl(a * e_j) * fl(1 + fl(n_j - y')) )     (= G p_j (1 + n_j - y'))
//   normalised_mean:    g_j = fl(G * w_j)
//
// These kernels only ever write the columns of their own aggregator (the entry points run the existing kernels with
// these codes replaced by PNA_AGGR_SKIP, then the moment kernels, then these, one aggregator after the other in stream
// order so that each reuses the scratch).  The thread layout is the moment kernels' (pna_aggregate_moments.cuh): one
// thread per (row or chunk, feature column), 32 lanes on 32 consecutive columns, no shared memory, no shuffles, no
// barriers (tests run them on the host thread by thread).  Rows at/above the split threshold are done chunk by chunk in
// fixed order, with no atomics: softmax / softmin (1) per chunk the max, (2) per split row the max of the chunk maxima
// -> M (exact), (3) per chunk (Z, S) against M, (4) per split row their chunk-order merge -> y (forward: the epilogue;
// backward: the coefficients); normalised_mean (3) per chunk the sum, (4) their chunk-order merge.  Backward only:
// (5) per chunk the slot gradients and the chunk's share of grad_row_bias, (6) per split row those shares added in
// chunk order (k_mom_bwd_hub_bias).
//
// Scratch (pna_agg_t.hub_partials) stays inside the existing contracts.  Forward, 4 * n_feat floats per chunk c:
// [0] chunk max (1), or the chunk sum of normalised_mean (3); [1] of the row's FIRST chunk: M (2); [2] Z; [3] S.
// Backward, 6 * n_feat per chunk: [0] chunk max, [1] Z, [2] S, [5] grad_row_bias share; and 6 * n_feat per split row h
// at (n_chunks + h): [0] M, [1] a (normalised_mean: G), [2] y'.
#pragma once

namespace pna {

__host__ __device__ __forceinline__ bool weighted_code(unsigned code) {
  return code >= PNA_AGGR_SOFTMAX && code <= PNA_AGGR_NORMALISED_MEAN;
}

// bit (code - PNA_AGGR_SOFTMAX) set for every weighted aggregator in the list
inline unsigned weighted_codes(unsigned codes, int n_aggr) {
  unsigned m = 0;
  for (int a = 0; a < n_aggr; ++a) {
    const unsigned c = (codes >> (4 * a)) & 15u;
    if (weighted_code(c)) m |= 1u << (c - PNA_AGGR_SOFTMAX);
  }
  return m;
}

// the list with every code the add-on kernels write (moments, weighted sums) replaced by PNA_AGGR_SKIP: what the
// existing kernels run
inline unsigned strip_addons(unsigned codes, int n_aggr) {
  for (int a = 0; a < n_aggr; ++a) {
    const unsigned c = (codes >> (4 * a)) & 15u;
    if (moment_order(c) || weighted_code(c)) codes |= 15u << (4 * a);
  }
  return codes;
}

// D^(-1/2), correctly rounded.  The host build of these kernels (tests/emu, which has no CUDA intrinsics) rounds the
// double quotient once instead: the same float for every integer D below 2^22 (checked exhaustively).
__device__ __forceinline__ float wsum_rsqrt(float D) {
#ifdef __CUDA_ARCH__
  return __frsqrt_rn(D);
#else
  return (float)(1.0 / sqrt((double)D));
#endif
}

// r_k = D_k^(-1/2), correctly rounded; 0 for D_k == 0 and for k outside the CSR's rows
__device__ __forceinline__ float wsum_rsqrt_deg(const MParams& p, long long k) {
  if (k < 0 || k >= p.n_rows) return 0.f;
  const int D = __ldg(p.rowptr + k + 1) - __ldg(p.rowptr + k);
  return D > 0 ? wsum_rsqrt((float)D) : 0.f;
}

// the node whose degree weighs slot e: pna_agg_t.degree_col when given, else the slot's source
__device__ __forceinline__ long long wsum_degree_node(const MParams& p, int e) {
  return p.dcol ? __ldg(p.dcol + e) : __ldg(p.col + e);
}

__device__ __forceinline__ float wsum_sigma(unsigned code) { return code == PNA_AGGR_SOFTMIN ? -1.f : 1.f; }

// max over slots [beg, end) of sigma * m
template <typename T>
__device__ __forceinline__ float wsum_max(const MParams& p, int beg, int end, int f, float b, bool hb, float sigma) {
  float M = -INFINITY;
  for (int e = beg; e < end; ++e) M = fmaxf(M, sigma * mom_msg<T>(p, e, f, b, hb));
  return M;
}

struct WZS { float Z, S; };

// slot-order (Z, S) over slots [beg, end) against the row maximum M
template <typename T>
__device__ __forceinline__ WZS wsum_zs(const MParams& p, int beg, int end, int f, float b, bool hb, float sigma, float M) {
  WZS r = {0.f, 0.f};
  for (int e = beg; e < end; ++e) {
    const float n = sigma * mom_msg<T>(p, e, f, b, hb);
    const float ex = expf(__fsub_rn(n, M));
    r.Z = __fadd_rn(r.Z, ex);
    r.S = __fadd_rn(r.S, __fmul_rn(ex, n));
  }
  return r;
}

// slot-order sum of fl(m_s * w_s) over slots [beg, end) of row `row` (r_i = its D^(-1/2))
template <typename T>
__device__ __forceinline__ float wsum_nmean(const MParams& p, int beg, int end, int f, float b, bool hb, float ri) {
  float s = 0.f;
  for (int e = beg; e < end; ++e) {
    const float w = __fmul_rn(ri, wsum_rsqrt_deg(p, wsum_degree_node(p, e)));
    s = __fadd_rn(s, __fmul_rn(mom_msg<T>(p, e, f, b, hb), w));
  }
  return s;
}

// the epilogue: y of every list position holding `code`, for every scaler
template <typename T>
__device__ __forceinline__ void wsum_store(const MParams& p, long long row, int deg, int f, unsigned code, float y) {
  const DegScales ds = deg_scales(p.sdeg ? __ldg(p.sdeg + row) : deg, p.avg_log, p.avg_lin);
  const bool zero_all = deg == 0 && (p.flags & PNA_FLAG_ZERO_ISOLATED);
  T* orow = static_cast<T*>(p.out) + row * p.ldo + mom_base_col(p, f);
  for (int a = 0; a < p.nA; ++a) {
    if (((p.acodes >> (4 * a)) & 15u) != code) continue;
    for (int s = 0; s < p.nS; ++s) {
      const unsigned sc = (p.scodes >> (4 * s)) & 15u;
      float o[1] = {zero_all ? 0.f : (sc == PNA_SCALE_IDENTITY ? y : __fmul_rn(y, ds.of(sc)))};
      Io<T, 1>::store(orow + (s * p.nA + a) * p.Ft, o);
    }
  }
}

// ---- forward ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_wsum_rows(const MParams p, const unsigned code) {
  long long row; int f;
  if (!mom_thread(p, p.n_rows, row, f)) return;
  const int beg = __ldg(p.rowptr + row), end = __ldg(p.rowptr + row + 1), deg = end - beg;
  if (deg >= p.split) return;                             // split rows: the chunk kernels
  if (p.ldeg && __ldg(p.ldeg + row) < 0) return;          // not in the masked view
  float y = 0.f;
  if (deg > 0) {
    const bool hb = p.bias != nullptr;
    const float b = mom_bias<T>(p, row, f);
    if (code == PNA_AGGR_NORMALISED_MEAN) {
      y = wsum_nmean<T>(p, beg, end, f, b, hb, wsum_rsqrt((float)deg));
    } else {
      const float sigma = wsum_sigma(code);
      const WZS zs = wsum_zs<T>(p, beg, end, f, b, hb, sigma, wsum_max<T>(p, beg, end, f, b, hb, sigma));
      y = sigma * __fdiv_rn(zs.S, zs.Z);
    }
  }
  wsum_store<T>(p, row, deg, f, code, y);
}

// per chunk: the max of sigma * m into [0]
template <typename T, int W>
__global__ void __launch_bounds__(kMomThreads) k_wsum_chunk_max(const MParams p, const unsigned code) {
  long long c; int f;
  if (!mom_thread(p, p.n_chunks, c, f)) return;
  const MomChunk m = mom_chunk(p, c);
  *mom_part<W>(p, c, 0, f) = wsum_max<T>(p, m.beg, m.end, f, mom_bias<T>(p, m.row, f), p.bias != nullptr, wsum_sigma(code));
}

// per split row: the max of the chunk maxima -> M, forward into [1] of the row's first chunk, backward into [0] of the
// row's slot
template <int W>
__global__ void __launch_bounds__(kMomThreads) k_wsum_hub_max(const MParams p) {
  long long h; int f;
  if (!mom_thread(p, p.n_hubs, h, f)) return;
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2);
  float M = -INFINITY;
  for (int j = 0; j < nch; ++j) M = fmaxf(M, *mom_part<W>(p, first + j, 0, f));
  if (W == 4) *mom_part<W>(p, first, 1, f) = M;
  else *mom_part<W>(p, p.n_chunks + h, 0, f) = M;
}

// per chunk: (Z, S) against M (softmax / softmin), or the chunk sum (normalised_mean).  Forward: Z, S into [2], [3],
// the sum into [0]; backward: Z, S into [1], [2] (normalised_mean needs no chunk pass in the backward).
template <typename T, int W>
__global__ void __launch_bounds__(kMomThreads) k_wsum_chunk_zs(const MParams p, const unsigned code) {
  long long c; int f;
  if (!mom_thread(p, p.n_chunks, c, f)) return;
  const MomChunk m = mom_chunk(p, c);
  const bool hb = p.bias != nullptr;
  const float b = mom_bias<T>(p, m.row, f);
  if (code == PNA_AGGR_NORMALISED_MEAN) {
    *mom_part<W>(p, c, 0, f) = wsum_nmean<T>(p, m.beg, m.end, f, b, hb, wsum_rsqrt((float)__ldg(p.hub_info + 4 * m.h + 3)));
    return;
  }
  const float M = W == 4 ? *mom_part<W>(p, m.first, 1, f) : *mom_part<W>(p, p.n_chunks + m.h, 0, f);
  const WZS zs = wsum_zs<T>(p, m.beg, m.end, f, b, hb, wsum_sigma(code), M);
  *mom_part<W>(p, c, W == 4 ? 2 : 1, f) = zs.Z;
  *mom_part<W>(p, c, W == 4 ? 3 : 2, f) = zs.S;
}

// per split row: the chunk-order merge -> y, stored
template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_wsum_hub_final(const MParams p, const unsigned code) {
  long long h; int f;
  if (!mom_thread(p, p.n_hubs, h, f)) return;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2), deg = __ldg(p.hub_info + 4 * h + 3);
  float y;
  if (code == PNA_AGGR_NORMALISED_MEAN) {
    y = 0.f;
    for (int j = 0; j < nch; ++j) y = __fadd_rn(y, *mom_part<4>(p, first + j, 0, f));
  } else {
    float Z = 0.f, S = 0.f;
    for (int j = 0; j < nch; ++j) {
      Z = __fadd_rn(Z, *mom_part<4>(p, first + j, 2, f));
      S = __fadd_rn(S, *mom_part<4>(p, first + j, 3, f));
    }
    y = wsum_sigma(code) * __fdiv_rn(S, Z);
  }
  wsum_store<T>(p, row, deg, f, code, y);
}

// ---- backward --------------------------------------------------------------------------------------------------------
// G: the upstream gradient of y, summed over the list positions holding `code` and over the scalers
template <typename T>
__device__ __forceinline__ float wsum_upstream(const MParams& p, long long row, int deg, int f, unsigned code) {
  const DegScales ds = deg_scales(p.sdeg ? __ldg(p.sdeg + row) : deg, p.avg_log, p.avg_lin);
  const long long gbase = row * p.ldgo + mom_base_col(p, f);
  float G = 0.f;
  for (int a = 0; a < p.nA; ++a) {
    if (((p.acodes >> (4 * a)) & 15u) != code) continue;
    for (int s = 0; s < p.nS; ++s) {
      const unsigned sc = (p.scodes >> (4 * s)) & 15u;
      const float go = mom_load<T>(p.go, gbase + (s * p.nA + a) * p.Ft);
      G = __fadd_rn(G, sc == PNA_SCALE_IDENTITY ? go : __fmul_rn(ds.of(sc), go));
    }
  }
  return G;
}

// per-row coefficients of the slot gradients: (M, a, y') for softmax / softmin, (-, G, -) with the row's r_i for
// normalised_mean
struct WCoef { float M, a, y, ri; };

// add the term of every slot in [beg, end) to its gradient; returns the slot-order sum (grad_row_bias share).
// SLOTS: grad_slots[slot] += g (plain load-add-store; this thread owns the element).  Otherwise grad_gathered[col[slot]]
// gets an atomic add, or with col == NULL (per-slot rows) a plain add.
template <typename T, bool SLOTS>
__device__ __forceinline__ float wsum_emit(const MParams& p, int beg, int end, int f, float b, bool hb, unsigned code,
                                           const WCoef& c) {
  const float sigma = wsum_sigma(code);
  float acc = 0.f;
  for (int e = beg; e < end; ++e) {
    float g;
    if (code == PNA_AGGR_NORMALISED_MEAN) {
      g = __fmul_rn(c.a, __fmul_rn(c.ri, wsum_rsqrt_deg(p, wsum_degree_node(p, e))));
    } else {
      const float n = sigma * mom_msg<T>(p, e, f, b, hb);
      const float ex = expf(__fsub_rn(n, c.M));
      g = __fmul_rn(__fmul_rn(c.a, ex), __fadd_rn(1.f, __fsub_rn(n, c.y)));
    }
    acc = __fadd_rn(acc, g);
    if constexpr (SLOTS) {
      float* dst = p.gs + (long long)e * p.ldgs + (f - p.f0);
      *dst = __fadd_rn(*dst, g);
    } else {
      if (p.col) {
        atomicAdd(p.gg + (long long)__ldg(p.col + e) * p.ldgg + f, g);
      } else {
        float* dst = p.gg + (long long)e * p.ldgg + f;
        *dst = __fadd_rn(*dst, g);
      }
    }
  }
  return acc;
}

template <typename T, bool SLOTS>
__global__ void __launch_bounds__(kMomThreads) k_wsum_bwd_rows(const MParams p, const unsigned code) {
  long long row; int f;
  if (!mom_thread(p, p.n_rows, row, f)) return;
  const int beg = __ldg(p.rowptr + row), end = __ldg(p.rowptr + row + 1), deg = end - beg;
  if (deg == 0 || deg >= p.split) return;
  const bool hb = p.bias != nullptr;
  const float b = mom_bias<T>(p, row, f);
  const float G = wsum_upstream<T>(p, row, deg, f, code);
  WCoef c = {0.f, G, 0.f, 0.f};
  if (code == PNA_AGGR_NORMALISED_MEAN) {
    c.ri = wsum_rsqrt((float)deg);
  } else {
    const float sigma = wsum_sigma(code);
    c.M = wsum_max<T>(p, beg, end, f, b, hb, sigma);
    const WZS zs = wsum_zs<T>(p, beg, end, f, b, hb, sigma, c.M);
    c.y = __fdiv_rn(zs.S, zs.Z);
    c.a = __fdiv_rn(G, zs.Z);
  }
  const float gbs = wsum_emit<T, SLOTS>(p, beg, end, f, b, hb, code, c);
  if (p.gb) {
    float* dst = p.gb + row * p.ldgb + f;
    *dst = __fadd_rn(*dst, gbs);
  }
}

// per split row: (Z, S) merged in chunk order -> a = G / Z and y' (softmax / softmin), or a = G (normalised_mean)
template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_wsum_bwd_hub_coef(const MParams p, const unsigned code) {
  long long h; int f;
  if (!mom_thread(p, p.n_hubs, h, f)) return;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2), deg = __ldg(p.hub_info + 4 * h + 3);
  const float G = wsum_upstream<T>(p, row, deg, f, code);
  const long long hs = p.n_chunks + h;
  if (code == PNA_AGGR_NORMALISED_MEAN) {
    *mom_part<6>(p, hs, 1, f) = G;
    return;
  }
  float Z = 0.f, S = 0.f;
  for (int j = 0; j < nch; ++j) {
    Z = __fadd_rn(Z, *mom_part<6>(p, first + j, 1, f));
    S = __fadd_rn(S, *mom_part<6>(p, first + j, 2, f));
  }
  *mom_part<6>(p, hs, 1, f) = __fdiv_rn(G, Z);
  *mom_part<6>(p, hs, 2, f) = __fdiv_rn(S, Z);
}

template <typename T, bool SLOTS>
__global__ void __launch_bounds__(kMomThreads) k_wsum_bwd_chunk_grad(const MParams p, const unsigned code) {
  long long c; int f;
  if (!mom_thread(p, p.n_chunks, c, f)) return;
  const MomChunk m = mom_chunk(p, c);
  const long long hs = p.n_chunks + m.h;
  WCoef cf;
  cf.a = *mom_part<6>(p, hs, 1, f);
  if (code == PNA_AGGR_NORMALISED_MEAN) {
    cf.M = cf.y = 0.f;
    cf.ri = wsum_rsqrt((float)__ldg(p.hub_info + 4 * m.h + 3));
  } else {
    cf.M = *mom_part<6>(p, hs, 0, f);
    cf.y = *mom_part<6>(p, hs, 2, f);
    cf.ri = 0.f;
  }
  *mom_part<6>(p, c, 5, f) = wsum_emit<T, SLOTS>(p, m.beg, m.end, f, mom_bias<T>(p, m.row, f), p.bias != nullptr, code, cf);
}

}  // namespace pna
