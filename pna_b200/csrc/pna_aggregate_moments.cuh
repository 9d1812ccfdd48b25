// The moment3 / moment4 / moment5 aggregators (reference models/pytorch/pna/aggregators.py:122-146), forward and backward.
//
// For destination row i with messages m_s (row_bias added when given), d = |In(i)| and k in {3, 4, 5}:
//   mu    = fp32 sum of m_s in slot order, divided by d (mom_div: the correctly rounded quotient)
//   delta = fl(m_s - mu);  delta^2 = fl(delta * delta), delta^(j+1) = fl(delta^j * delta)   (one rounding per product)
//   M_k   = (fp32 sum of delta^k in slot order) / d          (correctly rounded)
//   r_k   = sign(M_k) * (|M_k| + 1e-5)^(1/k)                 (powf, exponent 1/k rounded to fp32);  d == 0: r_k = 0
// r_k is scaled by the row's scaler factors and stored in its column slot like every other aggregator.  Gradient:
//   dr_k/dm_j = rho_k * (k/d) * (delta_j^(k-1) - C_(k-1)),   C_(k-1) = (1/d) sum_s delta_s^(k-1),
//   rho_k     = (1/k) * (|M_k| + 1e-5)^(1/k - 1)  (0 where M_k == 0: the autograd of sign * pow in the reference).
// With G_k = sum over the list positions of moment k and over the scalers of  scale * grad_out  (positions, then scalers,
// in order) the per-row coefficients are  a_k = fl(fl(G_k * rho_k) * fl(k / d))  and  c0 = a_3 C_2 + a_4 C_3 + a_5 C_4
// (left to right, requested k only), and the gradient of slot j is
//   g_j = fl( fl(a_3 delta_j^2) + fl(a_4 delta_j^3) + fl(a_5 delta_j^4) ) - c0        (requested k only, left to right).
//
// These kernels only ever write the moment columns (the entry points run the existing kernels with the moment codes
// replaced by PNA_AGGR_SKIP, then these).  One thread per (row or chunk, feature column): 32 lanes of a warp cover 32
// consecutive columns of one row, so every gathered row is read coalesced; no shared memory, no shuffles, no barriers
// (tests run them on the host thread by thread).  Rows at/above the split threshold are done chunk by chunk in fixed
// order, with no atomics: (1) per chunk the slot-order sum, (2) per split row the chunk sums in chunk order -> mu,
// (3) per chunk the central sums, (4) per split row their chunk-order merge -> M_k (forward: the epilogue; backward: the
// coefficients), backward only: (5) per chunk the slot gradients and the chunk's share of grad_row_bias, (6) per split
// row those shares added in chunk order.
//
// Scratch (pna_agg_t.hub_partials) stays inside the existing contracts.  Forward, 4 * n_feat floats per chunk c:
// [0] chunk sum (1), later the delta^3 sum (3); [1] of the row's FIRST chunk: mu (2); [2] delta^4 sum; [3] delta^5 sum.
// Backward, 6 * n_feat per chunk: [0] chunk sum, [1..4] delta^2..delta^5 sums, [5] grad_row_bias share; and 6 * n_feat
// per split row h at (n_chunks + h): [0] mu, [1..3] a_3, a_4, a_5, [4] c0.
#pragma once
#include <string.h>

namespace pna {

// aggregator code -> moment order (0 = not a moment)
__host__ __device__ __forceinline__ int moment_order(unsigned code) {
  return (code >= PNA_AGGR_MOMENT3 && code <= PNA_AGGR_MOMENT5) ? (int)(code - PNA_AGGR_MOMENT3) + 3 : 0;
}

// bit k-3 set for every moment order k in the list
inline unsigned moment_orders(unsigned codes, int n_aggr) {
  unsigned m = 0;
  for (int a = 0; a < n_aggr; ++a) {
    const int k = moment_order((codes >> (4 * a)) & 15u);
    if (k) m |= 1u << (k - 3);
  }
  return m;
}

struct MParams {
  const void* x; long long ldx;
  const int* rowptr; const int* col;
  const void* bias; long long ldb;
  void* out; long long ldo;
  long long n_rows;
  int F, Ft, Wt, has_self, nA, nS;
  unsigned acodes, scodes, orders;    // orders: moment_orders()
  float avg_log, avg_lin;
  unsigned flags;
  int split, chunk;
  const int* hub_info; const int* chunk_items; long long n_hubs, n_chunks;
  float* partials;
  const int* ldeg;                    // masked light view in row order (-1 = row not selected), or NULL
  const int* sdeg;                    // degree seen by the scalers, or NULL
  // backward
  const void* go; long long ldgo;     // grad_out (layout of out)
  float* gg; long long ldgg;          // atomic mode: grad_gathered (per-slot rows when col == NULL)
  float* gs; long long ldgs;          // deterministic mode: grad_slots [E, f1 - f0]
  float* gb; long long ldgb;          // grad_row_bias, nullable
  int f0, f1;                         // feature columns handled by this call
  const int* dcol;                    // normalised_mean: the node whose degree weighs each slot (pna_agg_t.degree_col), or NULL
};

inline MParams moment_params(const pna_agg_t* d) {
  MParams p;
  memset(&p, 0, sizeof(p));
  p.x = d->gathered; p.ldx = d->ld_gathered;
  p.rowptr = d->rowptr; p.col = d->col;
  p.bias = d->row_bias; p.ldb = d->ld_row_bias;
  p.out = d->out; p.ldo = d->ld_out;
  p.n_rows = d->n_rows;
  p.F = d->n_feat; p.Ft = d->n_feat / d->n_towers;
  p.has_self = d->self_feat ? 1 : 0;
  p.nA = d->n_aggr; p.nS = d->n_scalers; p.acodes = d->aggr_codes; p.scodes = d->scaler_codes;
  p.orders = moment_orders(d->aggr_codes, d->n_aggr);
  p.Wt = (p.has_self + p.nA * p.nS) * p.Ft;
  p.avg_log = d->avg_log; p.avg_lin = d->avg_lin;
  p.flags = d->flags; p.split = d->split_threshold; p.chunk = d->chunk_edges;
  p.hub_info = d->hub_info; p.chunk_items = d->chunk_items; p.n_hubs = d->n_hubs; p.n_chunks = d->n_chunks;
  p.partials = d->hub_partials;
  // the row selection of pna_aggregate_fwd's light kernels: a usable view that lists the real rows in order (no chunk
  // pseudo-rows) skips the rows whose light_deg is -1
  const bool view = d->light_rowptr && d->light_deg && d->part && d->n_part >= 1 && (d->light_col || !d->col);
  p.ldeg = (view && d->n_view_rows <= d->n_rows) ? d->light_deg : nullptr;
  p.sdeg = d->scaler_degree;
  p.f0 = 0; p.f1 = d->n_feat;
  p.dcol = d->degree_col;
  return p;
}

constexpr int kMomThreads = 256;      // 8 warps: 8 rows (or chunks) x 32 feature columns per CTA

template <typename T>
__device__ __forceinline__ float mom_load(const void* base, long long idx) {
  float v[1];
  Io<T, 1>::load(static_cast<const T*>(base) + idx, v);
  return v[0];
}

// message of slot s at feature f
template <typename T>
__device__ __forceinline__ float mom_msg(const MParams& p, int s, int f, float b, bool has_bias) {
  const int src = p.col ? __ldg(p.col + s) : s;
  const float m = mom_load<T>(p.x, (long long)src * p.ldx + f);
  return has_bias ? __fadd_rn(m, b) : m;
}

template <typename T>
__device__ __forceinline__ float mom_sum(const MParams& p, int beg, int end, int f, float b, bool has_bias) {
  float s = 0.f;
  for (int e = beg; e < end; ++e) s = __fadd_rn(s, mom_msg<T>(p, e, f, b, has_bias));
  return s;
}

// delta^2 .. delta^5 of one message, one rounding per product
struct Pow4 { float q[4]; };
__device__ __forceinline__ Pow4 central_powers(float delta) {
  Pow4 r;
  r.q[0] = __fmul_rn(delta, delta);
  r.q[1] = __fmul_rn(r.q[0], delta);
  r.q[2] = __fmul_rn(r.q[1], delta);
  r.q[3] = __fmul_rn(r.q[2], delta);
  return r;
}

// slot-order sums of delta^2 .. delta^5 over slots [beg, end)
template <typename T>
__device__ __forceinline__ Pow4 mom_central(const MParams& p, int beg, int end, int f, float b, bool has_bias, float mu) {
  Pow4 acc;
#pragma unroll
  for (int j = 0; j < 4; ++j) acc.q[j] = 0.f;
  for (int e = beg; e < end; ++e) {
    const Pow4 w = central_powers(__fsub_rn(mom_msg<T>(p, e, f, b, has_bias), mu));
#pragma unroll
    for (int j = 0; j < 4; ++j) acc.q[j] = __fadd_rn(acc.q[j], w.q[j]);
  }
  return acc;
}

// x / d correctly rounded (IEEE division).  Not SharedDivisor: its reciprocal-and-correction sequence gives NaN for an
// infinite numerator (a sum of overflowed powers, inf - inf in the correction) and may miss a subnormal quotient by one
// ulp; these kernels divide a handful of times per row, so the full division costs nothing measurable.
__device__ __forceinline__ float mom_div(float x, int d) { return __fdiv_rn(x, (float)d); }

__device__ __forceinline__ float moment_inv(int k) { return k == 3 ? (1.0f / 3.0f) : k == 4 ? 0.25f : 0.2f; }

// sign(M) * (|M| + 1e-5)^(1/k); 0 (and NaN) pass through
__device__ __forceinline__ float moment_root(float M, int k) {
  if (!(M > 0.f) && !(M < 0.f)) return M;
  const float r = powf(__fadd_rn(fabsf(M), 1e-5f), moment_inv(k));
  return M > 0.f ? r : -r;
}

// d r_k / d M_k
__device__ __forceinline__ float moment_slope(float M, int k) {
  if (!(M > 0.f) && !(M < 0.f)) return M == 0.f ? 0.f : M;
  const float e = k == 3 ? (1.0f / 3.0f - 1.0f) : k == 4 ? -0.75f : -0.8f;
  return __fmul_rn(moment_inv(k), powf(__fadd_rn(fabsf(M), 1e-5f), e));
}

// column of feature f for (scaler 0, aggregator 0) in the output row
__device__ __forceinline__ long long mom_base_col(const MParams& p, int f) {
  const int t = f / p.Ft, ft = f - t * p.Ft;
  return (long long)t * p.Wt + p.has_self * p.Ft + ft;
}

// the epilogue: r_k of every moment position for every scaler.  M[k-3] = M_k (ignored when deg == 0)
template <typename T>
__device__ __forceinline__ void mom_store(const MParams& p, long long row, int deg, int f, const float (&M)[3]) {
  const DegScales ds = deg_scales(p.sdeg ? __ldg(p.sdeg + row) : deg, p.avg_log, p.avg_lin);
  const bool zero_all = deg == 0 && (p.flags & PNA_FLAG_ZERO_ISOLATED);
  T* orow = static_cast<T*>(p.out) + row * p.ldo + mom_base_col(p, f);
  for (int a = 0; a < p.nA; ++a) {
    const int k = moment_order((p.acodes >> (4 * a)) & 15u);
    if (!k) continue;
    const float r = deg == 0 ? 0.f : moment_root(M[k - 3], k);
    for (int s = 0; s < p.nS; ++s) {
      const unsigned sc = (p.scodes >> (4 * s)) & 15u;
      float o[1] = {zero_all ? 0.f : (sc == PNA_SCALE_IDENTITY ? r : __fmul_rn(r, ds.of(sc)))};
      Io<T, 1>::store(orow + (s * p.nA + a) * p.Ft, o);
    }
  }
}

// thread -> (item, feature column); false when out of range
__device__ __forceinline__ bool mom_thread(const MParams& p, long long n_items, long long& item, int& f) {
  item = (long long)blockIdx.x * (kMomThreads / 32) + (threadIdx.x >> 5);
  f = p.f0 + (int)blockIdx.y * 32 + (int)(threadIdx.x & 31);
  return item < n_items && f < p.f1;
}

template <typename T>
__device__ __forceinline__ float mom_bias(const MParams& p, long long row, int f) {
  return p.bias ? mom_load<T>(p.bias, row * p.ldb + f) : 0.f;
}

// ---- forward ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_mom_rows(const MParams p) {
  long long row; int f;
  if (!mom_thread(p, p.n_rows, row, f)) return;
  const int beg = __ldg(p.rowptr + row), end = __ldg(p.rowptr + row + 1), deg = end - beg;
  if (deg >= p.split) return;                             // split rows: the chunk kernels
  if (p.ldeg && __ldg(p.ldeg + row) < 0) return;          // not in the masked view
  float M[3] = {0.f, 0.f, 0.f};
  if (deg > 0) {
    const bool hb = p.bias != nullptr;
    const float b = mom_bias<T>(p, row, f);
    const float mu = mom_div(mom_sum<T>(p, beg, end, f, b, hb), deg);
    const Pow4 c = mom_central<T>(p, beg, end, f, b, hb, mu);
#pragma unroll
    for (int j = 0; j < 3; ++j) M[j] = mom_div(c.q[j + 1], deg);
  }
  mom_store<T>(p, row, deg, f, M);
}

// chunk c of split row h: (h, row, slot range)
struct MomChunk { int h, first; long long row; int beg, end; };
__device__ __forceinline__ MomChunk mom_chunk(const MParams& p, long long c) {
  MomChunk m;
  m.h = __ldg(p.chunk_items + 2 * c);
  const int j = __ldg(p.chunk_items + 2 * c + 1);
  m.row = __ldg(p.hub_info + 4 * m.h);
  m.first = __ldg(p.hub_info + 4 * m.h + 1);
  const int rbeg = __ldg(p.rowptr + m.row), rend = __ldg(p.rowptr + m.row + 1);
  m.beg = rbeg + j * p.chunk;
  m.end = min(m.beg + p.chunk, rend);
  return m;
}

// scratch slot j of chunk c (W floats per feature row: 4 forward, 6 backward)
template <int W>
__device__ __forceinline__ float* mom_part(const MParams& p, long long c, int j, int f) {
  return p.partials + (c * W + j) * (long long)p.F + f;
}

template <typename T, int W>
__global__ void __launch_bounds__(kMomThreads) k_mom_chunk_sum(const MParams p) {
  long long c; int f;
  if (!mom_thread(p, p.n_chunks, c, f)) return;
  const MomChunk m = mom_chunk(p, c);
  *mom_part<W>(p, c, 0, f) = mom_sum<T>(p, m.beg, m.end, f, mom_bias<T>(p, m.row, f), p.bias != nullptr);
}

// chunk sums in chunk order -> mu: forward into [1] of the row's first chunk, backward into [0] of the row's slot
template <int W>
__global__ void __launch_bounds__(kMomThreads) k_mom_hub_mean(const MParams p) {
  long long h; int f;
  if (!mom_thread(p, p.n_hubs, h, f)) return;
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2), deg = __ldg(p.hub_info + 4 * h + 3);
  float s = 0.f;
  for (int j = 0; j < nch; ++j) s = __fadd_rn(s, *mom_part<W>(p, first + j, 0, f));
  const float mu = mom_div(s, deg);
  if (W == 4) *mom_part<W>(p, first, 1, f) = mu;
  else *mom_part<W>(p, p.n_chunks + h, 0, f) = mu;
}

template <int W>
__device__ __forceinline__ float mom_hub_mu(const MParams& p, const MomChunk& m, int f) {
  return W == 4 ? *mom_part<W>(p, m.first, 1, f) : *mom_part<W>(p, p.n_chunks + m.h, 0, f);
}

template <typename T, int W>
__global__ void __launch_bounds__(kMomThreads) k_mom_chunk_central(const MParams p) {
  long long c; int f;
  if (!mom_thread(p, p.n_chunks, c, f)) return;
  const MomChunk m = mom_chunk(p, c);
  const Pow4 q = mom_central<T>(p, m.beg, m.end, f, mom_bias<T>(p, m.row, f), p.bias != nullptr, mom_hub_mu<W>(p, m, f));
  if (W == 4) {        // [1] of the first chunk holds mu: delta^3, ^4, ^5 sums go to [0], [2], [3]
    *mom_part<W>(p, c, 0, f) = q.q[1]; *mom_part<W>(p, c, 2, f) = q.q[2]; *mom_part<W>(p, c, 3, f) = q.q[3];
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) *mom_part<W>(p, c, 1 + j, f) = q.q[j];
  }
}

template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_mom_hub_final(const MParams p) {
  long long h; int f;
  if (!mom_thread(p, p.n_hubs, h, f)) return;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2), deg = __ldg(p.hub_info + 4 * h + 3);
  float s3 = 0.f, s4 = 0.f, s5 = 0.f;
  for (int j = 0; j < nch; ++j) {
    s3 = __fadd_rn(s3, *mom_part<4>(p, first + j, 0, f));
    s4 = __fadd_rn(s4, *mom_part<4>(p, first + j, 2, f));
    s5 = __fadd_rn(s5, *mom_part<4>(p, first + j, 3, f));
  }
  const float M[3] = {mom_div(s3, deg), mom_div(s4, deg), mom_div(s5, deg)};
  mom_store<T>(p, row, deg, f, M);
}

// ---- backward --------------------------------------------------------------------------------------------------------
struct MomCoef { float a3, a4, a5, c0; };

// upstream gradient of the row's moment columns + the central sums (P.q = sums of delta^2..delta^5) -> coefficients
template <typename T>
__device__ __forceinline__ MomCoef mom_coef(const MParams& p, long long row, int deg, int f, const Pow4& P) {
  const DegScales ds = deg_scales(p.sdeg ? __ldg(p.sdeg + row) : deg, p.avg_log, p.avg_lin);
  const long long gbase = row * p.ldgo + mom_base_col(p, f);
  float G[3] = {0.f, 0.f, 0.f};
  for (int a = 0; a < p.nA; ++a) {
    const int k = moment_order((p.acodes >> (4 * a)) & 15u);
    if (!k) continue;
    for (int s = 0; s < p.nS; ++s) {
      const unsigned sc = (p.scodes >> (4 * s)) & 15u;
      const float go = mom_load<T>(p.go, gbase + (s * p.nA + a) * p.Ft);
      G[k - 3] = __fadd_rn(G[k - 3], sc == PNA_SCALE_IDENTITY ? go : __fmul_rn(ds.of(sc), go));
    }
  }
  float a[3], C[3];
  for (int i = 0; i < 3; ++i) {
    const int k = i + 3;
    C[i] = mom_div(P.q[i], deg);                           // C_(k-1)
    a[i] = (p.orders >> i) & 1u ? __fmul_rn(__fmul_rn(G[i], moment_slope(mom_div(P.q[i + 1], deg), k)), mom_div((float)k, deg)) : 0.f;
  }
  MomCoef c;
  c.a3 = a[0]; c.a4 = a[1]; c.a5 = a[2];
  c.c0 = 0.f;
  for (int i = 0; i < 3; ++i)
    if ((p.orders >> i) & 1u) c.c0 = __fadd_rn(c.c0, __fmul_rn(a[i], C[i]));
  return c;
}

__device__ __forceinline__ float mom_slot_grad(const MParams& p, const MomCoef& c, float delta) {
  const Pow4 w = central_powers(delta);
  float g = 0.f;
  if (p.orders & 1u) g = __fadd_rn(g, __fmul_rn(c.a3, w.q[0]));
  if (p.orders & 2u) g = __fadd_rn(g, __fmul_rn(c.a4, w.q[1]));
  if (p.orders & 4u) g = __fadd_rn(g, __fmul_rn(c.a5, w.q[2]));
  return __fsub_rn(g, c.c0);
}

// add the moment term of every slot in [beg, end) to its gradient; returns the slot-order sum (grad_row_bias share).
// SLOTS: grad_slots[slot] += g (plain load-add-store; this thread owns the element).  Otherwise grad_gathered[col[slot]]
// gets an atomic add, or with col == NULL (per-slot rows) a plain add.
template <typename T, bool SLOTS>
__device__ __forceinline__ float mom_emit(const MParams& p, int beg, int end, int f, float b, bool has_bias, float mu,
                                          const MomCoef& c) {
  float acc = 0.f;
  for (int e = beg; e < end; ++e) {
    const float g = mom_slot_grad(p, c, __fsub_rn(mom_msg<T>(p, e, f, b, has_bias), mu));
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
__global__ void __launch_bounds__(kMomThreads) k_mom_bwd_rows(const MParams p) {
  long long row; int f;
  if (!mom_thread(p, p.n_rows, row, f)) return;
  const int beg = __ldg(p.rowptr + row), end = __ldg(p.rowptr + row + 1), deg = end - beg;
  if (deg == 0 || deg >= p.split) return;
  const bool hb = p.bias != nullptr;
  const float b = mom_bias<T>(p, row, f);
  const float mu = mom_div(mom_sum<T>(p, beg, end, f, b, hb), deg);
  const MomCoef c = mom_coef<T>(p, row, deg, f, mom_central<T>(p, beg, end, f, b, hb, mu));
  const float gbs = mom_emit<T, SLOTS>(p, beg, end, f, b, hb, mu, c);
  if (p.gb) {
    float* dst = p.gb + row * p.ldgb + f;
    *dst = __fadd_rn(*dst, gbs);
  }
}

template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_mom_bwd_hub_coef(const MParams p) {
  long long h; int f;
  if (!mom_thread(p, p.n_hubs, h, f)) return;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2), deg = __ldg(p.hub_info + 4 * h + 3);
  Pow4 P;
#pragma unroll
  for (int j = 0; j < 4; ++j) P.q[j] = 0.f;
  for (int i = 0; i < nch; ++i) {
#pragma unroll
    for (int j = 0; j < 4; ++j) P.q[j] = __fadd_rn(P.q[j], *mom_part<6>(p, first + i, 1 + j, f));
  }
  const MomCoef c = mom_coef<T>(p, row, deg, f, P);
  const long long hs = p.n_chunks + h;
  *mom_part<6>(p, hs, 1, f) = c.a3; *mom_part<6>(p, hs, 2, f) = c.a4; *mom_part<6>(p, hs, 3, f) = c.a5;
  *mom_part<6>(p, hs, 4, f) = c.c0;
}

template <typename T, bool SLOTS>
__global__ void __launch_bounds__(kMomThreads) k_mom_bwd_chunk_grad(const MParams p) {
  long long c; int f;
  if (!mom_thread(p, p.n_chunks, c, f)) return;
  const MomChunk m = mom_chunk(p, c);
  const long long hs = p.n_chunks + m.h;
  MomCoef cf;
  cf.a3 = *mom_part<6>(p, hs, 1, f); cf.a4 = *mom_part<6>(p, hs, 2, f); cf.a5 = *mom_part<6>(p, hs, 3, f);
  cf.c0 = *mom_part<6>(p, hs, 4, f);
  const float share = mom_emit<T, SLOTS>(p, m.beg, m.end, f, mom_bias<T>(p, m.row, f), p.bias != nullptr,
                                         *mom_part<6>(p, hs, 0, f), cf);
  *mom_part<6>(p, c, 5, f) = share;
}

// grad_row_bias of a split row += the chunks' shares, added in chunk order (W = 6; a template so that every translation
// unit including this header may instantiate it)
template <int W>
__global__ void __launch_bounds__(kMomThreads) k_mom_bwd_hub_bias(const MParams p) {
  long long h; int f;
  if (!mom_thread(p, p.n_hubs, h, f)) return;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2);
  float acc = 0.f;
  for (int j = 0; j < nch; ++j) acc = __fadd_rn(acc, *mom_part<W>(p, first + j, 5, f));
  float* dst = p.gb + row * p.ldgb + f;
  *dst = __fadd_rn(*dst, acc);
}

}  // namespace pna
