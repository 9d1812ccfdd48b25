// Slot-weighted aggregation (pna_aggregate_fwd_weighted / _bwd_weighted / _bwd_slots_weighted: slot_weight and
// scaler_degree_f): sum / mean / min / max / var / std over a real-valued adjacency, as the dense reference computes them (models/pytorch/pna/aggregators.py:17-84, scalers.py:8-38).  Forward here,
// backward in pna_aggregate_bwd.cu (it reuses that file's coefficients and message_grad).
//
// For destination row i with slots s, message m_s (row_bias added when given) and weight w_s (1 where slot_weight is NULL):
//   W_i = fp32 sum of w_s in slot order (every row, split rows included)
//   S   = fp32 sum of fl(m_s * w_s) in slot order,  Q = fp32 sum of fl(fl(m_s * m_s) * w_s) in slot order
//   sum = S;  mean = __fdiv_rn(S, W_i);  var = fl(__fdiv_rn(Q, W_i) - fl(mean * mean))  (clamped at 0 with RELU_VAR)
//   std = __fsqrt_rn(fl(max(var, 0) + 1e-5))
//   min / max over the slots with w_s > 0 of the unweighted m_s (the reference's adj > 0 mask); 0 when there is none
// A row without slots is written as the existing kernels write it (0, std = sqrt(1e-5), all 0 with ZERO_ISOLATED).  The
// scalers see D = scaler_degree_f[i], else scaler_degree[i], else the slot count, through deg_scales_f.  With every w_s = 1
// these are the unweighted kernels' values bit for bit on rows below the split threshold (fl(m * 1) = m, W_i = d exactly,
// and SharedDivisor is the correctly rounded quotient there).
//
// Thread layout of the moment kernels (pna_aggregate_moments.cuh): one thread per (row or chunk, feature column), no shared
// memory, no shuffles, no barriers, no atomics.  Split rows: (1) per chunk S, Q, min, max into hub_partials [0..3] (4 * n_feat
// floats per chunk, the forward's contract), (2) per split row the chunk partials merged in chunk order, W_i over the row's
// slots in slot order, the epilogue.  These kernels write every column of the call (self block included); the existing
// kernels do not run for a weighted call.
#pragma once

namespace pna {

// the aggregators a weighted call takes (and PNA_AGGR_SKIP)
__host__ __device__ __forceinline__ bool adj_weight_code(unsigned code) {
  return code <= PNA_AGGR_STD || code == PNA_AGGR_SKIP;
}

struct AWParams {
  MParams m;
  const float* w;                     // slot weights, or NULL (all 1)
  const float* sdf;                   // real-valued scaler degree, or NULL
  const void* self; long long lds, self_tstride;
};

inline AWParams adj_weight_params(const pna_agg_t* d, const float* slot_weight, const float* scaler_degree_f) {
  AWParams a;
  a.m = moment_params(d);
  a.w = slot_weight; a.sdf = scaler_degree_f;
  a.self = d->self_feat; a.lds = d->ld_self; a.self_tstride = d->self_tower_stride;
  return a;
}

__device__ __forceinline__ float aw_weight(const float* w, int e) { return w ? __ldg(w + e) : 1.0f; }

// W_i: the row's weights summed in slot order
__device__ __forceinline__ float aw_weight_sum(const float* w, int beg, int end) {
  if (!w) return (float)(end - beg);
  float W = 0.f;
  for (int e = beg; e < end; ++e) W = __fadd_rn(W, __ldg(w + e));
  return W;
}

// the scalers' degree of a row
__device__ __forceinline__ float aw_scaler_degree(const MParams& p, const float* sdf, long long row, int deg) {
  return sdf ? __ldg(sdf + row) : (float)(p.sdeg ? __ldg(p.sdeg + row) : deg);
}

struct AwSums { float S, Q, mn, mx; };

// slot-order S and Q over slots [beg, end), min / max over the positive-weight slots (+inf / -inf when there is none)
template <typename T>
__device__ __forceinline__ AwSums aw_sums(const MParams& p, const float* w, int beg, int end, int f, float b, bool hb) {
  AwSums r = {0.f, 0.f, INFINITY, -INFINITY};
  for (int e = beg; e < end; ++e) {
    const float m = mom_msg<T>(p, e, f, b, hb), ws = aw_weight(w, e);
    r.S = __fadd_rn(r.S, __fmul_rn(m, ws));
    r.Q = __fadd_rn(r.Q, __fmul_rn(__fmul_rn(m, m), ws));
    if (ws > 0.f) { r.mn = fminf(r.mn, m); r.mx = fmaxf(r.mx, m); }
  }
  return r;
}

// self block of this thread's column (the existing kernels' plain copy)
template <typename T>
__device__ __forceinline__ void aw_copy_self(const AWParams& a, long long row, int f) {
  if (!a.self) return;
  const MParams& p = a.m;
  const int t = f / p.Ft, ft = f - t * p.Ft;
  float v[1];
  Io<T, 1>::load(static_cast<const T*>(a.self) + row * a.lds + t * a.self_tstride + ft, v);
  Io<T, 1>::store(static_cast<T*>(p.out) + row * p.ldo + (long long)t * p.Wt + ft, v);
}

// the epilogue: every (scaler, aggregator) column of the row at feature f
template <typename T>
__device__ __forceinline__ void aw_store(const AWParams& a, long long row, int deg, int f, float W, const AwSums& r) {
  const MParams& p = a.m;
  const DegScales ds = deg_scales_f(aw_scaler_degree(p, a.sdf, row, deg), p.avg_log, p.avg_lin);
  const bool iso = deg == 0;
  const bool zero_all = iso && (p.flags & PNA_FLAG_ZERO_ISOLATED);
  float mean = 0.f, var = 0.f, mn = 0.f, mx = 0.f;
  if (!iso) {
    mean = __fdiv_rn(r.S, W);
    var = __fsub_rn(__fdiv_rn(r.Q, W), __fmul_rn(mean, mean));
    if (!(r.mx < r.mn)) { mn = r.mn; mx = r.mx; }       // some slot has a positive weight
  }
  const float sd = __fsqrt_rn(__fadd_rn(fmaxf(var, 0.0f), 1e-5f));
  T* orow = static_cast<T*>(p.out) + row * p.ldo + mom_base_col(p, f);
  for (int k = 0; k < p.nA; ++k) {
    const unsigned ac = (p.acodes >> (4 * k)) & 15u;
    if (ac == PNA_AGGR_SKIP) continue;
    float y;
    switch (ac) {
      case PNA_AGGR_SUM: y = iso ? 0.f : r.S; break;
      case PNA_AGGR_MEAN: y = mean; break;
      case PNA_AGGR_MIN: y = mn; break;
      case PNA_AGGR_MAX: y = mx; break;
      case PNA_AGGR_VAR: y = (p.flags & PNA_FLAG_RELU_VAR) ? fmaxf(var, 0.0f) : var; break;
      default: y = sd; break;
    }
    if (zero_all) y = 0.f;
    for (int s = 0; s < p.nS; ++s) {
      const unsigned sc = (p.scodes >> (4 * s)) & 15u;
      float o[1] = {sc == PNA_SCALE_IDENTITY ? y : __fmul_rn(y, ds.of(sc))};
      Io<T, 1>::store(orow + (s * p.nA + k) * p.Ft, o);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_aw_rows(const AWParams a) {
  const MParams& p = a.m;
  long long row; int f;
  if (!mom_thread(p, p.n_rows, row, f)) return;
  const int beg = __ldg(p.rowptr + row), end = __ldg(p.rowptr + row + 1), deg = end - beg;
  if (deg >= p.split) return;                             // split rows: the chunk kernels
  if (p.ldeg && __ldg(p.ldeg + row) < 0) return;          // not in the masked view
  aw_copy_self<T>(a, row, f);
  const bool hb = p.bias != nullptr;
  const AwSums r = aw_sums<T>(p, a.w, beg, end, f, mom_bias<T>(p, row, f), hb);
  aw_store<T>(a, row, deg, f, aw_weight_sum(a.w, beg, end), r);
}

// per chunk: S, Q, min, max into [0..3]
template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_aw_chunk(const AWParams a) {
  const MParams& p = a.m;
  long long c; int f;
  if (!mom_thread(p, p.n_chunks, c, f)) return;
  const MomChunk m = mom_chunk(p, c);
  const AwSums r = aw_sums<T>(p, a.w, m.beg, m.end, f, mom_bias<T>(p, m.row, f), p.bias != nullptr);
  *mom_part<4>(p, c, 0, f) = r.S; *mom_part<4>(p, c, 1, f) = r.Q;
  *mom_part<4>(p, c, 2, f) = r.mn; *mom_part<4>(p, c, 3, f) = r.mx;
}

// per split row: the chunk partials in chunk order, the epilogue
template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_aw_hub_final(const AWParams a) {
  const MParams& p = a.m;
  long long h; int f;
  if (!mom_thread(p, p.n_hubs, h, f)) return;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2), deg = __ldg(p.hub_info + 4 * h + 3);
  AwSums r = {0.f, 0.f, INFINITY, -INFINITY};
  for (int j = 0; j < nch; ++j) {
    r.S = __fadd_rn(r.S, *mom_part<4>(p, first + j, 0, f));
    r.Q = __fadd_rn(r.Q, *mom_part<4>(p, first + j, 1, f));
    r.mn = fminf(r.mn, *mom_part<4>(p, first + j, 2, f));
    r.mx = fmaxf(r.mx, *mom_part<4>(p, first + j, 3, f));
  }
  aw_copy_self<T>(a, row, f);
  const int beg = __ldg(p.rowptr + row);
  aw_store<T>(a, row, deg, f, aw_weight_sum(a.w, beg, beg + deg), r);
}

}  // namespace pna
