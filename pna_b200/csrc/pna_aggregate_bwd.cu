// pna_aggregate_bwd: gradient of the aggregation w.r.t. the gathered rows (and the destination-side row_bias).
//
// Autograd of reference models/pytorch_geometric/aggregators.py:9-32 + scalers.py:8-29, as every training loop needs
// (multitask_benchmark/util/train.py:148, realworld_benchmark/train/*.py:31):
//   g_a   = sum over scalers s of scale_s(d) * grad_out[(s*A + a)*F + f]                        (per aggregator a)
//   d sum/dm = 1;  d mean/dm = 1/cnt;  d var/dm = 2 (m - mean)/cnt;  d std/dm = [var > 0] (m - mean)/(cnt * std)
//   min / max route to the FIRST slot attaining the extremum (torch_scatter's arg semantics)
// so that  grad_m(slot) = c0 + c1 * m + [slot == argmin] g_min + [slot == argmax] g_max  with two per-row coefficients.
// Two passes over the slots of a row: (A) recompute sum, sumsq, min, max and the first arg slots exactly as the forward
// does; (C) evaluate grad_m per slot, accumulate it into grad_gathered[col[slot]] (vector atomics -- several
// destinations share a source) and into grad_row_bias[row].  Rows at/above the split threshold are processed chunk by
// chunk by three small kernels (statistics, coefficients, scatter), like the forward.
//
// pna_aggregate_bwd_coef (gathered rows, col != NULL): pass C and its one vector atomic per (slot, feature chunk) are what
// bound the kernel above (the issue rate of the REDG atomics).  Per SOURCE row j the same gradient is
//   grad_gathered[j] = sum_{i <- j} (c0_i + c1_i * bias_i)  +  gathered[j] * sum_{i <- j} c1_i  +  routed min / max terms,
// so this entry point stops after the coefficients: it writes the row [c0' | c1] per destination, routes min / max with ONE
// scalar atomic per (row, feature) and writes grad_row_bias in closed form (deg * c0 + c1 * sum_m + gmin + gmax).  The two
// sums over the out-edges are a 'sum' aggregation of those rows over the transposed graph (pna_aggregate_fwd, no atomics),
// folded into grad_gathered by pna_aggregate_bwd_combine.
//
// pna_aggregate_bwd_slots (the deterministic backward): the same kernels compiled with SLOTS = true.  Pass C STORES grad_m of
// every slot into grad_slots[slot] (one feature slab [f_begin, f_begin + f_count) per call) instead of adding it into
// grad_gathered[col[slot]]; the caller sums those rows over the reversed edges with the forward kernel (fixed order).  Split
// rows store each chunk's share of grad_row_bias in scratch and k_bwd_hub_bias adds the shares in chunk order.  No
// floating-point atomics in any kernel of this variant.
//
// pna_aggregate_bwd_peer_slots (the peer plane's backward): the bodies of the per-slot kernels that read source rows
// (bwd_rows, bwd_hub_stats, bwd_hub_scatter) compiled with PEER = true into k_peer_bwd_*, so that col = owner << shift |
// row is read from the owner's buffer through the peer pointer table (NVLink) exactly as the forward's PEER instances
// read it.  Nothing else differs: each slot's gradient and grad_row_bias are the
// bits pna_aggregate_bwd_slots stores for the same slot of the unpartitioned graph.  k_bwd_hub_coef and k_bwd_hub_bias
// read only scratch and grad_out, so their per-slot instances serve both.  The existing k_bwd_* kernels are thin wrappers
// around the same bodies with PEER = false: their symbols and SASS are what they were before the peer instances existed.
#include "pna_aggregate.cuh"
#include <string.h>

namespace pna {

struct BParams {
  KParams k;
  const void* go; long long ldgo;     // grad_out, layout of out
  float* gg; long long ldgg;          // grad_gathered [n_src, F] fp32, accumulated
  float* gb; long long ldgb;          // grad_row_bias [n_rows, F] fp32, written (nullable)
  int vec_atomics;                    // grad_gathered rows are 16-byte aligned
  float* coef; long long ldc;         // coefficient mode (pna_aggregate_bwd_coef): [n_rows, ldc] rows [c0' | c1], c1 at column coef_c1
  int coef_c1, coef_vec;
  float* gs; long long ldgs;          // per-slot mode (pna_aggregate_bwd_slots): grad_slots [E, f1 - f0] fp32, written
  int f0, f1;                         // feature slab [f0, f1) of the per-slot mode
  int gs_vec;                         // grad_slots rows are 16-byte aligned
};

// Gradient of one message, grad_m = c0 + c1 * m + [slot == argmin] gmin + [slot == argmax] gmax, every operation rounded on
// its own and added left to right.  The atomic and the per-slot kernels share it, so both see the same value of every slot.
__device__ __forceinline__ float message_grad(float c0, float c1, float m, bool is_min, float gmin, bool is_max, float gmax) {
  return __fadd_rn(__fadd_rn(__fadd_rn(c0, __fmul_rn(c1, m)), is_min ? gmin : 0.f), is_max ? gmax : 0.f);
}

template <int VEC>
struct Stats {
  float sum[VEC], sq[VEC], mn[VEC], mx[VEC];
  int amn[VEC], amx[VEC];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int i = 0; i < VEC; ++i) { sum[i] = 0.f; sq[i] = 0.f; mn[i] = CUDART_INF_F; mx[i] = -CUDART_INF_F; amn[i] = -1; amx[i] = -1; }
  }
  __device__ __forceinline__ void add(const float (&m)[VEC], int slot) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      sum[i] = __fadd_rn(sum[i], m[i]);
      sq[i] = __fadd_rn(sq[i], __fmul_rn(m[i], m[i]));
      if (m[i] < mn[i]) { mn[i] = m[i]; amn[i] = slot; }   // strict: the first slot attaining the extremum wins
      if (m[i] > mx[i]) { mx[i] = m[i]; amx[i] = slot; }
    }
  }
};

template <int VEC>
struct Coef {
  float c0[VEC], c1[VEC], gmin[VEC], gmax[VEC];
};

// Source row `c` of a slot.  PEER (pna_aggregate_bwd_peer_slots): c = owner << shift | row, read from the owner's buffer
// through the peer pointer table as the forward's PEER instances read it; otherwise a row of the local buffer.
template <typename T, bool PEER>
__device__ __forceinline__ const T* source_row(const KParams& p, int c) {
  if constexpr (PEER) return gathered_row<T>(p, c);
  else return local_row<T>(p, c);
}

template <typename T, int VEC>
__device__ __forceinline__ void load_m(const KParams& p, int src, int f, const float (&bias)[VEC], bool has_bias, float (&m)[VEC]) {
  Io<T, VEC>::load(local_row<T>(p, src) + f, m);
  if (has_bias) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) m[i] = __fadd_rn(m[i], bias[i]);
  }
}

// upstream gradients of one row -> the two coefficients and the min / max gradients.  cnt: what the row's moments divide by
// (the slot count, clamped at 1; W_i for slot weights); sdegf: the scalers' degree, siso = (it is 0).
template <typename T, int VEC>
__device__ __forceinline__ void coefficients_at(const BParams& b, long long row, float cnt, bool siso, float sdegf, int ooff,
                                                const Stats<VEC>& st, Coef<VEC>& c) {
  const KParams& p = b.k;
  const float lg = logf(sdegf + 1.0f);
  const float s_amp = lg / p.avg_log, s_att = siso ? 1.0f : p.avg_log / lg;
  const float s_lin = sdegf / p.avg_lin, s_ilin = siso ? 1.0f : p.avg_lin / sdegf;
  const T* __restrict__ gorow = static_cast<const T*>(b.go) + row * b.ldgo + ooff;
#pragma unroll
  for (int i = 0; i < VEC; ++i) { c.c0[i] = 0.f; c.c1[i] = 0.f; c.gmin[i] = 0.f; c.gmax[i] = 0.f; }
  float mean[VEC], var[VEC], sd[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    mean[i] = st.sum[i] / cnt;
    var[i] = st.sq[i] / cnt - mean[i] * mean[i];
    sd[i] = sqrtf(fmaxf(var[i], 0.f) + 1e-5f);
  }
  for (int a = 0; a < p.nA; ++a) {
    const unsigned ac = (p.acodes >> (4 * a)) & 15u;
    if (ac == PNA_AGGR_SKIP) continue;
    float g[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) g[i] = 0.f;
    for (int s = 0; s < p.nS; ++s) {
      const unsigned sc = (p.scodes >> (4 * s)) & 15u;
      const float scale = sc == PNA_SCALE_IDENTITY ? 1.0f : sc == PNA_SCALE_AMPLIFICATION ? s_amp : sc == PNA_SCALE_ATTENUATION ? s_att
                          : sc == PNA_SCALE_LINEAR ? s_lin : s_ilin;
      float go[VEC];
      Io<T, VEC>::load(gorow + (s * p.nA + a) * p.Ft, go);
#pragma unroll
      for (int i = 0; i < VEC; ++i) g[i] += scale * go[i];
    }
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      switch (ac) {
        case PNA_AGGR_SUM: c.c0[i] += g[i]; break;
        case PNA_AGGR_MEAN: c.c0[i] += g[i] / cnt; break;
        case PNA_AGGR_MIN: c.gmin[i] += g[i]; break;
        case PNA_AGGR_MAX: c.gmax[i] += g[i]; break;
        case PNA_AGGR_VAR: {   // relu'(var) = [var > 0] in the DGL / dense flavours (PNA_FLAG_RELU_VAR)
          const float t = ((p.flags & PNA_FLAG_RELU_VAR) && !(var[i] > 0.f)) ? 0.f : 2.0f * g[i] / cnt;
          c.c1[i] += t; c.c0[i] -= t * mean[i];
        } break;
        default: { const float t = var[i] > 0.f ? g[i] / (cnt * sd[i]) : 0.f; c.c1[i] += t; c.c0[i] -= t * mean[i]; } break;
      }
    }
  }
}

template <typename T, int VEC>
__device__ __forceinline__ void coefficients(const BParams& b, long long row, int deg, int ooff, const Stats<VEC>& st, Coef<VEC>& c) {
  const KParams& p = b.k;
  const bool iso = deg == 0;
  const float degf = (float)deg, cnt = iso ? 1.0f : degf;
  const int sdeg = p.sdeg ? __ldg(p.sdeg + row) : deg;      // degree seen by the scalers (pna_agg_t.scaler_degree)
  coefficients_at<T, VEC>(b, row, cnt, sdeg == 0, (float)sdeg, ooff, st, c);
}

template <int VEC>
__device__ __forceinline__ void scatter_grad(const BParams& b, long long src_row, int f, const float (&gm)[VEC], bool atomic) {
  float* dst = b.gg + src_row * b.ldgg + f;
  if (!atomic) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) dst[i] = gm[i];
    return;
  }
  if constexpr (VEC % 4 == 0) {
    if (b.vec_atomics) {
#pragma unroll
      for (int i = 0; i < VEC; i += 4) atomicAdd(reinterpret_cast<float4*>(dst + i), make_float4(gm[i], gm[i + 1], gm[i + 2], gm[i + 3]));
      return;
    }
  }
#pragma unroll
  for (int i = 0; i < VEC; ++i) atomicAdd(dst + i, gm[i]);
}

// feature column / output column of this lane
struct LaneCols { int f, ooff; bool ok; };
template <int VEC>
__device__ __forceinline__ LaneCols lane_cols(const KParams& p, int gl, int fblock) {
  LaneCols c;
  c.f = fblock + gl * VEC;
  c.ok = c.f < p.F;
  if (!c.ok) { c.f = 0; }
  const int t = c.f / p.Ft, ft = c.f - t * p.Ft;
  c.ooff = t * p.Wt + p.has_self * p.Ft + ft;
  return c;
}

// columns of this lane in this block: all n_feat columns, or (per-slot mode) the slab [f0, f1)
template <int VEC, int G, bool SLOTS>
__device__ __forceinline__ LaneCols block_cols(const BParams& b, int gl) {
  if constexpr (SLOTS) {
    LaneCols c = lane_cols<VEC>(b.k, gl, b.f0 + (int)blockIdx.y * (G * VEC));
    if (c.f >= b.f1) c.ok = false;
    return c;
  } else {
    return lane_cols<VEC>(b.k, gl, blockIdx.y * (G * VEC));
  }
}

// per-slot mode: grad_slots[slot, f - f0] = gm (plain stores)
template <int VEC>
__device__ __forceinline__ void store_slot(const BParams& b, int slot, int f, const float (&gm)[VEC]) {
  float* dst = b.gs + (long long)slot * b.ldgs + (f - b.f0);
  if constexpr (VEC % 4 == 0) {
    if (b.gs_vec) {
#pragma unroll
      for (int i = 0; i < VEC; i += 4) *reinterpret_cast<float4*>(dst + i) = make_float4(gm[i], gm[i + 1], gm[i + 2], gm[i + 3]);
      return;
    }
  }
#pragma unroll
  for (int i = 0; i < VEC; ++i) dst[i] = gm[i];
}

// coefficient mode: what one destination row hands to its sources.  c0' = c0 + c1 * bias; min / max go to the source of the
// one slot that attained them (st.amn / st.amx: absolute CSR slots, -1 = none); grad_row_bias in closed form.
template <int VEC>
__device__ __forceinline__ void emit_row(const BParams& b, long long row, int deg, const LaneCols& lc, const Stats<VEC>& st,
                                         const Coef<VEC>& c, const float (&bias)[VEC], bool has_bias) {
  const KParams& p = b.k;
  float* crow = b.coef + row * b.ldc + lc.f;
  float c0p[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) c0p[i] = has_bias ? fmaf(c.c1[i], bias[i], c.c0[i]) : c.c0[i];
  bool stored = false;
  if constexpr (VEC % 4 == 0) {
    if (b.coef_vec) {     // 16-byte aligned rows and halves
#pragma unroll
      for (int i = 0; i < VEC; i += 4) {
        *reinterpret_cast<float4*>(crow + i) = make_float4(c0p[i], c0p[i + 1], c0p[i + 2], c0p[i + 3]);
        *reinterpret_cast<float4*>(crow + b.coef_c1 + i) = make_float4(c.c1[i], c.c1[i + 1], c.c1[i + 2], c.c1[i + 3]);
      }
      stored = true;
    }
  }
  if (!stored) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) { crow[i] = c0p[i]; crow[b.coef_c1 + i] = c.c1[i]; }
  }
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    if (c.gmin[i] != 0.f && st.amn[i] >= 0) atomicAdd(b.gg + (long long)__ldg(p.col + st.amn[i]) * b.ldgg + lc.f + i, c.gmin[i]);
    if (c.gmax[i] != 0.f && st.amx[i] >= 0) atomicAdd(b.gg + (long long)__ldg(p.col + st.amx[i]) * b.ldgg + lc.f + i, c.gmax[i]);
  }
  if (b.gb) {
    const float degf = (float)deg;
#pragma unroll
    for (int i = 0; i < VEC; ++i) b.gb[row * b.ldgb + lc.f + i] = degf * c.c0[i] + c.c1[i] * st.sum[i] + c.gmin[i] + c.gmax[i];
  }
}

constexpr int kBwdThreads = 256;

// ---- rows below the split threshold: one lane group per row --------------------------------------------------------
template <typename T, int VEC, int G, bool SLOTS, bool PEER>
__device__ __forceinline__ void bwd_rows(const BParams& b) {
  const KParams& p = b.k;
  constexpr int RPW = 32 / G;
  const int lane = threadIdx.x & 31, gl = lane % G;
  const long long row = ((long long)blockIdx.x * (kBwdThreads / 32) + (threadIdx.x >> 5)) * RPW + lane / G;
  if (row >= p.n_rows) return;
  const LaneCols lc = block_cols<VEC, G, SLOTS>(b, gl);
  if (!lc.ok) return;
  const int beg = __ldg(p.rowptr + row), end = __ldg(p.rowptr + row + 1), deg = end - beg;
  if (deg >= p.split) return;
  const bool has_bias = p.bias != nullptr;
  float bias[VEC];
  if (has_bias) Io<T, VEC>::load(static_cast<const T*>(p.bias) + row * p.ldb + lc.f, bias);
  if (deg == 0) {
    if (b.gb) {
      float z[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) z[i] = 0.f;
#pragma unroll
      for (int i = 0; i < VEC; ++i) b.gb[row * b.ldgb + lc.f + i] = z[i];
    }
    return;
  }
  constexpr int UB = 4;   // neighbour rows in flight per lane in each pass
  Stats<VEC> st;
  st.init();
  for (int e = beg; e < end; e += UB) {
    int src[UB];
    typename Io<T, VEC>::Raw raw[UB];
#pragma unroll
    for (int u = 0; u < UB; ++u) src[u] = (e + u < end) ? (p.col ? __ldg(p.col + e + u) : e + u) : -1;
#pragma unroll
    for (int u = 0; u < UB; ++u) if (src[u] >= 0) raw[u] = Io<T, VEC>::load_raw(source_row<T, PEER>(p, src[u]) + lc.f);
#pragma unroll
    for (int u = 0; u < UB; ++u) {
      if (src[u] >= 0) {
        float m[VEC];
        Io<T, VEC>::unpack(raw[u], m);
        if (has_bias) {
#pragma unroll
          for (int i = 0; i < VEC; ++i) m[i] = __fadd_rn(m[i], bias[i]);
        }
        st.add(m, e + u);
      }
    }
  }
  Coef<VEC> c;
  coefficients<T, VEC>(b, row, deg, lc.ooff, st, c);
  if constexpr (!SLOTS) {
    if (b.coef) {   // coefficient mode: no second pass over the slots
      emit_row<VEC>(b, row, deg, lc, st, c, bias, has_bias);
      return;
    }
  }
  float gbs[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) gbs[i] = 0.f;
  for (int e = beg; e < end; e += UB) {
    int src[UB];
    typename Io<T, VEC>::Raw raw[UB];
#pragma unroll
    for (int u = 0; u < UB; ++u) src[u] = (e + u < end) ? (p.col ? __ldg(p.col + e + u) : e + u) : -1;
#pragma unroll
    for (int u = 0; u < UB; ++u) if (src[u] >= 0) raw[u] = Io<T, VEC>::load_raw(source_row<T, PEER>(p, src[u]) + lc.f);
#pragma unroll
    for (int u = 0; u < UB; ++u) {
      if (src[u] >= 0) {
        float m[VEC], gm[VEC];
        Io<T, VEC>::unpack(raw[u], m);
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          if (has_bias) m[i] = __fadd_rn(m[i], bias[i]);
          gm[i] = message_grad(c.c0[i], c.c1[i], m[i], e + u == st.amn[i], c.gmin[i], e + u == st.amx[i], c.gmax[i]);
          gbs[i] += gm[i];
        }
        if constexpr (SLOTS) store_slot<VEC>(b, e + u, lc.f, gm);
        else scatter_grad<VEC>(b, src[u], lc.f, gm, p.col != nullptr);
      }
    }
  }
  if (b.gb) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) b.gb[row * b.ldgb + lc.f + i] = gbs[i];
  }
}

template <typename T, int VEC, int G, bool SLOTS>
__global__ void __launch_bounds__(kBwdThreads) k_bwd_rows(const BParams b) { bwd_rows<T, VEC, G, SLOTS, false>(b); }

// the peer plane's instance (pna_aggregate_bwd_peer_slots): per-slot, source rows read through the peer pointer table
template <typename T, int VEC, int G>
__global__ void __launch_bounds__(kBwdThreads) k_peer_bwd_rows(const BParams b) { bwd_rows<T, VEC, G, true, true>(b); }

// ---- split rows: chunk-parallel, like the forward ---------------------------------------------------------------
// (1) k_bwd_hub_stats: one lane group per 128-slot chunk -> partial sum, sumsq, min, max, first argmin / argmax slot;
// (2) k_bwd_hub_coef:  one lane group per split row merges its chunks in chunk order (strict < keeps the first slot)
//                      and turns the upstream gradient into (c0, c1, gmin, gmax, argmin, argmax) per feature;
// (3) k_bwd_hub_scatter: one lane group per chunk evaluates grad_m per slot, scatters it, and adds its share of the
//                      row_bias gradient.  Scratch (descriptor field hub_partials): 6*F floats per chunk + per split row.
// Per-slot mode: (3) stores grad_m per slot and parks the chunk's row_bias share in the chunk's (consumed) sum partial;
// (4) k_bwd_hub_bias: one lane group per split row adds those shares in chunk order.
template <typename T, int VEC, int G, bool SLOTS, bool PEER>
__device__ __forceinline__ void bwd_hub_stats(const BParams& b) {
  const KParams& p = b.k;
  constexpr int RPW = 32 / G;
  const int lane = threadIdx.x & 31, gl = lane % G;
  const long long c = ((long long)blockIdx.x * (kBwdThreads / 32) + (threadIdx.x >> 5)) * RPW + lane / G;
  if (c >= p.n_chunks) return;
  const LaneCols lc = block_cols<VEC, G, SLOTS>(b, gl);
  if (!lc.ok) return;
  const int h = __ldg(p.chunk_items + 2 * c), j = __ldg(p.chunk_items + 2 * c + 1);
  const long long row = __ldg(p.hub_info + 4 * h);
  const int rbeg = __ldg(p.rowptr + row), rend = __ldg(p.rowptr + row + 1);
  const int beg = rbeg + j * p.chunk, end = min(beg + p.chunk, rend);
  const bool has_bias = p.bias != nullptr;
  float bias[VEC];
  if (has_bias) Io<T, VEC>::load(static_cast<const T*>(p.bias) + row * p.ldb + lc.f, bias);
  constexpr int UB = 4;
  Stats<VEC> st;
  st.init();
  for (int e = beg; e < end; e += UB) {
    int src[UB];
    typename Io<T, VEC>::Raw raw[UB];
#pragma unroll
    for (int u = 0; u < UB; ++u) src[u] = (e + u < end) ? (p.col ? __ldg(p.col + e + u) : e + u) : -1;
#pragma unroll
    for (int u = 0; u < UB; ++u) if (src[u] >= 0) raw[u] = Io<T, VEC>::load_raw(source_row<T, PEER>(p, src[u]) + lc.f);
#pragma unroll
    for (int u = 0; u < UB; ++u) {
      if (src[u] >= 0) {
        float m[VEC];
        Io<T, VEC>::unpack(raw[u], m);
        if (has_bias) {
#pragma unroll
          for (int i = 0; i < VEC; ++i) m[i] = __fadd_rn(m[i], bias[i]);
        }
        st.add(m, e + u);
      }
    }
  }
  float* part = p.partials + c * 6ll * p.F + lc.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    part[0ll * p.F + i] = st.sum[i]; part[1ll * p.F + i] = st.sq[i]; part[2ll * p.F + i] = st.mn[i]; part[3ll * p.F + i] = st.mx[i];
    part[4ll * p.F + i] = __int_as_float(st.amn[i]); part[5ll * p.F + i] = __int_as_float(st.amx[i]);
  }
}

template <typename T, int VEC, int G, bool SLOTS>
__global__ void __launch_bounds__(kBwdThreads) k_bwd_hub_stats(const BParams b) { bwd_hub_stats<T, VEC, G, SLOTS, false>(b); }

// the peer plane's instance (pna_aggregate_bwd_peer_slots): per-slot, source rows read through the peer pointer table
template <typename T, int VEC, int G>
__global__ void __launch_bounds__(kBwdThreads) k_peer_bwd_hub_stats(const BParams b) { bwd_hub_stats<T, VEC, G, true, true>(b); }

template <typename T, int VEC, int G, bool SLOTS>
__global__ void __launch_bounds__(kBwdThreads) k_bwd_hub_coef(const BParams b) {
  const KParams& p = b.k;
  constexpr int RPW = 32 / G;
  const int lane = threadIdx.x & 31, gl = lane % G;
  const long long h = ((long long)blockIdx.x * (kBwdThreads / 32) + (threadIdx.x >> 5)) * RPW + lane / G;
  if (h >= p.n_hubs) return;
  const LaneCols lc = block_cols<VEC, G, SLOTS>(b, gl);
  if (!lc.ok) return;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2), deg = __ldg(p.hub_info + 4 * h + 3);
  Stats<VEC> st;
  st.init();
  for (int j = 0; j < nch; ++j) {
    const float* part = p.partials + (long long)(first + j) * 6ll * p.F + lc.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      st.sum[i] += part[0ll * p.F + i]; st.sq[i] += part[1ll * p.F + i];
      const float mn = part[2ll * p.F + i], mx = part[3ll * p.F + i];
      if (mn < st.mn[i]) { st.mn[i] = mn; st.amn[i] = __float_as_int(part[4ll * p.F + i]); }
      if (mx > st.mx[i]) { st.mx[i] = mx; st.amx[i] = __float_as_int(part[5ll * p.F + i]); }
    }
  }
  Coef<VEC> c;
  coefficients<T, VEC>(b, row, deg, lc.ooff, st, c);
  if constexpr (!SLOTS) {
    if (b.coef) {   // coefficient mode: the split row ends here, like every other row
      const bool has_bias = p.bias != nullptr;
      float bias[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) bias[i] = 0.f;
      if (has_bias) Io<T, VEC>::load(static_cast<const T*>(p.bias) + row * p.ldb + lc.f, bias);
      emit_row<VEC>(b, row, deg, lc, st, c, bias, has_bias);
      return;
    }
  }
  float* co = p.partials + (p.n_chunks + h) * 6ll * p.F + lc.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    co[0ll * p.F + i] = c.c0[i]; co[1ll * p.F + i] = c.c1[i]; co[2ll * p.F + i] = c.gmin[i]; co[3ll * p.F + i] = c.gmax[i];
    co[4ll * p.F + i] = __int_as_float(st.amn[i]); co[5ll * p.F + i] = __int_as_float(st.amx[i]);
  }
  if constexpr (!SLOTS) {
    if (b.gb) {   // the chunks add their shares atomically in pass 3
#pragma unroll
      for (int i = 0; i < VEC; ++i) b.gb[row * b.ldgb + lc.f + i] = 0.f;
    }
  }
}

template <typename T, int VEC, int G, bool SLOTS, bool PEER>
__device__ __forceinline__ void bwd_hub_scatter(const BParams& b) {
  const KParams& p = b.k;
  constexpr int RPW = 32 / G;
  const int lane = threadIdx.x & 31, gl = lane % G;
  const long long c = ((long long)blockIdx.x * (kBwdThreads / 32) + (threadIdx.x >> 5)) * RPW + lane / G;
  if (c >= p.n_chunks) return;
  const LaneCols lc = block_cols<VEC, G, SLOTS>(b, gl);
  if (!lc.ok) return;
  const int h = __ldg(p.chunk_items + 2 * c), j = __ldg(p.chunk_items + 2 * c + 1);
  const long long row = __ldg(p.hub_info + 4 * h);
  const int rbeg = __ldg(p.rowptr + row), rend = __ldg(p.rowptr + row + 1);
  const int beg = rbeg + j * p.chunk, end = min(beg + p.chunk, rend);
  const bool has_bias = p.bias != nullptr;
  float bias[VEC];
  if (has_bias) Io<T, VEC>::load(static_cast<const T*>(p.bias) + row * p.ldb + lc.f, bias);
  const float* co = p.partials + (p.n_chunks + h) * 6ll * p.F + lc.f;
  Coef<VEC> cf;
  int amn[VEC], amx[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    cf.c0[i] = co[0ll * p.F + i]; cf.c1[i] = co[1ll * p.F + i]; cf.gmin[i] = co[2ll * p.F + i]; cf.gmax[i] = co[3ll * p.F + i];
    amn[i] = __float_as_int(co[4ll * p.F + i]); amx[i] = __float_as_int(co[5ll * p.F + i]);
  }
  constexpr int UB = 4;
  float gbs[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) gbs[i] = 0.f;
  for (int e = beg; e < end; e += UB) {
    int src[UB];
    typename Io<T, VEC>::Raw raw[UB];
#pragma unroll
    for (int u = 0; u < UB; ++u) src[u] = (e + u < end) ? (p.col ? __ldg(p.col + e + u) : e + u) : -1;
#pragma unroll
    for (int u = 0; u < UB; ++u) if (src[u] >= 0) raw[u] = Io<T, VEC>::load_raw(source_row<T, PEER>(p, src[u]) + lc.f);
#pragma unroll
    for (int u = 0; u < UB; ++u) {
      if (src[u] >= 0) {
        float m[VEC], gm[VEC];
        Io<T, VEC>::unpack(raw[u], m);
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          if (has_bias) m[i] = __fadd_rn(m[i], bias[i]);
          gm[i] = message_grad(cf.c0[i], cf.c1[i], m[i], e + u == amn[i], cf.gmin[i], e + u == amx[i], cf.gmax[i]);
          gbs[i] += gm[i];
        }
        if constexpr (SLOTS) store_slot<VEC>(b, e + u, lc.f, gm);
        else scatter_grad<VEC>(b, src[u], lc.f, gm, p.col != nullptr);
      }
    }
  }
  if (b.gb) {
    if constexpr (SLOTS) {   // this chunk's share, merged in chunk order by k_bwd_hub_bias (k_bwd_hub_coef has read the stats)
      float* part = p.partials + c * 6ll * p.F + lc.f;
#pragma unroll
      for (int i = 0; i < VEC; ++i) part[i] = gbs[i];
    } else {
#pragma unroll
      for (int i = 0; i < VEC; ++i) atomicAdd(b.gb + row * b.ldgb + lc.f + i, gbs[i]);
    }
  }
}

template <typename T, int VEC, int G, bool SLOTS>
__global__ void __launch_bounds__(kBwdThreads) k_bwd_hub_scatter(const BParams b) { bwd_hub_scatter<T, VEC, G, SLOTS, false>(b); }

// the peer plane's instance (pna_aggregate_bwd_peer_slots): per-slot, source rows read through the peer pointer table
template <typename T, int VEC, int G>
__global__ void __launch_bounds__(kBwdThreads) k_peer_bwd_hub_scatter(const BParams b) { bwd_hub_scatter<T, VEC, G, true, true>(b); }

// per-slot mode, split rows: grad_row_bias = the chunks' shares added in chunk order (each share in slot order)
template <int VEC, int G>
__global__ void __launch_bounds__(kBwdThreads) k_bwd_hub_bias(const BParams b) {
  const KParams& p = b.k;
  constexpr int RPW = 32 / G;
  const int lane = threadIdx.x & 31, gl = lane % G;
  const long long h = ((long long)blockIdx.x * (kBwdThreads / 32) + (threadIdx.x >> 5)) * RPW + lane / G;
  if (h >= p.n_hubs) return;
  const LaneCols lc = block_cols<VEC, G, true>(b, gl);
  if (!lc.ok) return;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2);
  float acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
  for (int j = 0; j < nch; ++j) {
    const float* part = p.partials + (long long)(first + j) * 6ll * p.F + lc.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = __fadd_rn(acc[i], part[i]);
  }
#pragma unroll
  for (int i = 0; i < VEC; ++i) b.gb[row * b.ldgb + lc.f + i] = acc[i];
}

template <typename T, int VEC, int G, bool SLOTS, bool PEER>
static int launch_bwd(const BParams& b, cudaStream_t st) {
  static_assert(SLOTS || !PEER, "peer-memory graphs have the per-slot backward only");
  const KParams& p = b.k;
  constexpr int RPW = 32 / G;
  const int width = SLOTS ? b.f1 - b.f0 : p.F;     // the per-slot mode covers one feature slab
  const unsigned gy = (unsigned)((width + G * VEC - 1) / (G * VEC));
  const long long per_block = (kBwdThreads / 32) * RPW;
  const long long gx = (p.n_rows + per_block - 1) / per_block;
  PNA_REQUIRE(gx <= 0x7fffffffll, PNA_ERR_UNSUPPORTED, "pna_aggregate_bwd: too many rows");
  if constexpr (PEER)
    k_peer_bwd_rows<T, VEC, G><<<dim3((unsigned)gx, gy), kBwdThreads, 0, st>>>(b);
  else
    k_bwd_rows<T, VEC, G, SLOTS><<<dim3((unsigned)gx, gy), kBwdThreads, 0, st>>>(b);
  PNA_CUDA_TRY(cudaGetLastError());
  if (p.n_hubs > 0) {
    const long long gc = (p.n_chunks + per_block - 1) / per_block, gh = (p.n_hubs + per_block - 1) / per_block;
    if constexpr (PEER)
      k_peer_bwd_hub_stats<T, VEC, G><<<dim3((unsigned)gc, gy), kBwdThreads, 0, st>>>(b);
    else
      k_bwd_hub_stats<T, VEC, G, SLOTS><<<dim3((unsigned)gc, gy), kBwdThreads, 0, st>>>(b);
    PNA_CUDA_TRY(cudaGetLastError());
    k_bwd_hub_coef<T, VEC, G, SLOTS><<<dim3((unsigned)gh, gy), kBwdThreads, 0, st>>>(b);
    PNA_CUDA_TRY(cudaGetLastError());
    if (!b.coef) {
      if constexpr (PEER)
        k_peer_bwd_hub_scatter<T, VEC, G><<<dim3((unsigned)gc, gy), kBwdThreads, 0, st>>>(b);
      else
        k_bwd_hub_scatter<T, VEC, G, SLOTS><<<dim3((unsigned)gc, gy), kBwdThreads, 0, st>>>(b);
      PNA_CUDA_TRY(cudaGetLastError());
    }
    if (SLOTS && b.gb) {
      k_bwd_hub_bias<VEC, G><<<dim3((unsigned)gh, gy), kBwdThreads, 0, st>>>(b);
      PNA_CUDA_TRY(cudaGetLastError());
    }
  }
  return PNA_OK;
}

template <typename T, int VEC, bool SLOTS, bool PEER = false>
static int launch_bwd_typed(const BParams& b, cudaStream_t st) {
  const int chunks = (SLOTS ? b.f1 - b.f0 : b.k.F) / VEC;
  if (chunks <= 1) return launch_bwd<T, VEC, 1, SLOTS, PEER>(b, st);
  if (chunks <= 2) return launch_bwd<T, VEC, 2, SLOTS, PEER>(b, st);
  if (chunks <= 4) return launch_bwd<T, VEC, 4, SLOTS, PEER>(b, st);
  if (chunks <= 8) return launch_bwd<T, VEC, 8, SLOTS, PEER>(b, st);
  if (chunks <= 16) return launch_bwd<T, VEC, 16, SLOTS, PEER>(b, st);
  return launch_bwd<T, VEC, 32, SLOTS, PEER>(b, st);     // wider rows: several feature blocks (gridDim.y)
}

static bool al16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0; }

// The moment term of every slot's gradient (pna_aggregate_moments.cuh), added after the existing kernels have written it.
template <typename T, bool SLOTS>
static int launch_moments_bwd(const MParams& p, cudaStream_t st) {
  const unsigned gy = (unsigned)((p.f1 - p.f0 + 31) / 32);
  constexpr long long per_block = kMomThreads / 32;
  const long long gx = (p.n_rows + per_block - 1) / per_block;
  PNA_REQUIRE(gx <= 0x7fffffffll, PNA_ERR_UNSUPPORTED, "pna_aggregate_bwd: too many rows");
  k_mom_bwd_rows<T, SLOTS><<<dim3((unsigned)gx, gy), kMomThreads, 0, st>>>(p);
  PNA_CUDA_TRY(cudaGetLastError());
  if (p.n_hubs > 0) {
    const unsigned gc = (unsigned)((p.n_chunks + per_block - 1) / per_block), gh = (unsigned)((p.n_hubs + per_block - 1) / per_block);
    k_mom_chunk_sum<T, 6><<<dim3(gc, gy), kMomThreads, 0, st>>>(p);
    PNA_CUDA_TRY(cudaGetLastError());
    k_mom_hub_mean<6><<<dim3(gh, gy), kMomThreads, 0, st>>>(p);
    PNA_CUDA_TRY(cudaGetLastError());
    k_mom_chunk_central<T, 6><<<dim3(gc, gy), kMomThreads, 0, st>>>(p);
    PNA_CUDA_TRY(cudaGetLastError());
    k_mom_bwd_hub_coef<T><<<dim3(gh, gy), kMomThreads, 0, st>>>(p);
    PNA_CUDA_TRY(cudaGetLastError());
    k_mom_bwd_chunk_grad<T, SLOTS><<<dim3(gc, gy), kMomThreads, 0, st>>>(p);
    PNA_CUDA_TRY(cudaGetLastError());
    if (p.gb) {
      k_mom_bwd_hub_bias<6><<<dim3(gh, gy), kMomThreads, 0, st>>>(p);
      PNA_CUDA_TRY(cudaGetLastError());
    }
  }
  return PNA_OK;
}

// The term of one weighted aggregator in every slot's gradient (pna_aggregate_weighted.cuh), after the moments'.
template <typename T, bool SLOTS>
static int launch_weighted_bwd(const MParams& p, unsigned code, cudaStream_t st) {
  const unsigned gy = (unsigned)((p.f1 - p.f0 + 31) / 32);
  constexpr long long per_block = kMomThreads / 32;
  const long long gx = (p.n_rows + per_block - 1) / per_block;
  PNA_REQUIRE(gx <= 0x7fffffffll, PNA_ERR_UNSUPPORTED, "pna_aggregate_bwd: too many rows");
  k_wsum_bwd_rows<T, SLOTS><<<dim3((unsigned)gx, gy), kMomThreads, 0, st>>>(p, code);
  PNA_CUDA_TRY(cudaGetLastError());
  if (p.n_hubs > 0) {
    const unsigned gc = (unsigned)((p.n_chunks + per_block - 1) / per_block), gh = (unsigned)((p.n_hubs + per_block - 1) / per_block);
    if (code != PNA_AGGR_NORMALISED_MEAN) {
      k_wsum_chunk_max<T, 6><<<dim3(gc, gy), kMomThreads, 0, st>>>(p, code);
      PNA_CUDA_TRY(cudaGetLastError());
      k_wsum_hub_max<6><<<dim3(gh, gy), kMomThreads, 0, st>>>(p);
      PNA_CUDA_TRY(cudaGetLastError());
      k_wsum_chunk_zs<T, 6><<<dim3(gc, gy), kMomThreads, 0, st>>>(p, code);
      PNA_CUDA_TRY(cudaGetLastError());
    }
    k_wsum_bwd_hub_coef<T><<<dim3(gh, gy), kMomThreads, 0, st>>>(p, code);
    PNA_CUDA_TRY(cudaGetLastError());
    k_wsum_bwd_chunk_grad<T, SLOTS><<<dim3(gc, gy), kMomThreads, 0, st>>>(p, code);
    PNA_CUDA_TRY(cudaGetLastError());
    if (p.gb) {
      k_mom_bwd_hub_bias<6><<<dim3(gh, gy), kMomThreads, 0, st>>>(p);
      PNA_CUDA_TRY(cudaGetLastError());
    }
  }
  return PNA_OK;
}

// The add-on aggregators' terms: the moments, then each weighted aggregator in turn (stream order: each reuses
// hub_partials).
template <typename T, bool SLOTS>
static int launch_addons_bwd(const pna_agg_t* d, const MParams& mp, cudaStream_t st) {
  if (mp.orders) {
    const int rc = launch_moments_bwd<T, SLOTS>(mp, st);
    if (rc != PNA_OK) return rc;
  }
  const unsigned w = weighted_codes(d->aggr_codes, d->n_aggr);
  for (unsigned c = PNA_AGGR_SOFTMAX; c <= PNA_AGGR_NORMALISED_MEAN; ++c) {
    if (!((w >> (c - PNA_AGGR_SOFTMAX)) & 1u)) continue;
    const int rc = launch_weighted_bwd<T, SLOTS>(mp, c, st);
    if (rc != PNA_OK) return rc;
  }
  return PNA_OK;
}

// ---- slot weights (pna_aggregate_bwd_weighted / _bwd_slots_weighted; forward and formulas: pna_aggregate_adj_weight.cuh) --
// The gradient of slot s is  g_s = fl(w_s * fl(c0 + c1 * m_s)) + [s == argmin] gmin + [s == argmax] gmax,  with c0, c1, gmin,
// gmax from coefficients_at at cnt = W_i (and the scalers at D), the statistics S, Q of the weighted forward and min / max
// over the positive-weight slots (first slot attaining them); message_grad evaluates both steps, so all-ones weights give
// the unweighted per-slot bits.  One thread per (row or chunk, feature column) as in the forward; split rows:
// (1) per chunk S, Q, min, max, arg slots into [0..5]; (2) per split row their chunk-order merge -> the coefficients into
// the row's slot (n_chunks + h) [0..5]; (3) per chunk the slot gradients and the chunk's slot-order share of grad_row_bias
// into [0]; (4) per split row those shares added in chunk order.  SLOTS stores g_s into grad_slots; the atomic instance
// adds it into grad_gathered[col[s]] (per-slot rows, col == NULL: stores).  grad_row_bias is stored, never accumulated.
struct AWBParams {
  AWParams a;
  BParams b;
};

__device__ __forceinline__ float aw_slot_grad(const Coef<1>& c, float w, float m, bool is_min, bool is_max) {
  return message_grad(0.f, w, message_grad(c.c0[0], c.c1[0], m, false, 0.f, false, 0.f), is_min, c.gmin[0], is_max, c.gmax[0]);
}

// statistics of slots [beg, end) in the layout of the unweighted backward (Stats<1>: S, Q, min, max and their first slot)
template <typename T>
__device__ __forceinline__ Stats<1> aw_stats(const AWParams& a, int beg, int end, int f, float b, bool hb) {
  Stats<1> st;
  st.init();
  for (int e = beg; e < end; ++e) {
    const float m = mom_msg<T>(a.m, e, f, b, hb), ws = aw_weight(a.w, e);
    st.sum[0] = __fadd_rn(st.sum[0], __fmul_rn(m, ws));
    st.sq[0] = __fadd_rn(st.sq[0], __fmul_rn(__fmul_rn(m, m), ws));
    if (ws > 0.f) {
      if (m < st.mn[0]) { st.mn[0] = m; st.amn[0] = e; }
      if (m > st.mx[0]) { st.mx[0] = m; st.amx[0] = e; }
    }
  }
  return st;
}

template <typename T>
__device__ __forceinline__ void aw_coef(const AWBParams& q, long long row, int beg, int deg, int f, const Stats<1>& st, Coef<1>& c) {
  const MParams& p = q.a.m;
  const float D = aw_scaler_degree(p, q.a.sdf, row, deg);
  coefficients_at<T, 1>(q.b, row, aw_weight_sum(q.a.w, beg, beg + deg), D == 0.0f, D, (int)mom_base_col(p, f), st, c);
}

// add every slot's gradient of [beg, end) to its destination; returns their slot-order sum
template <typename T, bool SLOTS>
__device__ __forceinline__ float aw_emit(const AWParams& a, int beg, int end, int f, float b, bool hb, const Coef<1>& c, int amn,
                                         int amx) {
  const MParams& p = a.m;
  float acc = 0.f;
  for (int e = beg; e < end; ++e) {
    const float g = aw_slot_grad(c, aw_weight(a.w, e), mom_msg<T>(p, e, f, b, hb), e == amn, e == amx);
    acc = __fadd_rn(acc, g);
    if constexpr (SLOTS) {
      p.gs[(long long)e * p.ldgs + (f - p.f0)] = g;
    } else {
      if (p.col) atomicAdd(p.gg + (long long)__ldg(p.col + e) * p.ldgg + f, g);
      else p.gg[(long long)e * p.ldgg + f] = g;
    }
  }
  return acc;
}

template <typename T, bool SLOTS>
__global__ void __launch_bounds__(kMomThreads) k_aw_bwd_rows(const AWBParams q) {
  const MParams& p = q.a.m;
  long long row; int f;
  if (!mom_thread(p, p.n_rows, row, f)) return;
  const int beg = __ldg(p.rowptr + row), end = __ldg(p.rowptr + row + 1), deg = end - beg;
  if (deg >= p.split) return;
  float gbs = 0.f;
  if (deg > 0) {
    const bool hb = p.bias != nullptr;
    const float b = mom_bias<T>(p, row, f);
    const Stats<1> st = aw_stats<T>(q.a, beg, end, f, b, hb);
    Coef<1> c;
    aw_coef<T>(q, row, beg, deg, f, st, c);
    gbs = aw_emit<T, SLOTS>(q.a, beg, end, f, b, hb, c, st.amn[0], st.amx[0]);
  }
  if (p.gb) p.gb[row * p.ldgb + f] = gbs;
}

template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_aw_bwd_chunk_stats(const AWBParams q) {
  const MParams& p = q.a.m;
  long long c; int f;
  if (!mom_thread(p, p.n_chunks, c, f)) return;
  const MomChunk m = mom_chunk(p, c);
  const Stats<1> st = aw_stats<T>(q.a, m.beg, m.end, f, mom_bias<T>(p, m.row, f), p.bias != nullptr);
  *mom_part<6>(p, c, 0, f) = st.sum[0]; *mom_part<6>(p, c, 1, f) = st.sq[0];
  *mom_part<6>(p, c, 2, f) = st.mn[0]; *mom_part<6>(p, c, 3, f) = st.mx[0];
  *mom_part<6>(p, c, 4, f) = __int_as_float(st.amn[0]); *mom_part<6>(p, c, 5, f) = __int_as_float(st.amx[0]);
}

template <typename T>
__global__ void __launch_bounds__(kMomThreads) k_aw_bwd_hub_coef(const AWBParams q) {
  const MParams& p = q.a.m;
  long long h; int f;
  if (!mom_thread(p, p.n_hubs, h, f)) return;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2), deg = __ldg(p.hub_info + 4 * h + 3);
  Stats<1> st;
  st.init();
  for (int j = 0; j < nch; ++j) {
    st.sum[0] = __fadd_rn(st.sum[0], *mom_part<6>(p, first + j, 0, f));
    st.sq[0] = __fadd_rn(st.sq[0], *mom_part<6>(p, first + j, 1, f));
    const float mn = *mom_part<6>(p, first + j, 2, f), mx = *mom_part<6>(p, first + j, 3, f);
    if (mn < st.mn[0]) { st.mn[0] = mn; st.amn[0] = __float_as_int(*mom_part<6>(p, first + j, 4, f)); }
    if (mx > st.mx[0]) { st.mx[0] = mx; st.amx[0] = __float_as_int(*mom_part<6>(p, first + j, 5, f)); }
  }
  Coef<1> c;
  aw_coef<T>(q, row, __ldg(p.rowptr + row), deg, f, st, c);
  const long long hs = p.n_chunks + h;
  *mom_part<6>(p, hs, 0, f) = c.c0[0]; *mom_part<6>(p, hs, 1, f) = c.c1[0];
  *mom_part<6>(p, hs, 2, f) = c.gmin[0]; *mom_part<6>(p, hs, 3, f) = c.gmax[0];
  *mom_part<6>(p, hs, 4, f) = __int_as_float(st.amn[0]); *mom_part<6>(p, hs, 5, f) = __int_as_float(st.amx[0]);
}

template <typename T, bool SLOTS>
__global__ void __launch_bounds__(kMomThreads) k_aw_bwd_chunk_grad(const AWBParams q) {
  const MParams& p = q.a.m;
  long long c; int f;
  if (!mom_thread(p, p.n_chunks, c, f)) return;
  const MomChunk m = mom_chunk(p, c);
  const long long hs = p.n_chunks + m.h;
  Coef<1> cf;
  cf.c0[0] = *mom_part<6>(p, hs, 0, f); cf.c1[0] = *mom_part<6>(p, hs, 1, f);
  cf.gmin[0] = *mom_part<6>(p, hs, 2, f); cf.gmax[0] = *mom_part<6>(p, hs, 3, f);
  const int amn = __float_as_int(*mom_part<6>(p, hs, 4, f)), amx = __float_as_int(*mom_part<6>(p, hs, 5, f));
  *mom_part<6>(p, c, 0, f) = aw_emit<T, SLOTS>(q.a, m.beg, m.end, f, mom_bias<T>(p, m.row, f), p.bias != nullptr, cf, amn, amx);
}

__global__ void __launch_bounds__(kMomThreads) k_aw_bwd_hub_bias(const AWBParams q) {
  const MParams& p = q.a.m;
  long long h; int f;
  if (!mom_thread(p, p.n_hubs, h, f)) return;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2);
  float acc = 0.f;
  for (int j = 0; j < nch; ++j) acc = __fadd_rn(acc, *mom_part<6>(p, first + j, 0, f));
  p.gb[row * p.ldgb + f] = acc;
}

template <typename T, bool SLOTS>
static int launch_adj_weight_bwd(const AWBParams& q, cudaStream_t st) {
  const MParams& p = q.a.m;
  const unsigned gy = (unsigned)((p.f1 - p.f0 + 31) / 32);
  constexpr long long per_block = kMomThreads / 32;
  const long long gx = (p.n_rows + per_block - 1) / per_block;
  PNA_REQUIRE(gx <= 0x7fffffffll, PNA_ERR_UNSUPPORTED, "pna_aggregate_bwd: too many rows");
  k_aw_bwd_rows<T, SLOTS><<<dim3((unsigned)gx, gy), kMomThreads, 0, st>>>(q);
  PNA_CUDA_TRY(cudaGetLastError());
  if (p.n_hubs > 0) {
    const unsigned gc = (unsigned)((p.n_chunks + per_block - 1) / per_block), gh = (unsigned)((p.n_hubs + per_block - 1) / per_block);
    k_aw_bwd_chunk_stats<T><<<dim3(gc, gy), kMomThreads, 0, st>>>(q);
    PNA_CUDA_TRY(cudaGetLastError());
    k_aw_bwd_hub_coef<T><<<dim3(gh, gy), kMomThreads, 0, st>>>(q);
    PNA_CUDA_TRY(cudaGetLastError());
    k_aw_bwd_chunk_grad<T, SLOTS><<<dim3(gc, gy), kMomThreads, 0, st>>>(q);
    PNA_CUDA_TRY(cudaGetLastError());
    if (p.gb) {
      k_aw_bwd_hub_bias<<<dim3(gh, gy), kMomThreads, 0, st>>>(q);
      PNA_CUDA_TRY(cudaGetLastError());
    }
  }
  return PNA_OK;
}

// ---- phase 3 of the coefficient path: grad_gathered[j] += S0[j] + gathered[j] * S1[j] ------------------------------------
// sums[j] = [S0 | S1] (S1 at column c1): the 'sum' of the coefficient rows over the out-edges of source row j.
template <typename T>
__global__ void __launch_bounds__(256) k_bwd_combine(const float* __restrict__ sums, long long lds, int c1, const T* __restrict__ x,
                                                     long long ldx, float* __restrict__ gg, long long ldgg, long long n_src, int F) {
  const long long total = n_src * F;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / F;
    const int f = (int)(i - r * F);
    const float s0 = sums[r * lds + f], s1 = sums[r * lds + c1 + f];
    float xv;
    if constexpr (sizeof(T) == 4) xv = x[r * ldx + f];
    else xv = __bfloat162float(x[r * ldx + f]);
    gg[r * ldgg + f] += s0 + xv * s1;
  }
}

}  // namespace pna

using namespace pna;

// grad_slots != NULL: the per-slot mode (pna_aggregate_bwd_slots) over the feature slab [f_begin, f_begin + f_count);
// peer: the same over a peer-memory graph (pna_aggregate_bwd_peer_slots), source rows read through desc->peer_gathered
static int bwd_entry(const pna_agg_t* d, const void* grad_out, int64_t ld_grad_out, float* grad_gathered, int64_t ld_grad_gathered,
                     float* grad_row_bias, int64_t ld_grad_row_bias, float* coef, int64_t ld_coef, int32_t coef_c1,
                     pna_stream_t stream, float* grad_slots = nullptr, int64_t ld_grad_slots = 0, int32_t f_begin = 0,
                     int32_t f_count = 0, bool peer = false, const float* sw = nullptr, const float* sdf = nullptr) {
  PNA_REQUIRE(d != nullptr, PNA_ERR_BAD_ARG, "pna_aggregate_bwd: null descriptor");
  PNA_REQUIRE(d->n_rows >= 0 && d->n_feat > 0 && d->n_towers > 0 && d->n_feat % d->n_towers == 0, PNA_ERR_BAD_ARG,
              "pna_aggregate_bwd: bad sizes");
  PNA_REQUIRE(d->n_aggr >= 1 && d->n_aggr <= PNA_MAX_AGGR && d->n_scalers >= 1 && d->n_scalers <= PNA_MAX_SCALERS, PNA_ERR_BAD_ARG,
              "pna_aggregate_bwd: n_aggr / n_scalers out of range");
  PNA_REQUIRE(d->dtype == PNA_F32 || d->dtype == PNA_BF16, PNA_ERR_UNSUPPORTED, "pna_aggregate_bwd: dtype %d", d->dtype);
  const bool slots = grad_slots != nullptr;
  if (slots) {   // slabs start and (but for the last) end on a 16-byte boundary of the element type
    const int al = d->dtype == PNA_F32 ? 4 : 8;
    PNA_REQUIRE(f_begin >= 0 && f_count >= 1 && (long long)f_begin + f_count <= d->n_feat && f_begin % al == 0 &&
                    (f_count % al == 0 || f_begin + f_count == d->n_feat),
                PNA_ERR_BAD_ARG, "pna_aggregate_bwd_slots: bad feature slab [%d, +%d) of %d features", f_begin, f_count, d->n_feat);
    PNA_REQUIRE(ld_grad_slots >= f_count, PNA_ERR_BAD_ARG, "pna_aggregate_bwd_slots: ld_grad_slots < f_count");
  }
  const bool moments = moment_orders(d->aggr_codes, d->n_aggr) != 0;
  // a moment's per-slot gradient is a polynomial of degree k-1 in m, not the c0 + c1 * m the coefficient rows regroup
  PNA_REQUIRE(!moments || !coef, PNA_ERR_UNSUPPORTED,
              "pna_aggregate_bwd_coef: moment aggregators have no coefficient form; use pna_aggregate_bwd or pna_aggregate_bwd_slots");
  PNA_REQUIRE(!moments || (!d->peer_gathered && !d->row_ids), PNA_ERR_UNSUPPORTED,
              "pna_aggregate_bwd: moment aggregators are not available with peer_gathered or row_ids");
  const unsigned weighted = weighted_codes(d->aggr_codes, d->n_aggr);
  const bool addons = moments || weighted;
  // softmax / softmin: p_j (1 + m_j - y) is not linear in m_j; normalised_mean's weight depends on the source's degree
  PNA_REQUIRE(!weighted || !coef, PNA_ERR_UNSUPPORTED,
              "pna_aggregate_bwd_coef: softmax / softmin / normalised_mean have no coefficient form; use pna_aggregate_bwd or "
              "pna_aggregate_bwd_slots");
  PNA_REQUIRE(!weighted || (!d->peer_gathered && !d->row_ids), PNA_ERR_UNSUPPORTED,
              "pna_aggregate_bwd: softmax / softmin / normalised_mean are not available with peer_gathered or row_ids");
  PNA_REQUIRE(!((weighted >> (PNA_AGGR_NORMALISED_MEAN - PNA_AGGR_SOFTMAX)) & 1u) || d->col || d->degree_col,
              PNA_ERR_UNSUPPORTED, "pna_aggregate_bwd: normalised_mean needs col or degree_col (the source of every slot)");
  // the *_weighted entry points (they have no coefficient or peer-memory form: coef == NULL and peer == false here)
  const bool adj_weight = sw || sdf;
  if (adj_weight) {
    for (int a = 0; a < d->n_aggr; ++a)
      PNA_REQUIRE(adj_weight_code((d->aggr_codes >> (4 * a)) & 15u), PNA_ERR_UNSUPPORTED,
                  "pna_aggregate_bwd: slot_weight / scaler_degree_f take sum, mean, min, max, var and std only");
    PNA_REQUIRE(!d->peer_gathered && !d->row_ids, PNA_ERR_UNSUPPORTED,
                "pna_aggregate_bwd: slot_weight / scaler_degree_f are not available with peer_gathered or row_ids");
  }
  if (d->n_rows == 0) return PNA_OK;
  PNA_REQUIRE(d->gathered && d->rowptr && grad_out && (slots || grad_gathered), PNA_ERR_BAD_ARG, "pna_aggregate_bwd: null pointer");
  if (peer) {
    PNA_REQUIRE(d->peer_gathered != nullptr, PNA_ERR_BAD_ARG, "pna_aggregate_bwd_peer_slots: no peer_gathered table");
    PNA_REQUIRE(d->peer_shift >= 1 && d->peer_shift <= 30, PNA_ERR_BAD_ARG, "pna_aggregate_bwd_peer_slots: peer_shift out of range");
    PNA_REQUIRE(d->row_ids == nullptr, PNA_ERR_UNSUPPORTED, "pna_aggregate_bwd_peer_slots: row_ids are not available");
    PNA_REQUIRE(d->col != nullptr, PNA_ERR_UNSUPPORTED,
                "pna_aggregate_bwd_peer_slots: col is required (it names the owner and row of every source)");
  } else {
    PNA_REQUIRE(d->peer_gathered == nullptr, PNA_ERR_UNSUPPORTED,
                "pna_aggregate_bwd: peer-memory graphs have pna_aggregate_bwd_peer_slots only");
  }
  PNA_REQUIRE(d->ld_gathered < 0x3fffffffll, PNA_ERR_UNSUPPORTED, "pna_aggregate_bwd: row pitch too large");
  PNA_REQUIRE(d->split_threshold >= 2, PNA_ERR_BAD_ARG, "pna_aggregate_bwd: bad split threshold");
  if (d->n_hubs > 0)
    PNA_REQUIRE(d->hub_info && d->chunk_items && d->hub_partials && d->chunk_edges >= 1, PNA_ERR_BAD_ARG,
                "pna_aggregate_bwd: split rows need hub_info, chunk_items and hub_partials ((n_chunks + n_hubs) * 6 * n_feat floats)");

  BParams b;
  memset(&b, 0, sizeof(b));
  KParams& p = b.k;
  p.x = d->gathered; p.ldx = d->ld_gathered;
  p.rowptr = d->rowptr; p.col = d->col;
  p.bias = d->row_bias; p.ldb = d->ld_row_bias;
  p.n_rows = d->n_rows;
  p.F = d->n_feat; p.T = d->n_towers; p.Ft = d->n_feat / d->n_towers;
  p.has_self = d->self_feat ? 1 : 0;
  p.nA = d->n_aggr; p.nS = d->n_scalers; p.scodes = d->scaler_codes;
  p.acodes = addons ? strip_addons(d->aggr_codes, d->n_aggr) : d->aggr_codes;   // the add-on kernels add their term
  p.Wt = (p.has_self + p.nA * p.nS) * p.Ft;
  p.avg_log = d->avg_log; p.avg_lin = d->avg_lin;
  p.flags = d->flags; p.split = d->split_threshold; p.chunk = d->chunk_edges;
  p.hub_info = d->hub_info; p.n_hubs = d->n_hubs; p.chunk_items = d->chunk_items; p.n_chunks = d->n_chunks;
  p.partials = d->hub_partials;
  p.sdeg = d->scaler_degree;
  if (peer) { p.peer_x = reinterpret_cast<const void* const*>(d->peer_gathered); p.peer_shift = d->peer_shift; }
  b.go = grad_out; b.ldgo = ld_grad_out;
  b.gg = grad_gathered; b.ldgg = ld_grad_gathered;
  b.gb = grad_row_bias; b.ldgb = ld_grad_row_bias;
  PNA_REQUIRE(b.ldgo >= (long long)p.T * p.Wt, PNA_ERR_BAD_ARG, "pna_aggregate_bwd: ld_grad_out too small");
  b.vec_atomics = al16(grad_gathered) && (ld_grad_gathered % 4 == 0);
  if (coef) {
    PNA_REQUIRE(d->col != nullptr, PNA_ERR_UNSUPPORTED, "pna_aggregate_bwd_coef: per-edge messages (col == NULL) have no shared sources");
    PNA_REQUIRE(coef_c1 >= p.F && ld_coef >= (long long)coef_c1 + p.F, PNA_ERR_BAD_ARG,
                "pna_aggregate_bwd_coef: coefficient rows need c1_column >= n_feat and ld_coef >= c1_column + n_feat");
    b.coef = coef; b.ldc = ld_coef; b.coef_c1 = coef_c1;
    b.coef_vec = al16(coef) && (ld_coef % 4 == 0) && (coef_c1 % 4 == 0);
  }
  if (slots) {
    b.gs = grad_slots; b.ldgs = ld_grad_slots;
    b.f0 = f_begin; b.f1 = f_begin + f_count;
    b.gs_vec = al16(grad_slots) && (ld_grad_slots % 4 == 0);
  }

  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool f32 = d->dtype == PNA_F32;
  if (adj_weight) {   // every slot's gradient from the weighted kernels alone
    AWBParams q;
    q.a = adj_weight_params(d, sw, sdf);
    q.b = b;
    MParams& mp = q.a.m;
    mp.go = grad_out; mp.ldgo = ld_grad_out;
    mp.gb = grad_row_bias; mp.ldgb = ld_grad_row_bias;
    if (slots) {
      mp.gs = grad_slots; mp.ldgs = ld_grad_slots;
      mp.f0 = f_begin; mp.f1 = f_begin + f_count;
      return f32 ? launch_adj_weight_bwd<float, true>(q, st) : launch_adj_weight_bwd<__nv_bfloat16, true>(q, st);
    }
    mp.gg = grad_gathered; mp.ldgg = ld_grad_gathered;
    return f32 ? launch_adj_weight_bwd<float, false>(q, st) : launch_adj_weight_bwd<__nv_bfloat16, false>(q, st);
  }
  const int esz = d->dtype == PNA_F32 ? 4 : 2;
  const int vec = 16 / esz;
  bool vec_ok = (p.Ft % vec == 0) && al16(p.x) && al16(grad_out) && (p.ldx % vec == 0) && (b.ldgo % vec == 0);
  if (p.bias) vec_ok = vec_ok && al16(p.bias) && (p.ldb % vec == 0);
  int rc;
  if (peer) {
    if (f32) rc = vec_ok ? launch_bwd_typed<float, 4, true, true>(b, st) : launch_bwd_typed<float, 1, true, true>(b, st);
    else rc = vec_ok ? launch_bwd_typed<__nv_bfloat16, 8, true, true>(b, st) : launch_bwd_typed<__nv_bfloat16, 1, true, true>(b, st);
  } else if (slots) {
    if (f32) rc = vec_ok ? launch_bwd_typed<float, 4, true>(b, st) : launch_bwd_typed<float, 1, true>(b, st);
    else rc = vec_ok ? launch_bwd_typed<__nv_bfloat16, 8, true>(b, st) : launch_bwd_typed<__nv_bfloat16, 1, true>(b, st);
  } else {
    if (f32) rc = vec_ok ? launch_bwd_typed<float, 4, false>(b, st) : launch_bwd_typed<float, 1, false>(b, st);
    else rc = vec_ok ? launch_bwd_typed<__nv_bfloat16, 8, false>(b, st) : launch_bwd_typed<__nv_bfloat16, 1, false>(b, st);
  }
  if (rc != PNA_OK || !addons) return rc;
  MParams mp = moment_params(d);
  mp.go = grad_out; mp.ldgo = ld_grad_out;
  mp.gb = grad_row_bias; mp.ldgb = ld_grad_row_bias;
  if (slots) {
    mp.gs = grad_slots; mp.ldgs = ld_grad_slots;
    mp.f0 = f_begin; mp.f1 = f_begin + f_count;
    return f32 ? launch_addons_bwd<float, true>(d, mp, st) : launch_addons_bwd<__nv_bfloat16, true>(d, mp, st);
  }
  mp.gg = grad_gathered; mp.ldgg = ld_grad_gathered;
  return f32 ? launch_addons_bwd<float, false>(d, mp, st) : launch_addons_bwd<__nv_bfloat16, false>(d, mp, st);
}

extern "C" int pna_aggregate_bwd(const pna_agg_t* d, const void* grad_out, int64_t ld_grad_out, float* grad_gathered,
                                 int64_t ld_grad_gathered, float* grad_row_bias, int64_t ld_grad_row_bias, pna_stream_t stream) {
  return bwd_entry(d, grad_out, ld_grad_out, grad_gathered, ld_grad_gathered, grad_row_bias, ld_grad_row_bias, nullptr, 0, 0, stream);
}

extern "C" int pna_aggregate_bwd_slots(const pna_agg_t* d, const void* grad_out, int64_t ld_grad_out, int32_t f_begin, int32_t f_count,
                                       float* grad_slots, int64_t ld_grad_slots, float* grad_row_bias, int64_t ld_grad_row_bias,
                                       pna_stream_t stream) {
  PNA_REQUIRE(grad_slots != nullptr, PNA_ERR_BAD_ARG, "pna_aggregate_bwd_slots: null grad_slots");
  return bwd_entry(d, grad_out, ld_grad_out, nullptr, 0, grad_row_bias, ld_grad_row_bias, nullptr, 0, 0, stream, grad_slots,
                   ld_grad_slots, f_begin, f_count);
}

extern "C" int pna_aggregate_bwd_weighted(const pna_agg_t* d, const float* slot_weight, const float* scaler_degree_f,
                                          const void* grad_out, int64_t ld_grad_out, float* grad_gathered, int64_t ld_grad_gathered,
                                          float* grad_row_bias, int64_t ld_grad_row_bias, pna_stream_t stream) {
  return bwd_entry(d, grad_out, ld_grad_out, grad_gathered, ld_grad_gathered, grad_row_bias, ld_grad_row_bias, nullptr, 0, 0, stream,
                   nullptr, 0, 0, 0, false, slot_weight, scaler_degree_f);
}

extern "C" int pna_aggregate_bwd_slots_weighted(const pna_agg_t* d, const float* slot_weight, const float* scaler_degree_f,
                                                const void* grad_out, int64_t ld_grad_out, int32_t f_begin, int32_t f_count,
                                                float* grad_slots, int64_t ld_grad_slots, float* grad_row_bias,
                                                int64_t ld_grad_row_bias, pna_stream_t stream) {
  PNA_REQUIRE(grad_slots != nullptr, PNA_ERR_BAD_ARG, "pna_aggregate_bwd_slots_weighted: null grad_slots");
  return bwd_entry(d, grad_out, ld_grad_out, nullptr, 0, grad_row_bias, ld_grad_row_bias, nullptr, 0, 0, stream, grad_slots,
                   ld_grad_slots, f_begin, f_count, false, slot_weight, scaler_degree_f);
}

extern "C" int pna_aggregate_bwd_peer_slots(const pna_agg_t* d, const void* grad_out, int64_t ld_grad_out, int32_t f_begin,
                                            int32_t f_count, float* grad_slots, int64_t ld_grad_slots, float* grad_row_bias,
                                            int64_t ld_grad_row_bias, pna_stream_t stream) {
  PNA_REQUIRE(grad_slots != nullptr, PNA_ERR_BAD_ARG, "pna_aggregate_bwd_peer_slots: null grad_slots");
  return bwd_entry(d, grad_out, ld_grad_out, nullptr, 0, grad_row_bias, ld_grad_row_bias, nullptr, 0, 0, stream, grad_slots,
                   ld_grad_slots, f_begin, f_count, true);
}

extern "C" int pna_aggregate_bwd_coef(const pna_agg_t* d, const void* grad_out, int64_t ld_grad_out, float* coef, int64_t ld_coef,
                                      int32_t c1_column, float* grad_gathered, int64_t ld_grad_gathered, float* grad_row_bias,
                                      int64_t ld_grad_row_bias, pna_stream_t stream) {
  PNA_REQUIRE(coef != nullptr, PNA_ERR_BAD_ARG, "pna_aggregate_bwd_coef: null coefficient buffer");
  return bwd_entry(d, grad_out, ld_grad_out, grad_gathered, ld_grad_gathered, grad_row_bias, ld_grad_row_bias, coef, ld_coef,
                   c1_column, stream);
}

extern "C" int pna_aggregate_bwd_combine(const float* coef_sums, int64_t ld_sums, int32_t c1_column, const void* gathered,
                                         int64_t ld_gathered, int32_t dtype, float* grad_gathered, int64_t ld_grad_gathered,
                                         int64_t n_src, int32_t n_feat, pna_stream_t stream) {
  PNA_REQUIRE(n_src >= 0 && n_feat > 0 && c1_column >= n_feat, PNA_ERR_BAD_ARG, "pna_aggregate_bwd_combine: bad sizes");
  PNA_REQUIRE(dtype == PNA_F32 || dtype == PNA_BF16, PNA_ERR_UNSUPPORTED, "pna_aggregate_bwd_combine: dtype %d", dtype);
  if (n_src == 0) return PNA_OK;
  PNA_REQUIRE(coef_sums && gathered && grad_gathered, PNA_ERR_BAD_ARG, "pna_aggregate_bwd_combine: null pointer");
  PNA_REQUIRE(ld_sums >= (long long)c1_column + n_feat && ld_gathered >= n_feat && ld_grad_gathered >= n_feat, PNA_ERR_BAD_ARG,
              "pna_aggregate_bwd_combine: row pitch too small");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total = n_src * (long long)n_feat;
  int dev = 0, sms = 0;
  PNA_CUDA_TRY(cudaGetDevice(&dev));
  PNA_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  long long blocks = (total + 255) / 256;
  if (blocks > sms * 8LL) blocks = sms * 8LL;    // grid-stride: 8 CTAs of 256 threads fill an SM (2048 threads)
  if (dtype == PNA_F32)
    k_bwd_combine<float><<<(unsigned)blocks, 256, 0, st>>>(coef_sums, ld_sums, c1_column, static_cast<const float*>(gathered),
                                                           ld_gathered, grad_gathered, ld_grad_gathered, n_src, n_feat);
  else
    k_bwd_combine<__nv_bfloat16><<<(unsigned)blocks, 256, 0, st>>>(coef_sums, ld_sums, c1_column,
                                                                   static_cast<const __nv_bfloat16*>(gathered), ld_gathered,
                                                                   grad_gathered, ld_grad_gathered, n_src, n_feat);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}
