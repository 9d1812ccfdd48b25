// Device-side building blocks of the PNA aggregation (forward).
//
// Work decomposition (GPU-first, not a translation of torch_scatter's atomics):
//   * destination rows are independent; a row is owned by a group of G lanes (G = 1..32, a power of two),
//     32/G rows per warp.  Lanes map to FEATURE columns: lane g owns the 16-byte chunks g, g+G, .. (K of them), so
//     every gathered neighbour row is read as fully coalesced 128-bit loads and NO cross-lane reduction is needed;
//   * the slots of a row are walked in CSR order, U at a time (U independent 128-bit loads in flight per lane),
//     and accumulated sequentially in fp32 with unfused mul/add -- the same order and rounding as the reference's
//     CPU scatter_add path, so rows below the split threshold reproduce it bit for bit up to log/div rounding;
//   * rows at/above the split threshold ("hubs", power-law graphs) are cut into chunks of `chunk` slots; each chunk
//     is reduced by its own lane group into fp32 partials, and a finalize pass merges a hub's partials in chunk
//     order (deterministic, no atomics on the output) and runs the same epilogue;
//   * the epilogue computes mean / var / std and the degree scalers in registers and writes the S*A row segments
//     with streaming 128-bit stores, in the reference's scaler-major column order.
#pragma once
#include "common.cuh"
#include <math_constants.h>

namespace pna {

struct KParams {
  const void* x; long long ldx;
  const int* rowptr; const int* col;
  const void* bias; long long ldb;
  const void* self; long long lds; long long self_tstride;
  void* out; long long ldo;
  long long n_rows;
  int F, T, Ft, Wt, has_self;
  int nA, nS; unsigned acodes, scodes;
  float avg_log, avg_lin;
  unsigned flags;
  int split, chunk;
  const int* hub_info; const int* chunk_items; long long n_hubs, n_chunks;
  float* partials;
  int* hub_done;           // nullable: per split row 8 group counters + 1 row counter (finalize folded into the stream kernel)
  const int* row_ids; long long n_row_ids;
  const int* lrowptr; const int* ldeg; const int* lcol; const int* part; int n_part;   // light view (nullable)
  long long n_view_rows;   // > n_rows: view rows n_rows + c are chunk pseudo-rows reduced into partials[c]
  int* work_ctr;           // nullable: counter through which the last partitions are handed out dynamically
  int n_static;            // partitions [0, n_static) are dealt out statically (set by the launcher)
  int hub_merged;          // 1: every split row's total already sits in its first partial slot (k_hub_tree ran)
  const int* sdeg;         // nullable [n_rows]: degree seen by the scalers (default: the in-degree of the row)
  const void* const* peer_x; int peer_shift;   // multi-GPU: x of every rank (NVLink peer pointers), col = owner << shift | row
};

// First element of gathered row `c`.  Single GPU: x + c*ldx.  Destination-partitioned multi-GPU graph: `c` encodes
// (owner rank, row on that rank) and the row is read straight from the owner's HBM over NVLink (peer pointer) --
// the gather and the "halo exchange" are the same load, there is no pack / all-to-all / unpack step.
// row `c` of the local buffer: one unsigned 32 x 32 -> 64-bit multiply-add (pna_aggregate_fwd checks ldx * sizeof(T) < 2^32)
template <typename T>
__device__ __forceinline__ const T* local_row(const KParams& p, int c) {
  return reinterpret_cast<const T*>(static_cast<const char*>(p.x) + (unsigned long long)(unsigned)c * ((unsigned)p.ldx * (unsigned)sizeof(T)));
}

template <typename T>
__device__ __forceinline__ const T* gathered_row(const KParams& p, int c) {
  if (p.peer_x == nullptr) return local_row<T>(p, c);
  const unsigned owner = (unsigned)c >> p.peer_shift;
  const int r = c & ((1 << p.peer_shift) - 1);
  const unsigned long long base = __ldg(reinterpret_cast<const unsigned long long*>(p.peer_x) + owner);
  return reinterpret_cast<const T*>(base) + (long long)r * (int)p.ldx;
}

// Compile-time aggregator / scaler lists for the configurations the reference's configs use; Dynamic reads them from
// KParams.  A static list turns the epilogue into straight-line code (no uniform branches, no selects).
struct CfgDynamic {
  static constexpr bool kStatic = false;
  static constexpr int NA = PNA_MAX_AGGR, NS = PNA_MAX_SCALERS;
  static constexpr unsigned ACODES = 0, SCODES = 0;
};
template <int NA_, unsigned ACODES_, int NS_, unsigned SCODES_>
struct CfgStatic {
  static constexpr bool kStatic = true;
  static constexpr int NA = NA_, NS = NS_;
  static constexpr unsigned ACODES = ACODES_, SCODES = SCODES_;
};
// "mean max min std" x "identity amplification attenuation" (realworld_benchmark/configs/*.json) and the
// "mean min max std" order of models/pytorch_geometric/example.py:33
using CfgMeanMaxMinStd = CfgStatic<4, (1u) | (3u << 4) | (2u << 8) | (5u << 12), 3, (0u) | (1u << 4) | (2u << 8)>;
// the same aggregators with the identity scaler only: the compact [N, A*F] tensor of the scaled post-linear path
using CfgMeanMaxMinStdId = CfgStatic<4, (1u) | (3u << 4) | (2u << 8) | (5u << 12), 1, 0u>;
using CfgMeanMinMaxStd = CfgStatic<4, (1u) | (2u << 4) | (3u << 8) | (5u << 12), 3, (0u) | (1u << 4) | (2u << 8)>;

// ---- fp32 pair arithmetic.  Hopper has no packed fp32 add/multiply, so a pair is two IEEE-rounded scalar operations;
// __fadd_rn / __fmul_rn are never contracted into an FMA, so the accumulation stays bit-identical to the reference's
// "sum += m; sumsq += m*m" sequence (the product is rounded before it is added).
__device__ __forceinline__ float2 add2_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2_rn(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 sqr2(float2 m) { return make_float2(__fmul_rn(m.x, m.x), __fmul_rn(m.y, m.y)); }
__device__ __forceinline__ float min3f(float a, float b, float c) { return fminf(fminf(a, b), c); }
__device__ __forceinline__ float max3f(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

template <int VEC>
struct Acc {
  float sum[VEC], sq[VEC], mn[VEC], mx[VEC];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int v = 0; v < VEC; ++v) { sum[v] = 0.f; sq[v] = 0.f; mn[v] = CUDART_INF_F; mx[v] = -CUDART_INF_F; }
  }
  // one neighbour row m (BIAS: m += bias first): sum += m; sq += m*m (product rounded, then added); min; max
  template <bool BIAS>
  __device__ __forceinline__ void add1(float (&m)[VEC], const float (&bias)[VEC]) {
    if constexpr (VEC % 2 == 0) {
#pragma unroll
      for (int i = 0; i < VEC; i += 2) {
        float2 mm = make_float2(m[i], m[i + 1]);
        if (BIAS) mm = add2_rn(mm, make_float2(bias[i], bias[i + 1]));
        const float2 s = add2_rn(make_float2(sum[i], sum[i + 1]), mm);
        const float2 q = add2_rn(make_float2(sq[i], sq[i + 1]), sqr2(mm));
        sum[i] = s.x; sum[i + 1] = s.y; sq[i] = q.x; sq[i + 1] = q.y;
        mn[i] = fminf(mn[i], mm.x); mn[i + 1] = fminf(mn[i + 1], mm.y);
        mx[i] = fmaxf(mx[i], mm.x); mx[i + 1] = fmaxf(mx[i + 1], mm.y);
      }
    } else {
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        float mm = m[i];
        if (BIAS) mm = __fadd_rn(mm, bias[i]);
        sum[i] = __fadd_rn(sum[i], mm);
        sq[i] = __fadd_rn(sq[i], __fmul_rn(mm, mm));
        mn[i] = fminf(mn[i], mm);
        mx[i] = fmaxf(mx[i], mm);
      }
    }
  }
  // two neighbour rows, a then b (slot order is kept for the sums; min/max take both at once)
  template <bool BIAS>
  __device__ __forceinline__ void add2(float (&a)[VEC], float (&b)[VEC], const float (&bias)[VEC]) {
    if constexpr (VEC % 2 == 0) {
#pragma unroll
      for (int i = 0; i < VEC; i += 2) {
        float2 ma = make_float2(a[i], a[i + 1]), mb = make_float2(b[i], b[i + 1]);
        if (BIAS) {
          const float2 bb = make_float2(bias[i], bias[i + 1]);
          ma = add2_rn(ma, bb); mb = add2_rn(mb, bb);
        }
        float2 s = add2_rn(make_float2(sum[i], sum[i + 1]), ma);
        s = add2_rn(s, mb);
        float2 q = add2_rn(make_float2(sq[i], sq[i + 1]), sqr2(ma));
        q = add2_rn(q, sqr2(mb));
        sum[i] = s.x; sum[i + 1] = s.y; sq[i] = q.x; sq[i + 1] = q.y;
        mn[i] = min3f(mn[i], ma.x, mb.x); mn[i + 1] = min3f(mn[i + 1], ma.y, mb.y);
        mx[i] = max3f(mx[i], ma.x, mb.x); mx[i + 1] = max3f(mx[i + 1], ma.y, mb.y);
      }
    } else {
      add1<BIAS>(a, bias);
      add1<BIAS>(b, bias);
    }
  }
};

// Which feature columns a lane owns and where they land in the output row.
template <int VEC, int G, int K>
struct FeatMap {
  int f[K];     // first feature column of chunk k
  int ooff[K];  // output column of (scaler 0, aggregator 0) for that chunk
  int soff[K];  // output column of the self block for that chunk
  int sin[K];   // column inside self_feat
  bool ok[K];
  __device__ __forceinline__ void init(const KParams& p, int gl, int fblock) {
    if (p.T == 1 && !p.has_self) {   // one tower, no self block: the output column of a feature is the feature
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int ff = fblock + (gl + k * G) * VEC;
        ok[k] = ff < p.F;
        f[k] = ok[k] ? ff : 0;
        ooff[k] = f[k]; soff[k] = 0; sin[k] = 0;
      }
      return;
    }
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int ff = fblock + (gl + k * G) * VEC;
      ok[k] = ff < p.F;
      const int fc = ok[k] ? ff : 0;
      const int t = fc / p.Ft;
      const int ft = fc - t * p.Ft;
      f[k] = fc;
      soff[k] = t * p.Wt + ft;
      ooff[k] = soff[k] + p.has_self * p.Ft;
      sin[k] = (int)(t * p.self_tstride) + ft;
    }
  }
};

// One batch of U slots starting at e.  FULL: all U slots exist (no predicates in the instruction stream).
template <typename T, int VEC, int G, int K, int U, bool FULL>
__device__ __forceinline__ void accumulate_batch(const KParams& p, const int* __restrict__ col,
                                                 const FeatMap<VEC, G, K>& fm, int e, int end,
                                                 const float (&bias)[K][VEC], bool has_bias, Acc<VEC> (&acc)[K]) {
  int src[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int s = e + u;
    if (FULL) src[u] = col ? __ldg(col + s) : s;
    else src[u] = (s < end) ? (col ? __ldg(col + s) : s) : -1;
  }
  typename Io<T, VEC>::Raw raw[U][K];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    if (FULL || src[u] >= 0) {
#pragma unroll
      for (int k = 0; k < K; ++k)
        if (fm.ok[k]) raw[u][k] = Io<T, VEC>::load_raw(gathered_row<T>(p, src[u]) + fm.f[k]);
    }
  }
  static_assert(U % 2 == 0, "slots are reduced two at a time");
#pragma unroll
  for (int u = 0; u < U; u += 2) {
    const bool v0 = FULL || src[u] >= 0, v1 = FULL || src[u + 1] >= 0;
    if (v0) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        if (fm.ok[k]) {
          float m0[VEC], m1[VEC];
          Io<T, VEC>::unpack(raw[u][k], m0);
          if (v1) {
            Io<T, VEC>::unpack(raw[u + 1][k], m1);
            if (has_bias) acc[k].template add2<true>(m0, m1, bias[k]); else acc[k].template add2<false>(m0, m1, bias[k]);
          } else {
            if (has_bias) acc[k].template add1<true>(m0, bias[k]); else acc[k].template add1<false>(m0, bias[k]);
          }
        }
      }
    }
  }
}

// Reduce slots [beg, end) of one row into acc, U slots per step.
template <typename T, int VEC, int G, int K, int U>
__device__ __forceinline__ void accumulate_slots(const KParams& p, const FeatMap<VEC, G, K>& fm, int beg, int end,
                                                 const float (&bias)[K][VEC], bool has_bias, Acc<VEC> (&acc)[K]) {
  const int* __restrict__ col = p.col;
  int e = beg;
  for (; e + U <= end; e += U) accumulate_batch<T, VEC, G, K, U, true>(p, col, fm, e, end, bias, has_bias, acc);
  if (e < end) accumulate_batch<T, VEC, G, K, U, false>(p, col, fm, e, end, bias, has_bias, acc);
}

// Correctly rounded x / d for MANY numerators and ONE divisor (the in-degree): r = RN(1/d) once, then per numerator
// q = RN(x r), e = x - q d (exact, one FMA), x/d = RN(q + e r) -- Markstein's theorem: with a correctly rounded reciprocal and
// q within one ulp of the quotient the corrected q is the correctly rounded quotient (the sequence IEEE division itself ends
// with).  3 instructions per quotient instead of the ~9 of div.rn.f32; the same bits (tests/test_gpu_parity.py compares it
// with the CPU's division on random and adversarial operands).  Quotients below the normal range may differ by one
// subnormal ulp (1.4e-45).
struct SharedDivisor {
  float d, r;
#ifdef __CUDA_ARCH__   // (the host pass of nvcc parses this non-template struct but has no device intrinsics)
  __device__ __forceinline__ explicit SharedDivisor(float d_) : d(d_), r(__frcp_rn(d_)) {}
  __device__ __forceinline__ float operator()(float x) const {
    const float q = __fmul_rn(x, r);
    const float e = __fmaf_rn(-q, d, x);
    return __fmaf_rn(e, r, q);
  }
#else
  explicit SharedDivisor(float d_) : d(d_), r(1.0f / d_) {}
  float operator()(float x) const { return x / d; }
#endif
};

// A row without in-edges (PyG semantics, aggregators.py:13-32 / scalers.py:8-29 at d = 0): mean = min = max = sum = var = 0,
// std = sqrt(1e-5); amplification = log(1)/delta = 0, attenuation = linear-inverse = 1, linear = 0 -- every output segment is
// one constant splat.  Power-law graphs consist mostly of such rows (94 % in config 5), so they get their own short path.
// `ds0` = the scaler factors of in-degree 0 (from the kernel's shared-memory table: no division on this path).
template <typename T, int VEC, int G, int K, typename Cfg>
__device__ __forceinline__ void finalize_isolated_row(const KParams& p, const FeatMap<VEC, G, K>& fm, long long row,
                                                      const DegScales& ds0) {
  const int nA = Cfg::kStatic ? Cfg::NA : p.nA, nS = Cfg::kStatic ? Cfg::NS : p.nS;
  const unsigned acodes = Cfg::kStatic ? Cfg::ACODES : p.acodes, scodes = Cfg::kStatic ? Cfg::SCODES : p.scodes;
  const bool zero_all = (p.flags & PNA_FLAG_ZERO_ISOLATED) != 0;
  const float sd0 = __fsqrt_rn(__fadd_rn(0.0f, 1e-5f));      // constant-folded
  T* __restrict__ orow = static_cast<T*>(p.out) + row * p.ldo;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (!fm.ok[k]) continue;
    if (p.self) {
      float sv[VEC];
      Io<T, VEC>::load(static_cast<const T*>(p.self) + row * p.lds + fm.sin[k], sv);
      Io<T, VEC>::store(orow + fm.soff[k], sv);
    }
    T* __restrict__ obase = orow + fm.ooff[k];
#pragma unroll
    for (int a = 0; a < Cfg::NA; ++a) {
      if (!Cfg::kStatic && a >= nA) break;
      const unsigned ac = (acodes >> (4 * a)) & 15u;
      if (ac == PNA_AGGR_SKIP) continue;
      const float base = (ac == PNA_AGGR_STD && !zero_all) ? sd0 : 0.0f;
#pragma unroll
      for (int s = 0; s < Cfg::NS; ++s) {
        if (!Cfg::kStatic && s >= nS) break;
        const unsigned sc = (scodes >> (4 * s)) & 15u;
        const float v = (sc == PNA_SCALE_IDENTITY) ? base : __fmul_rn(base, ds0.of(sc));
        float o[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) o[i] = v;
        Io<T, VEC>::store(obase + (s * nA + a) * p.Ft, o);
      }
    }
  }
}

// mean/var/std + scalers + the S*A streaming stores of one row; `ds` = the row's degree-scaler factors.
template <typename T, int VEC, int G, int K, typename Cfg>
__device__ __forceinline__ void finalize_row_ds(const KParams& p, const FeatMap<VEC, G, K>& fm, long long row, int deg,
                                                const DegScales& ds, const Acc<VEC> (&acc)[K]);

// mean/var/std + scalers + the S*A streaming stores of one row.
template <typename T, int VEC, int G, int K, typename Cfg>
__device__ __forceinline__ void finalize_row(const KParams& p, const FeatMap<VEC, G, K>& fm, long long row, int deg,
                                             const Acc<VEC> (&acc)[K]) {
  // unused factors are dead code under a static Cfg; the scalers' degree may be supplied separately (dense layer)
  const DegScales ds = deg_scales(p.sdeg ? __ldg(p.sdeg + row) : deg, p.avg_log, p.avg_lin);
  finalize_row_ds<T, VEC, G, K, Cfg>(p, fm, row, deg, ds, acc);
}

template <typename T, int VEC, int G, int K, typename Cfg>
__device__ __forceinline__ void finalize_row_ds(const KParams& p, const FeatMap<VEC, G, K>& fm, long long row, int deg,
                                                const DegScales& ds, const Acc<VEC> (&acc)[K]) {
  const bool iso = deg == 0;
  const float degf = (float)deg;
  const float cnt = iso ? 1.0f : degf;                     // count.clamp_(1)
  const SharedDivisor by_cnt(cnt);
  const bool zero_all = iso && (p.flags & PNA_FLAG_ZERO_ISOLATED);
  const int nA = Cfg::kStatic ? Cfg::NA : p.nA, nS = Cfg::kStatic ? Cfg::NS : p.nS;
  const unsigned acodes = Cfg::kStatic ? Cfg::ACODES : p.acodes, scodes = Cfg::kStatic ? Cfg::SCODES : p.scodes;
  const int Ft = p.Ft;
  T* __restrict__ orow = static_cast<T*>(p.out) + row * p.ldo;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (!fm.ok[k]) continue;
    if (p.self) {
      float sv[VEC];
      Io<T, VEC>::load(static_cast<const T*>(p.self) + row * p.lds + fm.sin[k], sv);
      Io<T, VEC>::store(orow + fm.soff[k], sv);
    }
    float mean[VEC], var[VEC], sd[VEC], mn[VEC], mx[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      mean[i] = by_cnt(acc[k].sum[i]);                                           // aggregators.py:13-14 (true divide)
      const float msq = by_cnt(acc[k].sq[i]);
      var[i] = __fsub_rn(msq, __fmul_rn(mean[i], mean[i]));                      // aggregators.py:25-28
      sd[i] = __fsqrt_rn(__fadd_rn(fmaxf(var[i], 0.0f), 1e-5f));                 // aggregators.py:31-32
      mn[i] = iso ? 0.0f : acc[k].mn[i];                                         // aggregators.py:17-22 (empty -> 0)
      mx[i] = iso ? 0.0f : acc[k].mx[i];
    }
    T* __restrict__ obase = orow + fm.ooff[k];
#pragma unroll
    for (int a = 0; a < Cfg::NA; ++a) {
      if (!Cfg::kStatic && a >= nA) break;
      const unsigned ac = (acodes >> (4 * a)) & 15u;
      if (ac == PNA_AGGR_SKIP) continue;
      float val[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        float r;
        switch (ac) {
          case PNA_AGGR_SUM: r = acc[k].sum[i]; break;
          case PNA_AGGR_MEAN: r = mean[i]; break;
          case PNA_AGGR_MIN: r = mn[i]; break;
          case PNA_AGGR_MAX: r = mx[i]; break;
          case PNA_AGGR_VAR: r = (p.flags & PNA_FLAG_RELU_VAR) ? fmaxf(var[i], 0.0f) : var[i]; break;
          default: r = sd[i]; break;
        }
        val[i] = zero_all ? 0.0f : r;
      }
#pragma unroll
      for (int s = 0; s < Cfg::NS; ++s) {
        if (!Cfg::kStatic && s >= nS) break;
        const unsigned sc = (scodes >> (4 * s)) & 15u;
        const float scale = ds.of(sc);
        float o[VEC];
        if constexpr (VEC % 2 == 0) {
#pragma unroll
          for (int i = 0; i < VEC; i += 2) {
            const float2 r = (sc == PNA_SCALE_IDENTITY) ? make_float2(val[i], val[i + 1])
                                                        : mul2_rn(make_float2(val[i], val[i + 1]), make_float2(scale, scale));
            o[i] = r.x; o[i + 1] = r.y;
          }
        } else {
#pragma unroll
          for (int i = 0; i < VEC; ++i) o[i] = (sc == PNA_SCALE_IDENTITY) ? val[i] : __fmul_rn(val[i], scale);
        }
        Io<T, VEC>::store(obase + (s * nA + a) * Ft, o);
      }
    }
  }
}

}  // namespace pna

#include "pna_aggregate_moments.cuh"
#include "pna_aggregate_weighted.cuh"
#include "pna_aggregate_adj_weight.cuh"
