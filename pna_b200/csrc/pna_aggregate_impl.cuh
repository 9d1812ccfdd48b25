// pna_aggregate_fwd kernels + launch dispatch (templates).  Instantiated per dtype / vector width in
// pna_aggregate_{f32,bf16}_{vec,scalar}.cu so the translation units compile in parallel.
#pragma once
#include "pna_aggregate.cuh"

namespace pna {

constexpr int kThreads = 256;  // 8 warps per CTA
// Resident CTAs per SM the register allocator must leave room for (latency hiding for the gather needs warps):
// 16 accumulators per 128-bit chunk per lane bound what is possible.
constexpr int min_blocks(int vec, int k) { return vec * k <= 4 ? 4 : (vec * k <= 8 ? 3 : (vec * k <= 16 ? 2 : 1)); }

// fp32 partials of a chunk: default cache policy (re-read by k_hub_finalize right after).
template <int VEC>
__device__ __forceinline__ void store_f32(float* p, const float (&v)[VEC]) {
  if constexpr (VEC % 4 == 0) {
#pragma unroll
    for (int i = 0; i < VEC; i += 4) *reinterpret_cast<float4*>(p + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) p[i] = v[i];
  }
}

// ---- rows below the split threshold: one lane group per row ------------------------------------------------
template <typename T, int VEC, int G, int K, int U, typename Cfg>
__global__ void __launch_bounds__(kThreads, min_blocks(VEC, K)) k_rows(const KParams p) {
  constexpr int RPW = 32 / G;
  const int lane = threadIdx.x & 31;
  const int gl = lane % G;
  const long long slot = ((long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * RPW + lane / G;
  long long row;
  if (p.row_ids) {
    if (slot >= p.n_row_ids) return;
    row = __ldg(p.row_ids + slot);
  } else {
    if (slot >= p.n_rows) return;
    row = slot;
  }
  const int beg = __ldg(p.rowptr + row), end = __ldg(p.rowptr + row + 1);
  const int deg = end - beg;
  if (deg >= p.split) return;  // hubs are handled by k_hub_chunks + k_hub_finalize

  FeatMap<VEC, G, K> fm;
  fm.init(p, gl, blockIdx.y * (G * VEC * K));
  Acc<VEC> acc[K];
  float bias[K][VEC];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    acc[k].init();
    if (p.bias && fm.ok[k]) Io<T, VEC>::load(static_cast<const T*>(p.bias) + row * p.ldb + fm.f[k], bias[k]);
  }
  accumulate_slots<T, VEC, G, K, U>(p, fm, beg, end, bias, p.bias != nullptr, acc);
  finalize_row<T, VEC, G, K, Cfg>(p, fm, row, deg, acc);
}

// ---- rows below the split threshold, tiled + software pipelined (the main kernel) ----------------------------
// A warp owns a TILE of consecutive row slots and walks it in steps of 32/G rows (one row per lane group):
//   * lane l loads rowptr[slot l] / rowptr[slot l + 1] once for the whole tile (coalesced); each step gets its
//     (begin, degree) by shuffle -- no dependent rowptr load per row;
//   * the column indices of a row are loaded by the lanes of its group in one coalesced access and handed out by
//     shuffle -- no per-edge index load;
//   * the loop is software pipelined: the column block of step j+1 is requested before row j is reduced, and the
//     first U neighbour rows of step j+1 are requested BEFORE the divide/sqrt/scale/store epilogue of row j, so the
//     gather latency of one row hides behind the arithmetic of the previous one.
// The slot order inside a row is unchanged (sequential fp32 accumulation in CSR order).
constexpr int kTiledThreads = 128;   // 4 warps per CTA: small CTAs retire early, keeping more warps resident
constexpr int kScaleLut = 256;       // in-degrees with precomputed scaler factors (rows at/above it: computed per row)

// degree-scaler factors of every in-degree below kScaleLut in shared memory: one read per row instead of logf + two IEEE
// divisions per lane per row.  The same device function (deg_scales) fills the table, so the factors keep their bits.
__device__ __forceinline__ void fill_scale_lut(float4* lut, const KParams& p, int tid, int nthreads) {
  for (int i = tid; i < kScaleLut; i += nthreads) {
    const DegScales d = deg_scales(i, p.avg_log, p.avg_lin);
    lut[i] = make_float4(d.amp, d.att, d.lin, d.ilin);
  }
  __syncthreads();
}
__device__ __forceinline__ DegScales scales_of_row(const float4* lut, const KParams& p, long long row, int deg) {
  const int sd = p.sdeg ? __ldg(p.sdeg + row) : deg;      // the scalers' degree may be supplied separately (dense layer)
  DegScales ds;
  if (sd < kScaleLut) {
    const float4 t = lut[sd];
    ds.amp = t.x; ds.att = t.y; ds.lin = t.z; ds.ilin = t.w;
  } else {
    ds = deg_scales(sd, p.avg_log, p.avg_lin);
  }
  return ds;
}
// resident 128-thread CTAs the register allocator leaves room for: 6 -> <= 80 registers (no spills at one 128-bit
// chunk per lane), i.e. 24 warps/SM, each with U gathers in flight underneath its epilogue
#ifndef PNA_TILED_MINB
#define PNA_TILED_MINB 6
#endif
constexpr int tiled_min_blocks(int vec, int k) { return vec * k <= 4 ? PNA_TILED_MINB : (vec * k <= 8 ? 4 : (vec * k <= 16 ? 3 : 2)); }

// PEER: sources may live on other ranks (owner << shift | row).  A template flag because the run-time test costs ~20
// predicated instructions per gathered row in both modes.
template <typename T, int VEC, int G, int K, int U, typename Cfg, bool BIAS, bool PEER = false>
__global__ void __launch_bounds__(kTiledThreads, tiled_min_blocks(VEC, K)) k_rows_tiled(const KParams p) {
  static_assert(U <= G && G % U == 0, "a batch must not straddle column blocks");
  constexpr int RPW = 32 / G;                            // rows per step
  constexpr int TR = (8 * RPW < 32) ? 8 * RPW : 32;      // row slots per tile (<= 32: one rowptr pair per lane)
  constexpr int S = TR / RPW;                            // steps per tile
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int gl = lane % G;
  const int grp = lane / G;
  const int gbase = grp * G;
  const long long n_slots = p.row_ids ? p.n_row_ids : p.n_rows;
  const long long s0 = ((long long)blockIdx.x * (kTiledThreads / 32) + (threadIdx.x >> 5)) * TR;
  __shared__ float4 s_scale_lut[kScaleLut];
  fill_scale_lut(s_scale_lut, p, threadIdx.x, kTiledThreads);
  if (s0 >= n_slots) return;   // warp-uniform

  // tile metadata: one slot per lane.  dg: in-degree, -1 = nothing to do here (padding slot or split row)
  int my_row = 0, rp = 0, dg = -1;
  if (lane < TR && s0 + lane < n_slots) {
    my_row = p.row_ids ? __ldg(p.row_ids + s0 + lane) : (int)(s0 + lane);
    rp = __ldg(p.rowptr + my_row);
    dg = __ldg(p.rowptr + my_row + 1) - rp;
    if (dg >= p.split) dg = -1;
    // masked view in row order (no chunk pseudo-rows): rows outside it are skipped
    if (p.ldeg && !p.row_ids && p.n_view_rows == p.n_rows) dg = __ldg(p.ldeg + my_row);
  }

  const int* __restrict__ col = p.col;
  constexpr bool has_bias = BIAS;
  FeatMap<VEC, G, K> fm;
  fm.init(p, gl, blockIdx.y * (G * VEC * K));

  // ---- stage step 0
  int row = __shfl_sync(FULL, my_row, grp);
  int beg = __shfl_sync(FULL, rp, grp);
  int deg = __shfl_sync(FULL, dg, grp);
  int d = deg > 0 ? deg : 0;
  int cv = (gl < d) ? (col ? __ldg(col + beg + gl) : beg + gl) : 0;
  float bias[BIAS ? K : 1][VEC];
  if (has_bias && deg >= 0) {
#pragma unroll
    for (int k = 0; k < K; ++k)
      if (fm.ok[k]) Io<T, VEC>::load(static_cast<const T*>(p.bias) + (long long)row * p.ldb + fm.f[k], bias[BIAS ? k : 0]);
  }
  typename Io<T, VEC>::Raw raw[U][K];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int src = __shfl_sync(FULL, cv, gbase + u);
    if (u < d) {
#pragma unroll
      for (int k = 0; k < K; ++k)
        if (fm.ok[k]) raw[u][k] = Io<T, VEC>::load_raw((PEER ? gathered_row<T>(p, src) : local_row<T>(p, src)) + fm.f[k]);
    }
  }

#pragma unroll 1
  for (int j = 0; j < S; ++j) {
    // ---- request metadata + first column block of step j+1
    const int tn = (j + 1) * RPW + grp;
    const bool more = (j + 1 < S);
    const int rowN = __shfl_sync(FULL, my_row, tn & 31);
    const int begN = __shfl_sync(FULL, rp, tn & 31);
    int degN = __shfl_sync(FULL, dg, tn & 31);
    if (!more) degN = -1;
    const int dN = degN > 0 ? degN : 0;
    const int cvN = (gl < dN) ? (col ? __ldg(col + begN + gl) : begN + gl) : 0;
    float biasN[BIAS ? K : 1][VEC];
    if (has_bias && degN >= 0) {
#pragma unroll
      for (int k = 0; k < K; ++k)
        if (fm.ok[k]) Io<T, VEC>::load(static_cast<const T*>(p.bias) + (long long)rowN * p.ldb + fm.f[k], biasN[BIAS ? k : 0]);
    }

    // ---- reduce row j: first batch is already in flight
    Acc<VEC> acc[K];
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k].init();
#pragma unroll
    for (int u = 0; u < U; u += 2) {
      if (u < d) {
#pragma unroll
        for (int k = 0; k < K; ++k)
          if (fm.ok[k]) {
            float m0[VEC], m1[VEC];
            Io<T, VEC>::unpack(raw[u][k], m0);
            if (u + 1 < d) {
              Io<T, VEC>::unpack(raw[u + 1][k], m1);
              acc[k].template add2<BIAS>(m0, m1, bias[BIAS ? k : 0]);
            } else {
              acc[k].template add1<BIAS>(m0, bias[BIAS ? k : 0]);
            }
          }
      }
    }
    // remaining slots of the longest row of this step (warp-uniform trip count; shorter rows are predicated off)
    const int dmax = __reduce_max_sync(FULL, d);
    for (int eb = U; eb < dmax; eb += U) {
      if ((eb % G) == 0) cv = (eb + gl < d) ? (col ? __ldg(col + beg + eb + gl) : beg + eb + gl) : 0;
      typename Io<T, VEC>::Raw r2[U][K];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int src = __shfl_sync(FULL, cv, gbase + ((eb + u) % G));
        if (eb + u < d) {
#pragma unroll
          for (int k = 0; k < K; ++k)
            if (fm.ok[k]) r2[u][k] = Io<T, VEC>::load_raw((PEER ? gathered_row<T>(p, src) : local_row<T>(p, src)) + fm.f[k]);
        }
      }
#pragma unroll
      for (int u = 0; u < U; u += 2) {
        if (eb + u < d) {
#pragma unroll
          for (int k = 0; k < K; ++k)
            if (fm.ok[k]) {
              float m0[VEC], m1[VEC];
              Io<T, VEC>::unpack(r2[u][k], m0);
              if (eb + u + 1 < d) {
                Io<T, VEC>::unpack(r2[u + 1][k], m1);
                acc[k].template add2<BIAS>(m0, m1, bias[BIAS ? k : 0]);
              } else {
                acc[k].template add1<BIAS>(m0, bias[BIAS ? k : 0]);
              }
            }
        }
      }
    }

    // ---- request the first batch of step j+1, then run the epilogue of row j underneath its latency
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int src = __shfl_sync(FULL, cvN, gbase + u);
      if (u < dN) {
#pragma unroll
        for (int k = 0; k < K; ++k)
          if (fm.ok[k]) raw[u][k] = Io<T, VEC>::load_raw((PEER ? gathered_row<T>(p, src) : local_row<T>(p, src)) + fm.f[k]);
      }
    }
    if (deg >= 0) finalize_row_ds<T, VEC, G, K, Cfg>(p, fm, (long long)row, deg, scales_of_row(s_scale_lut, p, row, deg), acc);

    row = rowN; beg = begN; deg = degN; d = dN; cv = cvN;
    if (has_bias) {
#pragma unroll
      for (int k = 0; k < K; ++k)
#pragma unroll
        for (int i = 0; i < VEC; ++i) bias[BIAS ? k : 0][i] = biasN[BIAS ? k : 0][i];
    }
  }
}

// ---- rows below the split threshold, streamed gather (rows of >= 17 128-bit chunks: F >= 68 fp32) ---------------
// Persistent warps: each owns a contiguous range of rows of the LIGHT VIEW (split rows removed, so the in-edges of
// the range are ONE contiguous stream of slots), the ranges cut at equal-cost boundaries precomputed with the CSR.
// The warp keeps a ring of neighbour feature rows in shared memory, cut into segments of H slots: every lane copies
// its own 16-byte chunk(s) of each row x[col[slot]] into the ring slot with cp.async (LDGSTS, L2 evict-last hint),
// one cp.async group per segment, and later reads back exactly those bytes (ld.shared.v4, lanes = feature chunks,
// slot order = CSR order), so completion is tracked per thread and no lane waits for another.  While one segment is
// being reduced the others are in flight.
// Gather latency is hidden by bytes in flight in shared memory instead of by registers or by more warps:
// 24 warps x 8 KB per SM versus 24 warps x 4 x 512 B with register staging.
constexpr int kStreamThreads = 128;

__device__ __forceinline__ unsigned smem_u32(const void* ptr) { return (unsigned)__cvta_generic_to_shared(ptr); }

// 128-bit shared-memory load through a 32-bit shared address (no generic-address conversion in the loop)
template <typename T, int VEC>
__device__ __forceinline__ typename Io<T, VEC>::Raw lds_raw(unsigned addr) {
  static_assert(sizeof(typename Io<T, VEC>::Raw) == 16, "the stream path moves 128-bit chunks");
  typename Io<T, VEC>::Raw r;
  unsigned* w = reinterpret_cast<unsigned*>(&r);
  unsigned a, b, c, d;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(addr));
  w[0] = a; w[1] = b; w[2] = c; w[3] = d;
  return r;
}

// DEPTH scales the ring: 1 for local HBM gathers; 2 when remote rows arrive over NVLink (2-3x the latency, and a row
// at the head of the in-order ring blocks the rows behind it)
template <typename T, int VEC, int K, int DEPTH = 1>
struct StreamGeom {
  static constexpr int kHalfBytes = 4096;   // bytes of neighbour rows per ring segment per warp (DEPTH 1)
  static constexpr int kStages = 2;         // ring segments per warp: one being reduced, the others in flight
  static constexpr int kBlockBytes = 32 * VEC * K * (int)sizeof(T);            // bytes of one ring slot
  static constexpr int kHalf = kHalfBytes * DEPTH;
  static constexpr int kH = (kHalf / kBlockBytes) < 4 ? 4 : ((kHalf / kBlockBytes) > 32 ? 32 : (kHalf / kBlockBytes));
  static constexpr int kWarpBytes = kStages * kH * kBlockBytes;
  static constexpr size_t kSmem = (size_t)(kStreamThreads / 32) * kWarpBytes;
};

// 16-byte async copy global -> shared (LDGSTS, L2-only caching) with an L2 eviction-priority hint
// L1 = true: the copy allocates in L1 (cp.async.ca).  A source row that many destinations of the same SM gather (power-law
// graphs: a handful of rows receive a third of all gathers) is then served by the SM's own L1 instead of the few L2 slices
// that hold its lines -- their bandwidth is what bounds such graphs otherwise.  For graphs without hot sources the L1
// detour costs time, hence a mode the caller selects (PNA_FLAG_GATHER_L1), not a default.
template <bool L1 = false>
__device__ __forceinline__ void cp_async16(unsigned dst, const void* src, unsigned long long policy) {
  if constexpr (L1)
    asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(__cvta_generic_to_global(src)), "l"(policy)
                 : "memory");
  else
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(__cvta_generic_to_global(src)), "l"(policy)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

// ---- hubs, pass 2: one CTA per hub merges its partials, then the common epilogue ---------------------------
// kFinGroups lane groups stride over the hub's chunks (group q takes chunks q, q+kFinGroups, ..), each merging in
// chunk order; the per-group results are parked in the groups' own first partial slots (scratch, rebuilt every call)
// and group 0 merges those in group order.  Deterministic; no atomics; a 20k-edge hub is ~20 chunk reads per group.
constexpr int kFinGroups = 8;

template <int VEC, int K, int UF>
__device__ __forceinline__ void merge_partials(const float* __restrict__ base, long long F, const int (&f)[K], const bool (&ok)[K],
                                               int first, int count, int stride, Acc<VEC> (&acc)[K]) {
  for (int j = 0; j < count; j += UF) {
    float ps[UF][K][4][VEC];
#pragma unroll
    for (int u = 0; u < UF; ++u) {
      if (j + u < count) {
        const float* part = base + (long long)(first + (long long)(j + u) * stride) * 4ll * F;
#pragma unroll
        for (int k = 0; k < K; ++k)
          if (ok[k]) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              // L2 loads (ld.global.cg): written earlier on this stream, by this CTA, or -- folded finalize -- by a warp of
              // another SM in the same launch, ordered by __threadfence + the completion counter
              const float* src = part + (long long)q * F + f[k];
              if constexpr (VEC % 4 == 0) {
#pragma unroll
                for (int i = 0; i < VEC; i += 4) {
                  const float4 t = __ldcg(reinterpret_cast<const float4*>(src + i));
                  ps[u][k][q][i] = t.x; ps[u][k][q][i + 1] = t.y; ps[u][k][q][i + 2] = t.z; ps[u][k][q][i + 3] = t.w;
                }
              } else {
#pragma unroll
                for (int i = 0; i < VEC; ++i) ps[u][k][q][i] = __ldcg(src + i);
              }
            }
          }
      }
    }
#pragma unroll
    for (int u = 0; u < UF; ++u) {
      if (j + u < count) {
#pragma unroll
        for (int k = 0; k < K; ++k)
          if (ok[k]) {
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
              acc[k].sum[i] = __fadd_rn(acc[k].sum[i], ps[u][k][0][i]);
              acc[k].sq[i] = __fadd_rn(acc[k].sq[i], ps[u][k][1][i]);
              acc[k].mn[i] = fminf(acc[k].mn[i], ps[u][k][2][i]);
              acc[k].mx[i] = fmaxf(acc[k].mx[i], ps[u][k][3][i]);
            }
          }
      }
    }
  }
}

// ---- folded finalize of the split rows (pna_agg_t.hub_done): completion counters instead of a second kernel ------------
// Called by the warp that has just stored the partial of chunk c.  The warp that completes the last chunk of merge
// group g (chunks g, g+8, .. of the split row) merges that group in chunk order and parks the result in the group's first
// slot; the warp that completes the last group merges the 8 group results in order and runs the row epilogue -- the same
// two-level order as k_hub_finalize, hence the same bits, deterministic.  Nobody waits: whoever arrives last does the
// work.  Counters are reset by their last visitor.  Out of line so that the streaming loop keeps its registers.
template <typename T, int VEC, int K, typename Cfg>
__device__ __noinline__ void fold_split_row(const KParams& p, int c, int fblock) {
  constexpr int G = 32;
  constexpr unsigned FULL = 0xffffffffu;
  constexpr int UFm = (K * VEC >= 8) ? 1 : 2;
  const int lane = threadIdx.x & 31;
  FeatMap<VEC, G, K> fm;
  fm.init(p, lane, fblock);
  Acc<VEC> acc[K];
  const int h = __ldg(p.chunk_items + 2 * c), jc = __ldg(p.chunk_items + 2 * c + 1);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2);
  int* cnt = p.hub_done + 9ll * h;
  auto arrive = [&](int* ctr) -> int {   // publishes this warp's stored partial, returns the arrival index
    __threadfence();
    __syncwarp();
    int t = 0;
    if (lane == 0) t = atomicAdd(ctr, 1);
    return __shfl_sync(FULL, t, 0);
  };
  if (nch > kFinGroups) {
    const int g = jc % kFinGroups;
    const int mine = (nch - g + kFinGroups - 1) / kFinGroups;
    if (arrive(cnt + g) != mine - 1) return;
    if (lane == 0) cnt[g] = 0;
    __threadfence();
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k].init();
    merge_partials<VEC, K, UFm>(p.partials, p.F, fm.f, fm.ok, first + g, mine, kFinGroups, acc);
    float* __restrict__ part = p.partials + (long long)(first + g) * 4ll * p.F;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (!fm.ok[k]) continue;
      store_f32<VEC>(part + 0ll * p.F + fm.f[k], acc[k].sum);
      store_f32<VEC>(part + 1ll * p.F + fm.f[k], acc[k].sq);
      store_f32<VEC>(part + 2ll * p.F + fm.f[k], acc[k].mn);
      store_f32<VEC>(part + 3ll * p.F + fm.f[k], acc[k].mx);
    }
    if (arrive(cnt + 8) != kFinGroups - 1) return;
  } else if (arrive(cnt + 8) != nch - 1) {
    return;
  }
  if (lane == 0) cnt[8] = 0;
  __threadfence();
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k].init();
  merge_partials<VEC, K, UFm>(p.partials, p.F, fm.f, fm.ok, first, nch > kFinGroups ? kFinGroups : nch, 1, acc);
  finalize_row<T, VEC, G, K, Cfg>(p, fm, (long long)__ldg(p.hub_info + 4 * h), __ldg(p.hub_info + 4 * h + 3), acc);
}

template <typename T, int VEC, int K, typename Cfg, bool BIAS, int DEPTH, bool FOLD = false, bool L1 = false>
__global__ void __launch_bounds__(kStreamThreads, tiled_min_blocks(VEC, K)) k_rows_stream(const __grid_constant__ KParams p) {
  constexpr int G = 32;
  constexpr int H = StreamGeom<T, VEC, K, DEPTH>::kH;
  constexpr int SLOT = StreamGeom<T, VEC, K, DEPTH>::kBlockBytes;
  constexpr int NST = StreamGeom<T, VEC, K, DEPTH>::kStages;
  constexpr int CB = 16;               // bytes per lane chunk
  constexpr unsigned FULL = 0xffffffffu;
  constexpr bool PEER = DEPTH > 1;     // the deep-ring instantiations are the ones launched with peer pointers
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ float4 s_scale_lut[kScaleLut];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  fill_scale_lut(s_scale_lut, p, threadIdx.x, kStreamThreads);

  // shared memory: per warp a ring of NST*H slots
  const unsigned ring = smem_u32(smem) + warp * StreamGeom<T, VEC, K, DEPTH>::kWarpBytes;
  const unsigned long long keep = l2_policy_evict_last();   // gathered rows are re-read by other destinations

  // this warp's rows: first a contiguous range of the light view cut at equal-cost partition boundaries -- the first
  // n_static partitions are dealt out statically, one contiguous range per warp (one uninterrupted slot stream).  The
  // remaining partitions are handed out one at a time through an atomic counter: the static ranges finish at different
  // times (17 % of the SM cycles were idle at the tail of configs 2 and 5), the dynamic ones fill the gap.
  const long long W = (long long)gridDim.x * (kStreamThreads / 32);
  const long long w = (long long)blockIdx.x * (kStreamThreads / 32) + warp;
  const int n_static = p.work_ctr ? p.n_static : p.n_part;
  int pi_a = (int)((w * n_static) / W), pi_b = (int)(((w + 1) * n_static) / W);
#pragma unroll 1
 for (;;) {
  const int pa = __ldg(p.part + pi_a);
  const int pb = __ldg(p.part + pi_b);
  const int Q0 = __ldg(p.lrowptr + pa);
  const int Te = __ldg(p.lrowptr + pb) - Q0;      // length of this slot stream
  if (pa < pb) {                                  // warp-uniform; no CTA-wide barrier is used below
  const int* __restrict__ lcol = p.lcol + Q0;
  const int fblock = blockIdx.y * (G * VEC * K);
  FeatMap<VEC, G, K> fm;
  fm.init(p, lane, fblock);

  // source row of stream position q for this lane.  Past the end of the stream (and for lanes >= H) it is row 0: the
  // ring slot is filled with a row nobody reads, which keeps every copy unconditional -- no per-slot branch
  auto source_of = [&](int q) -> int { return (lane < H && q < Te) ? __ldg(lcol + q) : 0; };
  // issue the copies of segment n (positions n*H .. n*H+H-1) whose sources were fetched one step earlier; each lane
  // copies only its own chunks (see above)
  const int lane_elems = fblock + lane * VEC;   // this lane's first 16-byte chunk inside a gathered row
  // byte address of this lane's chunk in row 0; a row is one unsigned 32 x 32 -> 64-bit multiply-add away (IMAD.WIDE.U32)
  const char* const xlane = reinterpret_cast<const char*>(static_cast<const T*>(p.x) + lane_elems);
  const unsigned ldxb = (unsigned)p.ldx * (unsigned)sizeof(T);
  auto issue_half = [&](int stage, int src) {
    unsigned dst = ring + (unsigned)(stage * H) * SLOT + lane * CB;
#pragma unroll
    for (int u = 0; u < H; ++u, dst += SLOT) {
      const int s_u = __shfl_sync(FULL, src, u);
      const char* sp;
      if constexpr (PEER) sp = reinterpret_cast<const char*>(gathered_row<T>(p, s_u) + lane_elems);
      else sp = xlane + (unsigned long long)(unsigned)s_u * ldxb;
#pragma unroll
      for (int k = 0; k < K; ++k)
        if (fm.ok[k]) cp_async16<L1>(dst + k * (32 * CB), sp + k * (32 * CB), keep);
    }
    cp_async_commit();
  };

  int pend = source_of(lane);                 // sources of segment 0
  if (Te > 0) {
    // fill the whole ring; segments past the end of the stream are copied too (row 0, never read): "one group per
    // segment" keeps wait_group<NST-1> exact
#pragma unroll
    for (int s0 = 0; s0 < NST; ++s0) {
      issue_half(s0, pend);
      pend = source_of((s0 + 1) * H + lane);
    }
  }
  int stage = 0;        // ring segment that holds stream positions [n*H, n*H + H) being consumed
  int n_issued = NST;   // segments issued so far

  // row metadata, 32 rows at a time, the next 32 prefetched while the current ones are reduced
  auto load_deg = [&](int r) -> int { return (r + lane < pb) ? __ldg(p.ldeg + r + lane) : -1; };
  const ViewMap vmap = {p.n_rows, (int)(p.n_view_rows - p.n_rows)};   // M > 0: chunk pseudo-rows interleaved in the view
  auto load_rid = [&](int r) -> int {
    if (p.row_ids) return (r + lane < pb) ? __ldg(p.row_ids + r + lane) : 0;
    return (int)vmap.to_row(r + lane);
  };
  int dg = load_deg(pa), rid = load_rid(pa);

  const unsigned lane_off = (unsigned)lane * (unsigned)CB;
  int q = 0;   // stream position being consumed
#pragma unroll 1
  for (int r0 = pa; r0 < pb; r0 += 32) {
    const int dgN = load_deg(r0 + 32), ridN = load_rid(r0 + 32);
    const int nj = min(32, pb - r0);
#pragma unroll 1
    for (int j = 0; j < nj; ++j) {
      const int deg = __shfl_sync(FULL, dg, j);
      if (deg < 0) continue;    // split row (warp-uniform)
      const int row = __shfl_sync(FULL, rid, j);
      const bool chunk_row = row >= p.n_rows;      // pseudo-row: one chunk of a split row, reduced into partials
      float bias[BIAS ? K : 1][VEC];
      if (BIAS) {
        long long brow = row;
        if (chunk_row) brow = __ldg(p.hub_info + 4 * __ldg(p.chunk_items + 2 * (row - (int)p.n_rows)));
#pragma unroll
        for (int k = 0; k < K; ++k)
          if (fm.ok[k]) Io<T, VEC>::load(static_cast<const T*>(p.bias) + brow * p.ldb + fm.f[k], bias[BIAS ? k : 0]);
      }
      Acc<VEC> acc[K];
#pragma unroll
      for (int k = 0; k < K; ++k) acc[k].init();

      int left = deg;
      while (left > 0) {
        // segment = slots of this row inside the current half
        const int inhalf = q & (H - 1);
        if (inhalf == 0) {       // entering a segment: wait for its copies
          cp_async_wait<NST - 1>();    // all groups but the NST-1 newest (the segments still in flight) have landed
        }
        const int seg = min(left, H - inhalf);
        unsigned sp = ring + (unsigned)(stage * H + inhalf) * SLOT + lane_off;
        int t = 0;
        for (; t + 2 <= seg; t += 2, sp += 2 * SLOT) {      // two slots per step: FADD2/FMUL2 + FMNMX3
#pragma unroll
          for (int k = 0; k < K; ++k) {
            if (fm.ok[k]) {
              float m0[VEC], m1[VEC];
              Io<T, VEC>::unpack(lds_raw<T, VEC>(sp + k * (32 * CB)), m0);
              Io<T, VEC>::unpack(lds_raw<T, VEC>(sp + SLOT + k * (32 * CB)), m1);
              acc[k].template add2<BIAS>(m0, m1, bias[BIAS ? k : 0]);
            }
          }
        }
        if (t < seg) {
#pragma unroll
          for (int k = 0; k < K; ++k) {
            if (fm.ok[k]) {
              float m0[VEC];
              Io<T, VEC>::unpack(lds_raw<T, VEC>(sp + k * (32 * CB)), m0);
              acc[k].template add1<BIAS>(m0, bias[BIAS ? k : 0]);
            }
          }
        }
        q += seg;
        left -= seg;
        if ((q & (H - 1)) == 0 || q == Te) {   // segment fully consumed: refill it with the segment NST further on
          issue_half(stage, pend);             // (a group of unread copies past the end of the stream)
          pend = source_of((n_issued + 1) * H + lane);
          ++n_issued;
          stage = (stage + 1 == NST) ? 0 : stage + 1;
        }
      }
      if (!chunk_row) {
        if (Cfg::kStatic && deg == 0 && !p.sdeg) {      // (the dynamic-configuration kernels keep one epilogue)
          finalize_isolated_row<T, VEC, G, K, Cfg>(p, fm, (long long)row, scales_of_row(s_scale_lut, p, row, 0));
        } else {
          finalize_row_ds<T, VEC, G, K, Cfg>(p, fm, (long long)row, deg, scales_of_row(s_scale_lut, p, row, deg), acc);
        }
      } else {
        float* __restrict__ part = p.partials + (long long)(row - (int)p.n_rows) * 4ll * p.F;
#pragma unroll
        for (int k = 0; k < K; ++k) {
          if (!fm.ok[k]) continue;
          store_f32<VEC>(part + 0ll * p.F + fm.f[k], acc[k].sum);
          store_f32<VEC>(part + 1ll * p.F + fm.f[k], acc[k].sq);
          store_f32<VEC>(part + 2ll * p.F + fm.f[k], acc[k].mn);
          store_f32<VEC>(part + 3ll * p.F + fm.f[k], acc[k].mx);
        }
        // FOLD is a separate instantiation: the out-of-line call costs the streaming loop registers (ABI partition)
        if constexpr (FOLD) fold_split_row<T, VEC, K, Cfg>(p, row - (int)p.n_rows, fblock);
      }
    }
    dg = dgN; rid = ridN;
  }
  if (p.work_ctr) { cp_async_wait<0>(); __syncwarp(); }    // the next range refills the ring from its first segment
  }  // pa < pb
  if (!p.work_ctr) break;
  int g = 0;
  if (lane == 0) g = atomicAdd(p.work_ctr, 1);
  g = __shfl_sync(FULL, g, 0);
  pi_a = n_static + g;
  if (pi_a >= p.n_part) break;
  pi_b = pi_a + 1;
 }  // ranges
}

// ---- hubs, pass 1: one lane group per chunk of `chunk` slots -> fp32 partials ------------------------------
template <typename T, int VEC, int G, int K, int U>
__global__ void __launch_bounds__(kThreads, min_blocks(VEC, K)) k_hub_chunks(const KParams p) {
  constexpr int RPW = 32 / G;
  const int lane = threadIdx.x & 31;
  const int gl = lane % G;
  const long long c = ((long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * RPW + lane / G;
  if (c >= p.n_chunks) return;
  const int h = __ldg(p.chunk_items + 2 * c), j = __ldg(p.chunk_items + 2 * c + 1);
  const long long row = __ldg(p.hub_info + 4 * h);
  const int rbeg = __ldg(p.rowptr + row), rend = __ldg(p.rowptr + row + 1);
  const int beg = rbeg + j * p.chunk;
  const int end = min(beg + p.chunk, rend);

  FeatMap<VEC, G, K> fm;
  fm.init(p, gl, blockIdx.y * (G * VEC * K));
  Acc<VEC> acc[K];
  float bias[K][VEC];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    acc[k].init();
    if (p.bias && fm.ok[k]) Io<T, VEC>::load(static_cast<const T*>(p.bias) + row * p.ldb + fm.f[k], bias[k]);
  }
  accumulate_slots<T, VEC, G, K, U>(p, fm, beg, end, bias, p.bias != nullptr, acc);

  float* __restrict__ part = p.partials + c * 4ll * p.F;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (!fm.ok[k]) continue;
    store_f32<VEC>(part + 0ll * p.F + fm.f[k], acc[k].sum);
    store_f32<VEC>(part + 1ll * p.F + fm.f[k], acc[k].sq);
    store_f32<VEC>(part + 2ll * p.F + fm.f[k], acc[k].mn);
    store_f32<VEC>(part + 3ll * p.F + fm.f[k], acc[k].mx);
  }
}

// ---- split rows with very many chunks (power-law graphs: millions of in-edges in one row) ---------------------------------
// One CTA walking a row's chunk partials (k_hub_finalize) is a serial tail of tens of thousands of dependent 4 KB reads.
// Instead the partials are merged by a radix tree over the GLOBAL chunk array: at the level with stride S a warp owns the
// block of R*S chunk positions [B*R*S, (B+1)*R*S) and visits its positions B*R*S + j*S, j = 1..R-1; a position that is a
// CONTINUATION of a split row (the row's first chunk lies before it) holds that row's parked partial for
// [pos, pos + S) from the level below and is added, in position order, into the row's head inside this block,
// max(first chunk of the row, B*R*S).  After ceil(log_R(n_chunks)) levels every row's total sits in its first chunk's slot.
// Fixed order for a given graph -> deterministic, no atomics; every level is one small launch.
constexpr int kTreeR = 32;

template <int VEC, int K>
__global__ void __launch_bounds__(128) k_hub_tree(const KParams p, long long S) {
  constexpr int G = 32;
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const long long B = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
  const long long base = B * kTreeR * S;
  if (base >= p.n_chunks) return;
  FeatMap<VEC, G, K> fm;
  fm.init(p, lane, blockIdx.y * (G * VEC * K));
  // lane j: is position base + j*S a continuation, and of which head?
  long long my_head = -1;
  {
    const long long pos = base + (long long)lane * S;
    if (lane > 0 && pos < p.n_chunks) {
      const int h = __ldg(p.chunk_items + 2 * pos);
      const long long first = __ldg(p.hub_info + 4 * h + 1);
      if (first < pos) my_head = first > base ? first : base;
    }
  }
  const long long F4 = 4ll * p.F;
  auto load = [&](long long c, Acc<VEC> (&a)[K]) {
    const float* part = p.partials + c * F4;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (!fm.ok[k]) continue;
      float* const dst[4] = {a[k].sum, a[k].sq, a[k].mn, a[k].mx};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float* src = part + (long long)q * p.F + fm.f[k];
        if constexpr (VEC % 4 == 0) {
#pragma unroll
          for (int i = 0; i < VEC; i += 4) {
            const float4 t4 = __ldcg(reinterpret_cast<const float4*>(src + i));
            dst[q][i] = t4.x; dst[q][i + 1] = t4.y; dst[q][i + 2] = t4.z; dst[q][i + 3] = t4.w;
          }
        } else {
#pragma unroll
          for (int i = 0; i < VEC; ++i) dst[q][i] = __ldcg(src + i);
        }
      }
    }
  };
  auto store = [&](long long c, const Acc<VEC> (&a)[K]) {
    float* part = p.partials + c * F4;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (!fm.ok[k]) continue;
      store_f32<VEC>(part + 0ll * p.F + fm.f[k], a[k].sum);
      store_f32<VEC>(part + 1ll * p.F + fm.f[k], a[k].sq);
      store_f32<VEC>(part + 2ll * p.F + fm.f[k], a[k].mn);
      store_f32<VEC>(part + 3ll * p.F + fm.f[k], a[k].mx);
    }
  };
  Acc<VEC> acc[K];
  long long cur = -1;
  auto fold = [&](long long head, const Acc<VEC> (&t)[K]) {
    if (head != cur) {
      if (cur >= 0) store(cur, acc);
      load(head, acc);
      cur = head;
    }
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        acc[k].sum[i] = __fadd_rn(acc[k].sum[i], t[k].sum[i]);
        acc[k].sq[i] = __fadd_rn(acc[k].sq[i], t[k].sq[i]);
        acc[k].mn[i] = fminf(acc[k].mn[i], t[k].mn[i]);
        acc[k].mx[i] = fmaxf(acc[k].mx[i], t[k].mx[i]);
      }
  };
  // UB partials are requested before the first dependent add: the walk is a chain of L2 round trips, UB of them overlap
  constexpr int UB = (K * VEC >= 16) ? 2 : 4;
#pragma unroll 1
  for (int j = 1; j < kTreeR; j += UB) {
    long long hd[UB];
    bool any = false;
#pragma unroll
    for (int u = 0; u < UB; ++u) {
      hd[u] = (j + u < kTreeR) ? __shfl_sync(FULL, my_head, (j + u) & 31) : -1;
      any |= hd[u] >= 0;
    }
    if (!any) continue;
    Acc<VEC> t[UB][K];
#pragma unroll
    for (int u = 0; u < UB; ++u)
      if (hd[u] >= 0) load(base + (long long)(j + u) * S, t[u]);
#pragma unroll
    for (int u = 0; u < UB; ++u)
      if (hd[u] >= 0) fold(hd[u], t[u]);
  }
  if (cur >= 0) store(cur, acc);
}

// ---- hubs, pass 2 (k_hub_finalize): merge_partials / kFinGroups are defined above k_rows_stream ------------------------
template <typename T, int VEC, int G, int K>
__global__ void __launch_bounds__(kFinGroups * 32) k_hub_finalize(const KParams p) {
  constexpr int UF = (K * VEC >= 16) ? 1 : (K * VEC >= 8 ? 2 : 4);  // partial sets in flight (register budget)
  const int gl = threadIdx.x % G;
  const int q = threadIdx.x / G;          // lane group within the CTA, 0..kFinGroups-1
  const long long h = blockIdx.x;
  const long long row = __ldg(p.hub_info + 4 * h);
  const int first = __ldg(p.hub_info + 4 * h + 1), nch = __ldg(p.hub_info + 4 * h + 2);
  const int deg = __ldg(p.hub_info + 4 * h + 3);

  FeatMap<VEC, G, K> fm;
  fm.init(p, gl, blockIdx.y * (G * VEC * K));
  Acc<VEC> acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k].init();

  const bool two_level = nch > kFinGroups && !p.hub_merged;
  if (p.hub_merged) {     // k_hub_tree left the row's total in its first chunk's slot
    if (q != 0) return;
    merge_partials<VEC, K, UF>(p.partials, p.F, fm.f, fm.ok, first, 1, 1, acc);
  } else if (two_level) {
    const int mine = (nch - q + kFinGroups - 1) / kFinGroups;     // chunks q, q+kFinGroups, ..
    merge_partials<VEC, K, UF>(p.partials, p.F, fm.f, fm.ok, first + q, mine, kFinGroups, acc);
    float* part = p.partials + (long long)(first + q) * 4ll * p.F;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (!fm.ok[k]) continue;
      store_f32<VEC>(part + 0ll * p.F + fm.f[k], acc[k].sum);
      store_f32<VEC>(part + 1ll * p.F + fm.f[k], acc[k].sq);
      store_f32<VEC>(part + 2ll * p.F + fm.f[k], acc[k].mn);
      store_f32<VEC>(part + 3ll * p.F + fm.f[k], acc[k].mx);
    }
    __syncthreads();   // CTA-scope visibility of the parked per-group results
    if (q != 0) return;
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k].init();
    merge_partials<VEC, K, UF>(p.partials, p.F, fm.f, fm.ok, first, kFinGroups, 1, acc);
  } else {
    if (q != 0) return;
    merge_partials<VEC, K, UF>(p.partials, p.F, fm.f, fm.ok, first, nch, 1, acc);
  }
  finalize_row<T, VEC, G, K, CfgDynamic>(p, fm, row, deg, acc);
}

// ---- host dispatch -----------------------------------------------------------------------------------------
template <typename T, int VEC, int G, int K, int U>
static int launch_config(const KParams& p_in, cudaStream_t st) {
  constexpr int RPW = 32 / G;
  constexpr int per_block = (kThreads / 32) * RPW;
  KParams p = p_in;
  const unsigned gy = (unsigned)((p.F + G * VEC * K - 1) / (G * VEC * K));
  // folded finalize: one counter set per split row, i.e. one feature block, and only the streamed kernel implements it
  if (gy != 1 || !(p.n_view_rows > p.n_rows) || p.hub_merged) p.hub_done = nullptr;
  bool folded = false;
  bool chunks_in_stream = false;   // the streamed kernel also reduced the chunks of the split rows
  if (!(p.flags & PNA_FLAG_SKIP_LIGHT)) {
    const long long slots = p.row_ids ? p.n_row_ids : p.n_rows;
    if (slots > 0) {
      const long long gx = (slots + per_block - 1) / per_block;
      PNA_REQUIRE(gx <= 0x7fffffffll, PNA_ERR_UNSUPPORTED, "too many rows for one launch: %lld", slots);
      const unsigned std_s = (0u) | (1u << 4) | (2u << 8);
      const bool s3 = p.nS == 3 && (p.scodes & 0xfffu) == std_s && p.nA == 4;
      // identity scaler only: the compact [N, A*F] result consumed by pna_linear_scaled_fwd
      const bool s1 = p.nS == 1 && (p.scodes & 0xfu) == PNA_SCALE_IDENTITY && p.nA == 4;
      const int cfg = (p.acodes & 0xffffu) != CfgMeanMaxMinStd::ACODES ? 0 : s3 ? 1 : s1 ? 2 : 0;
      if (G == 32 && VEC > 1 && p.lrowptr != nullptr && p.col != nullptr) {
       if constexpr (G == 32 && VEC > 1) {
        // streamed gather over the light view, persistent warps
        const bool b = p.bias != nullptr;
        const bool deep = p.peer_x != nullptr;
#define PNA_LAUNCH_STREAM_(CFG, B, DEPTH, FOLD) PNA_LAUNCH_STREAM__(CFG, B, DEPTH, FOLD, false)
#define PNA_LAUNCH_STREAM__(CFG, B, DEPTH, FOLD, L1)                                                                    \
  do {                                                                                                             \
    constexpr size_t smem = StreamGeom<T, VEC, K, DEPTH>::kSmem;                                                   \
    auto kern = k_rows_stream<T, VEC, K, CFG, B, DEPTH, FOLD, L1>;                                                     \
    static int resident = 0;  /* CTAs of this kernel that fit the device (every device of a process alike) */                \
    if (resident == 0) {  /* (static + dynamic shared memory of the K = 3 ring exceeds the 48 KB default) */       \
      PNA_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));            \
      int dev = 0, sms = 0, nb = 0;                                                                                \
      PNA_CUDA_TRY(cudaGetDevice(&dev));                                                                           \
      PNA_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));                             \
      PNA_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, kStreamThreads, smem));                \
      resident = (nb > 0 ? nb : 1) * sms;                                                                          \
    }                                                                                                              \
    long long gxs = (slots + 8 * (kStreamThreads / 32) - 1) / (8 * (kStreamThreads / 32)); /* >= 8 rows per warp */ \
    if (gxs > resident) gxs = resident;                                                                            \
    if (gxs < 1) gxs = 1;                                                                                          \
    if (p.work_ctr) {   /* dynamic tail: the last ~30 % of the partitions, if every warp still gets static work */  \
      const long long nw = gxs * (kStreamThreads / 32);                                                            \
      p.n_static = (int)((long long)p.n_part * 7 / 10);                                                            \
      if (gy != 1 || p.n_static < nw || gxs < resident) p.work_ctr = nullptr;                                      \
      else PNA_CUDA_TRY(cudaMemsetAsync(p.work_ctr, 0, sizeof(int), st));                                          \
    }                                                                                                              \
    kern<<<dim3((unsigned)gxs, gy), kStreamThreads, smem, st>>>(p);                                                \
  } while (0)
        // single-GPU kernels exist with and without the folded finalize; the peer (DEPTH 2) kernels without
#define PNA_LAUNCH_STREAM(CFG, B)                                        \
  do {                                                                   \
    if (p.hub_done) PNA_LAUNCH_STREAM_(CFG, B, 1, true);                 \
    else PNA_LAUNCH_STREAM_(CFG, B, 1, false);                           \
  } while (0)
        if (deep) {
          p.hub_done = nullptr;
          if (cfg == 1 && !b) PNA_LAUNCH_STREAM_(CfgMeanMaxMinStd, false, 2, false);
          else if (!b) PNA_LAUNCH_STREAM_(CfgDynamic, false, 2, false);
          else PNA_LAUNCH_STREAM_(CfgDynamic, true, 2, false);
        } else if ((p.flags & PNA_FLAG_GATHER_L1) && cfg == 1 && !b) {      // hot source rows: L1-allocating copies
          p.hub_done = nullptr;
          PNA_LAUNCH_STREAM__(CfgMeanMaxMinStd, false, 1, false, true);
        } else if ((p.flags & PNA_FLAG_GATHER_L1) && cfg == 2 && !b) {
          p.hub_done = nullptr;
          PNA_LAUNCH_STREAM__(CfgMeanMaxMinStdId, false, 1, false, true);
        } else if (cfg == 1 && !b) PNA_LAUNCH_STREAM(CfgMeanMaxMinStd, false);
        else if (cfg == 1) PNA_LAUNCH_STREAM(CfgMeanMaxMinStd, true);
        else if (cfg == 2 && !b) PNA_LAUNCH_STREAM(CfgMeanMaxMinStdId, false);
        else if (!b) PNA_LAUNCH_STREAM(CfgDynamic, false);
        else PNA_LAUNCH_STREAM(CfgDynamic, true);
        chunks_in_stream = p.n_view_rows > p.n_rows;
        folded = chunks_in_stream && p.hub_done != nullptr;
#undef PNA_LAUNCH_STREAM
#undef PNA_LAUNCH_STREAM_
#undef PNA_LAUNCH_STREAM__
       }
      } else if constexpr (G >= U && G % U == 0) {
        constexpr int TR = (8 * RPW < 32) ? 8 * RPW : 32;
        constexpr int tiles_per_block = kTiledThreads / 32;
        const long long tiles = (slots + TR - 1) / TR;
        const long long gt = (tiles + tiles_per_block - 1) / tiles_per_block;
        PNA_REQUIRE(gt <= 0x7fffffffll, PNA_ERR_UNSUPPORTED, "too many rows for one launch: %lld", slots);
        const dim3 grid((unsigned)gt, gy);
        const bool b = p.bias != nullptr;
        if (p.peer_x != nullptr) {   // narrow rows gathered over NVLink: the dynamic-configuration kernels only
          if (!b) k_rows_tiled<T, VEC, G, K, U, CfgDynamic, false, true><<<grid, kTiledThreads, 0, st>>>(p);
          else k_rows_tiled<T, VEC, G, K, U, CfgDynamic, true, true><<<grid, kTiledThreads, 0, st>>>(p);
        } else if (cfg == 1 && !b) k_rows_tiled<T, VEC, G, K, U, CfgMeanMaxMinStd, false><<<grid, kTiledThreads, 0, st>>>(p);
        else if (cfg == 1) k_rows_tiled<T, VEC, G, K, U, CfgMeanMaxMinStd, true><<<grid, kTiledThreads, 0, st>>>(p);
        else if (!b) k_rows_tiled<T, VEC, G, K, U, CfgDynamic, false><<<grid, kTiledThreads, 0, st>>>(p);
        else k_rows_tiled<T, VEC, G, K, U, CfgDynamic, true><<<grid, kTiledThreads, 0, st>>>(p);
      } else {
        k_rows<T, VEC, G, K, U, CfgDynamic><<<dim3((unsigned)gx, gy), kThreads, 0, st>>>(p);
      }
      PNA_CUDA_TRY(cudaGetLastError());
    }
  }
  if (!(p.flags & PNA_FLAG_SKIP_HUBS) && p.n_hubs > 0) {
    if (!chunks_in_stream) {
      const long long gc = (p.n_chunks + per_block - 1) / per_block;
      k_hub_chunks<T, VEC, G, K, U><<<dim3((unsigned)gc, gy), kThreads, 0, st>>>(p);
      PNA_CUDA_TRY(cudaGetLastError());
    }
    if (!folded) {
      if constexpr (G == 32) {
        if (p.hub_merged) {
          for (long long S = 1; S < p.n_chunks; S *= kTreeR) {
            const long long blocks = (p.n_chunks + kTreeR * S - 1) / (kTreeR * S);
            k_hub_tree<VEC, K><<<dim3((unsigned)((blocks + 3) / 4), gy), 128, 0, st>>>(p, S);
            PNA_CUDA_TRY(cudaGetLastError());
          }
        }
      } else {
        p.hub_merged = 0;     // narrow rows keep the CTA-per-row merge
      }
      k_hub_finalize<T, VEC, G, K><<<dim3((unsigned)p.n_hubs, gy), kFinGroups * G, 0, st>>>(p);
      PNA_CUDA_TRY(cudaGetLastError());
    }
  }
  return PNA_OK;
}

template <typename T, int VEC>
int launch_typed(const KParams& p, cudaStream_t st) {
  const int chunks = p.F / VEC;  // VEC divides F on the vector path; VEC == 1 on the scalar path
  if (chunks <= 1) return launch_config<T, VEC, 1, 1, 4>(p, st);
  if (chunks <= 2) return launch_config<T, VEC, 2, 1, 4>(p, st);
  if (chunks <= 4) return launch_config<T, VEC, 4, 1, 4>(p, st);
  if (chunks <= 8) return launch_config<T, VEC, 8, 1, 4>(p, st);
  if (chunks <= 16) return launch_config<T, VEC, 16, 1, 4>(p, st);
  if (chunks <= 32) return launch_config<T, VEC, 32, 1, 4>(p, st);
  if (chunks <= 64) return launch_config<T, VEC, 32, 2, 2>(p, st);
  if (chunks <= 96) return launch_config<T, VEC, 32, 3, 2>(p, st);
  return launch_config<T, VEC, 32, 4, 2>(p, st);  // wider rows: several feature blocks (gridDim.y)
}

}  // namespace pna
