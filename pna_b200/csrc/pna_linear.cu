// pna_linear_fwd: Y[N, O] = A[N, K] . W[O, K]^T + b in fp32 accuracy on the Hopper tensor cores (wgmma).
//
// This is the first dense linear of the post-aggregation MLP (reference models/pytorch_geometric/pna.py:222-227,
// post_nn[0]; models/dgl/pna_layer.py:31 posttrans), the one place of the PNA layer where tensor cores apply
// (north_star: "the post-MLP uses tensor cores only for its dense linear").  The 1e-5 parity bar rules out plain TF32
// (10-bit mantissa); every operand is therefore split  x = hi + lo  (hi = top 19 bits, lo = x - hi, exact) and three
// wgmma tf32 products are accumulated in registers:  hi.hi + hi.lo + lo.hi  (the dropped lo.lo term is 2^-22).
//
// Two warpgroups (256 threads), 3-stage (2 for O = 256) mbarrier ring of {A hi, A lo, W hi, W lo} tiles:
//   all warps  load A with coalesced 128-bit loads issued ahead, split hi / lo (cvt.rna.tf32: an unbiased split --
//              truncation accumulates its one-sided error linearly in K) and store into the 128-byte-swizzled K-major
//              layout wgmma reads (the operand has to pass through registers for the split, so no TMA here).  The same
//              warps then issue the stage's wgmmas (12 per 32-wide K block: 4 K-steps x 3 products) and, one stage
//              later, release it.  Warpgroup g owns a 64 x min(O, 128) block of the CTA's output: rows 64g.. of a
//              128-row tile for O <= 128, columns 128g.. of a 64-row tile for O = 256 (two fp32 accumulators of
//              64 x 256 would not fit the register file).  The epilogue adds the accumulators and the bias and stores.
//   thread 0   also issues the W tiles: the weight is pre-split once per call into the exact swizzled shared-memory image
//              of every K block, so a W tile is one contiguous cp.async.bulk (TMA 1-D) completing on the stage's mbarrier;
//              the tile of step t + kSt is requested as soon as step t has released its stage.  (A separate producer
//              warp would lower the per-thread register budget below the two accumulators.)
//
// Scaled ("compact") mode -- pna_linear_scaled_fwd.  The reference's post-MLP input is cat_s(c_s(i) * agg_i) over the
// degree scalers s (pna.py:247-249): S copies of the same [N, A*F] aggregate, each multiplied by a per-row factor.  In
// this mode A is the COMPACT aggregate (identity scaler only) and the loaders regenerate every scaled copy in registers,
// fl(c_s(i) * a) rounded exactly like the reference's multiply, right before the hi/lo split -- the [N, S*A*F] tensor
// never exists in HBM: the aggregation writes, and this kernel reads, 1/S of the bytes.  K blocks are visited
// compact-block-major, scaler-minor; the W tile of step (kb, s) is block s * (K/32) + kb of the reference's weight.
//
// Backward -- pna_linear_bwd_data / pna_linear_bwd_weight, at the same fp32 accuracy and deterministic (no atomics):
// dA runs the kernel above on dY with the transposed weight in column slabs; dW is k_linear_bwd_weight (below).
#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace pna {

constexpr int kLinBK = 32;          // fp32 per K block = one 128-byte swizzle row
constexpr int lin_rows(int o) { return o <= 128 ? 128 : 64; }      // rows per CTA
constexpr int lin_stages(int o) { return o <= 128 ? 3 : 2; }       // 48 / 64 / 80 KB per stage (O = 64 / 128 / 256)
constexpr int kLinThreads = 256;    // two warpgroups: A loaders and MMA issuers

__device__ __forceinline__ unsigned lin_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void lin_mbar_init(unsigned bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void lin_mbar_arrive(unsigned bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void lin_mbar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void lin_mbar_wait(unsigned bar, unsigned parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "LW_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra LD_%=;\n\t"
      "bra LW_%=;\n\t"
      "LD_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void lin_bulk_g2s(unsigned dst, const void* src, unsigned bytes, unsigned bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(__cvta_generic_to_global(src)), "r"(bytes), "r"(bar)
               : "memory");
}
// x -> nearest TF32 value (19 significant bits kept, round to nearest): the split must not be biased, a truncating
// split accumulates its one-sided error linearly in K
__device__ __forceinline__ float lin_tf32(float x) {
  unsigned r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// the hi part: cvt.rna rounds every finite |x| >= 0x7F7FF000 (within 2^-11 of FLT_MAX) up to inf, and x - hi would then
// be -inf (the product NaN); satfinite clamps hi to the largest TF32 value instead, so lo = x - hi stays exact and finite.
// An inf input gets hi = +-MAX and lo = +-inf (plain cvt.rna keeps lo infinite): the products give what fp32 gives.
__device__ __forceinline__ void lin_split(float x, float& hi, float& lo) {
  unsigned r;
  asm("cvt.rna.satfinite.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  hi = __uint_as_float(r);
  lo = lin_tf32(x - hi);
}

// wgmma shared-memory matrix descriptor: K-major, SWIZZLE_128B, rows of 128 bytes, 8-row groups 1024 bytes apart.
// A K step inside the 128-byte row advances the start address (the swizzle is applied to the computed addresses).
__device__ __forceinline__ unsigned long long lin_desc(unsigned smem_addr) {
  unsigned long long d = 0;
  d |= (unsigned long long)((smem_addr & 0x3ffffu) >> 4);        // start address, bits [0,14)
  d |= (unsigned long long)1 << 16;                               // leading byte offset (unused for swizzled K-major)
  d |= (unsigned long long)(1024 >> 4) << 32;                     // stride byte offset: 8 rows x 128 B
  d |= (unsigned long long)1 << 62;                               // SWIZZLE_128B
  return d;
}

#define LIN_F4(a, i) "+f"(a[i]), "+f"(a[i + 1]), "+f"(a[i + 2]), "+f"(a[i + 3])
#define LIN_F16(a, i) LIN_F4(a, i), LIN_F4(a, i + 4), LIN_F4(a, i + 8), LIN_F4(a, i + 12)

// D[64 x N] += A[64 x 8] . B[N x 8]^T, tf32 operands from shared memory, fp32 accumulator in registers (N/2 per thread:
// register 4j + q of lane l holds row l/4 + 8 (q/2) of the warp's 16 rows, column 8j + 2 (l%4) + q%2).  add == 0: D = A . B
// (restarts an accumulation chain without writing the registers outside the MMA pipeline)
template <int N>
__device__ __forceinline__ void lin_wgmma(float (&d)[N / 2], unsigned long long adesc, unsigned long long bdesc, int add = 1);
template <>
__device__ __forceinline__ void lin_wgmma<64>(float (&d)[32], unsigned long long adesc, unsigned long long bdesc, int add) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1;\n\t}"
      : LIN_F16(d, 0), LIN_F16(d, 16)
      : "l"(adesc), "l"(bdesc), "r"(add));
}
template <>
__device__ __forceinline__ void lin_wgmma<128>(float (&d)[64], unsigned long long adesc, unsigned long long bdesc, int add) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1;\n\t}"
      : LIN_F16(d, 0), LIN_F16(d, 16), LIN_F16(d, 32), LIN_F16(d, 48)
      : "l"(adesc), "l"(bdesc), "r"(add));
}
// keeps the compiler from moving accumulator registers across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void lin_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// byte offset of 16-byte unit j of row r inside a [rows][128 B] tile with the 128-byte swizzle (unit ^= row % 8)
__host__ __device__ __forceinline__ unsigned lin_swz(int r, int j) { return (unsigned)(r * 128 + ((j ^ (r & 7)) << 4)); }

template <int O>   // output width: 64, 128 or 256
struct LinSmem {
  static constexpr int kM = lin_rows(O);
  static constexpr int kSt = lin_stages(O);
  static constexpr int kN = O <= 128 ? O : 128;               // output columns per warpgroup
  static constexpr int kATile = kM * 128;                     // bytes of one A hi (or lo) stage
  static constexpr int kWTile = O * 128;
  static constexpr int kStage = 2 * kATile + 2 * kWTile;
  static constexpr size_t kBytes = 1024 /*align slack*/ + (size_t)kSt * kStage + 256;
};

// Wimg: for every K block the exact shared-memory images of the W hi and W lo tiles ([O rows][128 B], swizzled),
// produced once per call by k_split_weight -- so a tile is ONE contiguous bulk copy (TMA 1-D, no tensor map needed).
// Column slabs (the data gradient, whose width n_cols is not an O of its own): CTA b computes the O columns of slab
// b % n_slabs of row tile b / n_slabs -- the slabs of one row tile run side by side and read its A rows from L2 -- with
// the slab's own weight image (n_it K blocks each, zero rows past n_cols); stores to columns >= n_cols are dropped.
// The forward is n_slabs = 1, n_cols = O.
// FOLD (the data gradient): every kLinFoldSteps pipeline steps the warps wait for their MMAs and fold (acc + corr) into the
// CTA's own Y tile (stored the first time, added with one round-to-nearest add after), so no truncating tensor-core
// accumulation chain is longer than kLinFoldSteps * 32 products: with the S scalers the chain would be S * O long.
// (ptxas serializes this instance's wgmmas -- it cannot see that the accumulators are read only after a full drain -- so
// pna_linear_bwd_data launches it only where a fold happens.)
constexpr int kLinFoldSteps = 4;
template <int O, bool FOLD = false>
__global__ void __launch_bounds__(kLinThreads, 1)
k_linear_3xtf32(const float* __restrict__ A, long long lda, const float* __restrict__ row_scale, int n_rep,
                const float* __restrict__ Wimg, const float* __restrict__ bias, float* __restrict__ Y, long long ldy, long long N,
                int K, int n_slabs, int n_cols) {
  constexpr int kSt = LinSmem<O>::kSt, kM = LinSmem<O>::kM, kN = LinSmem<O>::kN;
  extern __shared__ unsigned char lin_raw[];
  const unsigned base = (lin_smem_u32(lin_raw) + 1023u) & ~1023u;          // swizzle atoms need 1024-byte alignment
  unsigned char* gbase = lin_raw + (base - lin_smem_u32(lin_raw));
  const unsigned bars = base + kSt * LinSmem<O>::kStage;                    // full[kSt], empty[kSt]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int slab = (int)(blockIdx.x % (unsigned)n_slabs);
  const long long row0 = (long long)(blockIdx.x / (unsigned)n_slabs) * kM;
  const int n_kb = K / kLinBK;          // K blocks of A (compact width)
  const int n_it = n_kb * n_rep;        // pipeline steps = K blocks of W (n_rep == 1 without row scales)
  Wimg += (long long)slab * n_it * (2 * O * kLinBK);
  Y += (long long)slab * O;
  const int c_end = n_cols - slab * O;  // columns of this slab that exist

  if (threadIdx.x == 0) {
    for (int s = 0; s < kSt; ++s) {
      lin_mbar_init(bars + 8 * s, kLinThreads / 32 + 1);    // full: one arrive per warp + the W request (with tx bytes)
      lin_mbar_init(bars + 8 * (kSt + s), kLinThreads / 32); // empty: one arrive per warp once its MMAs have read the stage
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // W tiles of pipeline step t: two bulk copies (hi, lo images) into stage t % kSt
  auto request_w = [&](int t) {
    const int sw = t % kSt;
    const int kb = (t % n_rep) * n_kb + t / n_rep;         // weight K block of (compact block t / n_rep, scaler t % n_rep)
    const unsigned st = base + sw * LinSmem<O>::kStage + 2 * LinSmem<O>::kATile;
    lin_mbar_expect_tx(bars + 8 * sw, 2u * LinSmem<O>::kWTile);
    const float* img = Wimg + (long long)kb * (2 * O * kLinBK);
    lin_bulk_g2s(st, img, LinSmem<O>::kWTile, bars + 8 * sw);
    lin_bulk_g2s(st + LinSmem<O>::kWTile, img + O * kLinBK, LinSmem<O>::kWTile, bars + 8 * sw);
  };
  __syncthreads();
  if (threadIdx.x == 0)
    for (int t = 0; t < kSt && t < n_it; ++t) request_w(t);   // every stage starts empty

  {
    // ---------------- A loaders + MMA issuers: LDG ahead -> split hi/lo -> swizzled STS -> wgmma ----------------
    const int tid = threadIdx.x;                            // 0..255
    const int j = tid & 7;                                  // 16-byte unit inside the 128-byte K block row
    const int r_in = tid >> 3;                              // 0..31: row inside a 32-row slab
    constexpr int kSlabs = kM / 32;                         // 4 (O <= 128) or 2 (O = 256)
    constexpr int kAhead = 8 / kSlabs;                      // K blocks of A kept in flight per thread (8 x 16 B)
    const int wg = warp >> 2;                               // warpgroup: which 64 x kN block of the output it owns
    const unsigned a_off = O <= 128 ? (unsigned)(wg * 64 * 128) : 0u;
    const unsigned w_off = O <= 128 ? 0u : (unsigned)(wg * kN * 128);
    // the tensor core adds into fp32 with truncation, a bias that grows with the number of accumulation steps times the
    // magnitude of the running sum: the two small cross terms (2^-11 of the main product) get their own accumulator
    float acc[kN / 2], corr[kN / 2];
#pragma unroll
    for (int i = 0; i < kN / 2; ++i) { acc[i] = 0.f; corr[i] = 0.f; }
    // ---------------- epilogue: (main + cross terms) + bias, two adjacent columns per store (FOLD: + the Y tile so far) -----
    const int wr = (warp & 3) * 16 + (lane >> 2);           // row of the warpgroup's 64 for registers 4j, 4j + 1
    const long long r_lo = row0 + (O <= 128 ? wg * 64 : 0) + wr, r_hi = r_lo + 8;
    bool folded = false, restart = false;
    auto emit = [&](const float* bs, bool add) {
#pragma unroll
      for (int jj = 0; jj < kN / 8; ++jj) {
        const int c = (O <= 128 ? 0 : wg * kN) + jj * 8 + 2 * (lane & 3);
        if (c >= c_end) continue;
        const float b0 = bs ? __ldg(bs + c) : 0.f, b1 = bs ? __ldg(bs + c + 1) : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long r = h ? r_hi : r_lo;
          if (r >= N) continue;
          float2* p = reinterpret_cast<float2*>(Y + r * ldy + c);
          float2 v = make_float2((acc[4 * jj + 2 * h] + corr[4 * jj + 2 * h]) + b0,
                                  (acc[4 * jj + 2 * h + 1] + corr[4 * jj + 2 * h + 1]) + b1);
          if (FOLD && add) {
            const float2 old = *p;
            v.x = old.x + v.x; v.y = old.y + v.y;
          }
          *p = v;
        }
      }
    };
    float4 pre[kAhead][kSlabs];
    auto fetch = [&](int kb, float4 (&dst)[kSlabs]) {
#pragma unroll
      for (int sl = 0; sl < kSlabs; ++sl) {
        const long long r = row0 + sl * 32 + r_in;
        dst[sl] = (kb < n_kb && r < N) ? __ldg(reinterpret_cast<const float4*>(A + r * lda + kb * kLinBK + j * 4))
                                      : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    };
#pragma unroll
    for (int u = 0; u < kAhead; ++u) fetch(u, pre[u]);
    unsigned phase = 0;
    int s = 0;                                              // ring stage of the next pipeline step
    int prev = -1;                                          // stage whose MMAs are still in flight
    int it = 0;                                             // pipeline step
    for (int kb0 = 0; kb0 < n_kb; kb0 += kAhead) {
#pragma unroll
      for (int u = 0; u < kAhead; ++u) {                    // unrolled so that pre[u] stays in registers
        const int kb = kb0 + u;
        if (kb >= n_kb) break;
        for (int rep = 0; rep < n_rep; ++rep) {             // the scaled copies of this K block (one pass without scales)
          float sc[kSlabs];
          if (row_scale) {                                  // issued before the wait: an L1 hit after the first K block
#pragma unroll
            for (int sl = 0; sl < kSlabs; ++sl) {
              const long long r = row0 + sl * 32 + r_in;
              sc[sl] = r < N ? __ldg(row_scale + r * n_rep + rep) : 0.f;
            }
          }
          lin_mbar_wait(bars + 8 * (kSt + s), phase ^ 1);   // stage free
          unsigned char* st = gbase + s * LinSmem<O>::kStage;
#pragma unroll
          for (int sl = 0; sl < kSlabs; ++sl) {
            float4 v = pre[u][sl];
            if (row_scale) {                                // scalers.py: src * scale, rounded to fp32 like the reference
              v.x = __fmul_rn(v.x, sc[sl]); v.y = __fmul_rn(v.y, sc[sl]);
              v.z = __fmul_rn(v.z, sc[sl]); v.w = __fmul_rn(v.w, sc[sl]);
            }
            float4 hi, lo;
            lin_split(v.x, hi.x, lo.x);
            lin_split(v.y, hi.y, lo.y);
            lin_split(v.z, hi.z, lo.z);
            lin_split(v.w, hi.w, lo.w);
            const unsigned off = lin_swz(sl * 32 + r_in, j);  // quarter-warps write whole swizzled 128-byte rows: conflict free
            *reinterpret_cast<float4*>(st + off) = hi;
            *reinterpret_cast<float4*>(st + LinSmem<O>::kATile + off) = lo;
          }
          if (rep == n_rep - 1) fetch(kb + kAhead, pre[u]);   // refill the slot just consumed
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic-proxy stores -> visible to the MMA (async proxy)
          __syncwarp();
          if (lane == 0) lin_mbar_arrive(bars + 8 * s);
          lin_mbar_wait(bars + 8 * s, phase);               // every warp's A rows and the W tiles have landed
          const unsigned sa = base + s * LinSmem<O>::kStage;
          const unsigned a_hi = sa + a_off, a_lo = sa + LinSmem<O>::kATile + a_off;
          const unsigned w_hi = sa + 2 * LinSmem<O>::kATile + w_off, w_lo = w_hi + LinSmem<O>::kWTile;
          lin_fence_acc(acc); lin_fence_acc(corr);
          asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
          for (int ks = 0; ks < kLinBK / 8; ++ks) {         // K = 8 tf32 = 32 bytes along the swizzled row
            const unsigned ko = ks * 32;
            const int add = FOLD ? (ks > 0 || !restart) : 1;  // FOLD: the first MMAs after a fold start a new chain
            lin_wgmma<kN>(corr, lin_desc(a_hi + ko), lin_desc(w_lo + ko), add);
            lin_wgmma<kN>(corr, lin_desc(a_lo + ko), lin_desc(w_hi + ko));
            lin_wgmma<kN>(acc, lin_desc(a_hi + ko), lin_desc(w_hi + ko), add);
          }
          restart = false;
          asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
          if (FOLD && (it + 1) % kLinFoldSteps == 0 && it + 1 < n_it) {
            asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");   // this step's too: fold the chain
            lin_fence_acc(acc); lin_fence_acc(corr);
            emit(nullptr, folded);
            folded = restart = true;
          } else {
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");   // the previous step's MMAs are done
            lin_fence_acc(acc); lin_fence_acc(corr);
          }
          if (prev >= 0) {
            if (lane == 0) lin_mbar_arrive(bars + 8 * (kSt + prev));
            const int t = it - 1 + kSt;                     // the next step that uses the released stage
            if (threadIdx.x == 0 && t < n_it) {
              lin_mbar_wait(bars + 8 * (kSt + prev), ((unsigned)((it - 1) / kSt)) & 1u);   // every warp is done with it
              request_w(t);
            }
            __syncwarp();
          }
          prev = s;
          ++it;
          if (++s == kSt) { s = 0; phase ^= 1; }
        }
      }
    }
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    lin_fence_acc(acc); lin_fence_acc(corr);
    emit(bias, FOLD && folded);
  }
}

// W [O, K] -> per K block the swizzled shared-memory images of its hi and lo TF32 parts
__global__ void k_split_weight(const float* __restrict__ W, int O, int K, float* __restrict__ img) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;    // one 16-byte unit of W
  const int units_per_row = K / 4;
  if (i >= (long long)O * units_per_row) return;
  const int r = (int)(i / units_per_row), u = (int)(i % units_per_row);
  const int kb = u / 8, j = u % 8;
  const float4 w = *reinterpret_cast<const float4*>(W + (long long)r * K + u * 4);
  float4 hi, lo;
  lin_split(w.x, hi.x, lo.x);
  lin_split(w.y, hi.y, lo.y);
  lin_split(w.z, hi.z, lo.z);
  lin_split(w.w, hi.w, lo.w);
  float* tile = img + (long long)kb * (2 * O * kLinBK);
  const unsigned off = lin_swz(r, j) / 4;
  *reinterpret_cast<float4*>(tile + off) = hi;
  *reinterpret_cast<float4*>(tile + O * kLinBK + off) = lo;
}

template <int O, bool FOLD = false>
static int launch_linear(const float* A, long long lda, const float* row_scale, int n_rep, const float* Wimg, const float* bias,
                         float* Y, long long ldy, long long N, int K, cudaStream_t st, int n_slabs = 1, int n_cols = O) {
  auto kern = k_linear_3xtf32<O, FOLD>;
  static bool attr_set = false;
  if (!attr_set) {
    PNA_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LinSmem<O>::kBytes));
    attr_set = true;
  }
  const long long grid = (N + LinSmem<O>::kM - 1) / LinSmem<O>::kM * n_slabs;
  kern<<<(unsigned)grid, kLinThreads, LinSmem<O>::kBytes, st>>>(A, lda, row_scale, n_rep, Wimg, bias, Y, ldy, N, K, n_slabs, n_cols);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

// ================================ backward (pna_linear_bwd_data / pna_linear_bwd_weight) ================================
//
// Data gradient: k_linear_3xtf32 with A = dY (K = O) and the weight W''[c, s * O + o] = W[o, s * n_cols + c]
// (n_cols = n_in / S), in column slabs of width Os.  With row scales the loaders form fl(c_s(i) * dY) like the forward's.

// slab width for n_cols output columns: 128, or 64 where that pads less (n_cols % 128 in (0, 64]).  Never 256: rounding
// up to 256 never pads less than rounding up to 128, and O = 256's 64-row tiles double the weight traffic per output.
static int bwd_data_slab(int n_cols) {
  return (n_cols + 63) / 64 * 64 < (n_cols + 127) / 128 * 128 ? 64 : 128;
}

// W [O, n_in] -> per slab of Os columns of W'' and per K block of W'' the swizzled hi / lo images (as k_split_weight)
__global__ void k_split_weight_t(const float* __restrict__ W, int O, int n_in, int n_rep, int Os, int n_slabs,
                                 float* __restrict__ img) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;    // one 16-byte unit of the image
  const int n_cols = n_in / n_rep, n_kbw = O * n_rep / kLinBK;
  if (i >= (long long)n_slabs * n_kbw * 8 * Os) return;
  const int r = (int)(i % Os);                      // consecutive threads: consecutive columns of W, coalesced reads
  const long long t = i / Os;
  const int j = (int)(t % 8), kbw = (int)(t / 8 % n_kbw), slab = (int)(t / 8 / n_kbw);
  const int c = slab * Os + r;
  const int kk = kbw * kLinBK + j * 4;              // first W'' column of the unit; O % 32 == 0: one scaler per unit
  const int s = kk / O, o = kk % O;
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) v[e] = c < n_cols ? __ldg(W + (long long)(o + e) * n_in + s * n_cols + c) : 0.f;
  float4 hi, lo;
  lin_split(v[0], hi.x, lo.x);
  lin_split(v[1], hi.y, lo.y);
  lin_split(v[2], hi.z, lo.z);
  lin_split(v[3], hi.w, lo.w);
  float* tile = img + ((long long)slab * n_kbw + kbw) * (2 * Os * kLinBK);
  const unsigned off = lin_swz(r, j) / 4;
  *reinterpret_cast<float4*>(tile + off) = hi;
  *reinterpret_cast<float4*>(tile + Os * kLinBK + off) = lo;
}

// Weight gradient dW[o, c] = sum_i dY[i, o] . a'[i, c]  (a' = a, or fl(row_scale[i, c / n_a] * a[i, c % n_a])).
// The reduction runs over the ROWS of both operands and tf32 wgmma reads K-major operands only, so the loaders transpose:
// a thread loads a 4-row x 4-column block (four coalesced 16-byte loads), splits it hi / lo and stores its four columns as
// four 16-byte K-major units (row = column of the operand, unit = its 4 rows) into the 128-byte-swizzled tiles; the 8
// threads of a quarter-warp hold the 8 units of one swizzled row, so the stores are conflict free.
// CTA tile: kTO outputs (rows of dW) x 128 columns, two warpgroups of 64 x kN.  A CTA owns one split of the rows; every
// kWgFoldRows rows it waits for its MMAs and folds (acc + corr) into an fp32 partial in shared memory (each thread its own
// words) with one round-to-nearest add, so no tensor-core accumulation chain (truncating adds) is longer than
// kWgFoldRows / 8 steps; the partial goes to HBM once at the end.  No atomics: it is stored into the CTA's own tile of the
// workspace (or into dW itself with one split), and k_sum_splits adds the splits in ascending order.
constexpr int kWgFoldRows = 64;
constexpr int kWgMinSplitRows = 512;
constexpr int kWgTargetCtas = 264;    // two waves of H100 SXM's 132 SMs at one CTA per SM
constexpr int kWgAhead = 2;           // K blocks of operands in flight per thread

template <int O>
struct WgSmem {
  static constexpr int kTO = O <= 128 ? O : 128;          // dW rows per CTA (O = 256: two tiles)
  static constexpr int kTC = 128;                          // dW columns per CTA
  static constexpr int kN = O == 64 ? 64 : 128;            // columns per warpgroup (O = 64: the warpgroups split columns)
  static constexpr int kYTile = kTO * 128, kATile = kTC * 128;
  static constexpr int kStage = 2 * kYTile + 2 * kATile;   // dY hi, dY lo, a hi, a lo
  static constexpr int kSt = 2;
  static constexpr int kPart = kTO * kTC * 4;               // the fp32 partial tile
  static constexpr int kBlocks = 2 * kTO + 2 * kTC;        // 4 x 4 blocks of a 32-row K block (dY, then a)
  static constexpr int kPer = (kBlocks + kLinThreads - 1) / kLinThreads;
  static constexpr size_t kBytes = 1024 /*align slack*/ + (size_t)kSt * kStage + kPart;
};

struct BwdWeightPlan {
  int col_tiles, o_tiles, n_split;
  long long rows;                     // rows per split, a multiple of 32
};
// depends on the shape alone (not on the device), so the partials -- and the bits of dW -- do too
static BwdWeightPlan bwd_weight_plan(long long n_rows, int n_in, int n_out) {
  BwdWeightPlan p;
  p.col_tiles = (n_in + 127) / 128;
  p.o_tiles = n_out > 128 ? 2 : 1;
  const long long tiles = (long long)p.col_tiles * p.o_tiles;
  long long sp = std::min((n_rows + kWgMinSplitRows - 1) / kWgMinSplitRows, std::max(1ll, (kWgTargetCtas + tiles - 1) / tiles));
  sp = std::max(sp, 1ll);
  p.rows = ((n_rows + sp - 1) / sp + 31) / 32 * 32;
  p.n_split = (int)((n_rows + p.rows - 1) / p.rows);     // no split is empty
  return p;
}

__device__ __forceinline__ float lin_comp(const float4& v, int e) { return e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w; }

template <int O>
__global__ void __launch_bounds__(kLinThreads, 1)
k_linear_bwd_weight(const float* __restrict__ dY, long long ldy, const float* __restrict__ A, long long lda,
                    const float* __restrict__ row_scale, int n_rep, long long N, int n_in, long long rows_per_split,
                    int col_tiles, float* __restrict__ partial) {
  using S = WgSmem<O>;
  constexpr int kTO = S::kTO, kN = S::kN, kSt = S::kSt, kPer = S::kPer;
  extern __shared__ unsigned char lin_raw[];
  const unsigned base = (lin_smem_u32(lin_raw) + 1023u) & ~1023u;
  unsigned char* gbase = lin_raw + (base - lin_smem_u32(lin_raw));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int col_tile = (int)(blockIdx.x % (unsigned)col_tiles);          // the column tiles of one split run side by side
  const int o_tile = (int)(blockIdx.x / (unsigned)col_tiles % (O / kTO));  // and share its dY rows through L2
  const int split = (int)(blockIdx.x / (unsigned)col_tiles / (O / kTO));
  const long long r_begin = split * rows_per_split, r_end = min(N, r_begin + rows_per_split);
  const int n_kb = (int)((r_end - r_begin + kLinBK - 1) / kLinBK);
  const int o0 = o_tile * kTO, c0 = col_tile * S::kTC, n_a = n_in / n_rep;
  partial += (long long)split * O * n_in;

  // block b of a K block: b < 2 kTO -> dY columns o0 + 4 (b >> 3), else a columns c0 + 4 ((b - 2 kTO) >> 3); rows 4 (b & 7)..+3
  auto fetch = [&](int kb, float4 (&dst)[kPer][4]) {
#pragma unroll
    for (int m = 0; m < kPer; ++m) {
      const int b = tid + m * kLinThreads;
      if (b >= S::kBlocks) break;
      const long long i0 = r_begin + (long long)kb * kLinBK + 4 * (b & 7);
      const bool is_y = b < 2 * kTO;
      const int q = (is_y ? b : b - 2 * kTO) >> 3;
      const int c = is_y ? o0 + 4 * q : c0 + 4 * q;
      const int sc = is_y ? 0 : c / n_a;                                  // n_a % 32 == 0: one scaler per unit
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const long long i = i0 + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (kb < n_kb && i < r_end) {
          if (is_y) {
            v = __ldg(reinterpret_cast<const float4*>(dY + i * ldy + c));
          } else if (c < n_in) {
            v = __ldg(reinterpret_cast<const float4*>(A + i * lda + (c - sc * n_a)));
            if (row_scale) {                                                 // the forward loaders' fl(c_s(i) * a)
              const float f = __ldg(row_scale + i * n_rep + sc);
              v.x = __fmul_rn(v.x, f); v.y = __fmul_rn(v.y, f); v.z = __fmul_rn(v.z, f); v.w = __fmul_rn(v.w, f);
            }
          }
        }
        dst[m][r] = v;
      }
    }
  };
  // transpose the 4 x 4 block in registers, split, store four K-major units
  auto stage_store = [&](const float4 (&src)[kPer][4], unsigned char* st) {
#pragma unroll
    for (int m = 0; m < kPer; ++m) {
      const int b = tid + m * kLinThreads;
      if (b >= S::kBlocks) break;
      const bool is_y = b < 2 * kTO;
      const int q = (is_y ? b : b - 2 * kTO) >> 3, jj = b & 7;
      unsigned char* hi_t = st + (is_y ? 0 : 2 * S::kYTile);
      unsigned char* lo_t = hi_t + (is_y ? S::kYTile : S::kATile);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float4 hi, lo;
        const float v0 = lin_comp(src[m][0], e), v1 = lin_comp(src[m][1], e), v2 = lin_comp(src[m][2], e), v3 = lin_comp(src[m][3], e);
        lin_split(v0, hi.x, lo.x);
        lin_split(v1, hi.y, lo.y);
        lin_split(v2, hi.z, lo.z);
        lin_split(v3, hi.w, lo.w);
        const unsigned off = lin_swz(4 * q + e, jj);
        *reinterpret_cast<float4*>(hi_t + off) = hi;
        *reinterpret_cast<float4*>(lo_t + off) = lo;
      }
    }
  };

  const unsigned y_off = O == 64 ? 0u : (unsigned)(wg * 64 * 128);           // this warpgroup's 64 dW rows
  const unsigned a_off = O == 64 ? (unsigned)(wg * 64 * 128) : 0u;           // and its kN columns
  float acc[kN / 2], corr[kN / 2];
#pragma unroll
  for (int i = 0; i < kN / 2; ++i) { acc[i] = 0.f; corr[i] = 0.f; }
  const int wr = (warp & 3) * 16 + (lane >> 2);
  const long long o_lo = o0 + (O == 64 ? 0 : wg * 64) + wr;                  // dW rows of registers 4j, 4j + 1 (+8: 4j + 2, 4j + 3)
  const int c_w = c0 + (O == 64 ? wg * 64 : 0) + 2 * (lane & 3);
  float* part = reinterpret_cast<float*>(gbase + kSt * S::kStage);          // word i * 256 + tid: thread-private
  bool first = true;
  auto fold = [&]() {                                                        // part (+)= acc + corr
#pragma unroll
    for (int i = 0; i < kN / 2; ++i) {
      const float v = acc[i] + corr[i];
      part[i * kLinThreads + tid] = first ? v : part[i * kLinThreads + tid] + v;
    }
    first = false;
  };
  float4 pre[kWgAhead][kPer][4];
#pragma unroll
  for (int u = 0; u < kWgAhead; ++u) fetch(u, pre[u]);
  int s = 0;
  for (int kb0 = 0; kb0 < n_kb; kb0 += kWgAhead) {
#pragma unroll
    for (int u = 0; u < kWgAhead; ++u) {
      const int kb = kb0 + u;
      if (kb >= n_kb) break;
      // stage s was last read by the MMAs of step kb - 2: every warp has waited for them (wait_group 1 after step kb - 1)
      __syncthreads();
      unsigned char* st = gbase + s * S::kStage;
      stage_store(pre[u], st);
      fetch(kb + kWgAhead, pre[u]);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
      const unsigned sa = base + s * S::kStage;
      const unsigned y_hi = sa + y_off, y_lo = sa + S::kYTile + y_off;
      const unsigned a_hi = sa + 2 * S::kYTile + a_off, a_lo = a_hi + S::kATile;
      lin_fence_acc(acc); lin_fence_acc(corr);
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int ks = 0; ks < kLinBK / 8; ++ks) {
        const unsigned ko = ks * 32;
        lin_wgmma<kN>(corr, lin_desc(y_hi + ko), lin_desc(a_lo + ko));
        lin_wgmma<kN>(corr, lin_desc(y_lo + ko), lin_desc(a_hi + ko));
        lin_wgmma<kN>(acc, lin_desc(y_hi + ko), lin_desc(a_hi + ko));
      }
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      if ((kb + 1) % (kWgFoldRows / kLinBK) == 0 || kb + 1 == n_kb) {
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        lin_fence_acc(acc); lin_fence_acc(corr);
        fold();
#pragma unroll
        for (int i = 0; i < kN / 2; ++i) { acc[i] = 0.f; corr[i] = 0.f; }
      } else {
        asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
        lin_fence_acc(acc); lin_fence_acc(corr);
      }
      if (++s == kSt) s = 0;
    }
  }
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");   // (the last step folded: nothing is in flight)
  // the partial tile -> the split's tile of the workspace (or dW), two adjacent columns per store
#pragma unroll
  for (int jj = 0; jj < kN / 8; ++jj) {
    const int c = c_w + jj * 8;
    if (c >= n_in) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(partial + (o_lo + 8 * h) * n_in + c) =
          make_float2(part[(4 * jj + 2 * h) * kLinThreads + tid], part[(4 * jj + 2 * h + 1) * kLinThreads + tid]);
  }
}

// dW = sum over the splits of their partials, in ascending split order (one float4 per thread)
__global__ void k_sum_splits(const float* __restrict__ P, int n_split, long long n4, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4* p = reinterpret_cast<const float4*>(P);
  float4 t = __ldg(p + i);
  for (int sp = 1; sp < n_split; ++sp) {
    const float4 v = __ldg(p + sp * n4 + i);
    t.x = t.x + v.x; t.y = t.y + v.y; t.z = t.z + v.z; t.w = t.w + v.w;
  }
  reinterpret_cast<float4*>(out)[i] = t;
}

template <int O>
static int launch_bwd_weight(const float* dY, long long ldy, const float* A, long long lda, const float* row_scale, int n_rep,
                             long long N, int n_in, const BwdWeightPlan& p, float* partial, cudaStream_t st) {
  auto kern = k_linear_bwd_weight<O>;
  static bool attr_set = false;
  if (!attr_set) {
    PNA_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WgSmem<O>::kBytes));
    attr_set = true;
  }
  const unsigned grid = (unsigned)p.n_split * p.o_tiles * p.col_tiles;
  kern<<<grid, kLinThreads, WgSmem<O>::kBytes, st>>>(dY, ldy, A, lda, row_scale, n_rep, N, n_in, p.rows, p.col_tiles, partial);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

// ============================ tower post linear (pna_linear_towers_scaled_fwd / pna_linear_towers_bwd_data) ============================
//
// PNAConv / the DGL PNALayer with T towers: tower t's first post Linear reads [self_t | cat_s(c_s(i) * agg_t)] (pna.py:131-132,
// pna_layer.py:67).  The aggregation writes the COMPACT per-tower block [self_t | agg_t] ((1 + A) * Fp columns, identity scaler
// only) and the loaders form every scaled copy in registers, as pna_linear_scaled_fwd does for one tower.  Each CTA computes a
// 128-row x 64-column tile of ONE tower's output from that tower's own columns only (no block-diagonal zero work).
//
// A tower's operand is a VIRTUAL K axis that the loaders gather column by column:
//     k < L0:               x[i, k]                                          (forward: the self block; data gradient: dY_t)
//     k = L0 + s * L1 + q:  fl(c_s(i) * x[i, c1 + q])   s < S, q < L1          (forward: agg_t; data gradient: dY_t again)
//     k >= L0 + S * L1:     0                                                 (the last K block's tail)
// Forward: x = a_t, (L0, L1, c1) = (Fp, A Fp, Fp): the virtual axis is exactly the reference weight's column axis
// [self | s-major blocks], so W_t is read as it is.  Data gradient: x = dY_t, (L0, L1, c1) = (O_t, O_t, 0): the unscaled
// copy feeds the self columns (W_t[o, c]), the scaled ones the aggregate columns (W_t[o, Fp + s A Fp + c - Fp]); the
// loaders put zeros in the pairs that do not meet.  The weight tiles are split hi / lo by the same threads straight from
// W_t (no image, no workspace: the weight of one tower is a few KB and stays in L1 / L2).  Element loads are 4-byte
// (tower widths such as 14 or 80 columns give rows that are not 16-byte aligned); 8 threads still cover 128 bytes of a row.
// Every kLinFoldSteps K blocks the chains are folded into an fp32 register total (t = v, then t = fl(t + v) with
// v = fl(fl(acc + corr) + b), b the bias after the last block and +0 before), in the forward as in the data gradient.
constexpr int kTwrM = 128;                 // rows per CTA: two warpgroups of 64
constexpr int kTwrN = 64;                  // output columns per CTA (wgmma n64)
constexpr int kTwrSt = 2;                  // stages: {A hi, A lo, W hi, W lo}
struct TwrSmem {
  static constexpr int kATile = kTwrM * 128, kWTile = kTwrN * 128;
  static constexpr int kStage = 2 * kATile + 2 * kWTile;
  static constexpr size_t kBytes = 1024 /*align slack*/ + (size_t)kTwrSt * kStage;
};

// X's element: fp32, or bf16 (the forward under bf16 autocast) widened to fp32 on load, which is exact; everything after the
// load is the fp32 kernel's, so the bf16 instance computes what the fp32 one computes on the widened aggregate
__device__ __forceinline__ float twr_ld(const float* p) { return __ldg(p); }
__device__ __forceinline__ float twr_ld(const __nv_bfloat16* p) {
  return __uint_as_float(static_cast<unsigned>(__ldg(reinterpret_cast<const unsigned short*>(p))) << 16);
}

template <bool BWD, typename TX>
__device__ __forceinline__ void towers_3xtf32(const TX* __restrict__ X, long long ldx, const float* __restrict__ row_scale, int S,
                                              const float* __restrict__ W, const float* __restrict__ bias, float* __restrict__ Y,
                                              long long ldy, long long N, int T, int Fp, int AF, int Ot, int n_slabs) {
  extern __shared__ unsigned char lin_raw[];
  const unsigned base = (lin_smem_u32(lin_raw) + 1023u) & ~1023u;
  unsigned char* gbase = lin_raw + (base - lin_smem_u32(lin_raw));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  // CTA -> (row tile, tower, column slab): the towers and slabs of one row tile run side by side and share its rows in L2
  const int slab = (int)(blockIdx.x % (unsigned)n_slabs);
  const int t = (int)(blockIdx.x / (unsigned)n_slabs % (unsigned)T);
  const long long row0 = (long long)(blockIdx.x / (unsigned)n_slabs / (unsigned)T) * kTwrM;
  const int L0 = BWD ? Ot : Fp, L1 = BWD ? Ot : AF, c1 = BWD ? 0 : Fp;
  const int Kv = L0 + S * L1;                                   // virtual K
  const int Kw = Fp + S * AF;                                   // columns of W_t
  const int n_kb = (Kv + kLinBK - 1) / kLinBK;
  const int n_out = BWD ? Fp + AF : Ot;                         // output columns of one tower
  X += (long long)t * (BWD ? Ot : Fp + AF);
  W += (long long)t * Ot * Kw;
  Y += (long long)t * n_out + slab * kTwrN;
  const int c_end = min(kTwrN, n_out - slab * kTwrN);           // columns of this slab that exist
  if (bias) bias += (long long)t * Ot;

  // ---- loaders: A unit (row r_in + 32 sl, 4 columns from 4 j), W units u = tid, tid + 256 (row u / 8, 4 columns from 4 (u % 8))
  const int j = tid & 7, r_in = tid >> 3;
  constexpr int kSlabs = kTwrM / 32;
  float xa[kSlabs][4], xs[kSlabs][4], xw[2][4];
  auto fetch = [&](int kb) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = kb * kLinBK + 4 * j + e;
      int col = k, s = -1;                                      // s: scaler of the element, -1 unscaled
      if (k >= L0) {
        const int q = k - L0;
        s = q / L1;
        col = c1 + (q - s * L1);
      }
      const bool live = k < Kv;
#pragma unroll
      for (int sl = 0; sl < kSlabs; ++sl) {
        const long long r = row0 + sl * 32 + r_in;
        const bool ok = live && r < N;
        xa[sl][e] = ok ? twr_ld(X + r * ldx + col) : 0.f;
        xs[sl][e] = (ok && s >= 0) ? __ldg(row_scale + r * S + s) : 1.f;
      }
    }
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const int u = tid + m * kLinThreads, wr = u >> 3, wj = u & 7;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int k = kb * kLinBK + 4 * wj + e;
        float v = 0.f;
        if (!BWD) {                                             // row wr = output o, column k of W_t
          if (wr < Ot && k < Kv) v = __ldg(W + (long long)wr * Kw + k);
        } else {                                                // row wr = grad_a column c of the slab, k virtual
          const int c = slab * kTwrN + wr;
          if (c < n_out && k < Kv) {
            if (k < Ot) {
              if (c < Fp) v = __ldg(W + (long long)k * Kw + c);
            } else if (c >= Fp) {
              const int q = k - Ot, s = q / Ot, o = q - s * Ot;
              v = __ldg(W + (long long)o * Kw + Fp + s * AF + (c - Fp));
            }
          }
        }
        xw[m][e] = v;
      }
    }
  };
  auto store = [&](unsigned char* st) {
#pragma unroll
    for (int sl = 0; sl < kSlabs; ++sl) {
      float4 hi, lo;                                            // scalers.py: src * scale, rounded to fp32 like the reference
      lin_split(__fmul_rn(xa[sl][0], xs[sl][0]), hi.x, lo.x);   // (x * 1 == x exactly: the unscaled and the zero elements)
      lin_split(__fmul_rn(xa[sl][1], xs[sl][1]), hi.y, lo.y);
      lin_split(__fmul_rn(xa[sl][2], xs[sl][2]), hi.z, lo.z);
      lin_split(__fmul_rn(xa[sl][3], xs[sl][3]), hi.w, lo.w);
      const unsigned off = lin_swz(sl * 32 + r_in, j);
      *reinterpret_cast<float4*>(st + off) = hi;
      *reinterpret_cast<float4*>(st + TwrSmem::kATile + off) = lo;
    }
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const int u = tid + m * kLinThreads;
      float4 hi, lo;
      lin_split(xw[m][0], hi.x, lo.x);
      lin_split(xw[m][1], hi.y, lo.y);
      lin_split(xw[m][2], hi.z, lo.z);
      lin_split(xw[m][3], hi.w, lo.w);
      const unsigned off = lin_swz(u >> 3, u & 7);
      *reinterpret_cast<float4*>(st + 2 * TwrSmem::kATile + off) = hi;
      *reinterpret_cast<float4*>(st + 2 * TwrSmem::kATile + TwrSmem::kWTile + off) = lo;
    }
  };

  float acc[kTwrN / 2], corr[kTwrN / 2], tot[kTwrN / 2];
#pragma unroll
  for (int i = 0; i < kTwrN / 2; ++i) { acc[i] = 0.f; corr[i] = 0.f; tot[i] = 0.f; }
  const unsigned a_off = (unsigned)(wg * 64 * 128);              // warpgroup g: rows 64 g.. of the tile, all 64 columns
  bool first = true;
  fetch(0);
  for (int kb = 0; kb < n_kb; ++kb) {
    const int s = kb & 1;
    // stage s was last read by the MMAs of step kb - 2: every warp has waited for them (wait_group 1 after step kb - 1)
    __syncthreads();
    store(gbase + s * TwrSmem::kStage);
    if (kb + 1 < n_kb) fetch(kb + 1);                             // in flight while this step's MMAs run
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const unsigned sa = base + s * TwrSmem::kStage;
    const unsigned a_hi = sa + a_off, a_lo = sa + TwrSmem::kATile + a_off;
    const unsigned w_hi = sa + 2 * TwrSmem::kATile, w_lo = w_hi + TwrSmem::kWTile;
    lin_fence_acc(acc); lin_fence_acc(corr);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int ks = 0; ks < kLinBK / 8; ++ks) {
      const unsigned ko = ks * 32;
      lin_wgmma<kTwrN>(corr, lin_desc(a_hi + ko), lin_desc(w_lo + ko));
      lin_wgmma<kTwrN>(corr, lin_desc(a_lo + ko), lin_desc(w_hi + ko));
      lin_wgmma<kTwrN>(acc, lin_desc(a_hi + ko), lin_desc(w_hi + ko));
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    if ((kb + 1) % kLinFoldSteps == 0 || kb + 1 == n_kb) {        // end of a chain: fold it into the total
      asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
      lin_fence_acc(acc); lin_fence_acc(corr);
      const bool last = kb + 1 == n_kb;
#pragma unroll
      for (int i = 0; i < kTwrN / 2; ++i) {
        const int c = (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
        const float b = (last && bias && c < Ot) ? __ldg(bias + c) : 0.f;
        const float v = (acc[i] + corr[i]) + b;
        tot[i] = first ? v : tot[i] + v;
        acc[i] = 0.f; corr[i] = 0.f;
      }
      first = false;
    } else {
      asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
      lin_fence_acc(acc); lin_fence_acc(corr);
    }
  }
  // register 4 jj + 2 h + q: row (warp % 4) * 16 + lane / 4 + 8 h of the warpgroup's 64, column 8 jj + 2 (lane % 4) + q
  const long long r_lo = row0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < kTwrN / 2; ++i) {
    const int c = (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
    const long long r = r_lo + 8 * ((i >> 1) & 1);
    if (c < c_end && r < N) Y[r * ldy + c] = tot[i];
  }
}

template <bool BWD>
__global__ void __launch_bounds__(kLinThreads, 1)
k_towers_3xtf32(const float* __restrict__ X, long long ldx, const float* __restrict__ row_scale, int S,
                const float* __restrict__ W, const float* __restrict__ bias, float* __restrict__ Y, long long ldy, long long N,
                int T, int Fp, int AF, int Ot, int n_slabs) {
  towers_3xtf32<BWD, float>(X, ldx, row_scale, S, W, bias, Y, ldy, N, T, Fp, AF, Ot, n_slabs);
}

// the forward on a bf16 compact aggregate (pna_linear_towers_scaled_fwd_bf16)
__global__ void __launch_bounds__(kLinThreads, 1)
k_towers_bf16_3xtf32(const __nv_bfloat16* __restrict__ X, long long ldx, const float* __restrict__ row_scale, int S,
                     const float* __restrict__ W, const float* __restrict__ bias, float* __restrict__ Y, long long ldy, long long N,
                     int T, int Fp, int AF, int Ot, int n_slabs) {
  towers_3xtf32<false, __nv_bfloat16>(X, ldx, row_scale, S, W, bias, Y, ldy, N, T, Fp, AF, Ot, n_slabs);
}

template <bool BWD, typename TX = float>
static int launch_towers(const TX* X, long long ldx, const float* row_scale, int S, const float* W, const float* bias, float* Y,
                         long long ldy, long long N, int T, int Fp, int AF, int Ot, cudaStream_t st) {
  void (*kern)(const TX*, long long, const float*, int, const float*, const float*, float*, long long, long long, int, int, int, int,
               int);
  if constexpr (std::is_same<TX, float>::value) kern = k_towers_3xtf32<BWD>;
  else kern = k_towers_bf16_3xtf32;
  static bool attr_set = false;
  if (!attr_set) {
    PNA_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TwrSmem::kBytes));
    attr_set = true;
  }
  const int n_slabs = BWD ? (Fp + AF + kTwrN - 1) / kTwrN : 1;
  const long long grid = (N + kTwrM - 1) / kTwrM * T * n_slabs;
  kern<<<(unsigned)grid, kLinThreads, TwrSmem::kBytes, st>>>(X, ldx, row_scale, S, W, bias, Y, ldy, N, T, Fp, AF, Ot, n_slabs);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

}  // namespace pna

using namespace pna;

extern "C" int pna_linear_workspace_bytes(int32_t n_in, int32_t n_out, size_t* bytes) {
  PNA_REQUIRE(bytes != nullptr && n_in > 0 && n_out > 0, PNA_ERR_BAD_ARG, "pna_linear_workspace_bytes: bad argument");
  *bytes = 2ull * (size_t)n_in * (size_t)n_out * sizeof(float);
  return PNA_OK;
}

// a: [n_rows, n_a] (n_a = n_in / n_rep); weight: [n_out, n_in]; row_scale: [n_rows, n_rep] or null (n_rep == 1)
static int linear_common(const float* a, int64_t lda, const float* row_scale, int32_t n_rep, const float* weight, const float* bias,
                         float* y, int64_t ldy, int64_t n_rows, int32_t n_in, int32_t n_out, void* workspace, size_t workspace_bytes,
                         pna_stream_t stream, const char* who) {
  PNA_REQUIRE(n_rows >= 0 && n_in > 0 && n_out > 0 && n_rep >= 1 && n_rep <= PNA_MAX_SCALERS, PNA_ERR_BAD_ARG, "%s: bad sizes", who);
  PNA_REQUIRE(n_in % n_rep == 0 && (n_in / n_rep) % kLinBK == 0, PNA_ERR_UNSUPPORTED,
              "%s: n_in / n_rep must be a multiple of %d", who, kLinBK);
  PNA_REQUIRE(n_out == 64 || n_out == 128 || n_out == 256, PNA_ERR_UNSUPPORTED, "%s: n_out must be 64, 128 or 256", who);
  if (n_rows == 0) return PNA_OK;
  PNA_REQUIRE(a && weight && y && workspace, PNA_ERR_BAD_ARG, "%s: null pointer", who);
  PNA_REQUIRE(workspace_bytes >= 2ull * n_in * n_out * sizeof(float), PNA_ERR_WORKSPACE, "%s: workspace too small", who);
  PNA_REQUIRE(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(workspace) |
                reinterpret_cast<uintptr_t>(weight)) & 15u) == 0 && lda % 4 == 0 && ldy % 4 == 0,
              PNA_ERR_UNSUPPORTED, "%s: a, y, weight, workspace must be 16-byte aligned with pitches that are multiples of 4", who);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* img = static_cast<float*>(workspace);
  const long long units = (long long)n_out * (n_in / 4);
  k_split_weight<<<(unsigned)((units + 255) / 256), 256, 0, st>>>(weight, n_out, n_in, img);
  PNA_CUDA_TRY(cudaGetLastError());
  const int n_a = n_in / n_rep;
  switch (n_out) {
    case 64: return launch_linear<64>(a, lda, row_scale, n_rep, img, bias, y, ldy, n_rows, n_a, st);
    case 128: return launch_linear<128>(a, lda, row_scale, n_rep, img, bias, y, ldy, n_rows, n_a, st);
    default: return launch_linear<256>(a, lda, row_scale, n_rep, img, bias, y, ldy, n_rows, n_a, st);
  }
}

extern "C" int pna_linear_fwd(const float* a, int64_t lda, const float* weight, const float* bias, float* y, int64_t ldy, int64_t n_rows,
                              int32_t n_in, int32_t n_out, void* workspace, size_t workspace_bytes, pna_stream_t stream) {
  return linear_common(a, lda, nullptr, 1, weight, bias, y, ldy, n_rows, n_in, n_out, workspace, workspace_bytes, stream,
                       "pna_linear_fwd");
}

extern "C" int pna_linear_scaled_fwd(const float* a, int64_t lda, const float* row_scale, int32_t n_scalers, const float* weight,
                                     const float* bias, float* y, int64_t ldy, int64_t n_rows, int32_t n_in, int32_t n_out,
                                     void* workspace, size_t workspace_bytes, pna_stream_t stream) {
  PNA_REQUIRE(row_scale != nullptr || n_rows == 0, PNA_ERR_BAD_ARG, "pna_linear_scaled_fwd: row_scale is null");
  return linear_common(a, lda, row_scale, n_scalers, weight, bias, y, ldy, n_rows, n_in, n_out, workspace, workspace_bytes, stream,
                       "pna_linear_scaled_fwd");
}

// ---- backward ----
static int bwd_check_shape(int64_t n_rows, int32_t n_in, int32_t n_out, int32_t n_rep, const char* who) {
  PNA_REQUIRE(n_rows >= 0 && n_in > 0 && n_out > 0 && n_rep >= 1 && n_rep <= PNA_MAX_SCALERS, PNA_ERR_BAD_ARG, "%s: bad sizes", who);
  PNA_REQUIRE(n_in % n_rep == 0 && (n_in / n_rep) % kLinBK == 0, PNA_ERR_UNSUPPORTED,
              "%s: n_in / n_scalers must be a multiple of %d", who, kLinBK);
  PNA_REQUIRE(n_out == 64 || n_out == 128 || n_out == 256, PNA_ERR_UNSUPPORTED, "%s: n_out must be 64, 128 or 256", who);
  return PNA_OK;
}
static size_t bwd_data_bytes(int32_t n_in, int32_t n_out, int32_t n_rep) {      // the slabs' weight images
  const int n_cols = n_in / n_rep, os = bwd_data_slab(n_cols);
  return 2ull * (size_t)n_out * n_rep * (size_t)((n_cols + os - 1) / os * os) * sizeof(float);
}
static size_t bwd_weight_bytes(int64_t n_rows, int32_t n_in, int32_t n_out) {   // the splits' partials (none for one split)
  const BwdWeightPlan p = bwd_weight_plan(n_rows, n_in, n_out);
  return p.n_split > 1 ? (size_t)p.n_split * n_out * n_in * sizeof(float) : 0;
}

extern "C" int pna_linear_bwd_workspace_bytes(int64_t n_rows, int32_t n_in, int32_t n_out, int32_t n_scalers, size_t* bytes) {
  PNA_REQUIRE(bytes != nullptr, PNA_ERR_BAD_ARG, "pna_linear_bwd_workspace_bytes: bytes is null");
  const int rc = bwd_check_shape(n_rows, n_in, n_out, n_scalers, "pna_linear_bwd_workspace_bytes");
  if (rc != PNA_OK) return rc;
  *bytes = std::max(bwd_data_bytes(n_in, n_out, n_scalers), n_rows > 0 ? bwd_weight_bytes(n_rows, n_in, n_out) : 0);
  return PNA_OK;
}

extern "C" int pna_linear_bwd_data(const float* grad_y, int64_t ld_grad_y, const float* row_scale, int32_t n_scalers, const float* weight,
                                   float* grad_a, int64_t ld_grad_a, int64_t n_rows, int32_t n_in, int32_t n_out, void* workspace,
                                   size_t workspace_bytes, pna_stream_t stream) {
  const char* who = "pna_linear_bwd_data";
  const int rc = bwd_check_shape(n_rows, n_in, n_out, n_scalers, who);
  if (rc != PNA_OK) return rc;
  if (n_rows == 0) return PNA_OK;
  PNA_REQUIRE(grad_y && weight && grad_a && workspace, PNA_ERR_BAD_ARG, "%s: null pointer", who);
  PNA_REQUIRE(row_scale || n_scalers == 1, PNA_ERR_BAD_ARG, "%s: row_scale is null with %d scalers", who, n_scalers);
  PNA_REQUIRE(workspace_bytes >= bwd_data_bytes(n_in, n_out, n_scalers), PNA_ERR_WORKSPACE, "%s: workspace too small", who);
  PNA_REQUIRE(((reinterpret_cast<uintptr_t>(grad_y) | reinterpret_cast<uintptr_t>(grad_a) | reinterpret_cast<uintptr_t>(workspace)) &
               15u) == 0 && ld_grad_y % 4 == 0 && ld_grad_a % 4 == 0,
              PNA_ERR_UNSUPPORTED, "%s: grad_y, grad_a, workspace must be 16-byte aligned with pitches that are multiples of 4", who);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int n_cols = n_in / n_scalers, os = bwd_data_slab(n_cols), n_slabs = (n_cols + os - 1) / os;
  float* img = static_cast<float*>(workspace);
  const long long units = (long long)n_slabs * (n_out * n_scalers / kLinBK) * 8 * os;
  k_split_weight_t<<<(unsigned)((units + 255) / 256), 256, 0, st>>>(weight, n_out, n_in, n_scalers, os, n_slabs, img);
  PNA_CUDA_TRY(cudaGetLastError());
  // a chain of at most kLinFoldSteps K blocks is never folded: the non-folding instance, whose wgmmas ptxas does not serialize
  const bool fold = n_out * n_scalers / kLinBK > kLinFoldSteps;
  if (os == 64)
    return fold ? launch_linear<64, true>(grad_y, ld_grad_y, row_scale, n_scalers, img, nullptr, grad_a, ld_grad_a, n_rows, n_out, st, n_slabs, n_cols)
                : launch_linear<64>(grad_y, ld_grad_y, row_scale, n_scalers, img, nullptr, grad_a, ld_grad_a, n_rows, n_out, st, n_slabs, n_cols);
  return fold ? launch_linear<128, true>(grad_y, ld_grad_y, row_scale, n_scalers, img, nullptr, grad_a, ld_grad_a, n_rows, n_out, st, n_slabs, n_cols)
              : launch_linear<128>(grad_y, ld_grad_y, row_scale, n_scalers, img, nullptr, grad_a, ld_grad_a, n_rows, n_out, st, n_slabs, n_cols);
}

extern "C" int pna_linear_bwd_weight(const float* grad_y, int64_t ld_grad_y, const float* a, int64_t lda, const float* row_scale,
                                     int32_t n_scalers, float* grad_weight, int64_t n_rows, int32_t n_in, int32_t n_out, void* workspace,
                                     size_t workspace_bytes, pna_stream_t stream) {
  const char* who = "pna_linear_bwd_weight";
  const int rc = bwd_check_shape(n_rows, n_in, n_out, n_scalers, who);
  if (rc != PNA_OK) return rc;
  if (n_rows == 0) return PNA_OK;
  PNA_REQUIRE(grad_y && a && grad_weight, PNA_ERR_BAD_ARG, "%s: null pointer", who);
  PNA_REQUIRE(row_scale || n_scalers == 1, PNA_ERR_BAD_ARG, "%s: row_scale is null with %d scalers", who, n_scalers);
  const size_t need = bwd_weight_bytes(n_rows, n_in, n_out);
  PNA_REQUIRE(workspace_bytes >= need && (workspace || need == 0), PNA_ERR_WORKSPACE, "%s: workspace too small", who);
  PNA_REQUIRE(((reinterpret_cast<uintptr_t>(grad_y) | reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(grad_weight) |
                reinterpret_cast<uintptr_t>(workspace)) & 15u) == 0 && ld_grad_y % 4 == 0 && lda % 4 == 0,
              PNA_ERR_UNSUPPORTED, "%s: grad_y, a, grad_weight, workspace must be 16-byte aligned with pitches that are multiples of 4", who);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const BwdWeightPlan p = bwd_weight_plan(n_rows, n_in, n_out);
  float* partial = p.n_split > 1 ? static_cast<float*>(workspace) : grad_weight;
  int r;
  switch (n_out) {
    case 64: r = launch_bwd_weight<64>(grad_y, ld_grad_y, a, lda, row_scale, n_scalers, n_rows, n_in, p, partial, st); break;
    case 128: r = launch_bwd_weight<128>(grad_y, ld_grad_y, a, lda, row_scale, n_scalers, n_rows, n_in, p, partial, st); break;
    default: r = launch_bwd_weight<256>(grad_y, ld_grad_y, a, lda, row_scale, n_scalers, n_rows, n_in, p, partial, st); break;
  }
  if (r != PNA_OK || p.n_split == 1) return r;
  const long long n4 = (long long)n_out * n_in / 4;
  k_sum_splits<<<(unsigned)((n4 + 255) / 256), 256, 0, st>>>(partial, p.n_split, n4, grad_weight);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

// ---- tower layers ----
static int towers_check(int64_t n_rows, int32_t n_towers, int32_t n_feat, int32_t n_aggr, int32_t n_out, int32_t n_scalers,
                        const char* who) {
  PNA_REQUIRE(n_rows >= 0 && n_towers >= 1 && n_feat > 0 && n_aggr >= 1 && n_aggr <= PNA_MAX_AGGR && n_out >= 1 && n_scalers >= 1 &&
                  n_scalers <= PNA_MAX_SCALERS,
              PNA_ERR_BAD_ARG, "%s: bad sizes", who);
  PNA_REQUIRE(n_towers <= 8 && n_out <= 64 && n_towers * n_out <= 256 && n_feat % 4 == 0, PNA_ERR_UNSUPPORTED,
              "%s: needs n_towers <= 8, n_out <= 64, n_towers * n_out <= 256 and n_feat %% 4 == 0", who);
  return PNA_OK;
}

extern "C" int pna_linear_towers_scaled_fwd(const float* a, int64_t lda, const float* row_scale, int32_t n_scalers, const float* weight,
                                            const float* bias, float* y, int64_t ldy, int64_t n_rows, int32_t n_towers, int32_t n_feat,
                                            int32_t n_aggr, int32_t n_out, pna_stream_t stream) {
  const char* who = "pna_linear_towers_scaled_fwd";
  const int rc = towers_check(n_rows, n_towers, n_feat, n_aggr, n_out, n_scalers, who);
  if (rc != PNA_OK) return rc;
  if (n_rows == 0) return PNA_OK;
  PNA_REQUIRE(a && row_scale && weight && y, PNA_ERR_BAD_ARG, "%s: null pointer", who);
  PNA_REQUIRE(lda >= (int64_t)n_towers * (1 + n_aggr) * n_feat && ldy >= (int64_t)n_towers * n_out, PNA_ERR_BAD_ARG,
              "%s: row pitch smaller than the row", who);
  return launch_towers<false>(a, lda, row_scale, n_scalers, weight, bias, y, ldy, n_rows, n_towers, n_feat, n_aggr * n_feat, n_out,
                              static_cast<cudaStream_t>(stream));
}

extern "C" int pna_linear_towers_scaled_fwd_bf16(const void* a, int64_t lda, const float* row_scale, int32_t n_scalers,
                                                 const float* weight, const float* bias, float* y, int64_t ldy, int64_t n_rows,
                                                 int32_t n_towers, int32_t n_feat, int32_t n_aggr, int32_t n_out, pna_stream_t stream) {
  const char* who = "pna_linear_towers_scaled_fwd_bf16";
  const int rc = towers_check(n_rows, n_towers, n_feat, n_aggr, n_out, n_scalers, who);
  if (rc != PNA_OK) return rc;
  if (n_rows == 0) return PNA_OK;
  PNA_REQUIRE(a && row_scale && weight && y, PNA_ERR_BAD_ARG, "%s: null pointer", who);
  PNA_REQUIRE(lda >= (int64_t)n_towers * (1 + n_aggr) * n_feat && ldy >= (int64_t)n_towers * n_out, PNA_ERR_BAD_ARG,
              "%s: row pitch smaller than the row", who);
  return launch_towers<false>(static_cast<const __nv_bfloat16*>(a), lda, row_scale, n_scalers, weight, bias, y, ldy, n_rows, n_towers,
                              n_feat, n_aggr * n_feat, n_out, static_cast<cudaStream_t>(stream));
}

extern "C" int pna_linear_towers_bwd_data(const float* grad_y, int64_t ld_grad_y, const float* row_scale, int32_t n_scalers,
                                          const float* weight, float* grad_a, int64_t ld_grad_a, int64_t n_rows, int32_t n_towers,
                                          int32_t n_feat, int32_t n_aggr, int32_t n_out, pna_stream_t stream) {
  const char* who = "pna_linear_towers_bwd_data";
  const int rc = towers_check(n_rows, n_towers, n_feat, n_aggr, n_out, n_scalers, who);
  if (rc != PNA_OK) return rc;
  if (n_rows == 0) return PNA_OK;
  PNA_REQUIRE(grad_y && row_scale && weight && grad_a, PNA_ERR_BAD_ARG, "%s: null pointer", who);
  PNA_REQUIRE(ld_grad_y >= (int64_t)n_towers * n_out && ld_grad_a >= (int64_t)n_towers * (1 + n_aggr) * n_feat, PNA_ERR_BAD_ARG,
              "%s: row pitch smaller than the row", who);
  return launch_towers<true>(grad_y, ld_grad_y, row_scale, n_scalers, weight, nullptr, grad_a, ld_grad_a, n_rows, n_towers, n_feat,
                             n_aggr * n_feat, n_out, static_cast<cudaStream_t>(stream));
}

namespace pna {
__global__ void k_row_scales(const int* __restrict__ rowptr, long long n_rows, int n_scalers, unsigned codes, float avg_log,
                             float avg_lin, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows) return;
  const DegScales ds = deg_scales(__ldg(rowptr + i + 1) - __ldg(rowptr + i), avg_log, avg_lin);
  for (int s = 0; s < n_scalers; ++s) out[i * n_scalers + s] = ds.of((codes >> (4 * s)) & 15u);
}
}  // namespace pna

extern "C" int pna_row_scales(const int32_t* rowptr, int64_t n_rows, int32_t n_scalers, uint32_t scaler_codes, float avg_log,
                              float avg_lin, float* scales, pna_stream_t stream) {
  PNA_REQUIRE(n_rows >= 0 && n_scalers >= 1 && n_scalers <= PNA_MAX_SCALERS, PNA_ERR_BAD_ARG, "pna_row_scales: bad sizes");
  for (int s = 0; s < n_scalers; ++s)
    PNA_REQUIRE(((scaler_codes >> (4 * s)) & 15u) <= PNA_SCALE_INVERSE_LINEAR, PNA_ERR_BAD_ARG, "pna_row_scales: bad scaler code");
  if (n_rows == 0) return PNA_OK;
  PNA_REQUIRE(rowptr && scales, PNA_ERR_BAD_ARG, "pna_row_scales: null pointer");
  k_row_scales<<<(unsigned)((n_rows + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(rowptr, n_rows, n_scalers, scaler_codes,
                                                                                            avg_log, avg_lin, scales);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}
