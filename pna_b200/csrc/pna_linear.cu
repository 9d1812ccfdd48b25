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
// register 4j + q of lane l holds row l/4 + 8 (q/2) of the warp's 16 rows, column 8j + 2 (l%4) + q%2)
template <int N>
__device__ __forceinline__ void lin_wgmma(float (&d)[N / 2], unsigned long long adesc, unsigned long long bdesc);
template <>
__device__ __forceinline__ void lin_wgmma<64>(float (&d)[32], unsigned long long adesc, unsigned long long bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1;\n\t}"
      : LIN_F16(d, 0), LIN_F16(d, 16)
      : "l"(adesc), "l"(bdesc));
}
template <>
__device__ __forceinline__ void lin_wgmma<128>(float (&d)[64], unsigned long long adesc, unsigned long long bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1;\n\t}"
      : LIN_F16(d, 0), LIN_F16(d, 16), LIN_F16(d, 32), LIN_F16(d, 48)
      : "l"(adesc), "l"(bdesc));
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
template <int O>
__global__ void __launch_bounds__(kLinThreads, 1)
k_linear_3xtf32(const float* __restrict__ A, long long lda, const float* __restrict__ row_scale, int n_rep,
                const float* __restrict__ Wimg, const float* __restrict__ bias, float* __restrict__ Y, long long ldy, long long N,
                int K) {
  constexpr int kSt = LinSmem<O>::kSt, kM = LinSmem<O>::kM, kN = LinSmem<O>::kN;
  extern __shared__ unsigned char lin_raw[];
  const unsigned base = (lin_smem_u32(lin_raw) + 1023u) & ~1023u;          // swizzle atoms need 1024-byte alignment
  unsigned char* gbase = lin_raw + (base - lin_smem_u32(lin_raw));
  const unsigned bars = base + kSt * LinSmem<O>::kStage;                    // full[kSt], empty[kSt]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row0 = (long long)blockIdx.x * kM;
  const int n_kb = K / kLinBK;          // K blocks of A (compact width)
  const int n_it = n_kb * n_rep;        // pipeline steps = K blocks of W (n_rep == 1 without row scales)

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
            hi.x = lin_tf32(v.x); lo.x = lin_tf32(v.x - hi.x);
            hi.y = lin_tf32(v.y); lo.y = lin_tf32(v.y - hi.y);
            hi.z = lin_tf32(v.z); lo.z = lin_tf32(v.z - hi.z);
            hi.w = lin_tf32(v.w); lo.w = lin_tf32(v.w - hi.w);
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
            lin_wgmma<kN>(corr, lin_desc(a_hi + ko), lin_desc(w_lo + ko));
            lin_wgmma<kN>(corr, lin_desc(a_lo + ko), lin_desc(w_hi + ko));
            lin_wgmma<kN>(acc, lin_desc(a_hi + ko), lin_desc(w_hi + ko));
          }
          asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
          asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");     // the previous step's MMAs are done
          lin_fence_acc(acc); lin_fence_acc(corr);
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
    // ---------------- epilogue: (main + cross terms) + bias, two adjacent columns per store ----------------
    const int wr = (warp & 3) * 16 + (lane >> 2);           // row of the warpgroup's 64 for registers 4j, 4j + 1
    const long long r_lo = row0 + (O <= 128 ? wg * 64 : 0) + wr, r_hi = r_lo + 8;
#pragma unroll
    for (int jj = 0; jj < kN / 8; ++jj) {
      const int c = (O <= 128 ? 0 : wg * kN) + jj * 8 + 2 * (lane & 3);
      const float b0 = bias ? __ldg(bias + c) : 0.f, b1 = bias ? __ldg(bias + c + 1) : 0.f;
      if (r_lo < N)
        *reinterpret_cast<float2*>(Y + r_lo * ldy + c) = make_float2((acc[4 * jj] + corr[4 * jj]) + b0, (acc[4 * jj + 1] + corr[4 * jj + 1]) + b1);
      if (r_hi < N)
        *reinterpret_cast<float2*>(Y + r_hi * ldy + c) =
            make_float2((acc[4 * jj + 2] + corr[4 * jj + 2]) + b0, (acc[4 * jj + 3] + corr[4 * jj + 3]) + b1);
    }
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
  hi.x = lin_tf32(w.x); lo.x = lin_tf32(w.x - hi.x);
  hi.y = lin_tf32(w.y); lo.y = lin_tf32(w.y - hi.y);
  hi.z = lin_tf32(w.z); lo.z = lin_tf32(w.z - hi.z);
  hi.w = lin_tf32(w.w); lo.w = lin_tf32(w.w - hi.w);
  float* tile = img + (long long)kb * (2 * O * kLinBK);
  const unsigned off = lin_swz(r, j) / 4;
  *reinterpret_cast<float4*>(tile + off) = hi;
  *reinterpret_cast<float4*>(tile + O * kLinBK + off) = lo;
}

template <int O>
static int launch_linear(const float* A, long long lda, const float* row_scale, int n_rep, const float* Wimg, const float* bias,
                         float* Y, long long ldy, long long N, int K, cudaStream_t st) {
  auto kern = k_linear_3xtf32<O>;
  static bool attr_set = false;
  if (!attr_set) {
    PNA_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LinSmem<O>::kBytes));
    attr_set = true;
  }
  const long long grid = (N + LinSmem<O>::kM - 1) / LinSmem<O>::kM;
  kern<<<(unsigned)grid, kLinThreads, LinSmem<O>::kBytes, st>>>(A, lda, row_scale, n_rep, Wimg, bias, Y, ldy, N, K);
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
