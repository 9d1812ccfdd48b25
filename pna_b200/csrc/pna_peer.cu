// Peer-memory data plane of the destination-partitioned multi-GPU path (SURVEY section 8e; DESIGN.md section 6).
//
//   pna_halo_pull     the halo exchange as ONE kernel of peer loads: every rank pulls the de-duplicated remote source
//                     rows it needs straight out of the owners' HBM over NVLink into the tail of its own
//                     [local ; halo] feature buffer.  It replaces pack (pna_gather_rows) -> NCCL all-to-all-v -> unpack:
//                     no send buffer, no collective, each remote row crosses NVLink once per layer.
//   pna_halo_grad_pull  its transpose for the backward: every owner pulls the gradients its peers hold for their halo
//                     copies of its rows and adds them into its own rows' gradient, in a fixed order (no atomics).
//   pna_peer_barrier  device-side barrier between the ranks: one flag store per peer + a spin on the own flags
//                     (instead of a host-driven collective): "every rank has finished writing its feature rows".
//
// The reference has no distributed code (SURVEY section 2); BASELINE.json's north_star names the exchange
// ("single NCCL all-to-all for halo source features per layer"), which stays available as the `halo` plane in
// pna_b200/dist.py and is what this kernel is measured against.
#include "common.cuh"

namespace pna {

constexpr int kPullThreads = 256;
constexpr int kPullRowsInFlight = 4;   // rows per warp iteration: 4 x (row bytes) of NVLink loads in flight per warp

// dst[i, :] = rank (enc[i] >> shift)'s row (enc[i] & mask); 16-byte chunks, CHUNKS of them per lane per row.
// ld.global.cg semantics (__ldcg): peer lines are never kept in this SM's L1 across steps.
template <int CHUNKS>
__global__ void __launch_bounds__(kPullThreads) k_halo_pull(const unsigned long long* __restrict__ peer_base, long long ld_bytes,
                                                            const int* __restrict__ enc, int shift, long long n,
                                                            char* __restrict__ dst, long long ld_dst_bytes, int row_bytes) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kPullThreads / 32);
  const long long w = (long long)blockIdx.x * (kPullThreads / 32) + (threadIdx.x >> 5);
  const int mask = (1 << shift) - 1;
  for (long long r0 = w * kPullRowsInFlight; r0 < n; r0 += warps * kPullRowsInFlight) {
    uint4 v[kPullRowsInFlight][CHUNKS];
#pragma unroll
    for (int u = 0; u < kPullRowsInFlight; ++u) {
      if (r0 + u < n) {
        const int e = __ldg(enc + r0 + u);
        const char* sp = reinterpret_cast<const char*>(__ldg(peer_base + ((unsigned)e >> shift))) + (long long)(e & mask) * ld_bytes;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
          const int b = (lane + c * 32) * 16;
          if (b < row_bytes) v[u][c] = __ldcg(reinterpret_cast<const uint4*>(sp + b));
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kPullRowsInFlight; ++u) {
      if (r0 + u < n) {
        char* dp = dst + (r0 + u) * ld_dst_bytes;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
          const int b = (lane + c * 32) * 16;
          if (b < row_bytes) *reinterpret_cast<uint4*>(dp + b) = v[u][c];
        }
      }
    }
  }
}

// rows that are not a multiple of 16 bytes or not 16-byte aligned: 4- or 2-byte elements
template <typename W>
__global__ void __launch_bounds__(kPullThreads) k_halo_pull_narrow(const unsigned long long* __restrict__ peer_base, long long ld_bytes,
                                                                   const int* __restrict__ enc, int shift, long long n,
                                                                   char* __restrict__ dst, long long ld_dst_bytes, int row_bytes) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kPullThreads / 32);
  const long long w = (long long)blockIdx.x * (kPullThreads / 32) + (threadIdx.x >> 5);
  const int mask = (1 << shift) - 1;
  for (long long r = w; r < n; r += warps) {
    const int e = __ldg(enc + r);
    const char* sp = reinterpret_cast<const char*>(__ldg(peer_base + ((unsigned)e >> shift))) + (long long)(e & mask) * ld_bytes;
    char* dp = dst + r * ld_dst_bytes;
    for (int b = lane * (int)sizeof(W); b < row_bytes; b += 32 * (int)sizeof(W))
      *reinterpret_cast<W*>(dp + b) = __ldcg(reinterpret_cast<const W*>(sp + b));
  }
}

// The transpose of k_halo_pull (the backward of the pull plane): the owner adds the gradients its peers hold for copies of
// its rows.  grad[rows[i], :] += rank (enc[s] >> shift)'s halo-gradient row (enc[s] & mask) for s in [rowptr[i], rowptr[i+1]),
// in slot order, one fp32 rounding per add.  A row is owned by one warp and no two list entries name the same row, so there
// are no atomics and the result is the same bits on every run.  Lanes map to 16-byte chunks (CHUNKS per lane), several rows
// are in flight per warp: the k-th slots of all of them are loaded before any is added.
template <int CHUNKS>
__global__ void __launch_bounds__(kPullThreads) k_halo_grad_pull(const unsigned long long* __restrict__ peer_base, long long ld_bytes,
                                                                 const int* __restrict__ rows, const int* __restrict__ rowptr,
                                                                 const int* __restrict__ enc, int shift, long long n,
                                                                 float* __restrict__ grad, long long ld_grad, int n_vec) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kPullThreads / 32);
  const long long w = (long long)blockIdx.x * (kPullThreads / 32) + (threadIdx.x >> 5);
  const int mask = (1 << shift) - 1;
  for (long long r0 = w * kPullRowsInFlight; r0 < n; r0 += warps * kPullRowsInFlight) {
    float4 acc[kPullRowsInFlight][CHUNKS];
    int s0[kPullRowsInFlight], cnt[kPullRowsInFlight];
    float* gp[kPullRowsInFlight];
    int k_max = 0;
#pragma unroll
    for (int u = 0; u < kPullRowsInFlight; ++u) {
      s0[u] = 0;
      cnt[u] = 0;
      gp[u] = grad;
      if (r0 + u < n) {
        s0[u] = __ldg(rowptr + r0 + u);
        cnt[u] = __ldg(rowptr + r0 + u + 1) - s0[u];
        gp[u] = grad + (long long)__ldg(rows + r0 + u) * ld_grad;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
          const int q = lane + c * 32;
          if (q < n_vec) acc[u][c] = *reinterpret_cast<const float4*>(gp[u] + 4 * q);
        }
        k_max = max(k_max, cnt[u]);
      }
    }
    for (int k = 0; k < k_max; ++k) {
      float4 v[kPullRowsInFlight][CHUNKS];
#pragma unroll
      for (int u = 0; u < kPullRowsInFlight; ++u) {
        if (k < cnt[u]) {
          const int e = __ldg(enc + s0[u] + k);
          const float* sp = reinterpret_cast<const float*>(reinterpret_cast<const char*>(__ldg(peer_base + ((unsigned)e >> shift))) +
                                                           (long long)(e & mask) * ld_bytes);
#pragma unroll
          for (int c = 0; c < CHUNKS; ++c) {
            const int q = lane + c * 32;
            if (q < n_vec) v[u][c] = __ldcg(reinterpret_cast<const float4*>(sp + 4 * q));
          }
        }
      }
#pragma unroll
      for (int u = 0; u < kPullRowsInFlight; ++u) {
        if (k < cnt[u]) {
#pragma unroll
          for (int c = 0; c < CHUNKS; ++c) {
            if (lane + c * 32 < n_vec) {
              acc[u][c].x = __fadd_rn(acc[u][c].x, v[u][c].x);
              acc[u][c].y = __fadd_rn(acc[u][c].y, v[u][c].y);
              acc[u][c].z = __fadd_rn(acc[u][c].z, v[u][c].z);
              acc[u][c].w = __fadd_rn(acc[u][c].w, v[u][c].w);
            }
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kPullRowsInFlight; ++u) {
      if (r0 + u < n && cnt[u] > 0) {
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
          const int q = lane + c * 32;
          if (q < n_vec) *reinterpret_cast<float4*>(gp[u] + 4 * q) = acc[u][c];
        }
      }
    }
  }
}

// widths that are not a multiple of 4 floats or pitches / pointers that are not 16-byte aligned: one row per warp, 4-byte lanes
__global__ void __launch_bounds__(kPullThreads) k_halo_grad_pull_narrow(const unsigned long long* __restrict__ peer_base, long long ld_bytes,
                                                                        const int* __restrict__ rows, const int* __restrict__ rowptr,
                                                                        const int* __restrict__ enc, int shift, long long n,
                                                                        float* __restrict__ grad, long long ld_grad, int n_feat) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kPullThreads / 32);
  const long long w = (long long)blockIdx.x * (kPullThreads / 32) + (threadIdx.x >> 5);
  const int mask = (1 << shift) - 1;
  for (long long r = w; r < n; r += warps) {
    const int s0 = __ldg(rowptr + r), s1 = __ldg(rowptr + r + 1);
    if (s1 <= s0) continue;
    float* gp = grad + (long long)__ldg(rows + r) * ld_grad;
    for (int f = lane; f < n_feat; f += 32) {
      float a = gp[f];
      for (int s = s0; s < s1; ++s) {
        const int e = __ldg(enc + s);
        const float* sp = reinterpret_cast<const float*>(reinterpret_cast<const char*>(__ldg(peer_base + ((unsigned)e >> shift))) +
                                                         (long long)(e & mask) * ld_bytes);
        a = __fadd_rn(a, __ldcg(sp + f));
      }
      gp[f] = a;
    }
  }
}

// One CTA, one thread per peer.  flags[r] (on every rank) = the last epoch rank r has announced to this rank.
// status[0] is set to 1 if a peer did not arrive within timeout_ns (the kernel then returns instead of hanging the GPU).
__global__ void k_peer_barrier(const unsigned long long* __restrict__ flag_base, int rank, int world, unsigned long long epoch,
                               unsigned long long timeout_ns, int* status) {
  const int p = threadIdx.x;
  if (p >= world) return;
  // everything earlier kernels of this stream wrote (the rank's feature rows) is visible system-wide before the flag is
  __threadfence_system();
  unsigned long long* theirs = reinterpret_cast<unsigned long long*>(flag_base[p]) + rank;
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(theirs), "l"(epoch) : "memory");
  const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(flag_base[rank]) + p;
  unsigned long long t0, t1, seen;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (;;) {
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(mine) : "memory");
    if (seen >= epoch) break;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (t1 - t0 > timeout_ns) {
      if (status) atomicExch(status, 1);
      break;
    }
    __nanosleep(100);
  }
}

}  // namespace pna

using namespace pna;

extern "C" int pna_halo_pull(const void* const* peer_rows, int64_t ld_rows, const int32_t* enc, int32_t peer_shift, int64_t n_idx,
                             void* dst, int64_t ld_dst, int32_t n_feat, int32_t dtype, pna_stream_t stream) {
  PNA_REQUIRE(n_idx >= 0 && n_feat > 0 && ld_rows >= n_feat && ld_dst >= n_feat, PNA_ERR_BAD_ARG, "pna_halo_pull: bad sizes");
  PNA_REQUIRE(dtype == PNA_F32 || dtype == PNA_BF16, PNA_ERR_UNSUPPORTED, "pna_halo_pull: dtype %d", dtype);
  PNA_REQUIRE(peer_shift >= 1 && peer_shift <= 30, PNA_ERR_BAD_ARG, "pna_halo_pull: peer_shift out of range");
  if (n_idx == 0) return PNA_OK;
  PNA_REQUIRE(peer_rows && enc && dst, PNA_ERR_BAD_ARG, "pna_halo_pull: null pointer");
  const int esz = dtype == PNA_F32 ? 4 : 2;
  const int row_bytes = n_feat * esz;
  const long long ldb = ld_rows * esz, lddb = ld_dst * esz;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    PNA_CUDA_TRY(cudaGetDevice(&dev));
    PNA_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const long long warps_needed = (n_idx + kPullRowsInFlight - 1) / kPullRowsInFlight;
  long long grid = (warps_needed + (kPullThreads / 32) - 1) / (kPullThreads / 32);
  if (grid > 4ll * sms) grid = 4ll * sms;
  const auto* base = reinterpret_cast<const unsigned long long*>(peer_rows);
  const bool vec = (row_bytes % 16 == 0) && (ldb % 16 == 0) && (lddb % 16 == 0) && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0);
  if (vec && row_bytes <= 512)
    k_halo_pull<1><<<(unsigned)grid, kPullThreads, 0, st>>>(base, ldb, enc, peer_shift, n_idx, (char*)dst, lddb, row_bytes);
  else if (vec && row_bytes <= 1024)
    k_halo_pull<2><<<(unsigned)grid, kPullThreads, 0, st>>>(base, ldb, enc, peer_shift, n_idx, (char*)dst, lddb, row_bytes);
  else if (vec && row_bytes <= 2048)
    k_halo_pull<4><<<(unsigned)grid, kPullThreads, 0, st>>>(base, ldb, enc, peer_shift, n_idx, (char*)dst, lddb, row_bytes);
  else if (row_bytes % 4 == 0 && ldb % 4 == 0 && lddb % 4 == 0)
    k_halo_pull_narrow<unsigned><<<(unsigned)grid, kPullThreads, 0, st>>>(base, ldb, enc, peer_shift, n_idx, (char*)dst, lddb, row_bytes);
  else
    k_halo_pull_narrow<unsigned short><<<(unsigned)grid, kPullThreads, 0, st>>>(base, ldb, enc, peer_shift, n_idx, (char*)dst, lddb, row_bytes);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

extern "C" int pna_halo_grad_pull(const void* const* peer_rows, int64_t ld_rows, const int32_t* rows, const int32_t* rowptr,
                                  const int32_t* enc, int32_t enc_shift, int64_t n_rows, float* grad, int64_t ld_grad, int32_t n_feat,
                                  pna_stream_t stream) {
  PNA_REQUIRE(n_rows >= 0 && n_feat > 0 && ld_rows >= n_feat && ld_grad >= n_feat, PNA_ERR_BAD_ARG, "pna_halo_grad_pull: bad sizes");
  PNA_REQUIRE(enc_shift >= 1 && enc_shift <= 30, PNA_ERR_BAD_ARG, "pna_halo_grad_pull: enc_shift out of range");
  if (n_rows == 0) return PNA_OK;
  PNA_REQUIRE(peer_rows && rows && rowptr && enc && grad, PNA_ERR_BAD_ARG, "pna_halo_grad_pull: null pointer");
  const long long ldb = ld_rows * 4;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    PNA_CUDA_TRY(cudaGetDevice(&dev));
    PNA_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const long long warps_needed = (n_rows + kPullRowsInFlight - 1) / kPullRowsInFlight;
  long long grid = (warps_needed + (kPullThreads / 32) - 1) / (kPullThreads / 32);
  if (grid > 4ll * sms) grid = 4ll * sms;
  const auto* base = reinterpret_cast<const unsigned long long*>(peer_rows);
  const bool vec = (n_feat % 4 == 0) && (ld_rows % 4 == 0) && (ld_grad % 4 == 0) && ((reinterpret_cast<uintptr_t>(grad) & 15u) == 0);
  const int n_vec = n_feat / 4;
  if (vec && n_feat <= 128)
    k_halo_grad_pull<1><<<(unsigned)grid, kPullThreads, 0, st>>>(base, ldb, rows, rowptr, enc, enc_shift, n_rows, grad, ld_grad, n_vec);
  else if (vec && n_feat <= 256)
    k_halo_grad_pull<2><<<(unsigned)grid, kPullThreads, 0, st>>>(base, ldb, rows, rowptr, enc, enc_shift, n_rows, grad, ld_grad, n_vec);
  else if (vec && n_feat <= 512)
    k_halo_grad_pull<4><<<(unsigned)grid, kPullThreads, 0, st>>>(base, ldb, rows, rowptr, enc, enc_shift, n_rows, grad, ld_grad, n_vec);
  else
    k_halo_grad_pull_narrow<<<(unsigned)grid, kPullThreads, 0, st>>>(base, ldb, rows, rowptr, enc, enc_shift, n_rows, grad, ld_grad, n_feat);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

extern "C" int pna_peer_barrier(const void* const* peer_flags, int32_t rank, int32_t world, uint64_t epoch, uint64_t timeout_ns,
                                int32_t* status, pna_stream_t stream) {
  PNA_REQUIRE(peer_flags != nullptr && world >= 1 && world <= 64 && rank >= 0 && rank < world, PNA_ERR_BAD_ARG,
              "pna_peer_barrier: bad arguments (world %d, rank %d)", world, rank);
  k_peer_barrier<<<1, 64, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const unsigned long long*>(peer_flags), rank,
                                                                   world, epoch, timeout_ns ? timeout_ns : 2000000000ull, status);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}
