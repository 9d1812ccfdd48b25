// Error reporting, queries and the halo row-gather (send-buffer pack) kernel.
#include "common.cuh"

namespace pna {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
  (void)cudaGetLastError();  // clear the sticky-free error so the next call starts clean
  return PNA_ERR_CUDA;
}

// dst[i, :] = src[idx[i], :]; one lane group per row, 16-byte chunks when aligned.
template <int BYTES>
__global__ void __launch_bounds__(256) k_gather_rows(const char* __restrict__ src, long long src_pitch, const int* __restrict__ idx,
                                                     long long n, char* __restrict__ dst, long long dst_pitch, int row_bytes) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const long long s = __ldg(idx + row);
  const char* sp = src + s * src_pitch;
  char* dp = dst + row * dst_pitch;
  for (int b = lane * BYTES; b < row_bytes; b += 32 * BYTES) {
    if constexpr (BYTES == 16) {
      *reinterpret_cast<uint4*>(dp + b) = __ldg(reinterpret_cast<const uint4*>(sp + b));
    } else if constexpr (BYTES == 4) {
      *reinterpret_cast<unsigned*>(dp + b) = __ldg(reinterpret_cast<const unsigned*>(sp + b));
    } else {
      *reinterpret_cast<unsigned short*>(dp + b) = __ldg(reinterpret_cast<const unsigned short*>(sp + b));
    }
  }
}

}  // namespace pna

using namespace pna;

extern "C" const char* pna_last_error(void) { return g_err; }

extern "C" int pna_query(int what) {
  switch (what) {
    case PNA_QUERY_ABI_VERSION: return PNA_ABI_VERSION;
    case PNA_QUERY_SM_ARCH: return 90;
    case PNA_QUERY_DEFAULT_SPLIT: return 256;
    case PNA_QUERY_DEFAULT_CHUNK: return 128;
    case PNA_QUERY_MAX_FEATURES: return 16384;
    case PNA_QUERY_SIZEOF_CSR: return (int)sizeof(pna_csr_t);
    case PNA_QUERY_SIZEOF_AGG: return (int)sizeof(pna_agg_t);
    case PNA_QUERY_DEVICE_SM_COUNT: {
      int dev = 0, sms = 0;
      if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
        (void)cudaGetLastError();
        set_error("pna_query: no CUDA device");
        return PNA_ERR_CUDA;
      }
      return sms;
    }
    default:
      set_error("pna_query: unknown selector %d", what);
      return PNA_ERR_BAD_ARG;
  }
}

extern "C" int pna_gather_rows(const void* src, int64_t ld_src, const int32_t* idx, int64_t n_idx, void* dst, int64_t ld_dst,
                               int32_t n_feat, int32_t dtype, pna_stream_t stream) {
  PNA_REQUIRE(n_idx >= 0 && n_feat > 0, PNA_ERR_BAD_ARG, "pna_gather_rows: bad sizes");
  PNA_REQUIRE(dtype == PNA_F32 || dtype == PNA_BF16, PNA_ERR_UNSUPPORTED, "pna_gather_rows: dtype %d", dtype);
  if (n_idx == 0) return PNA_OK;
  PNA_REQUIRE(src && idx && dst, PNA_ERR_BAD_ARG, "pna_gather_rows: null pointer");
  const int esz = dtype == PNA_F32 ? 4 : 2;
  const long long sp = ld_src * esz, dp = ld_dst * esz;
  const int rb = n_feat * esz;
  const bool a16 = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst) | (uintptr_t)sp | (uintptr_t)dp | (uintptr_t)rb) & 15u) == 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned grid = (unsigned)((n_idx + 7) / 8);
  if (a16)
    k_gather_rows<16><<<grid, 256, 0, st>>>((const char*)src, sp, idx, n_idx, (char*)dst, dp, rb);
  else if (esz == 4)
    k_gather_rows<4><<<grid, 256, 0, st>>>((const char*)src, sp, idx, n_idx, (char*)dst, dp, rb);
  else
    k_gather_rows<2><<<grid, 256, 0, st>>>((const char*)src, sp, idx, n_idx, (char*)dst, dp, rb);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}
