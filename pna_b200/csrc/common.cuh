// Shared helpers for libpna_sm90.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/pna_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libpna_sm90 is written for sm_90a (H100) only"
#endif

namespace pna {

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define PNA_CUDA_TRY(expr)                                   \
  do {                                                       \
    cudaError_t _e = (expr);                                 \
    if (_e != cudaSuccess) return ::pna::cuda_fail(_e, #expr); \
  } while (0)

#define PNA_REQUIRE(cond, code, ...)      \
  do {                                    \
    if (!(cond)) {                        \
      ::pna::set_error(__VA_ARGS__);      \
      return (code);                      \
    }                                     \
  } while (0)

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---- order of the rows of a "view" ------------------------------------------------------------------------------
// A view lists the N real rows and, interleaved evenly among them, the M chunk pseudo-rows of the split rows (one
// chunk row after every N/M real rows), so that every warp's contiguous range of view rows mixes epilogue-heavy real
// rows with gather-heavy chunk rows.  view_to_row returns the real row index, or N + c for chunk c.
struct ViewMap {
  long long N;
  int M;
  __host__ __device__ long long rows() const { return N + M; }
  __host__ __device__ long long to_row(long long v) const {
    if (M <= 0) return v;
    const long long s = N / M, g = s + 1;
    if (v < g * M) {
      const long long b = v / g, o = v - b * g;
      return o < s ? b * s + o : N + b;
    }
    return s * M + (v - g * M);
  }
};

// ---- degree scalers (reference models/pytorch_geometric/scalers.py:8-29) --------------------------------------------
// The ONE place the per-row scale factors are computed: the aggregation epilogue and pna_row_scales (the compact
// post-linear path) must produce bit-identical factors.
struct DegScales {
  float amp, att, lin, ilin;
  __device__ __forceinline__ float of(unsigned code) const {
    switch (code) {
      case PNA_SCALE_IDENTITY: return 1.0f;
      case PNA_SCALE_AMPLIFICATION: return amp;
      case PNA_SCALE_ATTENUATION: return att;
      case PNA_SCALE_LINEAR: return lin;
      default: return ilin;
    }
  }
};
__device__ __forceinline__ DegScales deg_scales_of(bool iso, float degf, float avg_log, float avg_lin) {
  const float lg = logf(degf + 1.0f);
  DegScales s;
  s.amp = __fdiv_rn(lg, avg_log);                      // scalers.py:12-13  (0 for an isolated row)
  s.att = iso ? 1.0f : __fdiv_rn(avg_log, lg);         // scalers.py:16-19  (scale := 1 where deg == 0)
  s.lin = __fdiv_rn(degf, avg_lin);                    // scalers.py:22-23
  s.ilin = iso ? 1.0f : __fdiv_rn(avg_lin, degf);      // scalers.py:26-29
  return s;
}
__device__ __forceinline__ DegScales deg_scales(int deg, float avg_log, float avg_lin) {
  return deg_scales_of(deg == 0, (float)deg, avg_log, avg_lin);
}
// a real-valued degree (scaler_degree_f of pna_aggregate_fwd_weighted: D = adj.sum(-1) of a weighted dense adjacency)
__device__ __forceinline__ DegScales deg_scales_f(float deg, float avg_log, float avg_lin) {
  return deg_scales_of(deg == 0.0f, deg, avg_log, avg_lin);
}

// ---- element load/store with fp32 math -------------------------------------------------------------------
// Gathered rows go through the read-only path (ld.global.nc); the [N, S*A*F] result is written once and never
// re-read by this library, so it is stored with the streaming (evict-first) policy to keep source rows in L2.
template <typename V>
__device__ __forceinline__ void store_out(V* p, V v) { __stcs(p, v); }

template <typename T, int VEC>
struct Io;

template <>
struct Io<float, 4> {
  typedef float4 Raw;
  static __device__ __forceinline__ Raw load_raw(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
  static __device__ __forceinline__ void unpack(const Raw& r, float (&v)[4]) { v[0] = r.x; v[1] = r.y; v[2] = r.z; v[3] = r.w; }
  static __device__ __forceinline__ void load(const float* p, float (&v)[4]) { unpack(load_raw(p), v); }
  static __device__ __forceinline__ void store(float* p, const float (&v)[4]) {
    store_out(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
  }
};

template <>
struct Io<float, 1> {
  typedef float Raw;
  static __device__ __forceinline__ Raw load_raw(const float* p) { return __ldg(p); }
  static __device__ __forceinline__ void unpack(const Raw& r, float (&v)[1]) { v[0] = r; }
  static __device__ __forceinline__ void load(const float* p, float (&v)[1]) { v[0] = __ldg(p); }
  static __device__ __forceinline__ void store(float* p, const float (&v)[1]) { __stcs(p, v[0]); }
};

template <>
struct Io<__nv_bfloat16, 8> {
  typedef uint4 Raw;
  static __device__ __forceinline__ Raw load_raw(const __nv_bfloat16* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float (&v)[8]) { unpack(load_raw(p), v); }
  static __device__ __forceinline__ void unpack(const Raw& r, float (&v)[8]) {
    v[0] = __uint_as_float(r.x << 16); v[1] = __uint_as_float(r.x & 0xffff0000u);
    v[2] = __uint_as_float(r.y << 16); v[3] = __uint_as_float(r.y & 0xffff0000u);
    v[4] = __uint_as_float(r.z << 16); v[5] = __uint_as_float(r.z & 0xffff0000u);
    v[6] = __uint_as_float(r.w << 16); v[7] = __uint_as_float(r.w & 0xffff0000u);
  }
  static __device__ __forceinline__ unsigned pack(float lo, float hi) {
    const __nv_bfloat162 b = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const unsigned*>(&b);
  }
  static __device__ __forceinline__ void store(__nv_bfloat16* p, const float (&v)[8]) {
    uint4 r;
    r.x = pack(v[0], v[1]); r.y = pack(v[2], v[3]); r.z = pack(v[4], v[5]); r.w = pack(v[6], v[7]);
    store_out(reinterpret_cast<uint4*>(p), r);
  }
};

template <>
struct Io<__nv_bfloat16, 1> {
  typedef unsigned short Raw;
  static __device__ __forceinline__ Raw load_raw(const __nv_bfloat16* p) { return __ldg(reinterpret_cast<const unsigned short*>(p)); }
  static __device__ __forceinline__ void unpack(const Raw& r, float (&v)[1]) { v[0] = __uint_as_float(static_cast<unsigned>(r) << 16); }
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float (&v)[1]) { unpack(load_raw(p), v); }
  static __device__ __forceinline__ void store(__nv_bfloat16* p, const float (&v)[1]) {
    const __nv_bfloat16 b = __float2bfloat16_rn(v[0]);
    __stcs(reinterpret_cast<unsigned short*>(p), *reinterpret_cast<const unsigned short*>(&b));
  }
};

}  // namespace pna
