// The device's powf / expf over arrays: the one pair of roundings the add-on aggregators' fp32 restatement
// (tests/addon_paths_ref.py) cannot state, so it takes them from the device.  Built with the library's own nvcc flags
// (pna_b200._lib.NVCC_FLAGS) and none of its headers, so that a change in the library cannot leak into this oracle.
// Every argument arrives at run time, as it does in the kernels: no exponent can be specialised at compile time.
#include <cuda_runtime.h>

__global__ void k_devmath_powf(const float* x, const float* y, float* out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = powf(x[i], y[i]);
}

__global__ void k_devmath_expf(const float* x, float* out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = expf(x[i]);
}

static unsigned blocks_for(long long n) { return (unsigned)(n < 256 * 1024 ? (n + 255) / 256 : 1024); }

// out[i] = powf(x[i], y[i]) for i < n (device pointers); returns the cudaError_t of the launch
extern "C" int devmath_powf(const float* x, const float* y, float* out, long long n, void* stream) {
  if (n <= 0) return 0;
  k_devmath_powf<<<blocks_for(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, out, n);
  return (int)cudaGetLastError();
}

// out[i] = expf(x[i]) for i < n (device pointers); returns the cudaError_t of the launch
extern "C" int devmath_expf(const float* x, float* out, long long n, void* stream) {
  if (n <= 0) return 0;
  k_devmath_expf<<<blocks_for(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, out, n);
  return (int)cudaGetLastError();
}
