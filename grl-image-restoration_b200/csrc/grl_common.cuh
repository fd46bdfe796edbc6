// grl_common.cuh -- error plumbing and small device helpers shared by all translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/grl_b200.h"
#include "grl_geometry.h"

namespace grl {

char* error_buffer();  // thread-local, defined in capi.cu
unsigned long long& launch_counter();  // kernels launched by this library since load (defined in capi.cu)

inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(error_buffer(), 512, fmt, ap);
  va_end(ap);
  return code;
}

#define GRL_REQUIRE(cond, ...)                                   \
  do {                                                           \
    if (!(cond)) return ::grl::fail(GRL_ERR_INVALID, __VA_ARGS__); \
  } while (0)

#define GRL_CUDA(expr)                                                                                  \
  do {                                                                                                  \
    cudaError_t e__ = (expr);                                                                           \
    if (e__ != cudaSuccess)                                                                             \
      return ::grl::fail(GRL_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, \
                         __LINE__);                                                                     \
  } while (0)

#define GRL_LAUNCH_CHECK(name)                                                                        \
  do {                                                                                                \
    ++::grl::launch_counter();                                                                        \
    cudaError_t e__ = cudaGetLastError();                                                             \
    if (e__ != cudaSuccess)                                                                           \
      return ::grl::fail(GRL_ERR_CUDA, "launch of %s failed: %s", name, cudaGetErrorString(e__));      \
  } while (0)

// channel_gate_kernel (ops_f32.cu) on per-chunk channel sums (B, chunks, C): the second half of grl_channel_gate_f32,
// shared with grl_tc_channel_gate (misc_tc.cu), which computes the sums from 16-bit features.
int channel_gate_from_partial(const float* partial, int chunks, int B, long long L, int C, const float* w1, const float* b1,
                              const float* w2, const float* b2, int R, float* gate, cudaStream_t st);

constexpr int kMaxDevices = 64;  // per-device one-time kernel attributes (cudaFuncSetAttribute is per device)

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  if (act == GRL_ACT_GELU) return gelu_erf(v);
  if (act == GRL_ACT_LEAKY) return v > 0.f ? v : v * slope;
  return v;
}

}  // namespace grl
