// Shared device/host helpers for the styletts2_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/styletts2_b200.h"

namespace st2 {

// Error plumbing: every extern "C" entry point returns 0 or a cudaError_t value and
// records a message retrievable with st2_last_error().
void set_error(const char* where, cudaError_t e);
void set_error_msg(const char* where, const char* msg);

// Range flag of the tensor-core convs (conv_tc.cu): reads and clears it; st2_range_flag_fetch reports it with the GEMMs' flag.
cudaError_t conv_tc_range_flag_fetch(int* flag);
// The same for the tensor-core attention (attention_tc.cu).
cudaError_t attention_tc_range_flag_fetch(int* flag);

#define ST2_CHECK_LAUNCH(where)                         \
  do {                                                  \
    cudaError_t _e = cudaGetLastError();                \
    if (_e != cudaSuccess) {                            \
      st2::set_error(where, _e);                        \
      return (int)_e;                                   \
    }                                                   \
  } while (0)

#define ST2_REQUIRE(cond, where, msg)                   \
  do {                                                  \
    if (!(cond)) {                                      \
      st2::set_error_msg(where, msg);                   \
      return (int)cudaErrorInvalidValue;                \
    }                                                   \
  } while (0)

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
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Activations used on the path.  ACT_* codes are part of the C ABI (include/styletts2_b200.h).
__device__ __forceinline__ float act_apply(float v, int act, float slope, float alpha) {
  if (act == ST2_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == ST2_ACT_SNAKE) {
    // x + (1/alpha) * sin(alpha x)^2  (Modules/istftnet.py:69)
    float sn = sinf(alpha * v);
    return v + (1.0f / alpha) * (sn * sn);
  }
  return v;
}

__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}

__device__ __forceinline__ float gelu_tanh(float x) {
  // 0.5*x*(1+tanh(sqrt(2/pi)*(x+0.044715*x^3)))  (transformers NewGELUActivation)
  return 0.5f * x * (1.0f + tanhf(0.79788456080286535588f * (x + 0.044715f * x * x * x)));
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// One-time host-side setup (cudaFuncSetAttribute, __constant__ tables, device queries) is PER DEVICE: a process that
// drives several GPUs must repeat it on each.  Usage: static PerDevice once; if (once.first()) { ...setup for current device... }
struct PerDevice {
  bool done[64] = {false};
  int value[64] = {0};
  int dev() const {
    int d = 0;
    cudaGetDevice(&d);
    return d & 63;
  }
  bool first() {
    const int d = dev();
    if (done[d]) return false;
    done[d] = true;
    return true;
  }
};

}  // namespace st2
