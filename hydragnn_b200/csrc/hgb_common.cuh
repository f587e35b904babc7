// Shared helpers for libhgb.so (sm_90a).  See include/hgb.h for the C-ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/hgb.h"

void hgb_set_error(const char* fmt, ...);
void hgb_count_launch(int n = 1);

#define HGB_REQUIRE(cond, ...)            \
  do {                                    \
    if (!(cond)) {                        \
      hgb_set_error(__VA_ARGS__);         \
      return HGB_EINVAL;                  \
    }                                     \
  } while (0)

// checks the launch (not the execution: nothing here synchronises)
#define HGB_LAUNCH_CHECK(name)                                                   \
  do {                                                                           \
    cudaError_t e__ = cudaPeekAtLastError();                                     \
    if (e__ != cudaSuccess) {                                                    \
      hgb_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));     \
      return HGB_ECUDA;                                                          \
    }                                                                            \
    hgb_count_launch();                                                          \
  } while (0)

#define HGB_NUM_SMS 132   // H100 SXM

static inline int hgb_grid_for(int64_t work_items, int per_block, int max_blocks = HGB_NUM_SMS * 16) {
  int64_t b = (work_items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}

__device__ __forceinline__ float hgb_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- activations -----------------------------------------------------------------------------
__device__ __forceinline__ float hgb_sigmoid(float x) { return 1.f / (1.f + __expf(-x)); }

__device__ __forceinline__ float hgb_act(float x, int act, float p) {
  switch (act) {
    case HGB_ACT_RELU: return x > 0.f ? x : 0.f;
    case HGB_ACT_SILU: return x * hgb_sigmoid(x);
    case HGB_ACT_TANH: return tanhf(x);
    case HGB_ACT_SIGMOID: return hgb_sigmoid(x);
    case HGB_ACT_LRELU: return x > 0.f ? x : p * x;
    case HGB_ACT_ELU: return x > 0.f ? x : expm1f(x);
    case HGB_ACT_SELU: {
      const float a = 1.6732632423543772848170429916717f, s = 1.0507009873554804934193349852946f;
      return s * (x > 0.f ? x : a * expm1f(x));
    }
    default: return x;
  }
}

// derivative of act at pre-activation z, given y = act(z) (z is only read for SiLU)
__device__ __forceinline__ float hgb_act_grad(float y, float z, int act, float p) {
  switch (act) {
    case HGB_ACT_RELU: return y > 0.f ? 1.f : 0.f;
    case HGB_ACT_DERIV: return z;   // the tensor already holds the derivative
    case HGB_ACT_SILU: { float s = hgb_sigmoid(z); return s * (1.f + z * (1.f - s)); }
    case HGB_ACT_TANH: return 1.f - y * y;
    case HGB_ACT_SIGMOID: return y * (1.f - y);
    case HGB_ACT_LRELU: return y > 0.f ? 1.f : p;
    case HGB_ACT_ELU: return y > 0.f ? 1.f : y + 1.f;
    case HGB_ACT_SELU: {
      const float a = 1.6732632423543772848170429916717f, s = 1.0507009873554804934193349852946f;
      return y > 0.f ? s : y + s * a;
    }
    default: return 1.f;
  }
}
