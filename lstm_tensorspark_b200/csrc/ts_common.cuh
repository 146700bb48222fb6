// Shared helpers for the sm_90a kernels of lstm_tensorspark_b200.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#define TS_DEVICE __device__ __forceinline__

namespace ts {

TS_DEVICE float tanhf_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// sigmoid(x) = 0.5*tanh(0.5x)+0.5 : ONE MUFU op (tanh.approx) instead of ex2 + rcp
TS_DEVICE float sigmoidf_fast(float x) { return fmaf(0.5f, tanhf_fast(0.5f * x), 0.5f); }
// accurate variants for the fp32 parity path
TS_DEVICE float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

template <typename T> struct Cvt;
template <> struct Cvt<float> {
  TS_DEVICE static float to_f(float v) { return v; }
  TS_DEVICE static float from_f(float v) { return v; }
};
template <> struct Cvt<__nv_bfloat16> {
  TS_DEVICE static float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  TS_DEVICE static __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};

TS_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
TS_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace ts
