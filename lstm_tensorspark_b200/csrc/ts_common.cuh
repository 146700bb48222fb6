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
// Accurate variants for the fp32 path: computed in fp64 and rounded once.  build.py compiles with --use_fast_math, which turns
// the fp32 tanhf / expf / division into tanh.approx / ex2.approx / rcp.approx (relative error up to about 2^-11, no better than
// bf16); it leaves fp64 math alone.
TS_DEVICE float tanhf_acc(float x) { return (float)tanh((double)x); }
TS_DEVICE float sigmoidf_acc(float x) { return (float)(1.0 / (1.0 + exp(-(double)x))); }

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

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11; the Random123 constants).
TS_DEVICE uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) { k.x += 0x9E3779B9u; k.y += 0xBB67AE85u; }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

// Dropout between stacked layers: the mask of one output sequence (one layer, one direction) of one training step.  The
// definition is shared with ops/reference.py dropout_mask; change both or neither.
//   key (key0, key1) = (seed, partition); counter = (b * ceil(H/8) + j/8, t, c2 = 2 * layer + reverse, step).
//   The 4 words give eight 16-bit values: unit 8g + i uses word i/2, low half for even i.  Kept iff value >= thr.
//   A kept value is multiplied by scale = 65536 / (65536 - thr) in fp32 (exact expectation for the quantised P).
// c2 also tells the other mask sites apart (bits above the layer index): weight drop, the embedding's input and row masks.
// kDropLocked in c2 makes the mask locked (AWD-LSTM's LockedDropout): the time word is 0, so every step shares one mask.
constexpr uint32_t kDropLocked = 0x20000000u;
constexpr uint32_t kDropInput = 0x40000000u;     // the embedding output x_t (counter over its E units)
constexpr uint32_t kDropRows = 0x10000000u;      // whole rows of the embedding table (one time step, one row of V units)
struct DropSpec {
  const int* step;        // device-resident step counter (c3): a captured CUDA graph reads the current value
  uint32_t key0, key1;
  uint32_t thr;           // min(round(P * 65536), 65535)
  uint32_t c2;
  int row0;               // batch row of local row 0 (batch chunks pass their offset)
  float scale;
};

// Host side: the descriptor of a launch from the step counter (null = no dropout) and host {key0, key1, thr, c2, row0}.
inline DropSpec make_drop_spec(const int* step, const unsigned int* desc) {
  DropSpec d{};
  if (step == nullptr) return d;
  d.step = step;
  d.key0 = desc[0]; d.key1 = desc[1]; d.thr = desc[2]; d.c2 = desc[3]; d.row0 = (int)desc[4];
  d.scale = 65536.0f / (float)(65536u - d.thr);
  return d;
}

// Keep bits of the 8 hidden units [j, j + 8) (j % 8 == 0) of local batch row b at time t: bit i = unit j + i.
TS_DEVICE uint32_t dropout_keep8(const DropSpec& d, uint32_t step, int b, int j, int t, int H) {
  const uint32_t c0 = (uint32_t)(b + d.row0) * (uint32_t)((H + 7) / 8) + (uint32_t)(j >> 3);
  const uint32_t tw = (d.c2 & kDropLocked) ? 0u : (uint32_t)t;
  const uint4 r = philox4x32_10(make_uint4(c0, tw, d.c2, step), make_uint2(d.key0, d.key1));
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
  uint32_t keep = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (((w[i >> 1] >> (16 * (i & 1))) & 0xffffu) >= d.thr) keep |= 1u << i;
  return keep;
}

// 8 bf16 values (a 16 B chunk, unit i in bits [16 (i & 1), +16) of word i / 2) -> bf16_rn(float(h) * scale) where kept, +0
// where dropped.
TS_DEVICE uint4 dropout_bf16x8(uint4 h, uint32_t keep, float scale) {
  uint32_t w[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float lo = __fmul_rn(__uint_as_float(w[i] << 16), scale), hi = __fmul_rn(__uint_as_float(w[i] & 0xffff0000u), scale);
    const uint32_t blo = ((keep >> (2 * i)) & 1u) ? (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(lo)) : 0u;
    const uint32_t bhi = ((keep >> (2 * i + 1)) & 1u) ? (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(hi)) : 0u;
    w[i] = blo | (bhi << 16);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// Zero the dropped units of 8 bf16 values (the backward pass scales the kept ones in fp32 later)
TS_DEVICE uint4 dropout_zero_bf16x8(uint4 h, uint32_t keep) {
  uint32_t w[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
  for (int i = 0; i < 4; ++i)
    w[i] &= (((keep >> (2 * i)) & 1u) ? 0x0000ffffu : 0u) | (((keep >> (2 * i + 1)) & 1u) ? 0xffff0000u : 0u);
  return make_uint4(w[0], w[1], w[2], w[3]);
}

}  // namespace ts
