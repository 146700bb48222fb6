// K-OPT: ONE launch over the flat fp32 master buffer (Adam, TF-1.0 "epsilon-hat" formulation, or SGD) that
// also refreshes the bf16 shadow the tensor-core kernels read.  Replaces the reference's one ApplyAdam
// kernel per variable (14*L+2 launches per step; original src/rnn.py:207,224).
// Memory-bound: 16 B vector loads/stores, grid = 132 SMs (H100) x 8 resident CTAs, grid-stride.
#include "ts_common.cuh"

namespace {

TS_DEVICE uint2 pack_bf16x4(float4 v) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y);
  __nv_bfloat162 hi = __floats2bfloat162_rn(v.z, v.w);
  uint2 r;
  r.x = *reinterpret_cast<uint32_t*>(&lo);
  r.y = *reinterpret_cast<uint32_t*>(&hi);
  return r;
}

// step_dev != null: lr_t is derived in-kernel from the device-resident step counter (bumped by inc_step_kernel right
// before), so a CUDA-graph replay of the training step applies the correct Adam bias correction every time.
__global__ void inc_step_kernel(int* step) { *step += 1; }

__global__ void __launch_bounds__(256) flat_adam_kernel(float4* __restrict__ p, const float4* __restrict__ g,
                                                        float4* __restrict__ m, float4* __restrict__ v,
                                                        uint2* __restrict__ shadow, size_t n4, float lr_t, float b1,
                                                        float b2, float eps, float wd, float gscale,
                                                        const int* __restrict__ step_dev, size_t wd_n4) {
  if (step_dev != nullptr) {
    const float t = (float)(*step_dev);
    lr_t = lr_t * sqrtf(1.f - powf(b2, t)) / (1.f - powf(b1, t));      // lr_t arrives as the base learning rate
  }
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 pv = p[i], gv = g[i], mv = m[i], vv = v[i];
    float* pp = &pv.x; float* gp = &gv.x; float* mp = &mv.x; float* vp = &vv.x;
    const float wdi = i < wd_n4 ? wd : 0.f;        // the L2 term of create_variable covers the LSTM variables only (K12)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float gg = gp[k] * gscale + wdi * pp[k];
      mp[k] = b1 * mp[k] + (1.f - b1) * gg;
      vp[k] = b2 * vp[k] + (1.f - b2) * gg * gg;
      pp[k] -= lr_t * mp[k] / (sqrtf(vp[k]) + eps);
    }
    p[i] = pv; m[i] = mv; v[i] = vv;
    if (shadow) shadow[i] = pack_bf16x4(pv);
  }
}

__global__ void __launch_bounds__(256) flat_sgd_kernel(float4* __restrict__ p, const float4* __restrict__ g,
                                                       uint2* __restrict__ shadow, size_t n4, float lr, float wd,
                                                       float gscale, size_t wd_n4) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 pv = p[i], gv = g[i];
    const float wdi = i < wd_n4 ? wd : 0.f;
    pv.x -= lr * (gv.x * gscale + wdi * pv.x);
    pv.y -= lr * (gv.y * gscale + wdi * pv.y);
    pv.z -= lr * (gv.z * gscale + wdi * pv.z);
    pv.w -= lr * (gv.w * gscale + wdi * pv.w);
    p[i] = pv;
    if (shadow) shadow[i] = pack_bf16x4(pv);
  }
}

__global__ void __launch_bounds__(256) cast_bf16_kernel(const float4* __restrict__ p, uint2* __restrict__ shadow,
                                                        size_t n4) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) shadow[i] = pack_bf16x4(p[i]);
}

int grid_for(size_t n4) {
  size_t want = (n4 + 255) / 256;
  size_t cap = 132 * 8;
  return (int)(want < cap ? (want ? want : 1) : cap);
}

}  // namespace

extern "C" int ts_flat_adam(float* p, const float* g, float* m, float* v, void* shadow, long long n, float lr_t,
                            float b1, float b2, float eps, float wd, float gscale, cudaStream_t st, int* step_dev, long long wd_n) {
  if (n % 4) return -2;
  size_t n4 = (size_t)n / 4;
  if (step_dev) inc_step_kernel<<<1, 1, 0, st>>>(step_dev);
  flat_adam_kernel<<<grid_for(n4), 256, 0, st>>>((float4*)p, (const float4*)g, (float4*)m, (float4*)v, (uint2*)shadow,
                                                 n4, lr_t, b1, b2, eps, wd, gscale, step_dev, wd_n < 0 ? n4 : (size_t)wd_n / 4);
  return (int)cudaGetLastError();
}

extern "C" int ts_flat_sgd(float* p, const float* g, void* shadow, long long n, float lr, float wd, float gscale,
                           cudaStream_t st, long long wd_n) {
  if (n % 4) return -2;
  size_t n4 = (size_t)n / 4;
  flat_sgd_kernel<<<grid_for(n4), 256, 0, st>>>((float4*)p, (const float4*)g, (uint2*)shadow, n4, lr, wd, gscale, wd_n < 0 ? n4 : (size_t)wd_n / 4);
  return (int)cudaGetLastError();
}

extern "C" int ts_cast_bf16(const float* p, void* shadow, long long n, cudaStream_t st) {
  if (n % 4) return -2;
  size_t n4 = (size_t)n / 4;
  cast_bf16_kernel<<<grid_for(n4), 256, 0, st>>>((const float4*)p, (uint2*)shadow, n4);
  return (int)cudaGetLastError();
}
