// K-OPT: ONE launch over the flat fp32 master buffer (Adam, TF-1.0 "epsilon-hat" formulation, SGD, or SGD with the ASGD
// average of the iterates) that also refreshes the bf16 shadow the tensor-core kernels read.  Replaces the reference's one ApplyAdam
// kernel per variable (14*L+2 launches per step; original src/rnn.py:207,224).
// Memory-bound: 16 B vector loads/stores, grid = 132 SMs (H100) x 8 resident CTAs, grid-stride.
#include "launchers.h"
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

// CLIP: the update kernels use coef * g_total, coef = clip[1] as flat_grad_norm_kernel wrote it.  The multiply is __fmul_rn, so
// it is never contracted into the m / v / p expressions: coef == 1 gives the bits of the kernel without CLIP, and that kernel
// (clip unused) compiles to the same instructions as it did before clipping existed.
template <bool CLIP>
TS_DEVICE float clipped(float gg, float coef) {
  if constexpr (CLIP) return __fmul_rn(coef, gg);
  else return gg;
}

template <bool CLIP>
__global__ void __launch_bounds__(256) flat_adam_kernel(float4* __restrict__ p, const float4* __restrict__ g,
                                                        float4* __restrict__ m, float4* __restrict__ v,
                                                        uint2* __restrict__ shadow, size_t n4, float lr_t, float b1,
                                                        float b2, float eps, float wd, float gscale,
                                                        const int* __restrict__ step_dev, size_t wd_n4,
                                                        const float* __restrict__ clip) {
  float coef = 1.f;
  if constexpr (CLIP) coef = clip[1];
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
      if constexpr (CLIP) {
        // the roundings the compiler picked for the expressions below (CLIP = false), spelled out, so that coef == 1 gives
        // the same bits: gg = fma(g, s, wd p), m = fma(m, b1, (1 - b1) gg), v = fma(v, b2, gg ((1 - b2) gg))
        const float gg = __fmul_rn(coef, __fmaf_rn(gp[k], gscale, __fmul_rn(wdi, pp[k])));
        mp[k] = __fmaf_rn(mp[k], b1, __fmul_rn(1.f - b1, gg));
        vp[k] = __fmaf_rn(vp[k], b2, __fmul_rn(gg, __fmul_rn(1.f - b2, gg)));
      } else {
        const float gg = gp[k] * gscale + wdi * pp[k];
        mp[k] = b1 * mp[k] + (1.f - b1) * gg;
        vp[k] = b2 * vp[k] + (1.f - b2) * gg * gg;
      }
      pp[k] -= lr_t * mp[k] / (sqrtf(vp[k]) + eps);
    }
    p[i] = pv; m[i] = mv; v[i] = vv;
    if (shadow) shadow[i] = pack_bf16x4(pv);
  }
}

// p -= lr * coef * (g * gscale + wd * p): the one SGD expression of flat_sgd_kernel and flat_asgd_kernel (inlined into both, so
// the compiler contracts it the same way in each)
template <bool CLIP>
TS_DEVICE float4 sgd_update(float4 pv, float4 gv, float lr, float wdi, float gscale, float coef) {
  pv.x -= lr * clipped<CLIP>(gv.x * gscale + wdi * pv.x, coef);
  pv.y -= lr * clipped<CLIP>(gv.y * gscale + wdi * pv.y, coef);
  pv.z -= lr * clipped<CLIP>(gv.z * gscale + wdi * pv.z, coef);
  pv.w -= lr * clipped<CLIP>(gv.w * gscale + wdi * pv.w, coef);
  return pv;
}

template <bool CLIP>
__global__ void __launch_bounds__(256) flat_sgd_kernel(float4* __restrict__ p, const float4* __restrict__ g,
                                                       uint2* __restrict__ shadow, size_t n4, float lr, float wd,
                                                       float gscale, size_t wd_n4, const float* __restrict__ clip) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  float coef = 1.f;
  if constexpr (CLIP) coef = clip[1];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 pv = sgd_update<CLIP>(p[i], g[i], lr, i < wd_n4 ? wd : 0.f, gscale, coef);
    p[i] = pv;
    if (shadow) shadow[i] = pack_bf16x4(pv);
  }
}

// ---- ASGD (torch.optim.ASGD with lambd = 0, t0 = 0): ax, the running average of the iterates -----------------------------
// avg = device int32 {on, k}.  bump_avg_kernel runs right before every averaging kernel (k counts the averaged updates, so a
// captured graph stays exact across replays; switching on is a fill_ of {1, 0} outside the graph).  The k-th averaged update
// uses torch's indexing mu_k = 1 / max(1, k - 1): k <= 2 copies ax = p, then ax = ax + (p - ax) * mu_k with each operation
// rounded on its own (torch's order, no FMA), mu_k = fp32(1.0 / (k - 1)) as torch rounds the Python double.
__global__ void bump_avg_kernel(int* avg) {
  if (avg[0]) avg[1] += 1;
}

TS_DEVICE float average_mu(int k) { return k <= 2 ? 1.f : (float)(1.0 / (double)(k - 1)); }

TS_DEVICE float4 average_step(float4 a, float4 pv, int k, float mu) {
  if (k <= 2) return pv;
  a.x = __fadd_rn(a.x, __fmul_rn(__fsub_rn(pv.x, a.x), mu));
  a.y = __fadd_rn(a.y, __fmul_rn(__fsub_rn(pv.y, a.y), mu));
  a.z = __fadd_rn(a.z, __fmul_rn(__fsub_rn(pv.z, a.z), mu));
  a.w = __fadd_rn(a.w, __fmul_rn(__fsub_rn(pv.w, a.w), mu));
  return a;
}

// flat_sgd_kernel's p and shadow (bit for bit: the same sgd_update), plus the average when on; with on == 0 ax is neither
// read nor written.  22 B per element against SGD's 14 B.
template <bool CLIP>
__global__ void __launch_bounds__(256) flat_asgd_kernel(float4* __restrict__ p, const float4* __restrict__ g,
                                                        float4* __restrict__ ax, const int* __restrict__ avg,
                                                        uint2* __restrict__ shadow, size_t n4, float lr, float wd,
                                                        float gscale, size_t wd_n4, const float* __restrict__ clip) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  float coef = 1.f;
  if constexpr (CLIP) coef = clip[1];
  const bool on = avg[0] != 0;
  const int k = avg[1];
  const float mu = average_mu(k);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 pv = sgd_update<CLIP>(p[i], g[i], lr, i < wd_n4 ? wd : 0.f, gscale, coef);
    p[i] = pv;
    if (shadow) shadow[i] = pack_bf16x4(pv);
    if (on) ax[i] = average_step(k <= 2 ? pv : ax[i], pv, k, mu);
  }
}

// The averaging half alone, for updates that ran elsewhere (the fused allreduce's bucket kernels): 12 B per element.
__global__ void __launch_bounds__(256) flat_average_kernel(const float4* __restrict__ p, float4* __restrict__ ax,
                                                           const int* __restrict__ avg, size_t n4) {
  if (!avg[0]) return;
  const int k = avg[1];
  const float mu = average_mu(k);
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 pv = p[i];
    ax[i] = average_step(k <= 2 ? pv : ax[i], pv, k, mu);
  }
}

// p <-> ax in place, shadow = bf16(new p): evaluating the average is swap, score, swap (two swaps restore all three bit for bit).
__global__ void __launch_bounds__(256) flat_swap_kernel(float4* __restrict__ p, float4* __restrict__ ax, uint2* __restrict__ shadow,
                                                        size_t n4) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 a = ax[i], pv = p[i];
    p[i] = a;
    ax[i] = pv;
    if (shadow) shadow[i] = pack_bf16x4(a);
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

// fp64 sum over the CTA in a fixed tree: shuffles within each warp, then warp 0 over the 8 warp sums.  -> thread 0.
TS_DEVICE double block_sum_256(double s, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < 8 ? red[threadIdx.x] : 0.0;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  }
  return s;
}

// Gradient clipping by the global norm: out = {norm, coef} of g_total = g * gscale + wd * p (the decay on float4s [0, wd_n4)
// only, p not read at all when wd == 0), norm = ||g_total||_2, coef = min(max_norm / (norm + 1e-6), 1) as clip_grad_norm_
// computes it in fp32 (a NaN norm gives a NaN coef, an infinite one 0).  Deterministic and SM-count independent: the grid
// depends on n alone (grid_for), each thread sums the squares of a fixed set of elements in fp64, the CTA sums in a fixed
// tree, and the last CTA to take a ticket sums the fp64 CTA partials in a fixed order and leaves the ticket 0 again (so a
// replayed graph starts from 0 too).  No host synchronisation.
__global__ void __launch_bounds__(256) flat_grad_norm_kernel(const float4* __restrict__ g, const float4* __restrict__ p,
                                                             size_t n4, float wd, float gscale, size_t wd_n4, float max_norm,
                                                             double* __restrict__ partial, unsigned int* __restrict__ ticket,
                                                             float* __restrict__ out) {
  __shared__ double red[8];
  __shared__ bool last_s;
  const size_t wd_end = wd != 0.f ? wd_n4 : 0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  double s = 0.0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 gv = g[i];
    float t[4] = {gv.x * gscale, gv.y * gscale, gv.z * gscale, gv.w * gscale};
    if (i < wd_end) {
      const float4 pv = p[i];
      t[0] = gv.x * gscale + wd * pv.x; t[1] = gv.y * gscale + wd * pv.y;
      t[2] = gv.z * gscale + wd * pv.z; t[3] = gv.w * gscale + wd * pv.w;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) s = fma((double)t[k], (double)t[k], s);
  }
  s = block_sum_256(s, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last_s = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last_s) return;
  __threadfence();
  double tot = 0.0;
  for (unsigned int j = threadIdx.x; j < gridDim.x; j += blockDim.x) tot += __ldcg(partial + j);
  __syncthreads();                                             // red is reused
  tot = block_sum_256(tot, red);
  if (threadIdx.x == 0) {
    const float norm = (float)sqrt(tot);
    const float c = __fdiv_rn(max_norm, __fadd_rn(norm, 1e-6f));
    out[0] = norm;
    out[1] = c > 1.f ? 1.f : c;                                // not fminf: fminf(NaN, 1) is 1
    *ticket = 0u;
  }
}

}  // namespace

extern "C" int ts_flat_adam(float* p, const float* g, float* m, float* v, void* shadow, long long n, float lr_t,
                            float b1, float b2, float eps, float wd, float gscale, cudaStream_t st, int* step_dev, long long wd_n,
                            const float* clip) {
  if (n % 4 || (wd_n >= 0 && wd_n % 4)) return -2;       // the decay is chosen per float4: [0, wd_n) must end on one
  size_t n4 = (size_t)n / 4;
  if (step_dev) inc_step_kernel<<<1, 1, 0, st>>>(step_dev);
  auto kern = clip ? flat_adam_kernel<true> : flat_adam_kernel<false>;
  kern<<<grid_for(n4), 256, 0, st>>>((float4*)p, (const float4*)g, (float4*)m, (float4*)v, (uint2*)shadow, n4, lr_t, b1, b2, eps,
                                     wd, gscale, step_dev, wd_n < 0 ? n4 : (size_t)wd_n / 4, clip);
  return (int)cudaGetLastError();
}

extern "C" int ts_flat_sgd(float* p, const float* g, void* shadow, long long n, float lr, float wd, float gscale,
                           cudaStream_t st, long long wd_n, const float* clip) {
  if (n % 4 || (wd_n >= 0 && wd_n % 4)) return -2;
  size_t n4 = (size_t)n / 4;
  auto kern = clip ? flat_sgd_kernel<true> : flat_sgd_kernel<false>;
  kern<<<grid_for(n4), 256, 0, st>>>((float4*)p, (const float4*)g, (uint2*)shadow, n4, lr, wd, gscale,
                                     wd_n < 0 ? n4 : (size_t)wd_n / 4, clip);
  return (int)cudaGetLastError();
}

extern "C" int ts_flat_asgd(float* p, const float* g, float* ax, int* avg, void* shadow, long long n, float lr, float wd,
                            float gscale, cudaStream_t st, long long wd_n, const float* clip) {
  if (n % 4 || (wd_n >= 0 && wd_n % 4)) return -2;
  size_t n4 = (size_t)n / 4;
  bump_avg_kernel<<<1, 1, 0, st>>>(avg);
  auto kern = clip ? flat_asgd_kernel<true> : flat_asgd_kernel<false>;
  kern<<<grid_for(n4), 256, 0, st>>>((float4*)p, (const float4*)g, (float4*)ax, avg, (uint2*)shadow, n4, lr, wd, gscale,
                                     wd_n < 0 ? n4 : (size_t)wd_n / 4, clip);
  return (int)cudaGetLastError();
}

extern "C" int ts_flat_average(const float* p, float* ax, int* avg, long long n, cudaStream_t st) {
  if (n % 4) return -2;
  size_t n4 = (size_t)n / 4;
  bump_avg_kernel<<<1, 1, 0, st>>>(avg);
  flat_average_kernel<<<grid_for(n4), 256, 0, st>>>((const float4*)p, (float4*)ax, avg, n4);
  return (int)cudaGetLastError();
}

extern "C" int ts_flat_swap(float* p, float* ax, void* shadow, long long n, cudaStream_t st) {
  if (n % 4) return -2;
  size_t n4 = (size_t)n / 4;
  flat_swap_kernel<<<grid_for(n4), 256, 0, st>>>((float4*)p, (float4*)ax, (uint2*)shadow, n4);
  return (int)cudaGetLastError();
}

// Scratch of flat_grad_norm in doubles: one fp64 partial per CTA, then the ticket word (zero before the first call; every call
// leaves it zero).
extern "C" long long ts_flat_grad_norm_scratch(long long n) { return grid_for((size_t)n / 4) + 1; }

// out: fp32 [2] = {norm, coef}; p is read only when wd != 0.
extern "C" int ts_flat_grad_norm(const float* g, const float* p, long long n, float wd, float gscale, long long wd_n, float max_norm,
                                 double* scratch, float* out, cudaStream_t st) {
  if (n % 4 || (wd_n >= 0 && wd_n % 4)) return -2;
  size_t n4 = (size_t)n / 4;
  const int grid = grid_for(n4);
  flat_grad_norm_kernel<<<grid, 256, 0, st>>>((const float4*)g, (const float4*)p, n4, wd, gscale,
                                              wd_n < 0 ? n4 : (size_t)wd_n / 4, max_norm, scratch,
                                              (unsigned int*)(scratch + grid), out);
  return (int)cudaGetLastError();
}

extern "C" int ts_cast_bf16(const float* p, void* shadow, long long n, cudaStream_t st) {
  if (n % 4) return -2;
  size_t n4 = (size_t)n / 4;
  cast_bf16_kernel<<<grid_for(n4), 256, 0, st>>>((const float4*)p, (uint2*)shadow, n4);
  return (int)cudaGetLastError();
}
