// Pooling of the top layer's output over time for sequence classification (--pooling mean | max | attention).
//
// h_seq [T,B,H] is read in place as T·B time-major rows; lengths (int32 [B], device) mark the counted steps t < len_b
// (every step without lengths).  Nothing at an uncounted step reaches a result or a gradient, and every reduction runs in
// a fixed order (two calls give identical bits).  Nothing is read back to the host, so a captured graph holds across batches
// with different lengths.
//
//   forward  mean       s_b = (1/len_b) sum_{t<len_b} h_t                       (fp32 sum in t order, one rounded division)
//            max        s_b[j] = max_{t<len_b} h_t[j], argmax = the smallest t attaining it
//            attention  u = tanh(h W_a + b_a) (h W_a: the wgmma GEMM, fp32 out), e_t = u_t . v, alpha = softmax over t < len_b
//                       (max-subtracted; alpha = 0 elsewhere), s_b = sum_t alpha_t h_t.  u is KEPT (fp32 [T·B, A], written
//                       over the GEMM's output in place) for the backward pass, not recomputed.
//   backward mean       dh_t = ds / len_b
//            max        dh_t[j] = ds[j] at t = argmax[j], 0 elsewhere
//            attention  dalpha_t = ds . h_t, de_t = alpha_t (dalpha_t - sum_t alpha_t dalpha_t), dU = de_t v (1 - u^2);
//                       dh_t = alpha_t ds + (dU W_a^T)_t, the second term from the GEMM in fp32, summed and rounded once here.
//                       dv = sum de_t u_t and db_a = sum dU_t (fp32 dU) come from per-CTA partials that the last CTA to take
//                       a ticket sums in batch-row order.
#include "ts_common.cuh"

namespace {

constexpr int kMean = 0, kMax = 1, kAttn = 2;
constexpr int kThreads = 256;

TS_DEVICE int row_len(const int* lengths, int b, int T) { return lengths ? lengths[b] : T; }

// Fixed-order block reductions over kThreads threads (warp butterflies, then warp 0 over the 8 warp results).
template <bool MAX>
TS_DEVICE float block_reduce(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = MAX ? ts::warp_max(v) : ts::warp_sum(v);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = lane < kThreads / 32 ? red[lane] : (MAX ? -INFINITY : 0.f);
  r = MAX ? ts::warp_max(r) : ts::warp_sum(r);
  __syncthreads();                                            // red is reused by the next call
  return r;
}

// One thread per (column j, row b): grid (B, ceil(H / 256)).  alpha [T,B] (attention only).
template <int MODE, typename TIn>
__global__ void __launch_bounds__(kThreads) seq_pool_fwd_kernel(const TIn* __restrict__ h, const int* __restrict__ lengths,
                                                                const float* __restrict__ alpha, int T, int B, int H,
                                                                float* __restrict__ s, int* __restrict__ argmax) {
  const int b = blockIdx.x;
  const int j = blockIdx.y * kThreads + threadIdx.x;
  if (j >= H) return;
  const int len = row_len(lengths, b, T);
  const size_t step = (size_t)B * H;
  const TIn* p = h + (size_t)b * H + j;
  if (MODE == kMax) {
    float m = ts::Cvt<TIn>::to_f(p[0]);
    int am = 0;
#pragma unroll 4
    for (int t = 1; t < len; ++t) {
      const float x = ts::Cvt<TIn>::to_f(p[t * step]);
      if (x > m) { m = x; am = t; }                           // strict: the first t that attains the max keeps it
    }
    s[(size_t)b * H + j] = m;
    argmax[(size_t)b * H + j] = am;
    return;
  }
  float acc = 0.f;
#pragma unroll 4
  for (int t = 0; t < len; ++t) {
    const float x = ts::Cvt<TIn>::to_f(p[t * step]);
    acc = MODE == kMean ? acc + x : fmaf(__ldg(alpha + (size_t)t * B + b), x, acc);
  }
  s[(size_t)b * H + j] = MODE == kMean ? __fdiv_rn(acc, (float)len) : acc;
}

// Attention scores, one CTA per batch row b.  u [T·B, A]: in h W_a (fp32), out tanh(h W_a + b_a) at counted steps, 0 at the
// others.  alpha [T,B]: first e_t, then the softmax weights (0 at uncounted steps).  kExact (fp32 h): tanh in fp64, rounded once
// (ts::tanhf_acc); otherwise tanh.approx, within the bf16 path's error.
template <bool kExact>
__global__ void __launch_bounds__(kThreads) attn_scores_kernel(float* __restrict__ u, const float* __restrict__ ba,
                                                               const float* __restrict__ v, const int* __restrict__ lengths,
                                                               int T, int B, int A, float* __restrict__ alpha) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int len = row_len(lengths, b, T);
  for (int t = warp; t < T; t += kThreads / 32) {
    float* row = u + ((size_t)t * B + b) * A;
    if (t >= len) {
      for (int k = lane; k < A; k += 32) row[k] = 0.f;
      continue;
    }
    float e = 0.f;
    for (int k = lane; k < A; k += 32) {
      const float x = kExact ? ts::tanhf_acc(row[k] + ba[k]) : ts::tanhf_fast(row[k] + ba[k]);
      row[k] = x;
      e = fmaf(x, v[k], e);
    }
    e = ts::warp_sum(e);
    if (lane == 0) alpha[(size_t)t * B + b] = e;
  }
  __syncthreads();                                            // e_t of every warp visible to the whole CTA
  float m = -INFINITY;
  for (int t = threadIdx.x; t < len; t += kThreads) m = fmaxf(m, alpha[(size_t)t * B + b]);
  m = block_reduce<true>(m, red);
  float z = 0.f;
  for (int t = threadIdx.x; t < len; t += kThreads) z += expf(alpha[(size_t)t * B + b] - m);
  z = block_reduce<false>(z, red);
  for (int t = threadIdx.x; t < T; t += kThreads) {
    float* a = alpha + (size_t)t * B + b;
    *a = t < len ? __fdiv_rn(expf(*a - m), z) : 0.f;
  }
}

// Attention backward up to dU, one CTA per batch row b.  dalpha [T,B] is scratch.  dU [T·B, A] in TU (bf16 for the tensor-core
// GEMMs that read it, fp32 on the fp32 path), 0 at uncounted steps.  partial [B, 2A]: this row's dv and db_a; the last CTA sums
// them over b in order into dv / dba (accumulating into them when acc_dv / acc_dba) and leaves the ticket 0.
template <typename TIn, typename TU>
__global__ void __launch_bounds__(kThreads) attn_bwd_kernel(const TIn* __restrict__ h, const float* __restrict__ ds,
                                                            const float* __restrict__ alpha, const float* __restrict__ u,
                                                            const float* __restrict__ v, const int* __restrict__ lengths,
                                                            int T, int B, int H, int A, float* __restrict__ dalpha,
                                                            TU* __restrict__ dU, float* __restrict__ partial,
                                                            unsigned int* __restrict__ ticket, float* __restrict__ dv,
                                                            float* __restrict__ dba, int acc_dv, int acc_dba) {
  __shared__ float red[32];
  __shared__ bool last_s;
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int len = row_len(lengths, b, T);
  const float* dsb = ds + (size_t)b * H;
  for (int t = warp; t < len; t += kThreads / 32) {
    const TIn* hr = h + ((size_t)t * B + b) * H;
    float d = 0.f;
    for (int j = lane; j < H; j += 32) d = fmaf(dsb[j], ts::Cvt<TIn>::to_f(hr[j]), d);
    d = ts::warp_sum(d);
    if (lane == 0) dalpha[(size_t)t * B + b] = d;
  }
  __syncthreads();
  float sad = 0.f;
  for (int t = threadIdx.x; t < len; t += kThreads) sad = fmaf(alpha[(size_t)t * B + b], dalpha[(size_t)t * B + b], sad);
  sad = block_reduce<false>(sad, red);
  for (int t = threadIdx.x; t < len; t += kThreads) {
    float* d = dalpha + (size_t)t * B + b;
    *d = alpha[(size_t)t * B + b] * (*d - sad);               // de_t
  }
  __syncthreads();
  for (int k = threadIdx.x; k < A; k += kThreads) {
    const float vk = v[k];
    float pv = 0.f, pb = 0.f;
    for (int t = 0; t < T; ++t) {
      const size_t r = ((size_t)t * B + b) * A + k;
      float g = 0.f;
      if (t < len) {
        const float de = dalpha[(size_t)t * B + b], uk = u[r];
        g = de * vk * (1.f - uk * uk);
        pv = fmaf(de, uk, pv);
        pb += g;
      }
      dU[r] = ts::Cvt<TU>::from_f(g);
    }
    partial[(size_t)b * 2 * A + k] = pv;
    partial[(size_t)b * 2 * A + A + k] = pb;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last_s = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last_s) return;
  __threadfence();
  for (int k = threadIdx.x; k < 2 * A; k += kThreads) {
    float tot = 0.f;
    for (int r = 0; r < B; ++r) tot += __ldcg(partial + (size_t)r * 2 * A + k);
    if (k < A) dv[k] = acc_dv ? dv[k] + tot : tot;
    else dba[k - A] = acc_dba ? dba[k - A] + tot : tot;
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

// dh_seq [T·B, H] in TOut, one CTA per row (t, b); 0 at uncounted steps.  G [T·B, H] fp32: dU W_a^T (attention only).
template <int MODE, typename TOut>
__global__ void __launch_bounds__(kThreads) seq_pool_bwd_kernel(const float* __restrict__ ds, const int* __restrict__ lengths,
                                                                const int* __restrict__ argmax, const float* __restrict__ alpha,
                                                                const float* __restrict__ G, int T, int B, int H,
                                                                TOut* __restrict__ dh) {
  const size_t row = blockIdx.x;
  const int t = (int)(row / B), b = (int)(row % B);
  const int len = row_len(lengths, b, T);
  const float* dsb = ds + (size_t)b * H;
  TOut* out = dh + row * H;
  if (t >= len) {
    for (int j = threadIdx.x; j < H; j += kThreads) out[j] = ts::Cvt<TOut>::from_f(0.f);
    return;
  }
  const float a = MODE == kAttn ? alpha[row] : 0.f;
  for (int j = threadIdx.x; j < H; j += kThreads) {
    float g;
    if (MODE == kMean) g = __fdiv_rn(dsb[j], (float)len);
    else if (MODE == kMax) g = argmax[(size_t)b * H + j] == t ? dsb[j] : 0.f;
    else g = fmaf(a, dsb[j], G[row * H + j]);
    out[j] = ts::Cvt<TOut>::from_f(g);
  }
}

template <int MODE, typename TIn>
int launch_fwd(const void* h, const int* lengths, const float* alpha, int T, int B, int H, float* s, int* argmax, cudaStream_t st) {
  dim3 grid(B, (H + kThreads - 1) / kThreads);
  seq_pool_fwd_kernel<MODE, TIn><<<grid, kThreads, 0, st>>>((const TIn*)h, lengths, alpha, T, B, H, s, argmax);
  return (int)cudaGetLastError();
}

template <int MODE, typename TOut>
int launch_bwd(const float* ds, const int* lengths, const int* argmax, const float* alpha, const float* G, int T, int B, int H,
               void* dh, cudaStream_t st) {
  seq_pool_bwd_kernel<MODE, TOut><<<(unsigned)((size_t)T * B), kThreads, 0, st>>>(ds, lengths, argmax, alpha, G, T, B, H, (TOut*)dh);
  return (int)cudaGetLastError();
}

}  // namespace

// mode: 0 mean, 1 max (argmax required), 2 attention (alpha required).  h_bf16: h is bf16, else fp32.
extern "C" int ts_seq_pool_fwd(const void* h, int h_bf16, const int* lengths, const float* alpha, int mode, int T, int B, int H,
                               float* s, int* argmax, cudaStream_t st) {
  if (T < 1 || B < 1 || H < 1) return -2;
  if (mode == kMax && !argmax) return -3;
  if (mode == kAttn && !alpha) return -3;
  if (h_bf16) {
    if (mode == kMean) return launch_fwd<kMean, __nv_bfloat16>(h, lengths, alpha, T, B, H, s, argmax, st);
    if (mode == kMax) return launch_fwd<kMax, __nv_bfloat16>(h, lengths, alpha, T, B, H, s, argmax, st);
    if (mode == kAttn) return launch_fwd<kAttn, __nv_bfloat16>(h, lengths, alpha, T, B, H, s, argmax, st);
  } else {
    if (mode == kMean) return launch_fwd<kMean, float>(h, lengths, alpha, T, B, H, s, argmax, st);
    if (mode == kMax) return launch_fwd<kMax, float>(h, lengths, alpha, T, B, H, s, argmax, st);
    if (mode == kAttn) return launch_fwd<kAttn, float>(h, lengths, alpha, T, B, H, s, argmax, st);
  }
  return -4;
}

extern "C" int ts_seq_pool_attn_scores(float* u, const float* ba, const float* v, const int* lengths, int T, int B, int A,
                                       float* alpha, int exact, cudaStream_t st) {
  if (T < 1 || B < 1 || A < 1) return -2;
  if (exact)
    attn_scores_kernel<true><<<B, kThreads, 0, st>>>(u, ba, v, lengths, T, B, A, alpha);
  else
    attn_scores_kernel<false><<<B, kThreads, 0, st>>>(u, ba, v, lengths, T, B, A, alpha);
  return (int)cudaGetLastError();
}

// partial: fp32 [B, 2A]; dalpha: fp32 [T, B]; ticket: one zeroed word (left zero).  dU bf16 iff h is bf16.
extern "C" int ts_seq_pool_attn_bwd(const void* h, int h_bf16, const float* ds, const float* alpha, const float* u, const float* v,
                                    const int* lengths, int T, int B, int H, int A, float* dalpha, void* dU, float* partial,
                                    unsigned int* ticket, float* dv, float* dba, int acc_dv, int acc_dba, cudaStream_t st) {
  if (T < 1 || B < 1 || H < 1 || A < 1) return -2;
  if (h_bf16)
    attn_bwd_kernel<__nv_bfloat16, __nv_bfloat16><<<B, kThreads, 0, st>>>((const __nv_bfloat16*)h, ds, alpha, u, v, lengths, T, B, H,
                                                                           A, dalpha, (__nv_bfloat16*)dU, partial, ticket, dv, dba,
                                                                           acc_dv, acc_dba);
  else
    attn_bwd_kernel<float, float><<<B, kThreads, 0, st>>>((const float*)h, ds, alpha, u, v, lengths, T, B, H, A, dalpha, (float*)dU,
                                                          partial, ticket, dv, dba, acc_dv, acc_dba);
  return (int)cudaGetLastError();
}

extern "C" int ts_seq_pool_bwd(const float* ds, const int* lengths, const int* argmax, const float* alpha, const float* G, int mode,
                               int T, int B, int H, void* dh, int out_bf16, cudaStream_t st) {
  if (T < 1 || B < 1 || H < 1) return -2;
  if ((mode == kMax && !argmax) || (mode == kAttn && (!alpha || !G))) return -3;
  if (out_bf16) {
    if (mode == kMean) return launch_bwd<kMean, __nv_bfloat16>(ds, lengths, argmax, alpha, G, T, B, H, dh, st);
    if (mode == kMax) return launch_bwd<kMax, __nv_bfloat16>(ds, lengths, argmax, alpha, G, T, B, H, dh, st);
    if (mode == kAttn) return launch_bwd<kAttn, __nv_bfloat16>(ds, lengths, argmax, alpha, G, T, B, H, dh, st);
  } else {
    if (mode == kMean) return launch_bwd<kMean, float>(ds, lengths, argmax, alpha, G, T, B, H, dh, st);
    if (mode == kMax) return launch_bwd<kMax, float>(ds, lengths, argmax, alpha, G, T, B, H, dh, st);
    if (mode == kAttn) return launch_bwd<kAttn, float>(ds, lengths, argmax, alpha, G, T, B, H, dh, st);
  }
  return -4;
}
