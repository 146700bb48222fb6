// AWD-LSTM's activation regularisation (Merity et al. 2017) on the top layer's output sequence, two launches per top-layer op:
//   act_reg_fwd_kernel: the op's unnormalised sums {sum out^2, sum (h_t - h_{t-1})^2} over its counted positions, fp32 [2];
//   act_reg_bwd_kernel: the gradient the top recurrence's backward then reads (unmasked),
//       dh_total = keep * s * (dh + 2 g0 out) + 2 g1 ((h_t - h_{t-1})[t >= 1] - (h_{t+1} - h_t)[t + 1 < len_b])
//     at counted positions (t < len_b), and keep * s * dh elsewhere (the padded positions carry the head's gradient, if any, and
//     no penalty term), g = d loss / d sums (the model's ALPHA / N_ar, BETA / N_tar).
// out is the sequence the head reads (the top layer's h_drop under --output_dropout, else h itself: then out == null and h is
// read once), h the raw output in time order, both [T,B,H] time-major in the compute dtype.  keep / s are the output dropout's
// mask and scale (ts::dropout_keep8, the top layer's DropSpec, locked or per step).
//
// Both kernels give each thread one column (batch row b, V units from j) and walk it through kSteps time steps, carrying
// h_{t-1} (and h_t, h_{t+1}) in registers: every array is read once, plus one row of h per chunk boundary.  V = 8 (16-byte
// loads and stores) for bf16 with H % 8 == 0, V = 1 otherwise (fp32, other H).
// The sums are deterministic and do not depend on the SM count: the grid depends on the shape alone, each thread sums the fp32
// squares of its fp32 values (differences of two bf16 values are exact in fp32) in fp64, each CTA sums in a fixed tree, and
// the last CTA to take a ticket sums the CTA partials in a fixed order and leaves the ticket 0 (flat_grad_norm_kernel's
// pattern, csrc/multi_tensor_opt.cu).
#include "ts_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kSteps = 16;         // time steps per CTA: the grid is [ceil(B H / V / 256), ceil(T / 16)]

template <int V, typename T>
TS_DEVICE void load_f(const T* __restrict__ p, float (&v)[V]) {
  if constexpr (V == 8) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      v[2 * i] = __uint_as_float(w[i] << 16);
      v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  } else {
    v[0] = ts::Cvt<T>::to_f(p[0]);
  }
}

template <int V, typename T>
TS_DEVICE void store_f(T* __restrict__ p, const float (&v)[V]) {
  if constexpr (V == 8) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      w[i] = (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v[2 * i])) |
             ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v[2 * i + 1])) << 16);
    *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
  } else {
    p[0] = ts::Cvt<T>::from_f(v[0]);
  }
}

// Two fp64 sums over the CTA in a fixed tree: shuffles within each warp, then warp 0 over the 8 warp sums.  -> thread 0.
TS_DEVICE void block_sum2(double& a, double& b, double (*red)[8]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_down_sync(0xffffffffu, a, o);
    b += __shfl_down_sync(0xffffffffu, b, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = a;
    red[1][threadIdx.x >> 5] = b;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    a = threadIdx.x < 8 ? red[0][threadIdx.x] : 0.0;
    b = threadIdx.x < 8 ? red[1][threadIdx.x] : 0.0;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      a += __shfl_down_sync(0xffffffffu, a, o);
      b += __shfl_down_sync(0xffffffffu, b, o);
    }
  }
}

// Column of thread: batch row b, units [j, j + V); false past the last column.
TS_DEVICE bool column(int B, int H, int V, int& b, int& j) {
  const long long col = (long long)blockIdx.x * kThreads + threadIdx.x;
  const int per_row = H / V;
  if (col >= (long long)B * per_row) return false;
  b = (int)(col / per_row);
  j = (int)(col % per_row) * V;
  return true;
}

TS_DEVICE int row_length(const int* __restrict__ lengths, int b, int T) {
  if (lengths == nullptr) return T;
  const int l = __ldg(lengths + b);
  return l < 0 ? 0 : (l > T ? T : l);
}

template <typename T, int V>
__global__ void __launch_bounds__(kThreads) act_reg_fwd_kernel(const T* __restrict__ out, const T* __restrict__ h,
                                                               const int* __restrict__ lengths, int Tn, int B, int H,
                                                               double* __restrict__ partial, unsigned int* __restrict__ ticket,
                                                               float* __restrict__ sums) {
  __shared__ double red[2][8];
  __shared__ bool last_s;
  double s_ar = 0.0, s_tar = 0.0;
  int b, j;
  if (column(B, H, V, b, j)) {
    const int len = row_length(lengths, b, Tn);
    const int t0 = blockIdx.y * kSteps, t1 = min(t0 + kSteps, len);
    const size_t stride = (size_t)B * H, base = (size_t)b * H + j;
    float prev[V];
    if (t0 >= 1 && t0 < len) load_f<V>(h + (size_t)(t0 - 1) * stride + base, prev);
#pragma unroll 4
    for (int t = t0; t < t1; ++t) {
      float cur[V], o[V];
      load_f<V>(h + (size_t)t * stride + base, cur);
      if (out != nullptr) load_f<V>(out + (size_t)t * stride + base, o);
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const float x = out != nullptr ? o[k] : cur[k];
        s_ar = fma((double)x, (double)x, s_ar);
        if (t >= 1) {
          const float d = cur[k] - prev[k];
          s_tar = fma((double)d, (double)d, s_tar);
        }
        prev[k] = cur[k];
      }
    }
  }
  block_sum2(s_ar, s_tar, red);
  const unsigned int nblk = gridDim.x * gridDim.y, blk = blockIdx.y * gridDim.x + blockIdx.x;
  if (threadIdx.x == 0) {
    partial[2 * blk] = s_ar;
    partial[2 * blk + 1] = s_tar;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last_s = atomicAdd(ticket, 1u) == nblk - 1;
  __syncthreads();
  if (!last_s) return;
  __threadfence();
  double a = 0.0, c = 0.0;
  for (unsigned int i = threadIdx.x; i < nblk; i += blockDim.x) {
    a += __ldcg(partial + 2 * i);
    c += __ldcg(partial + 2 * i + 1);
  }
  __syncthreads();                                             // red is reused
  block_sum2(a, c, red);
  if (threadIdx.x == 0) {
    sums[0] = (float)a;
    sums[1] = (float)c;
    *ticket = 0u;
  }
}

// (kThreads, 2): with the thread count alone ptxas holds the 16-byte variant to 64 registers and spills; it needs 80.
template <typename T, int V>
__global__ void __launch_bounds__(kThreads, 2) act_reg_bwd_kernel(const T* __restrict__ dh, const T* __restrict__ out,
                                                               const T* __restrict__ h, const int* __restrict__ lengths,
                                                               const float* __restrict__ g, int Tn, int B, int H, ts::DropSpec d,
                                                               T* __restrict__ dst) {
  int b, j;
  if (!column(B, H, V, b, j)) return;
  const int len = row_length(lengths, b, Tn);
  const int t0 = blockIdx.y * kSteps, t1 = min(t0 + kSteps, Tn);
  const size_t stride = (size_t)B * H, base = (size_t)b * H + j;
  const float g0 = 2.f * __ldg(g), g1 = 2.f * __ldg(g + 1);
  const bool drop = d.step != nullptr;
  const uint32_t step = drop ? (uint32_t)__ldg(d.step) : 0u;
  const int jg = j & ~7, sh = j & 7;                           // the Philox group of unit j, j's bit in it
  const bool locked = drop && (d.c2 & ts::kDropLocked);
  const uint32_t keep_locked = locked ? ts::dropout_keep8(d, step, b, jg, 0, H) >> sh : 0u;
  float prev[V], cur[V], next[V] = {};
  if (t0 >= 1 && t0 < len) load_f<V>(h + (size_t)(t0 - 1) * stride + base, prev);
  if (t0 < len) load_f<V>(h + (size_t)t0 * stride + base, cur);
  for (int t = t0; t < t1; ++t) {
    float r[V];
    if (t >= len) {                                            // no penalty term: the head's gradient, masked
      float dv[V];
      if (dh != nullptr) load_f<V>(dh + (size_t)t * stride + base, dv);
      const uint32_t keep = !drop ? 0xffu : (locked ? keep_locked : ts::dropout_keep8(d, step, b, jg, t, H) >> sh);
#pragma unroll
      for (int k = 0; k < V; ++k)
        r[k] = dh == nullptr || !((keep >> k) & 1u) ? 0.f : (drop ? __fmul_rn(dv[k], d.scale) : dv[k]);
      store_f<V>(dst + (size_t)t * stride + base, r);
      continue;
    }
    const bool has_next = t + 1 < len;
    if (has_next) load_f<V>(h + (size_t)(t + 1) * stride + base, next);
    float o[V], dv[V];
    if (out != nullptr) load_f<V>(out + (size_t)t * stride + base, o);
    if (dh != nullptr) load_f<V>(dh + (size_t)t * stride + base, dv);
    const uint32_t keep = !drop ? 0xffu : (locked ? keep_locked : ts::dropout_keep8(d, step, b, jg, t, H) >> sh);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float a = fmaf(g0, out != nullptr ? o[k] : cur[k], dh != nullptr ? dv[k] : 0.f);
      const float m = !drop ? a : (((keep >> k) & 1u) ? __fmul_rn(a, d.scale) : 0.f);
      float st = t >= 1 ? cur[k] - prev[k] : 0.f;
      if (has_next) st -= next[k] - cur[k];
      r[k] = fmaf(g1, st, m);
      prev[k] = cur[k];
      cur[k] = next[k];
    }
    store_f<V>(dst + (size_t)t * stride + base, r);
  }
}

dim3 grid_of(int T, int B, int H, int V) {
  const long long cols = (long long)B * (H / V);
  return dim3((unsigned int)((cols + kThreads - 1) / kThreads), (unsigned int)((T + kSteps - 1) / kSteps));
}

int vec_of(int is_bf16, int H) { return is_bf16 && H % 8 == 0 ? 8 : 1; }

}  // namespace

// Scratch of ts_act_reg_fwd in doubles: two fp64 partials per CTA, then the ticket word (zero before the first call; every call
// leaves it zero).
extern "C" long long ts_act_reg_scratch(int T, int B, int H, int is_bf16) {
  const dim3 g = grid_of(T, B, H, vec_of(is_bf16, H));
  return 2LL * g.x * g.y + 1;
}

// sums: fp32 [2] = {sum out^2, sum (h_t - h_{t-1})^2} over the counted positions; out null: out is h.
extern "C" int ts_act_reg_fwd(const void* out, const void* h, const int* lengths, int T, int B, int H, int is_bf16, double* scratch,
                              float* sums, cudaStream_t st) {
  if (T < 1 || B < 1 || H < 1) return -2;
  const int V = vec_of(is_bf16, H);
  const dim3 grid = grid_of(T, B, H, V);
  unsigned int* ticket = (unsigned int*)(scratch + 2LL * grid.x * grid.y);
  if (!is_bf16)
    act_reg_fwd_kernel<float, 1><<<grid, kThreads, 0, st>>>((const float*)out, (const float*)h, lengths, T, B, H, scratch, ticket, sums);
  else if (V == 8)
    act_reg_fwd_kernel<__nv_bfloat16, 8><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)out, (const __nv_bfloat16*)h, lengths, T, B,
                                                                   H, scratch, ticket, sums);
  else
    act_reg_fwd_kernel<__nv_bfloat16, 1><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)out, (const __nv_bfloat16*)h, lengths, T, B,
                                                                   H, scratch, ticket, sums);
  return (int)cudaGetLastError();
}

// dst [T,B,H] = the combined gradient (header comment); dh null: no gradient from the head; out null: out is h (no output
// dropout, drop_step null).  g: fp32 [2] on the device.
extern "C" int ts_act_reg_bwd(const void* dh, const void* out, const void* h, const int* lengths, const float* g, int T, int B, int H,
                              int is_bf16, const int* drop_step, const unsigned int* drop_desc, void* dst, cudaStream_t st) {
  if (T < 1 || B < 1 || H < 1) return -2;
  const ts::DropSpec d = ts::make_drop_spec(drop_step, drop_desc);
  const int V = vec_of(is_bf16, H);
  const dim3 grid = grid_of(T, B, H, V);
  if (!is_bf16)
    act_reg_bwd_kernel<float, 1><<<grid, kThreads, 0, st>>>((const float*)dh, (const float*)out, (const float*)h, lengths, g, T, B, H,
                                                            d, (float*)dst);
  else if (V == 8)
    act_reg_bwd_kernel<__nv_bfloat16, 8><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)dh, (const __nv_bfloat16*)out,
                                                                   (const __nv_bfloat16*)h, lengths, g, T, B, H, d,
                                                                   (__nv_bfloat16*)dst);
  else
    act_reg_bwd_kernel<__nv_bfloat16, 1><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)dh, (const __nv_bfloat16*)out,
                                                                   (const __nv_bfloat16*)h, lengths, g, T, B, H, d,
                                                                   (__nv_bfloat16*)dst);
  return (int)cudaGetLastError();
}
