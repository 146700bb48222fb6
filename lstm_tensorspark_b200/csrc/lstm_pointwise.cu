// Generic-shape LSTM cell epilogue kernels (any B, H): gate activations + c/h update (forward) and the
// gate-gradient math (backward), each ONE launch per time step instead of the reference's ~19 elementwise
// TF ops per layer per step (reference: original src/models/recurrent/lstm.py:93-109).
// The 4-gate GEMM that feeds them is a library GEMM on this path; shapes that fit the tensor-core tiling
// take the persistent wgmma kernel in lstm_seq_wgmma.cu instead.
//
// kFast (bf16): tanh.approx activations, within the bf16 storage's error; fp32 (kFast = false) computes them in fp64 and rounds
// once (ts::tanhf_acc / sigmoidf_acc), so the fp32 path is as accurate as fp32 storage.
// Layout: pre/act/dpre are [B, 4H] with column n = 4*j + g, g: 0=i 1=f 2=g(candidate) 3=o. c is fp32.
// kMasked (per-row lengths, right padding): at step t >= lengths[b] row b holds its state - forward h_t = h_{t-1}, c_t = c_{t-1};
// backward dpre = 0, dc passes through and the total dh is handed on (dh_out) instead of going through W_h.
#include "ts_common.cuh"

namespace {

template <typename T, bool kFast, bool kMasked = false>
__global__ void lstm_pointwise_fwd_kernel(const T* __restrict__ pre, const float* __restrict__ bias,
                                          const float* __restrict__ c_prev, T* __restrict__ h_out,
                                          float* __restrict__ c_out, T* __restrict__ act, int B, int H,
                                          const T* __restrict__ h_prev = nullptr, const int* __restrict__ lengths = nullptr,
                                          int t = 0) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * H) return;
  int j = idx % H;
  if constexpr (kMasked) {
    if (t >= lengths[idx / H]) {               // padded step: carry the state (act is never read back)
      c_out[idx] = c_prev[idx];
      h_out[idx] = h_prev[idx];
      return;
    }
  }
  const T* p = pre + (size_t)idx * 4;
  float pi = ts::Cvt<T>::to_f(p[0]) + bias[4 * j + 0];
  float pf = ts::Cvt<T>::to_f(p[1]) + bias[4 * j + 1];
  float pg = ts::Cvt<T>::to_f(p[2]) + bias[4 * j + 2];
  float po = ts::Cvt<T>::to_f(p[3]) + bias[4 * j + 3];
  float i, f, g, o;
  if (kFast) {
    i = ts::sigmoidf_fast(pi); f = ts::sigmoidf_fast(pf); g = ts::tanhf_fast(pg); o = ts::sigmoidf_fast(po);
  } else {
    i = ts::sigmoidf_acc(pi); f = ts::sigmoidf_acc(pf); g = ts::tanhf_acc(pg); o = ts::sigmoidf_acc(po);
  }
  float c = f * c_prev[idx] + i * g;
  float h = o * (kFast ? ts::tanhf_fast(c) : ts::tanhf_acc(c));
  c_out[idx] = c;
  h_out[idx] = ts::Cvt<T>::from_f(h);
  T* a = act + (size_t)idx * 4;
  a[0] = ts::Cvt<T>::from_f(i); a[1] = ts::Cvt<T>::from_f(f);
  a[2] = ts::Cvt<T>::from_f(g); a[3] = ts::Cvt<T>::from_f(o);
}

// dh_a / dh_b: the two sources of dL/dh_t (layer above, and the recurrent term); either may be null.
// kMasked: dh_out [B,H] fp32 = the dh handed to step t-1 directly (the total dh at a padded step, 0 otherwise); the caller
// adds dpre W_h to it.
template <typename T, bool kFast, bool kMasked = false>
__global__ void lstm_pointwise_bwd_kernel(const T* __restrict__ dh_a, const float* __restrict__ dh_b,
                                          const float* __restrict__ dc_in, const T* __restrict__ act,
                                          const float* __restrict__ c_prev, const float* __restrict__ c_new,
                                          T* __restrict__ dpre, float* __restrict__ dc_out, int B, int H,
                                          const int* __restrict__ lengths = nullptr, int t = 0, float* __restrict__ dh_out = nullptr) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * H) return;
  float dh = 0.f;
  if (dh_a) dh += ts::Cvt<T>::to_f(dh_a[idx]);
  if (dh_b) dh += dh_b[idx];
  if constexpr (kMasked) {
    const bool pad = t >= lengths[idx / H];
    dh_out[idx] = pad ? dh : 0.f;
    if (pad) {
      dc_out[idx] = dc_in ? dc_in[idx] : 0.f;
      T* d = dpre + (size_t)idx * 4;
      d[0] = d[1] = d[2] = d[3] = ts::Cvt<T>::from_f(0.f);
      return;
    }
  }
  const T* a = act + (size_t)idx * 4;
  float i = ts::Cvt<T>::to_f(a[0]), f = ts::Cvt<T>::to_f(a[1]);
  float g = ts::Cvt<T>::to_f(a[2]), o = ts::Cvt<T>::to_f(a[3]);
  float tc = kFast ? ts::tanhf_fast(c_new[idx]) : ts::tanhf_acc(c_new[idx]);
  float dc = (dc_in ? dc_in[idx] : 0.f) + dh * o * (1.f - tc * tc);
  float d_o = dh * tc;
  float d_i = dc * g, d_f = dc * c_prev[idx], d_g = dc * i;
  dc_out[idx] = dc * f;
  T* d = dpre + (size_t)idx * 4;
  d[0] = ts::Cvt<T>::from_f(d_i * i * (1.f - i));
  d[1] = ts::Cvt<T>::from_f(d_f * f * (1.f - f));
  d[2] = ts::Cvt<T>::from_f(d_g * (1.f - g * g));
  d[3] = ts::Cvt<T>::from_f(d_o * o * (1.f - o));
}

}  // namespace

extern "C" int ts_lstm_pointwise_fwd(const void* pre, const float* bias, const float* c_prev, void* h_out,
                                     float* c_out, void* act, int B, int H, int is_bf16, cudaStream_t st,
                                     const void* h_prev, const int* lengths, int t) {
  int n = B * H, thr = 256, blk = (n + thr - 1) / thr;
  if (lengths && is_bf16)
    lstm_pointwise_fwd_kernel<__nv_bfloat16, true, true><<<blk, thr, 0, st>>>(
        (const __nv_bfloat16*)pre, bias, c_prev, (__nv_bfloat16*)h_out, c_out, (__nv_bfloat16*)act, B, H,
        (const __nv_bfloat16*)h_prev, lengths, t);
  else if (lengths)
    lstm_pointwise_fwd_kernel<float, false, true><<<blk, thr, 0, st>>>((const float*)pre, bias, c_prev, (float*)h_out,
                                                                       c_out, (float*)act, B, H, (const float*)h_prev, lengths, t);
  else if (is_bf16)
    lstm_pointwise_fwd_kernel<__nv_bfloat16, true><<<blk, thr, 0, st>>>(
        (const __nv_bfloat16*)pre, bias, c_prev, (__nv_bfloat16*)h_out, c_out, (__nv_bfloat16*)act, B, H);
  else
    lstm_pointwise_fwd_kernel<float, false><<<blk, thr, 0, st>>>((const float*)pre, bias, c_prev, (float*)h_out,
                                                                 c_out, (float*)act, B, H);
  return (int)cudaGetLastError();
}

extern "C" int ts_lstm_pointwise_bwd(const void* dh_a, const float* dh_b, const float* dc_in, const void* act,
                                     const float* c_prev, const float* c_new, void* dpre, float* dc_out, int B,
                                     int H, int is_bf16, cudaStream_t st, const int* lengths, int t, float* dh_out) {
  int n = B * H, thr = 256, blk = (n + thr - 1) / thr;
  if (lengths && is_bf16)
    lstm_pointwise_bwd_kernel<__nv_bfloat16, true, true><<<blk, thr, 0, st>>>(
        (const __nv_bfloat16*)dh_a, dh_b, dc_in, (const __nv_bfloat16*)act, c_prev, c_new, (__nv_bfloat16*)dpre,
        dc_out, B, H, lengths, t, dh_out);
  else if (lengths)
    lstm_pointwise_bwd_kernel<float, false, true><<<blk, thr, 0, st>>>((const float*)dh_a, dh_b, dc_in, (const float*)act,
                                                                       c_prev, c_new, (float*)dpre, dc_out, B, H, lengths, t, dh_out);
  else if (is_bf16)
    lstm_pointwise_bwd_kernel<__nv_bfloat16, true><<<blk, thr, 0, st>>>(
        (const __nv_bfloat16*)dh_a, dh_b, dc_in, (const __nv_bfloat16*)act, c_prev, c_new, (__nv_bfloat16*)dpre,
        dc_out, B, H);
  else
    lstm_pointwise_bwd_kernel<float, false><<<blk, thr, 0, st>>>((const float*)dh_a, dh_b, dc_in, (const float*)act,
                                                                  c_prev, c_new, (float*)dpre, dc_out, B, H);
  return (int)cudaGetLastError();
}


// Dropout between stacked layers, standalone: y = x * mask * scale over [T,B,H] (time t0 + t), the mask of ts::dropout_keep8.
// The same launch serves the forward (x = h, stored in x's dtype) and the backward (x = dL/dy) of the shapes the persistent
// kernels do not fuse it into: the generic path (fp32, H % 64 != 0), the one-step [B,D] path and anything else.  One thread
// per Philox group (8 units of one row).
namespace {
template <typename T>
__global__ void dropout_kernel(const T* __restrict__ x, T* __restrict__ y, int steps, int B, int H, int t0, ts::DropSpec d) {
  const int groups = (H + 7) / 8;
  const long long total = (long long)steps * B * groups;
  const uint32_t step = (uint32_t)__ldg(d.step);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const long long tb = i / groups;
    const int b = (int)(tb % B), t = (int)(tb / B);
    const uint32_t keep = ts::dropout_keep8(d, step, b, 8 * g, t0 + t, H);
    const size_t base = (size_t)tb * H + 8 * g;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (8 * g + u >= H) break;
      y[base + u] = ((keep >> u) & 1u) ? ts::Cvt<T>::from_f(__fmul_rn(ts::Cvt<T>::to_f(x[base + u]), d.scale)) : ts::Cvt<T>::from_f(0.f);
    }
  }
}
}  // namespace

extern "C" int ts_dropout(const void* x, void* y, int steps, int B, int H, int t0, int is_bf16, const int* drop_step,
                          const unsigned int* drop_desc, cudaStream_t st) {
  if (drop_step == nullptr) return -2;
  const ts::DropSpec d = ts::make_drop_spec(drop_step, drop_desc);
  const long long total = (long long)steps * B * ((H + 7) / 8);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks < 1) return 0;
  if (is_bf16)
    dropout_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, steps, B, H, t0, d);
  else
    dropout_kernel<float><<<blocks, 256, 0, st>>>((const float*)x, (float*)y, steps, B, H, t0, d);
  return (int)cudaGetLastError();
}


// Weight drop (DropConnect on the recurrent weights): the gradient of W_h' = W_h * M * s reaching W_h, dst (+)= src * M * s over
// one fp32 [R, H] matrix (R = 4H stored rows).  M is the mask of ts::dropout_keep8 with the matrix taken as ONE time step of R
// rows (t = 0; the weight stream's c2 comes with the descriptor), the same mask ts_dropout applies to the [1, R, H] image in the
// forward pass.  One thread per Philox group (8 units of a row): one Philox call, 16 B loads and stores when H % 8 == 0.  src may
// be dst (overwrite, in place): every element is read by the thread that writes it.
namespace {
__global__ void weight_drop_grad_kernel(const float* src, float* dst, int R, int H, int accumulate, ts::DropSpec d) {
  const int groups = (H + 7) / 8;
  const long long total = (long long)R * groups;
  const uint32_t step = (uint32_t)__ldg(d.step);
  const bool vec = (H & 7) == 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups), r = (int)(i / groups);
    const uint32_t keep = ts::dropout_keep8(d, step, r, 8 * g, 0, H);
    const size_t base = (size_t)r * H + 8 * g;
    if (vec) {
      float4 v[2] = {*reinterpret_cast<const float4*>(src + base), *reinterpret_cast<const float4*>(src + base + 4)};
      float4 o[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
      if (accumulate) { o[0] = *reinterpret_cast<const float4*>(dst + base); o[1] = *reinterpret_cast<const float4*>(dst + base + 4); }
      float* vf = reinterpret_cast<float*>(v);
      float* of = reinterpret_cast<float*>(o);
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const float m = ((keep >> u) & 1u) ? __fmul_rn(vf[u], d.scale) : 0.f;
        of[u] = accumulate ? __fadd_rn(of[u], m) : m;
      }
      *reinterpret_cast<float4*>(dst + base) = o[0];
      *reinterpret_cast<float4*>(dst + base + 4) = o[1];
    } else {
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (8 * g + u >= H) break;
        const float m = ((keep >> u) & 1u) ? __fmul_rn(src[base + u], d.scale) : 0.f;
        dst[base + u] = accumulate ? __fadd_rn(dst[base + u], m) : m;
      }
    }
  }
}
}  // namespace

extern "C" int ts_weight_drop_grad(const float* src, float* dst, int R, int H, int accumulate, const int* drop_step,
                                   const unsigned int* drop_desc, cudaStream_t st) {
  if (drop_step == nullptr) return -2;
  if ((H & 7) == 0 && (((uintptr_t)src | (uintptr_t)dst) & 15) != 0) return -3;      // the 16 B path needs aligned rows
  const ts::DropSpec d = ts::make_drop_spec(drop_step, drop_desc);
  const long long total = (long long)R * ((H + 7) / 8);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks < 1) return 0;
  weight_drop_grad_kernel<<<blocks, 256, 0, st>>>(src, dst, R, H, accumulate, d);
  return (int)cudaGetLastError();
}


// [B,T,D] -> [T,B,D] for a row-contiguous tensor (row = D elements, row_bytes % 16 == 0): a pure row permutation, so it
// runs at copy speed with 16 B vectors (the framework's generic strided copy of the transposed view takes 3.5x longer).
// Replaces the batch-major -> time-major feed conversion in front of the first layer's x-projection GEMM.
namespace {
__global__ void transpose01_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int B, int T, int vec_per_row) {
  const long long total = (long long)B * T * vec_per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / vec_per_row;          // destination row = t * B + b
    const int v = (int)(i - row * vec_per_row);
    const int t = (int)(row / B), b = (int)(row - (long long)t * B);
    dst[i] = src[((long long)b * T + t) * vec_per_row + v];
  }
}
}  // namespace

extern "C" int ts_transpose01_rows(const void* src, void* dst, int B, int T, long long row_bytes, cudaStream_t st) {
  if (row_bytes % 16 != 0) return -2;
  const int vec = (int)(row_bytes / 16);
  const long long total = (long long)B * T * vec;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  transpose01_rows_kernel<<<blocks, 256, 0, st>>>((const uint4*)src, (uint4*)dst, B, T, vec);
  return (int)cudaGetLastError();
}


// [R,C] -> [C,R] for 2-byte elements through a padded 64x64 shared-memory tile (coalesced 128 B rows both ways).  The
// backward recurrence wants W_h^T (and the input-gradient GEMM W_x^T) K-major; the weights change every step, so this runs
// three times per training step: ~5 us each instead of ~21 us for the framework's generic strided copy.
namespace {
__global__ void transpose2d_b16_kernel(const unsigned short* __restrict__ src, unsigned short* __restrict__ dst, int R, int C) {
  __shared__ unsigned short tile[64][66];
  const int c0 = blockIdx.x * 64, r0 = blockIdx.y * 64;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 256 threads: 32 x 8
  for (int i = ty; i < 64; i += 8) {
    const int r = r0 + i;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int c = c0 + tx + 32 * k;
      if (r < R && c < C) tile[i][tx + 32 * k] = src[(size_t)r * C + c];
    }
  }
  __syncthreads();
  for (int i = ty; i < 64; i += 8) {
    const int c = c0 + i;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int r = r0 + tx + 32 * k;
      if (r < R && c < C) dst[(size_t)c * R + r] = tile[tx + 32 * k][i];
    }
  }
}
}  // namespace

extern "C" int ts_transpose2d_b16(const void* src, void* dst, int R, int C, cudaStream_t st) {
  dim3 grid((C + 63) / 64, (R + 63) / 64);
  transpose2d_b16_kernel<<<grid, 256, 0, st>>>((const unsigned short*)src, (unsigned short*)dst, R, C);
  return (int)cudaGetLastError();
}


// Column sums of a bf16 [rows, cols] matrix into fp32 (bias gradient = sum over T*B of the gate gradients): 16 B loads,
// 8 fp32 accumulators per thread, warps stride over rows, one shared-memory reduction and one atomicAdd per column per block.
// cols % 256 == 0.  Deterministic: every row slab writes its partial sums to a scratch row, the LAST slab to finish (ticket
// counter per column block) adds the slabs in fixed order and accumulates the result into out (beta = 1).
// The work is a grid of nx = cols / 256 column blocks x ny row slabs; a launch with fewer CTAs than that walks it in a
// grid-stride loop (same slabs, same order of additions: the result does not depend on the CTA count).
namespace {
__global__ void colsum_bf16_kernel(const uint4* __restrict__ src, float* __restrict__ out, float* __restrict__ partial,
                                   unsigned int* __restrict__ tickets, int rows, int cols, int rows_per_block, int accumulate, int pdl,
                                   int pitch_cols, int nx, int ny) {
  __shared__ float red[8][256];
  __shared__ unsigned int ticket_s;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int vec_per_row = pitch_cols / 8;                      // (src / out already point at the first column of this launch)
  for (int vb = blockIdx.x; vb < nx * ny; vb += gridDim.x) {
    const int bx = vb % nx, by = vb / nx;
    const int cv = bx * 32 + lane;                             // 16 B column-vector index (8 columns)
    const int r_begin = by * rows_per_block;
    const int r_end = min(rows, r_begin + rows_per_block);
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int r = r_begin + warp; r < r_end; r += 8) {
      const uint4 v = src[(size_t)r * vec_per_row + cv];
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        acc[2 * i] += __uint_as_float(w[i] << 16);
        acc[2 * i + 1] += __uint_as_float(w[i] & 0xffff0000u);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) red[warp][lane * 8 + i] = acc[i];
    __syncthreads();
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    const int col = bx * 256 + threadIdx.x;
    if (ny == 1) {
      out[col] = accumulate ? out[col] + s : s;
    } else {
      partial[(size_t)by * cols + col] = s;
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) ticket_s = atomicAdd(tickets + bx, 1u);
      __syncthreads();
      if (ticket_s == (unsigned int)ny - 1) {
        __threadfence();
        float t = 0.f;
        for (int y = 0; y < ny; ++y) t += __ldcg(partial + (size_t)y * cols + col);     // fixed order
        out[col] = accumulate ? out[col] + t : t;
        if (threadIdx.x == 0) tickets[bx] = 0u;                  // ready for the next launch
      }
    }
    __syncthreads();                                             // red / ticket_s are reused by the next work item
  }
  // launched as a programmatic dependent of a weight-gradient GEMM (it runs on the SMs that GEMM leaves idle and reads the same
  // dG): do not let anything behind us start before that GEMM has completed
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
}
}  // namespace

// scratch: u32 [kColsumTickets] tickets at a FIXED place (zero before first use; the kernel leaves them zero - partial sums of
// another shape must never alias them) followed by fp32 [slabs * cols] partials
constexpr int kColsumTickets = 4096;
extern "C" long long ts_colsum_scratch_bytes(int rows, int cols) {
  const int rows_per_block = 512;
  const long long slabs = (rows + rows_per_block - 1) / rows_per_block;
  return (long long)kColsumTickets * 4 + slabs * cols * 4;
}

// cols = columns summed by this launch (a 256-aligned sub-range of a matrix with row pitch pitch_cols; src / out point at its first column)
// max_ctas > 0 caps the grid: a programmatic dependent that runs next to kernels holding most SMs then gets all of its CTAs
// resident on the SMs left to it (a CTA that has finished waits for the previous kernel before it exits, so CTAs that do not
// fit would only start once that kernel is complete).
extern "C" int ts_colsum_bf16(const void* src, float* out, void* scratch, int rows, int cols, int pitch_cols, int accumulate, int pdl,
                              int max_ctas, cudaStream_t st) {
  if (cols % 256 != 0 || cols / 256 > kColsumTickets) return -2;
  const int rows_per_block = 512;
  const int nx = cols / 256, ny = (rows + rows_per_block - 1) / rows_per_block;
  int grid = nx * ny;
  if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
  unsigned int* tickets = (unsigned int*)scratch;
  float* partial = (float*)((char*)scratch + (size_t)kColsumTickets * 4);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
  return (int)cudaLaunchKernelEx(&cfg, colsum_bf16_kernel, (const uint4*)src, out, partial, tickets, rows, cols, rows_per_block, accumulate, pdl,
                                 pitch_cols, nx, ny);
}
