// K-HEAD on the tensor cores: dense head + bias + sparse softmax cross-entropy + accuracy + dlogits in ONE launch, and the
// whole head backward (dh, dW, db) in ONE launch.
//
// Forward replaces reshape -> matmul(dense, weights) + bias -> sparse softmax cross-entropy -> reduce_mean ->
// argmax / equal / cast / reduce_mean of the original TensorFlow graph:
//   * one CTA per 128 batch rows; h [B, H] (bf16) streams through a 4-stage TMA -> mbarrier ring (128 B swizzle);
//   * the weights [H, C] (fp32 master) are converted to bf16 and laid out ONCE per CTA as the K-major 128B-swizzled wgmma
//     operand image [k-block][C padded to NP rows][64] directly in shared memory (C is tiny: no tensor map, no padded copy);
//   * two consumer warpgroups (64 rows each) issue wgmma m64nNPk16, the logits accumulate in registers;
//   * epilogue straight from the accumulator fragments: a lane quad holds two rows' logits, + bias, max / argmax,
//     log-sum-exp, NLL, dlogits = (softmax - onehot) / B reduced over the quad; loss sum and correct count via one atomic
//     per warp.
// Backward replaces the autodiff of the same ops: dh = dlogits·W^T, dW = h^T·dlogits, db = sum_b dlogits in one CUDA-core
// kernel (K = C <= 32 is far below a tensor-core tile; the work is 2·B·H·C FMAs, bandwidth-trivial).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "hopper.cuh"
#include "tmap.h"
#include "ts_common.cuh"

namespace {

constexpr int HM = 128;      // rows per CTA
constexpr int HK = 64;       // k-block
constexpr int kHStages = 4;
constexpr int kHThreads = 384;      // warp 0 producer, warps 1..3 idle, warps 4..11 two consumer warpgroups
constexpr int kHBwdJ = 32;          // backward: hidden columns per block (x 4 row groups = 128 threads)

struct HeadParams {
  const float* W;            // [H, C] fp32
  const float* bias;         // [C]
  const long long* labels;   // [B]
  float* logits;             // [B, C]
  float* dlogits;            // [B, C]
  float* loss_sum;           // [1]
  int* correct;              // [1]
  int B, H, C;
};

template <int NP>
__global__ void __launch_bounds__(kHThreads, 1)
head_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmap_h, const HeadParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int num_kb = (p.H + HK - 1) / HK;
  constexpr int wblk = NP * 128;                                  // bytes of one weight k-block image [NP rows][64 bf16]
  uint8_t* smem_w = smem;                                         // num_kb * wblk (wblk is a multiple of 2048: 1024-aligned blocks)
  uint8_t* smem_a = smem + (size_t)num_kb * wblk;                 // kHStages x 16 KB
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_a + kHStages * (HM * HK * 2));
  uint64_t* full = bars;
  uint64_t* empty = bars + kHStages;
  float* bias_s = reinterpret_cast<float*>(empty + kHStages);     // [NP]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * HM;

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&tmap_h);
    for (int s = 0; s < kHStages; ++s) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], 8); }
    tc::fence_barrier_init();
  }
  // the first pass over the ring needs no empty-barrier wait: start streaming h while the weight image is being built
  const int pre_kb = num_kb < kHStages ? num_kb : kHStages;
  if (threadIdx.x == 0) {
    for (int kb = 0; kb < pre_kb; ++kb) {
      tc::mbar_expect_tx(&full[kb], HM * HK * 2);
      tc::tma_load_2d(smem_a + kb * (HM * HK * 2), &tmap_h, &full[kb], kb * HK, m0);
    }
  }
  for (int c = threadIdx.x; c < NP; c += kHThreads) bias_s[c] = c < p.C ? p.bias[c] : 0.f;
  // weight image: element (n = class, k) -> block k/64, row n, 16 B chunk ((k%64)/8) ^ (n&7), 2 B slot k%8.  First zero the
  // image (padding rows C..NP and a ragged last k-block), then walk W [H, C] linearly: coalesced fp32 reads, one bf16 store each.
  {
    const int img16 = (num_kb * wblk) >> 4;
    for (int i = threadIdx.x; i < img16; i += kHThreads) reinterpret_cast<uint4*>(smem_w)[i] = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();
    const int total = p.H * p.C;
    constexpr int kWU = 8;                                         // loads in flight per thread: the walk is pure L2 latency otherwise
    for (int i0 = threadIdx.x; i0 < total; i0 += kHThreads * kWU) {
      float w[kWU];
#pragma unroll
      for (int u = 0; u < kWU; ++u) { const int i = i0 + u * kHThreads; w[u] = i < total ? __ldg(p.W + i) : 0.f; }
#pragma unroll
      for (int u = 0; u < kWU; ++u) {
        const int i = i0 + u * kHThreads;
        if (i < total) {
          const int k = i / p.C, n = i - k * p.C;
          const int kb = k / HK, kk = k % HK;
          const uint32_t off = (uint32_t)kb * wblk + (uint32_t)n * 128 + (uint32_t)((((kk >> 3) ^ (n & 7)) << 4) + ((kk & 7) << 1));
          *reinterpret_cast<__nv_bfloat16*>(smem_w + off) = __float2bfloat16_rn(w[u]);
        }
      }
    }
  }
  tc::fence_proxy_async();                       // generic-proxy smem writes -> visible to the tensor core (async proxy)
  __syncthreads();

  if (warp == 0) {
    uint32_t stage = pre_kb == kHStages ? 0 : pre_kb, phase = pre_kb == kHStages ? 1 : 0;
    for (int kb = pre_kb; kb < num_kb; ++kb) {
      while (!tc::mbar_try_wait(&empty[stage], phase ^ 1)) {}
      if (tc::elect_one()) {
        tc::mbar_expect_tx(&full[stage], HM * HK * 2);
        tc::tma_load_2d(smem_a + stage * (HM * HK * 2), &tmap_h, &full[stage], kb * HK, m0);
      }
      __syncwarp();
      if (++stage == kHStages) { stage = 0; phase ^= 1; }
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2, wq = warp & 3;
    const uint64_t da0 = tc::desc_kmajor_sw128(tc::smem_u32(smem_a) + wg * 8192);
    const uint64_t dw0 = tc::desc_kmajor_sw128(tc::smem_u32(smem_w));
    float acc[NP / 2];
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) acc[i] = 0.f;
    uint32_t stage = 0, phase = 0, prev = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      while (!tc::mbar_try_wait(&full[stage], phase)) {}
      const uint64_t da = da0 + (uint64_t)(stage * ((HM * HK * 2) >> 4));
      const uint64_t dw = dw0 + (uint64_t)((uint32_t)kb * (uint32_t)(wblk >> 4));
      tc::fence_regs(acc);
      tc::wgmma_fence();
#pragma unroll
      for (int k = 0; k < HK / 16; ++k) tc::Wgmma<NP, 0, 0>::mma(acc, da + 2 * k, dw + 2 * k, (kb > 0 || k > 0) ? 1u : 0u);
      tc::wgmma_commit();
      tc::fence_regs(acc);
      if (kb > 0) { tc::wgmma_wait<1>(); if (lane == 0) tc::mbar_arrive(&empty[prev]); }
      prev = stage;
      if (++stage == kHStages) { stage = 0; phase ^= 1; }
    }
    tc::wgmma_wait<0>();
    tc::fence_regs(acc);
    // epilogue: this lane holds rows r (h = 0) and r + 8 (h = 1), NP / 4 columns of each; its quad (lanes 4q..4q+3) the rest
    const float invB = 1.0f / (float)p.B;
    float nll_sum = 0.f;
    int ok_sum = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m0 + 64 * wg + tc::acc_row(2 * h, wq, lane);
      const bool valid = row < p.B;
      const int y = valid ? (int)p.labels[row] : -1;
      float mx = -INFINITY, ly = 0.f;
      int arg = 0x7fffffff;
#pragma unroll
      for (int i = 2 * h; i < NP / 2; i += 4) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = tc::acc_col(i + e, lane);
          if (c < p.C) {
            const float l = acc[i + e] + bias_s[c];
            acc[i + e] = l;
            if (valid) p.logits[(size_t)row * p.C + c] = l;
            if (l > mx || (l == mx && c < arg)) { mx = l; arg = c; }
            if (c == y) ly = l;
          }
        }
      }
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {                 // quad: the larger logit, the smaller class index on ties
        const float m2 = __shfl_xor_sync(0xffffffffu, mx, o);
        const int a2 = __shfl_xor_sync(0xffffffffu, arg, o);
        if (m2 > mx || (m2 == mx && a2 < arg)) { mx = m2; arg = a2; }
        ly += __shfl_xor_sync(0xffffffffu, ly, o);
      }
      float se = 0.f;
#pragma unroll
      for (int i = 2 * h; i < NP / 2; i += 4)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (tc::acc_col(i + e, lane) < p.C) se += __expf(acc[i + e] - mx);
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
      const float lse = mx + __logf(se);
      if (valid) {
#pragma unroll
        for (int i = 2 * h; i < NP / 2; i += 4)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = tc::acc_col(i + e, lane);
            if (c < p.C) p.dlogits[(size_t)row * p.C + c] = (__expf(acc[i + e] - lse) - (c == y ? 1.f : 0.f)) * invB;
          }
      }
      if ((lane & 3) == 0 && valid) { nll_sum += lse - ly; ok_sum += arg == y ? 1 : 0; }
    }
    nll_sum = ts::warp_sum(nll_sum);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ok_sum += __shfl_xor_sync(0xffffffffu, ok_sum, o);
    if (lane == 0) { atomicAdd(p.loss_sum, nll_sum); if (ok_sum) atomicAdd(p.correct, ok_sum); }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// backward: block (jb, bb) = 32 hidden columns x a slab of batch rows, 4 row groups per column.  A thread keeps W[j, 0:C) and
// its dW[j, 0:C) partial in registers; per batch row: dh[b, j] = sum_c d[b,c] W[j,c] (written once), dW[j,c] += h[b,j] d[b,c].
// The dlogits slab sits in shared memory (broadcast reads).  One slab (the common case) is deterministic: no atomics.
// ---------------------------------------------------------------------------------------------------------------------
template <typename T, int CP, typename TDH>
__global__ void __launch_bounds__(128) head_bwd_kernel(const T* __restrict__ h, const float* __restrict__ W, const float* __restrict__ dlogits,
                                                       const float* __restrict__ dloss, TDH* __restrict__ dh, float* __restrict__ dW,
                                                       float* __restrict__ db, int B, int H, int C, int rows_per_block, int accumulate) {
  // thread = (hidden column j, row group q of 4): lanes 0..31 of a warp = 32 consecutive j (coalesced h / dh accesses), warp = q.
  // Row b of the slab is handled by group b % 4; the four partial dW rows are added in fixed order through shared memory.
  extern __shared__ float ds[];                         // [rows_per_block][CP] dlogits slab, then [4][kHBwdJ][CP] partials
  float* part = ds + (size_t)rows_per_block * CP;
  const int jl = threadIdx.x & 31, q = threadIdx.x >> 5;
  const int j = blockIdx.x * kHBwdJ + jl;
  const int b0 = blockIdx.y * rows_per_block;
  const int nb = min(rows_per_block, B - b0);
  const float scale = dloss ? *dloss : 1.f;
  {
    constexpr int kLU = 8;                              // slab loads in flight per thread
    for (int i0 = threadIdx.x; i0 < nb * CP; i0 += 128 * kLU) {
      float v[kLU];
#pragma unroll
      for (int u = 0; u < kLU; ++u) {
        const int i = i0 + u * 128, b = i / CP, c = i % CP;
        v[u] = (i < nb * CP && c < C) ? __ldg(dlogits + (size_t)(b0 + b) * C + c) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < kLU; ++u) { const int i = i0 + u * 128; if (i < nb * CP) ds[i] = v[u] * scale; }
    }
  }
  __syncthreads();
  float w[CP], acc[CP];
#pragma unroll
  for (int c = 0; c < CP; ++c) { w[c] = (j < H && c < C) ? W[(size_t)j * C + c] : 0.f; acc[c] = 0.f; }
  if (j < H) {
    constexpr int kU = 8;                                // h loads in flight per thread (the loop is L2-latency bound otherwise)
    for (int bb = q; bb < nb; bb += 4 * kU) {
      T hraw[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) { const int b = bb + 4 * u; hraw[u] = h[(size_t)(b0 + (b < nb ? b : bb)) * H + j]; }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int b = bb + 4 * u;
        if (b < nb) {
          const float hv = ts::Cvt<T>::to_f(hraw[u]);
          const float* d = ds + b * CP;
          float s = 0.f;
#pragma unroll
          for (int c = 0; c < CP; ++c) { s = fmaf(d[c], w[c], s); acc[c] = fmaf(hv, d[c], acc[c]); }
          dh[(size_t)(b0 + b) * H + j] = ts::Cvt<TDH>::from_f(s);
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < CP; ++c) part[(q * kHBwdJ + jl) * CP + c] = acc[c];
  __syncthreads();
  const bool atomic = gridDim.y > 1 || accumulate;
  for (int i = threadIdx.x; i < kHBwdJ * CP; i += 128) {            // fixed-order sum of the four row groups
    const int jj = i / CP, c = i % CP;
    const int jg = blockIdx.x * kHBwdJ + jj;
    if (jg < H && c < C) {
      const float t = ((part[(0 * kHBwdJ + jj) * CP + c] + part[(1 * kHBwdJ + jj) * CP + c]) + part[(2 * kHBwdJ + jj) * CP + c]) +
                      part[(3 * kHBwdJ + jj) * CP + c];
      if (atomic) atomicAdd(dW + (size_t)jg * C + c, t); else dW[(size_t)jg * C + c] = t;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < C) {
    float s = 0.f;
    for (int b = 0; b < nb; ++b) s += ds[b * CP + threadIdx.x];
    if (atomic) atomicAdd(db + threadIdx.x, s); else db[threadIdx.x] = s;
  }
}

// any C (classes beyond the register-resident path): plain per-output kernels
template <typename T, typename TDH>
__global__ void head_bwd_dh_generic(const float* __restrict__ W, const float* __restrict__ dlogits, const float* __restrict__ dloss,
                                    TDH* __restrict__ dh, int B, int H, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * H) return;
  const int b = (int)(i / H), j = (int)(i % H);
  const float scale = dloss ? *dloss : 1.f;
  float s = 0.f;
  for (int c = 0; c < C; ++c) s = fmaf(dlogits[(size_t)b * C + c], W[(size_t)j * C + c], s);
  dh[i] = ts::Cvt<TDH>::from_f(s * scale);
}
template <typename T>
__global__ void head_bwd_dw_generic(const T* __restrict__ h, const float* __restrict__ dlogits, const float* __restrict__ dloss,
                                    float* __restrict__ dW, float* __restrict__ db, int B, int H, int C, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const float scale = dloss ? *dloss : 1.f;
  if (i < (long long)H * C) {
    const int j = (int)(i / C), c = (int)(i % C);
    float s = 0.f;
    for (int b = 0; b < B; ++b) s = fmaf(ts::Cvt<T>::to_f(h[(size_t)b * H + j]), dlogits[(size_t)b * C + c], s);
    dW[i] = (accumulate ? dW[i] : 0.f) + s * scale;
  } else if (i < (long long)H * C + C) {
    const int c = (int)(i - (long long)H * C);
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += dlogits[(size_t)b * C + c];
    db[c] = (accumulate ? db[c] : 0.f) + s * scale;
  }
}
// logits for heads the tensor-core kernel does not take (fp32 activations, very wide heads): one thread per output
template <typename T>
__global__ void head_logits_generic(const T* __restrict__ h, const float* __restrict__ W, const float* __restrict__ bias,
                                    float* __restrict__ logits, int B, int H, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * C) return;
  const int b = (int)(i / C), c = (int)(i % C);
  float s = bias[c];
  for (int k = 0; k < H; ++k) s = fmaf(ts::Cvt<T>::to_f(h[(size_t)b * H + k]), W[(size_t)k * C + c], s);
  logits[i] = s;
}

template <typename T, typename TDH>
int launch_bwd(const void* h, const float* W, const float* dlogits, const float* dloss, void* dh, float* dW, float* db, int B, int H, int C,
               int accumulate, cudaStream_t st) {
  if (C > 32) {
    const long long n1 = (long long)B * H, n2 = (long long)H * C + C;
    head_bwd_dh_generic<T, TDH><<<(unsigned)((n1 + 255) / 256), 256, 0, st>>>(W, dlogits, dloss, (TDH*)dh, B, H, C);
    head_bwd_dw_generic<T><<<(unsigned)((n2 + 255) / 256), 256, 0, st>>>((const T*)h, dlogits, dloss, dW, db, B, H, C, accumulate);
    return (int)cudaGetLastError();
  }
  // one slab (no atomics: deterministic) while the dlogits slab fits in shared memory, 32-row slabs + fp32 atomics beyond
  const int cp = C <= 8 ? 8 : (C <= 16 ? 16 : 32);
  const int rows = (size_t)(B + 4 * kHBwdJ) * cp * sizeof(float) <= 48 * 1024 ? B : 32;
  dim3 grid((H + kHBwdJ - 1) / kHBwdJ, (B + rows - 1) / rows);
  if (grid.y > 1 && !accumulate) {
    cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)H * C, st);
    cudaMemsetAsync(db, 0, sizeof(float) * (size_t)C, st);
  }
#define HEAD_BWD(CP) head_bwd_kernel<T, CP, TDH><<<grid, 128, (rows + 4 * kHBwdJ) * CP * sizeof(float), st>>>((const T*)h, W, dlogits, dloss, (TDH*)dh, dW, db, B, H, C, rows, accumulate)
  if (C <= 8) HEAD_BWD(8); else if (C <= 16) HEAD_BWD(16); else HEAD_BWD(32);
#undef HEAD_BWD
  return (int)cudaGetLastError();
}

}  // namespace

extern "C" int ts_head_fwd_tc_smem(int H, int C) {
  int NP = 16;
  while (NP < C) NP <<= 1;
  const int num_kb = (H + HK - 1) / HK;
  return num_kb * NP * 128 + kHStages * HM * HK * 2 + 1024 + 128 + NP * 4;
}

template <int NP>
int launch_head_fwd(const CUtensorMap& th, const HeadParams& p, int smem, cudaStream_t st) {
  cudaError_t e = cudaFuncSetAttribute(head_fwd_tc_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  head_fwd_tc_kernel<NP><<<(p.B + HM - 1) / HM, kHThreads, smem, st>>>(th, p);
  return (int)cudaGetLastError();
}

// h: bf16 [B, H] with row pitch ldh (elements).  Returns -1 when the shape does not fit this kernel (caller falls back).
extern "C" int ts_head_fwd_tc(const void* h, int ldh, const float* W, const float* bias, const long long* labels, float* logits,
                              float* dlogits, float* loss_sum, int* correct, int B, int H, int C, cudaStream_t st) {
  const int smem = ts_head_fwd_tc_smem(H, C);
  if (C > 256 || smem > 200 * 1024 || H % 8 != 0 || ldh % 8 != 0) return -1;
  CUtensorMap th;
  if (int rc = ts::make_tmap_2d_bf16(&th, h, (uint64_t)B, (uint64_t)H, (uint64_t)ldh, HK, HM)) return rc;
  HeadParams p{W, bias, labels, logits, dlogits, loss_sum, correct, B, H, C};
  if (C <= 16) return launch_head_fwd<16>(th, p, smem, st);
  if (C <= 32) return launch_head_fwd<32>(th, p, smem, st);
  if (C <= 64) return launch_head_fwd<64>(th, p, smem, st);
  if (C <= 128) return launch_head_fwd<128>(th, p, smem, st);
  return launch_head_fwd<256>(th, p, smem, st);
}

extern "C" int ts_head_logits_generic(const void* h, const float* W, const float* bias, float* logits, int B, int H, int C, int is_bf16,
                                      cudaStream_t st) {
  const long long n = (long long)B * C;
  if (is_bf16) head_logits_generic<__nv_bfloat16><<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const __nv_bfloat16*)h, W, bias, logits, B, H, C);
  else head_logits_generic<float><<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const float*)h, W, bias, logits, B, H, C);
  return (int)cudaGetLastError();
}

// dh dtype follows h (bf16 -> bf16, fp32 -> fp32); dW [H, C] / db [C] fp32, accumulate = add into them.
extern "C" int ts_head_bwd(const void* h, const float* W, const float* dlogits, const float* dloss, void* dh, float* dW, float* db,
                           int B, int H, int C, int is_bf16, int accumulate, cudaStream_t st) {
  if (is_bf16) return launch_bwd<__nv_bfloat16, __nv_bfloat16>(h, W, dlogits, dloss, dh, dW, db, B, H, C, accumulate, st);
  return launch_bwd<float, float>(h, W, dlogits, dloss, dh, dW, db, B, H, C, accumulate, st);
}
