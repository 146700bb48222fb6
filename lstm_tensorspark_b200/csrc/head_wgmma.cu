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
// The per-step head (sequence labelling, below the last-state kernels) runs the same head at every time step of h_seq.
#include <algorithm>

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
// db of a dlogits slab ds [nb][CP] in shared memory: its column sums as a pairwise tree over the rows, in place (ds is not read
// again) -> ds[c].  A single fp32 chain over up to 1024 rows was 3.5x the fp32 budget of a db that cancels
// (tests/test_gpu_head_edges.py::test_per_step_row_edges, the fp32 case of 1023 rows); the tree's error grows with log2(rows).
// Called by every thread of the block.
template <int CP>
__device__ __forceinline__ void slab_colsum_tree(float* ds, int nb) {
  for (int w = 1; w < nb; w <<= 1) {
    const int pairs = (nb + 2 * w - 1) / (2 * w);
    for (int i = threadIdx.x; i < pairs * CP; i += blockDim.x) {
      const int b = (i / CP) * 2 * w, c = i % CP;
      if (b + w < nb) ds[b * CP + c] += ds[(b + w) * CP + c];
    }
    __syncthreads();
  }
}

template <typename T, int CP, typename TDH>
__global__ void __launch_bounds__(128) head_bwd_kernel(const T* __restrict__ h, const float* __restrict__ W, const float* __restrict__ dlogits,
                                                       const float* __restrict__ dloss, TDH* __restrict__ dh, float* __restrict__ dW,
                                                       float* __restrict__ db, int B, int H, int C, int rows_per_block, int acc_w,
                                                       int acc_b) {
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
  const bool atomic_w = gridDim.y > 1 || acc_w, atomic_b = gridDim.y > 1 || acc_b;
  for (int i = threadIdx.x; i < kHBwdJ * CP; i += 128) {            // fixed-order sum of the four row groups
    const int jj = i / CP, c = i % CP;
    const int jg = blockIdx.x * kHBwdJ + jj;
    if (jg < H && c < C) {
      const float t = ((part[(0 * kHBwdJ + jj) * CP + c] + part[(1 * kHBwdJ + jj) * CP + c]) + part[(2 * kHBwdJ + jj) * CP + c]) +
                      part[(3 * kHBwdJ + jj) * CP + c];
      if (atomic_w) atomicAdd(dW + (size_t)jg * C + c, t); else dW[(size_t)jg * C + c] = t;
    }
  }
  if (blockIdx.x == 0) {                                            // (uniform in the block: the tree synchronises it)
    slab_colsum_tree<CP>(ds, nb);
    if (threadIdx.x < C) {
      const float s = ds[threadIdx.x];
      if (atomic_b) atomicAdd(db + threadIdx.x, s); else db[threadIdx.x] = s;
    }
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
                                    float* __restrict__ dW, float* __restrict__ db, int B, int H, int C, int acc_w, int acc_b) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const float scale = dloss ? *dloss : 1.f;
  if (i < (long long)H * C) {
    const int j = (int)(i / C), c = (int)(i % C);
    float s = 0.f;
    for (int b = 0; b < B; ++b) s = fmaf(ts::Cvt<T>::to_f(h[(size_t)b * H + j]), dlogits[(size_t)b * C + c], s);
    dW[i] = (acc_w ? dW[i] : 0.f) + s * scale;
  } else if (i < (long long)H * C + C) {
    const int c = (int)(i - (long long)H * C);
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += dlogits[(size_t)b * C + c];
    db[c] = (acc_b ? db[c] : 0.f) + s * scale;
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
               int acc_w, int acc_b, cudaStream_t st) {
  if (C > 32) {
    const long long n1 = (long long)B * H, n2 = (long long)H * C + C;
    head_bwd_dh_generic<T, TDH><<<(unsigned)((n1 + 255) / 256), 256, 0, st>>>(W, dlogits, dloss, (TDH*)dh, B, H, C);
    head_bwd_dw_generic<T><<<(unsigned)((n2 + 255) / 256), 256, 0, st>>>((const T*)h, dlogits, dloss, dW, db, B, H, C, acc_w, acc_b);
    return (int)cudaGetLastError();
  }
  // one slab (no atomics: deterministic) while the dlogits slab fits in shared memory, 32-row slabs + fp32 atomics beyond
  const int cp = C <= 8 ? 8 : (C <= 16 ? 16 : 32);
  const int rows = (size_t)(B + 4 * kHBwdJ) * cp * sizeof(float) <= 48 * 1024 ? B : 32;
  dim3 grid((H + kHBwdJ - 1) / kHBwdJ, (B + rows - 1) / rows);
  if (grid.y > 1 && !acc_w) cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)H * C, st);
  if (grid.y > 1 && !acc_b) cudaMemsetAsync(db, 0, sizeof(float) * (size_t)C, st);
#define HEAD_BWD(CP) head_bwd_kernel<T, CP, TDH><<<grid, 128, (rows + 4 * kHBwdJ) * CP * sizeof(float), st>>>((const T*)h, W, dlogits, dloss, (TDH*)dh, dW, db, B, H, C, rows, acc_w, acc_b)
  if (C <= 8) HEAD_BWD(8); else if (C <= 16) HEAD_BWD(16); else HEAD_BWD(32);
#undef HEAD_BWD
  return (int)cudaGetLastError();
}

// =====================================================================================================================
// Per-step head (sequence labelling): the same head at every time step of the top layer's output h_seq [T, B, H], read in
// place as R = T·B time-major rows r = t·B + b.  Row r counts iff t < lengths[b] (every row without lengths); N = the number
// of counted rows.  Logits go to [B, T, C] (batch-major, like the labels), dlogits to row order r: (softmax - onehot) / N at
// counted rows, 0 elsewhere, so the backward needs no mask.  Loss, correct count and N, and in the backward dW and db, are
// reduced in a fixed order (per-CTA partials in scratch, summed by the last CTA through a ticket): two calls on the same
// inputs give the same bits.
// =====================================================================================================================
struct HeadStepParams {
  const float* W;            // [H, C] fp32
  const float* bias;         // [C]
  const long long* labels;   // [B, T]
  const int* lengths;        // [B] or null
  float* logits;             // [B, T, C]
  float* dlogits;            // [R, C]
  float* part_loss;          // [gridDim.x] scratch
  int* part_ok;              // [gridDim.x] scratch
  unsigned int* ticket;      // [1]: 0 on entry, left 0
  float* loss;               // [1] mean NLL over counted rows
  int* correct;              // [1]
  int* count;                // [1] N
  int T, B, H, C, R, num_tiles;
};

// N = sum of lengths (T·B without): every CTA sums the B ints itself (exact, so the order does not matter)
__device__ __forceinline__ int step_count_rows(const int* lengths, int T, int B, int* n_s) {
  if (lengths == nullptr) return T * B;
  if (threadIdx.x == 0) *n_s = 0;
  __syncthreads();
  int s = 0;
  for (int b = threadIdx.x; b < B; b += blockDim.x) s += lengths[b];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(n_s, s);
  __syncthreads();
  return *n_s;
}

// Called by every thread of the CTA after this CTA's partial is in part_loss / part_ok[blockIdx.x]: the last CTA to arrive
// sums all partials in index order and writes the results.
__device__ __forceinline__ void step_finish(const HeadStepParams& p, int N, int* last_s) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) *last_s = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (*last_s && threadIdx.x == 0) {
    __threadfence();
    const volatile float* pl = p.part_loss;
    const volatile int* po = p.part_ok;
    float s = 0.f;
    int ok = 0;
    for (int i = 0; i < (int)gridDim.x; ++i) { s += pl[i]; ok += po[i]; }
    *p.loss = s / (float)N;
    *p.correct = ok;
    *p.count = N;
    *p.ticket = 0u;
  }
}

// Forward on the tensor cores: a persistent grid, each CTA builds the bf16 weight image once and streams its row tiles
// (blockIdx.x, + gridDim.x, ...) through one TMA ring; the epilogue of a tile overlaps the loads of the next one.
template <int NP>
__global__ void __launch_bounds__(kHThreads, 1)
head_step_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmap_h, const HeadStepParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int num_kb = (p.H + HK - 1) / HK;
  constexpr int wblk = NP * 128;
  uint8_t* smem_w = smem;
  uint8_t* smem_a = smem + (size_t)num_kb * wblk;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_a + kHStages * (HM * HK * 2));
  uint64_t* full = bars;
  uint64_t* empty = bars + kHStages;
  float* bias_s = reinterpret_cast<float*>(empty + kHStages);     // [NP]
  float* red_f = bias_s + NP;                                     // [8] per consumer warp
  int* red_i = reinterpret_cast<int*>(red_f + 8);                 // [8]
  int* misc = red_i + 8;                                          // [0] N, [1] last-CTA flag

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int my_tiles = blockIdx.x < p.num_tiles ? (p.num_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
  const int total = my_tiles * num_kb;                            // ring items (tile, k-block) of this CTA, in order

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&tmap_h);
    for (int s = 0; s < kHStages; ++s) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], 8); }
    tc::fence_barrier_init();
  }
  const int pre = total < kHStages ? total : kHStages;
  if (threadIdx.x == 0) {
    for (int i = 0; i < pre; ++i) {
      tc::mbar_expect_tx(&full[i], HM * HK * 2);
      tc::tma_load_2d(smem_a + i * (HM * HK * 2), &tmap_h, &full[i], (i % num_kb) * HK, (blockIdx.x + (i / num_kb) * gridDim.x) * HM);
    }
  }
  for (int c = threadIdx.x; c < NP; c += kHThreads) bias_s[c] = c < p.C ? p.bias[c] : 0.f;
  {
    const int img16 = (num_kb * wblk) >> 4;
    for (int i = threadIdx.x; i < img16; i += kHThreads) reinterpret_cast<uint4*>(smem_w)[i] = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();
    const int hc = p.H * p.C;
    constexpr int kWU = 8;
    for (int i0 = threadIdx.x; i0 < hc; i0 += kHThreads * kWU) {
      float w[kWU];
#pragma unroll
      for (int u = 0; u < kWU; ++u) { const int i = i0 + u * kHThreads; w[u] = i < hc ? __ldg(p.W + i) : 0.f; }
#pragma unroll
      for (int u = 0; u < kWU; ++u) {
        const int i = i0 + u * kHThreads;
        if (i < hc) {
          const int k = i / p.C, n = i - k * p.C;
          const int kb = k / HK, kk = k % HK;
          const uint32_t off = (uint32_t)kb * wblk + (uint32_t)n * 128 + (uint32_t)((((kk >> 3) ^ (n & 7)) << 4) + ((kk & 7) << 1));
          *reinterpret_cast<__nv_bfloat16*>(smem_w + off) = __float2bfloat16_rn(w[u]);
        }
      }
    }
  }
  tc::fence_proxy_async();
  __syncthreads();
  const int N = step_count_rows(p.lengths, p.T, p.B, misc);
  const float invN = 1.0f / (float)N;

  if (warp == 0) {
    for (int i = pre; i < total; ++i) {
      const uint32_t stage = i % kHStages, phase = (i / kHStages) & 1;
      while (!tc::mbar_try_wait(&empty[stage], phase ^ 1)) {}
      if (tc::elect_one()) {
        tc::mbar_expect_tx(&full[stage], HM * HK * 2);
        tc::tma_load_2d(smem_a + stage * (HM * HK * 2), &tmap_h, &full[stage], (i % num_kb) * HK,
                        (blockIdx.x + (i / num_kb) * gridDim.x) * HM);
      }
      __syncwarp();
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2, wq = warp & 3;
    const uint64_t da0 = tc::desc_kmajor_sw128(tc::smem_u32(smem_a) + wg * 8192);
    const uint64_t dw0 = tc::desc_kmajor_sw128(tc::smem_u32(smem_w));
    float acc[NP / 2];
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) acc[i] = 0.f;
    float nll_sum = 0.f;
    int ok_sum = 0, it = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      uint32_t prev = 0;
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const uint32_t stage = it % kHStages, phase = (it / kHStages) & 1;
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
      }
      tc::wgmma_wait<0>();
      tc::fence_regs(acc);
      if (lane == 0) tc::mbar_arrive(&empty[prev]);              // the ring moves on to the next tile during this epilogue
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = tile * HM + 64 * wg + tc::acc_row(2 * h, wq, lane);
        const bool valid = row < p.R;
        const int t = row / p.B, b = row - t * p.B;
        const bool counted = valid && (p.lengths == nullptr || t < p.lengths[b]);
        const int y = counted ? (int)p.labels[(size_t)b * p.T + t] : -1;
        float* lrow = p.logits + ((size_t)b * p.T + t) * p.C;
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
              if (valid) lrow[c] = l;
              if (l > mx || (l == mx && c < arg)) { mx = l; arg = c; }
              if (c == y) ly = l;
            }
          }
        }
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
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
          float* drow = p.dlogits + (size_t)row * p.C;
#pragma unroll
          for (int i = 2 * h; i < NP / 2; i += 4)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = tc::acc_col(i + e, lane);
              if (c < p.C) drow[c] = counted ? (__expf(acc[i + e] - lse) - (c == y ? 1.f : 0.f)) * invN : 0.f;
            }
        }
        if ((lane & 3) == 0 && counted) { nll_sum += lse - ly; ok_sum += arg == y ? 1 : 0; }
      }
    }
    nll_sum = ts::warp_sum(nll_sum);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ok_sum += __shfl_xor_sync(0xffffffffu, ok_sum, o);
    if (lane == 0) { red_f[warp - 4] = nll_sum; red_i[warp - 4] = ok_sum; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    int ok = 0;
    for (int w = 0; w < 8; ++w) { s += red_f[w]; ok += red_i[w]; }
    p.part_loss[blockIdx.x] = s;
    p.part_ok[blockIdx.x] = ok;
  }
  step_finish(p, N, misc + 1);
}

// Generic forward (fp32 activations, more than 256 classes, weight image beyond shared memory): one thread per logit, then
// one warp per row for the cross-entropy.
template <typename T>
__global__ void head_step_logits_generic(const T* __restrict__ h, const float* __restrict__ W, const float* __restrict__ bias,
                                         float* __restrict__ logits, int Tn, int B, int H, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Tn * B * C) return;
  const int r = (int)(i / C), c = (int)(i % C);
  const int t = r / B, b = r - t * B;
  float s = bias[c];
  for (int k = 0; k < H; ++k) s = fmaf(ts::Cvt<T>::to_f(h[(size_t)r * H + k]), W[(size_t)k * C + c], s);
  logits[((size_t)b * Tn + t) * C + c] = s;
}

constexpr int kXentWarps = 8;                                      // rows per block of xent_steps_kernel

// kExact (fp32 activations): the accurate softmax of xent_rows_kernel<true> (head_xent.cu), for the same reasons
// (tests/test_gpu_head_edges.py::test_per_step_head, fp32 rows of the negative regime: dh up to 15x its budget before); the bf16
// instantiation keeps the fast intrinsics.
template <bool kExact>
__global__ void __launch_bounds__(kXentWarps * 32) xent_steps_kernel(const HeadStepParams p) {
  __shared__ int misc[2];
  __shared__ float red_f[kXentWarps];
  __shared__ int red_i[kXentWarps];
  const int N = step_count_rows(p.lengths, p.T, p.B, misc);
  const float invN = 1.0f / (float)N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * kXentWarps + warp;
  float nll = 0.f;
  int ok = 0;
  if (row < p.R) {
    const int t = row / p.B, b = row - t * p.B;
    float* d = p.dlogits + (size_t)row * p.C;
    if (p.lengths != nullptr && t >= p.lengths[b]) {
      for (int c = lane; c < p.C; c += 32) d[c] = 0.f;
    } else {
      const float* l = p.logits + ((size_t)b * p.T + t) * p.C;
      float mx = -INFINITY;
      int arg = 0x7fffffff;
      for (int c = lane; c < p.C; c += 32)
        if (l[c] > mx) { mx = l[c]; arg = c; }
      for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, mx, o);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
        if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
      }
      float se = 0.f;
      for (int c = lane; c < p.C; c += 32) se += kExact ? ts::expf_acc(l[c] - mx) : expf(l[c] - mx);
      se = ts::warp_sum(se);
      const float ls = kExact ? ts::logf_acc(se) : logf(se);
      const float lse = mx + ls;
      const int y = (int)p.labels[(size_t)b * p.T + t];
      for (int c = lane; c < p.C; c += 32)
        d[c] = ((kExact ? ts::expf_acc((l[c] - mx) - ls) : expf(l[c] - lse)) - (c == y ? 1.f : 0.f)) * invN;
      if (lane == 0) { nll = kExact ? (mx - l[y]) + ls : lse - l[y]; ok = arg == y ? 1 : 0; }
    }
  }
  if (lane == 0) { red_f[warp] = nll; red_i[warp] = ok; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    int k = 0;
    for (int w = 0; w < kXentWarps; ++w) { s += red_f[w]; k += red_i[w]; }
    p.part_loss[blockIdx.x] = s;
    p.part_ok[blockIdx.x] = k;
  }
  step_finish(p, N, misc + 1);
}

// Backward, C <= 32: block (jb, slab) = 32 hidden columns x one slab of rows, as head_bwd_kernel, but every slab writes its
// dW / db partial to scratch and the last slab of each column block (ticket) sums the partials in slab order: deterministic at
// any number of rows.
template <int CP>
constexpr int step_bwd_rows() { return CP <= 8 ? 1024 : (CP <= 16 ? 512 : 192); }   // (rows + 4·32)·CP floats < 48 KB

template <typename T, int CP, typename TDH>
__global__ void __launch_bounds__(128) head_step_bwd_kernel(const T* __restrict__ h, const float* __restrict__ W,
                                                            const float* __restrict__ dlogits, const float* __restrict__ dloss,
                                                            TDH* __restrict__ dh, float* __restrict__ dW, float* __restrict__ db,
                                                            float* __restrict__ pdw, float* __restrict__ pdb,
                                                            unsigned int* __restrict__ tickets, int R, int H, int C, int acc_w,
                                                            int acc_b) {
  constexpr int RPB = step_bwd_rows<CP>();
  extern __shared__ float ds[];                         // [RPB][CP] dlogits slab, then [4][kHBwdJ][CP] partials
  float* part = ds + (size_t)RPB * CP;
  __shared__ int last_s;
  const int jl = threadIdx.x & 31, q = threadIdx.x >> 5;
  const int j = blockIdx.x * kHBwdJ + jl;
  const int b0 = blockIdx.y * RPB;
  const int nb = min(RPB, R - b0);
  const float scale = dloss ? *dloss : 1.f;
  {
    constexpr int kLU = 8;
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
    constexpr int kU = 8;
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
  for (int i = threadIdx.x; i < kHBwdJ * C; i += 128) {            // fixed-order sum of the four row groups -> slab partial
    const int jj = i / C, c = i % C;
    const int jg = blockIdx.x * kHBwdJ + jj;
    if (jg < H)
      pdw[((size_t)blockIdx.y * H + jg) * C + c] = ((part[(0 * kHBwdJ + jj) * CP + c] + part[(1 * kHBwdJ + jj) * CP + c]) +
                                                    part[(2 * kHBwdJ + jj) * CP + c]) + part[(3 * kHBwdJ + jj) * CP + c];
  }
  if (blockIdx.x == 0) {                                            // (uniform in the block: the tree synchronises it)
    slab_colsum_tree<CP>(ds, nb);
    if (threadIdx.x < C) pdb[(size_t)blockIdx.y * C + threadIdx.x] = ds[threadIdx.x];
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last_s = atomicAdd(tickets + blockIdx.x, 1u) == gridDim.y - 1;
  __syncthreads();
  if (!last_s) return;
  __threadfence();
  const int ns = gridDim.y;
  for (int i = threadIdx.x; i < kHBwdJ * C; i += 128) {
    const int jg = blockIdx.x * kHBwdJ + i / C, c = i % C;
    if (jg < H) {
      const volatile float* src = pdw + (size_t)jg * C + c;
      float s = 0.f;
      for (int k = 0; k < ns; ++k) s += src[(size_t)k * H * C];
      dW[(size_t)jg * C + c] = (acc_w ? dW[(size_t)jg * C + c] : 0.f) + s;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < C) {
    const volatile float* src = pdb + threadIdx.x;
    float s = 0.f;
    for (int k = 0; k < ns; ++k) s += src[(size_t)k * C];
    db[threadIdx.x] = (acc_b ? db[threadIdx.x] : 0.f) + s;
  }
  if (threadIdx.x == 0) tickets[blockIdx.x] = 0u;
}

template <typename T, typename TDH>
int launch_step_bwd(const void* h, const float* W, const float* dlogits, const float* dloss, void* dh, float* dW, float* db,
                    float* scratch, unsigned int* tickets, int R, int H, int C, int acc_w, int acc_b, cudaStream_t st) {
  if (C > 32) return launch_bwd<T, TDH>(h, W, dlogits, dloss, dh, dW, db, R, H, C, acc_w, acc_b, st);   // per-output kernels: no atomics
#define STEP_BWD(CP)                                                                                                      \
  do {                                                                                                                    \
    constexpr int rows = step_bwd_rows<CP>();                                                                             \
    const int ns = (R + rows - 1) / rows;                                                                                 \
    dim3 grid((H + kHBwdJ - 1) / kHBwdJ, ns);                                                                             \
    head_step_bwd_kernel<T, CP, TDH><<<grid, 128, (rows + 4 * kHBwdJ) * CP * sizeof(float), st>>>(                         \
        (const T*)h, W, dlogits, dloss, (TDH*)dh, dW, db, scratch, scratch + (size_t)ns * H * C, tickets, R, H, C, acc_w, acc_b); \
  } while (0)
  if (C <= 8) STEP_BWD(8); else if (C <= 16) STEP_BWD(16); else STEP_BWD(32);
#undef STEP_BWD
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

// dh dtype follows h (bf16 -> bf16, fp32 -> fp32); dW [H, C] / db [C] fp32, acc_w / acc_b = add into dW / db.
extern "C" int ts_head_bwd(const void* h, const float* W, const float* dlogits, const float* dloss, void* dh, float* dW, float* db,
                           int B, int H, int C, int is_bf16, int acc_w, int acc_b, cudaStream_t st) {
  if (is_bf16) return launch_bwd<__nv_bfloat16, __nv_bfloat16>(h, W, dlogits, dloss, dh, dW, db, B, H, C, acc_w, acc_b, st);
  return launch_bwd<float, float>(h, W, dlogits, dloss, dh, dW, db, B, H, C, acc_w, acc_b, st);
}

// ---- per-step head ------------------------------------------------------------------------------------------------------
// Scratch of the forward: float part_loss[n] + int part_ok[n] with n = this bound on its grid; 1 zeroed ticket word.
extern "C" int ts_head_step_fwd_parts(int R) { return (R + HM - 1) / HM; }

template <int NP>
int launch_head_step_fwd(const CUtensorMap& th, HeadStepParams p, int smem, cudaStream_t st) {
  cudaError_t e = cudaFuncSetAttribute(head_step_fwd_tc_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  int dev = 0, sms = 0, occ = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, head_step_fwd_tc_kernel<NP>, kHThreads, smem);
  if (e != cudaSuccess) return (int)e;
  const int grid = std::max(1, std::min(p.num_tiles, sms * std::max(occ, 1)));
  head_step_fwd_tc_kernel<NP><<<grid, kHThreads, smem, st>>>(th, p);
  return (int)cudaGetLastError();
}

// h: [R = T·B, H] rows of h_seq [T, B, H] (row pitch ldh elements), labels int64 [B, T], lengths int32 [B] or null.
// logits [B, T, C], dlogits [R, C]; loss (mean), correct, count [1] each; part_* / ticket: scratch (ts_head_step_fwd_parts).
// bf16 h on the tensor cores where the shape fits the weight image; everything else on the generic kernels.
extern "C" int ts_head_step_fwd(const void* h, int ldh, int is_bf16, const float* W, const float* bias, const long long* labels,
                                const int* lengths, float* logits, float* dlogits, float* part_loss, int* part_ok,
                                unsigned int* ticket, float* loss, int* correct, int* count, int T, int B, int H, int C,
                                int* used_tc, cudaStream_t st) {
  const int R = T * B;
  HeadStepParams p{W, bias, labels, lengths, logits, dlogits, part_loss, part_ok, ticket, loss, correct, count,
                   T, B, H, C, R, (R + HM - 1) / HM};
  const int smem = ts_head_fwd_tc_smem(H, C) + 64;
  *used_tc = 0;
  if (is_bf16 && C <= 256 && smem <= 200 * 1024 && H % 8 == 0 && ldh % 8 == 0) {
    CUtensorMap th;
    if (int rc = ts::make_tmap_2d_bf16(&th, h, (uint64_t)R, (uint64_t)H, (uint64_t)ldh, HK, HM)) return rc;
    *used_tc = 1;
    if (C <= 16) return launch_head_step_fwd<16>(th, p, smem, st);
    if (C <= 32) return launch_head_step_fwd<32>(th, p, smem, st);
    if (C <= 64) return launch_head_step_fwd<64>(th, p, smem, st);
    if (C <= 128) return launch_head_step_fwd<128>(th, p, smem, st);
    return launch_head_step_fwd<256>(th, p, smem, st);
  }
  if (ldh != H) return -2;                                        // the generic kernels read packed rows
  const long long n = (long long)R * C;
  if (is_bf16) head_step_logits_generic<__nv_bfloat16><<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const __nv_bfloat16*)h, W, bias, logits, T, B, H, C);
  else head_step_logits_generic<float><<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const float*)h, W, bias, logits, T, B, H, C);
  p.num_tiles = (R + kXentWarps - 1) / kXentWarps;
  if (is_bf16) xent_steps_kernel<false><<<p.num_tiles, kXentWarps * 32, 0, st>>>(p);
  else xent_steps_kernel<true><<<p.num_tiles, kXentWarps * 32, 0, st>>>(p);
  return (int)cudaGetLastError();
}
extern "C" int ts_head_step_fwd_generic_parts(int R) { return (R + kXentWarps - 1) / kXentWarps; }

// Scratch of the backward in floats (C <= 32; 0 beyond) and its ticket words (zeroed, left zeroed).
extern "C" long long ts_head_step_bwd_scratch(int R, int H, int C) {
  if (C > 32) return 0;
  const int rows = C <= 8 ? step_bwd_rows<8>() : (C <= 16 ? step_bwd_rows<16>() : step_bwd_rows<32>());
  const long long ns = (R + rows - 1) / rows;
  return ns * H * C + ns * C;
}
extern "C" int ts_head_step_bwd_tickets(int H) { return (H + kHBwdJ - 1) / kHBwdJ; }

// h [R, H] (packed), dlogits [R, C] in row order -> dh [R, H] (dtype of h), dW [H, C] / db [C] (+)= (dloss-scaled) sums.
extern "C" int ts_head_step_bwd(const void* h, const float* W, const float* dlogits, const float* dloss, void* dh, float* dW, float* db,
                                float* scratch, unsigned int* tickets, int R, int H, int C, int is_bf16, int acc_w, int acc_b,
                                cudaStream_t st) {
  if (is_bf16)
    return launch_step_bwd<__nv_bfloat16, __nv_bfloat16>(h, W, dlogits, dloss, dh, dW, db, scratch, tickets, R, H, C, acc_w, acc_b, st);
  return launch_step_bwd<float, float>(h, W, dlogits, dloss, dh, dW, db, scratch, tickets, R, H, C, acc_w, acc_b, st);
}
