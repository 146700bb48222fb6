// Continuous cache pointer (Grave et al. 2017, "Improving Neural Language Models with a Continuous Cache") for stream evaluation.
//
// For the query at absolute stream position p (stream b) with label y_p and the model's log-probability log p_v(y_p):
//     J(p) = { j : max(0, p - W) <= j < p },   s_j = theta (h_p . h_j)   (dot accumulated in fp32, then scaled in fp32)
//     Z = sum_{j in J} exp(s_j - m),   M = sum_{j in J, y_j = y_p} exp(s_j - m),   m = max s_j
//     log p(y_p) = logaddexp(log1p(-lambda) + log p_v(y_p), log lambda + log M - log Z)      (J empty: log p_v(y_p))
// ops/reference.py cache_pointer holds the same definition in the input dtype.
//
//   * History: a per-stream ring keys [B, Cap, H] (compute dtype) + labels [B, Cap] int32; position j lives in slot j % Cap.
//     Cap is a multiple of the key tile and >= W + T, so every key of J(p) for a query of the current segment is still in the
//     ring once the segment has been appended (cache_append_kernel) - the kernels read every key from one place.
//   * cache_scores_tc_kernel (bf16, H % 64 == 0): S = Q K^T on the tensor cores, TMA + wgmma.  A CTA takes 64 query positions of
//     one stream (read in place from the time-major h [T, B, H] through a 3-D tensor map) against one chunk of 128-key tiles of
//     that stream's ring.  A producer warp streams {Q, K} 64-wide H slices through a ring of 128B-swizzled stages; the consumer
//     warpgroup's epilogue masks each score, keeps an online {max, Z, M} per row (the key tile's labels sit in shared memory) and
//     writes the chunk's partial.  No score matrix reaches global memory.
//   * cache_scores_generic_kernel (fp32, or bf16 with H % 64 != 0): the same grid, masks and partials, from a CUDA-core tile
//     product in fp32.
//   * cache_combine_kernel: merges a position's chunk partials in chunk order, applies the mixture, and reduces the segment's
//     cache and model loss sums (per-block partials summed by the last block, ticket).
// The grid depends on the shapes only (B, T, W, H), so two calls on the same inputs give the same bits on any GPU.
//   * cache_label_logprob_*: the model's log p_v(y) per position, from the large-vocabulary head's partials or from stored logits.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "hopper.cuh"
#include "launchers.h"
#include "tmap.h"
#include "ts_common.cuh"

namespace {

constexpr int BQ = 64;            // query positions per CTA
constexpr int BKEY = 128;         // keys per tile (the ring's capacity is a multiple of this)
constexpr int BH = 64;            // H slice per stage: 64 bf16 = 128 B = one swizzle atom
constexpr int kStages = 4;
constexpr int kQBytes = BQ * BH * 2;
constexpr int kKBytes = BKEY * BH * 2;
constexpr int kLabBytes = BKEY * 4;
constexpr int kStageBytes = kQBytes + kKBytes;             // a multiple of 1 KB: every stage keeps the swizzle atoms aligned
constexpr int kTcThreads = 160;   // warps 0..3: the consumer warpgroup, warp 4: the TMA producer
constexpr int kTcSmem = kStages * (kStageBytes + kLabBytes) + 1024 /*align*/ + 256 /*barriers*/;
constexpr int kTargetCtas = 528;  // key chunks are split until (streams x query tiles x chunks) reaches this (4 x 132 SMs)
constexpr int kVocabTileClasses = 256;   // classes per partial of csrc/head_vocab.cu (ts_vocab_head_parts)
constexpr float kLog2e = 1.4426950408889634f;

struct Shape {
  int T, B, H, W, Cap, tiles_q, nchunks, kc;    // kc: key tiles per chunk
  long long P0;                                 // positions of each stream before this segment
};

// Key tiles [kt_lo, kt_hi] (absolute, in units of BKEY positions) that hold keys of queries [q0, q0 + BQ).
__device__ __forceinline__ void key_tiles(const Shape& s, long long q0, long long& kt_lo, long long& kt_hi) {
  const long long lo = q0 - s.W > 0 ? q0 - s.W : 0;
  kt_lo = lo / BKEY;
  kt_hi = (q0 + BQ - 2) / BKEY;                 // the last query of the tile sees keys up to q0 + BQ - 2
}

// Online {max, Z, M} of one row in base-2 units: values are s * log2(e), so exp(s - m) = exp2(v - mv).
struct Acc3 {
  float m, z, mm;
  __device__ __forceinline__ void init() { m = -INFINITY; z = 0.f; mm = 0.f; }
  __device__ __forceinline__ void merge(float m2, float z2, float mm2) {
    const float n = fmaxf(m, m2);
    if (n == -INFINITY) return;
    const float a = exp2f(m - n), b = exp2f(m2 - n);
    z = z * a + z2 * b;
    mm = mm * a + mm2 * b;
    m = n;
  }
};

// ================================================================================================ tensor-core scores
__global__ void __launch_bounds__(kTcThreads, 1)
cache_scores_tc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k, const int* __restrict__ klab,
                       const long long* __restrict__ labels, const Shape s, float theta2, float4* __restrict__ part) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  int* labs = reinterpret_cast<int*>(smem + kStages * kStageBytes);            // [kStages][BKEY] key labels
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * (kStageBytes + kLabBytes));
  uint64_t* empty = full + kStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x, qt = blockIdx.y, b = blockIdx.z;
  const int t0 = qt * BQ;
  const long long q0 = s.P0 + t0;
  long long kt_lo, kt_hi;
  key_tiles(s, q0, kt_lo, kt_hi);
  const long long kt0 = kt_lo + (long long)chunk * s.kc;
  const long long kt1 = min(kt0 + s.kc - 1, kt_hi);
  const int ntiles = kt1 >= kt0 ? (int)(kt1 - kt0 + 1) : 0;
  const int nkb = s.H / BH;
  const int ring_tiles = s.Cap / BKEY;

  if (warp == 4 && lane == 0) {
    tc::prefetch_tmap(&tmap_q);
    tc::prefetch_tmap(&tmap_k);
    for (int i = 0; i < kStages; ++i) { tc::mbar_init(&full[i], 1); tc::mbar_init(&empty[i], 4); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ===================================================================== TMA producer
    uint32_t stage = 0, phase = 0;
    for (int kt = 0; kt < ntiles; ++kt) {
      const int slot0 = (int)((kt0 + kt) % ring_tiles) * BKEY;
      for (int kb = 0; kb < nkb; ++kb) {
        const uint32_t fb = tc::smem_u32(&full[stage]);
        while (!tc::mbar_try_wait_u32(tc::smem_u32(&empty[stage]), phase ^ 1)) {}
        if (tc::elect_one()) {
          const bool last = kb == nkb - 1;
          uint8_t* st = smem + stage * kStageBytes;
          tc::mbar_expect_tx_u32(fb, kQBytes + kKBytes + (last ? kLabBytes : 0));
          asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                       ::"r"(tc::smem_u32(st)), "l"((uint64_t)&tmap_q), "r"(fb), "r"(kb * BH), "r"(b), "r"(t0) : "memory");
          asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                       ::"r"(tc::smem_u32(st + kQBytes)), "l"((uint64_t)&tmap_k), "r"(fb), "r"(kb * BH), "r"(slot0), "r"(b) : "memory");
          if (last) tc::bulk_load_1d_u32(tc::smem_u32(labs + stage * BKEY), klab + (size_t)b * s.Cap + slot0, kLabBytes, fb);
        }
        __syncwarp();
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================================================================== consumer warpgroup
  int yq[2];
  long long pq[2];
  bool rv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = t0 + tc::acc_row(2 * h, warp, lane);
    rv[h] = t < s.T;
    pq[h] = s.P0 + t;
    yq[h] = rv[h] ? (int)labels[(size_t)b * s.T + t] : -1;
  }
  Acc3 a[2];
  a[0].init(); a[1].init();
  uint32_t stage = 0, phase = 0;
  const uint64_t dq0 = tc::desc_kmajor_sw128(tc::smem_u32(smem));
  const uint64_t dk0 = tc::desc_kmajor_sw128(tc::smem_u32(smem + kQBytes));
  for (int kt = 0; kt < ntiles; ++kt) {
    float acc[BKEY / 2];
#pragma unroll
    for (int i = 0; i < BKEY / 2; ++i) acc[i] = 0.f;
    uint32_t prev = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      while (!tc::mbar_try_wait_u32(tc::smem_u32(&full[stage]), phase)) {}
      const uint64_t so = (uint64_t)((stage * kStageBytes) >> 4);
      tc::fence_regs(acc);
      tc::wgmma_fence();
#pragma unroll
      for (int k = 0; k < BH / 16; ++k) tc::Wgmma<BKEY, 0, 0>::mma(acc, dq0 + so + 2 * k, dk0 + so + 2 * k, (kb > 0 || k > 0) ? 1u : 0u);
      tc::wgmma_commit();
      tc::fence_regs(acc);
      if (kb > 0) {
        tc::wgmma_wait<1>();
        if (lane == 0) tc::mbar_arrive(&empty[prev]);
      }
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    tc::wgmma_wait<0>();
    tc::fence_regs(acc);
    // epilogue: the tile's labels came with its last H slice (stage `prev`, still held)
    const int* lab = labs + prev * BKEY;
    const long long j0 = (kt0 + kt) * BKEY;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long jlo = pq[h] - s.W > 0 ? pq[h] - s.W : 0;
      float v[BKEY / 4];
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < BKEY / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const long long j = j0 + tc::acc_col(4 * i + e, lane);
          const bool ok = rv[h] && j >= jlo && j < pq[h];
          const float x = ok ? acc[4 * i + 2 * h + e] * theta2 : -INFINITY;
          v[2 * i + e] = x;
          mx = fmaxf(mx, x);
        }
      if (mx != -INFINITY) {
        float z = 0.f, mm = 0.f;
#pragma unroll
        for (int i = 0; i < BKEY / 8; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float w = exp2f(v[2 * i + e] - mx);
            z += w;
            if (lab[tc::acc_col(4 * i + e, lane)] == yq[h]) mm += w;
          }
        a[h].merge(mx, z, mm);
      }
    }
    __syncwarp();
    if (lane == 0) tc::mbar_arrive(&empty[prev]);
  }
  // the four lanes of a row merge in a fixed tree
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, a[h].m, o), z2 = __shfl_xor_sync(0xffffffffu, a[h].z, o),
                  mm2 = __shfl_xor_sync(0xffffffffu, a[h].mm, o);
      a[h].merge(m2, z2, mm2);
    }
    const int t = t0 + tc::acc_row(2 * h, warp, lane);
    if ((lane & 3) == 0 && t < s.T)
      part[((size_t)b * s.T + t) * s.nchunks + chunk] = make_float4(a[h].m, a[h].z, a[h].mm, 0.f);
  }
}

// ================================================================================================ generic scores
// 256 threads: thread (ty = tid / 16, tx = tid % 16) owns query rows 4 ty .. 4 ty + 3 and keys tx + 16 c (c < 8) of each tile.
constexpr int kGenThreads = 256;
constexpr int kGenBH = 32;

template <typename T>
__global__ void __launch_bounds__(kGenThreads)
cache_scores_generic_kernel(const T* __restrict__ h, const T* __restrict__ keys, const int* __restrict__ klab,
                            const long long* __restrict__ labels, const Shape s, float theta2, float4* __restrict__ part) {
  __shared__ float qs[BQ][kGenBH + 1];
  __shared__ float ks[BKEY][kGenBH + 1];
  __shared__ int labs[BKEY];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int chunk = blockIdx.x, qt = blockIdx.y, b = blockIdx.z;
  const int t0 = qt * BQ;
  const long long q0 = s.P0 + t0;
  long long kt_lo, kt_hi;
  key_tiles(s, q0, kt_lo, kt_hi);
  const long long kt0 = kt_lo + (long long)chunk * s.kc;
  const long long kt1 = min(kt0 + s.kc - 1, kt_hi);
  const int ntiles = kt1 >= kt0 ? (int)(kt1 - kt0 + 1) : 0;
  const int ring_tiles = s.Cap / BKEY;

  int yq[4];
  long long pq[4];
  bool rv[4];
  Acc3 a[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int t = t0 + 4 * ty + r;
    rv[r] = t < s.T;
    pq[r] = s.P0 + t;
    yq[r] = rv[r] ? (int)labels[(size_t)b * s.T + t] : -1;
    a[r].init();
  }
  for (int kt = 0; kt < ntiles; ++kt) {
    const int slot0 = (int)((kt0 + kt) % ring_tiles) * BKEY;
    float acc[4][8];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[r][c] = 0.f;
    for (int k0 = 0; k0 < s.H; k0 += kGenBH) {
      __syncthreads();
      for (int i = tid; i < BQ * kGenBH; i += kGenThreads) {
        const int r = i / kGenBH, k = i % kGenBH, t = t0 + r;
        qs[r][k] = (t < s.T && k0 + k < s.H) ? ts::Cvt<T>::to_f(h[((size_t)t * s.B + b) * s.H + k0 + k]) : 0.f;
      }
      for (int i = tid; i < BKEY * kGenBH; i += kGenThreads) {
        const int r = i / kGenBH, k = i % kGenBH;
        ks[r][k] = k0 + k < s.H ? ts::Cvt<T>::to_f(keys[((size_t)b * s.Cap + slot0 + r) * s.H + k0 + k]) : 0.f;
      }
      if (k0 == 0 && tid < BKEY) labs[tid] = klab[(size_t)b * s.Cap + slot0 + tid];
      __syncthreads();
#pragma unroll 8
      for (int k = 0; k < kGenBH; ++k) {
        float q[4], kv[8];
#pragma unroll
        for (int r = 0; r < 4; ++r) q[r] = qs[4 * ty + r][k];
#pragma unroll
        for (int c = 0; c < 8; ++c) kv[c] = ks[tx + 16 * c][k];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 8; ++c) acc[r][c] = fmaf(q[r], kv[c], acc[r][c]);
      }
    }
    const long long j0 = (kt0 + kt) * BKEY;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const long long jlo = pq[r] - s.W > 0 ? pq[r] - s.W : 0;
      float v[8], mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const long long j = j0 + tx + 16 * c;
        v[c] = (rv[r] && j >= jlo && j < pq[r]) ? acc[r][c] * theta2 : -INFINITY;
        mx = fmaxf(mx, v[c]);
      }
      if (mx != -INFINITY) {
        float z = 0.f, mm = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float w = exp2f(v[c] - mx);
          z += w;
          if (labs[tx + 16 * c] == yq[r]) mm += w;
        }
        a[r].merge(mx, z, mm);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, a[r].m, o), z2 = __shfl_xor_sync(0xffffffffu, a[r].z, o),
                  mm2 = __shfl_xor_sync(0xffffffffu, a[r].mm, o);
      a[r].merge(m2, z2, mm2);
    }
    const int t = t0 + 4 * ty + r;
    if (tx == 0 && t < s.T) part[((size_t)b * s.T + t) * s.nchunks + chunk] = make_float4(a[r].m, a[r].z, a[r].mm, 0.f);
  }
}

// ================================================================================================ combine
constexpr int kCombThreads = 256;

struct CombineParams {
  const float4* part;          // [B, T, nchunks]
  const float* logp_model;     // [T·B] time-major rows
  const int* lengths;          // [B] or null
  float* logp;                 // [T·B] the mixture's log p(y) (0 at uncounted positions)
  float2* block_sums;          // [gridDim.x]
  unsigned int* ticket;        // [1]: 0 on entry, left 0
  float* sums;                 // [2] {sum -log p, sum -log p_v} over the counted positions
  int T, B, nchunks;
  float log_keep, log_lambda;  // log1p(-lambda), log(lambda) (-inf at lambda = 0)
};

// One thread per position r = t·B + b: merges the chunks in order, then a fixed-shape block tree and the last block's sum.
__global__ void __launch_bounds__(kCombThreads) cache_combine_kernel(const CombineParams p) {
  __shared__ float2 red[kCombThreads];
  __shared__ int last_s;
  const int r = blockIdx.x * kCombThreads + threadIdx.x;
  float2 mine = make_float2(0.f, 0.f);
  if (r < p.T * p.B) {
    const int t = r / p.B, b = r - t * p.B;
    float out = 0.f;
    if (p.lengths == nullptr || t < p.lengths[b]) {
      Acc3 a;
      a.init();
      const float4* pp = p.part + ((size_t)b * p.T + t) * p.nchunks;
      for (int c = 0; c < p.nchunks; ++c) { const float4 v = pp[c]; a.merge(v.x, v.y, v.z); }
      const float lv = p.logp_model[r];
      float lp = lv;
      if (a.m != -INFINITY) {
        const float x = p.log_keep + lv;
        if (a.mm > 0.f && p.log_lambda != -INFINITY) {
          const float c = p.log_lambda + (logf(a.mm) - logf(a.z));
          const float hi = fmaxf(x, c), lo = fminf(x, c);
          lp = hi + log1pf(expf(lo - hi));
        } else {
          lp = x;
        }
      }
      out = lp;
      mine = make_float2(-lp, -lv);
    }
    p.logp[r] = out;
  }
  red[threadIdx.x] = mine;
  __syncthreads();
  for (int o = kCombThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) { red[threadIdx.x].x += red[threadIdx.x + o].x; red[threadIdx.x].y += red[threadIdx.x + o].y; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    p.block_sums[blockIdx.x] = red[0];
    __threadfence();
    last_s = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last_s && threadIdx.x < 32) {                // the last block sums every block's partial: lane-strided, then a fixed tree
    __threadfence();
    const volatile float2* bs = p.block_sums;
    float x = 0.f, y = 0.f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += 32) { x += bs[i].x; y += bs[i].y; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { x += __shfl_xor_sync(0xffffffffu, x, o); y += __shfl_xor_sync(0xffffffffu, y, o); }
    if (threadIdx.x == 0) {
      p.sums[0] = x;
      p.sums[1] = y;
      *p.ticket = 0u;
    }
  }
}

// ================================================================================================ history and log p_v
// keys[b, (P0 + t) % Cap, :] = h[t, b, :], klab[b, (P0 + t) % Cap] = labels[b, t]: one block per (t, b), in words of V (16, 4
// or 2 bytes: the widest that divides the row and both base addresses).
template <typename V>
__global__ void __launch_bounds__(128) cache_append_kernel(const V* __restrict__ h, V* __restrict__ keys, int* __restrict__ klab,
                                                          const long long* __restrict__ labels, int T, int B, int row_words, int Cap,
                                                          long long P0) {
  const int t = blockIdx.x / B, b = blockIdx.x - t * B;
  const int slot = (int)((P0 + t) % Cap);
  const V* src = h + (size_t)blockIdx.x * row_words;
  V* dst = keys + ((size_t)b * Cap + slot) * row_words;
  for (int i = threadIdx.x; i < row_words; i += blockDim.x) dst[i] = src[i];
  if (threadIdx.x == 0) klab[(size_t)b * Cap + slot] = (int)labels[(size_t)b * T + t];
}

// From the large-vocabulary head's forward: part[r, tile].w holds the label's logit in the label's class tile (0 elsewhere).
__global__ void cache_label_logprob_parts_kernel(const float4* __restrict__ part, const float* __restrict__ lse,
                                                 const long long* __restrict__ labels, float* __restrict__ logp, int T, int B, int nt) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= T * B) return;
  const int t = r / B, b = r - t * B;
  const long long y = labels[(size_t)b * T + t];
  logp[r] = (y >= 0 && y < (long long)nt * kVocabTileClasses) ? part[(size_t)r * nt + y / kVocabTileClasses].w - lse[r] : 0.f;
}

// From stored fp32 logits [B, T, C]: one warp per position r = t·B + b.
__global__ void __launch_bounds__(256) cache_label_logprob_logits_kernel(const float* __restrict__ logits, const long long* __restrict__ labels,
                                                                         float* __restrict__ logp, int T, int B, int C) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= T * B) return;
  const int t = r / B, b = r - t * B;
  const float* row = logits + ((size_t)b * T + t) * C;
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
  mx = ts::warp_max(mx);
  float se = 0.f;
  for (int c = lane; c < C; c += 32) se += expf(row[c] - mx);
  se = ts::warp_sum(se);
  const long long y = labels[(size_t)b * T + t];
  if (lane == 0) logp[r] = (y >= 0 && y < C) ? row[y] - mx - logf(se) : 0.f;     // a label outside [0, C) marks a padded position
}

Shape make_shape(int T, int B, int H, int W, int Cap, long long P0) {
  Shape s;
  s.T = T; s.B = B; s.H = H; s.W = W; s.Cap = Cap; s.P0 = P0;
  s.tiles_q = (T + BQ - 1) / BQ;
  const int kt = (W + BQ - 2) / BKEY + 2;                      // key tiles a query tile can touch, at any alignment
  const long long pairs = (long long)B * s.tiles_q;
  int n = (int)((kTargetCtas + pairs - 1) / pairs);
  n = n < 1 ? 1 : (n > kt ? kt : n);
  s.kc = (kt + n - 1) / n;
  s.nchunks = (kt + s.kc - 1) / s.kc;
  return s;
}

}  // namespace

extern "C" int ts_cache_key_tile() { return BKEY; }
extern "C" int ts_cache_chunks(int T, int B, int H, int W) { return make_shape(T, B, H, W, BKEY, 0).nchunks; }
extern "C" int ts_cache_combine_blocks(int R) { return (R + kCombThreads - 1) / kCombThreads; }

// h [T, B, H] (bf16 or fp32, packed), keys [B, Cap, H] same dtype, klab int32 [B, Cap], labels int64 [B, T], logp_model fp32 [T·B],
// lengths int32 [B] or null; part float4 [B·T·ts_cache_chunks], block_sums float2 [ts_cache_combine_blocks(T·B)], ticket 1 zeroed
// word (left zeroed) -> logp fp32 [T·B], sums fp32 [2].  tc: the tensor-core path (bf16, H % 64 == 0).
extern "C" int ts_cache_pointer(const void* h, const void* keys, const int* klab, const long long* labels, const float* logp_model,
                                const int* lengths, int T, int B, int H, int W, int Cap, long long P0, float theta, float lambda,
                                int bf16, int tc, void* part, void* block_sums, unsigned int* ticket, float* logp, float* sums,
                                cudaStream_t st) {
  if (T < 1 || B < 1 || H < 1 || W < 1 || Cap % BKEY != 0 || Cap < W + T) return -1;
  if (tc && (!bf16 || H % BH != 0)) return -2;
  const Shape s = make_shape(T, B, H, W, Cap, P0);
  const float theta2 = theta * kLog2e;
  const dim3 grid(s.nchunks, s.tiles_q, B);
  float4* pt = reinterpret_cast<float4*>(part);
  if (tc) {
    CUtensorMap tq, tk;
    if (int rc = ts::make_tmap_3d_bf16(&tq, h, (uint64_t)H, (uint64_t)B, (uint64_t)T, (uint64_t)H, (uint64_t)B * H, BH, 1, BQ)) return rc;
    if (int rc = ts::make_tmap_3d_bf16(&tk, keys, (uint64_t)H, (uint64_t)Cap, (uint64_t)B, (uint64_t)H, (uint64_t)Cap * H, BH, BKEY, 1)) return rc;
    static bool attr_set = false;
    if (!attr_set) {
      cudaFuncSetAttribute(cache_scores_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmem);
      attr_set = true;
    }
    cache_scores_tc_kernel<<<grid, kTcThreads, kTcSmem, st>>>(tq, tk, klab, labels, s, theta2, pt);
  } else if (bf16) {
    cache_scores_generic_kernel<__nv_bfloat16><<<grid, kGenThreads, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(h), reinterpret_cast<const __nv_bfloat16*>(keys), klab, labels, s, theta2, pt);
  } else {
    cache_scores_generic_kernel<float><<<grid, kGenThreads, 0, st>>>(reinterpret_cast<const float*>(h),
                                                                     reinterpret_cast<const float*>(keys), klab, labels, s, theta2, pt);
  }
  if (cudaError_t e = cudaGetLastError()) return (int)e;
  CombineParams c{pt, logp_model, lengths, logp, reinterpret_cast<float2*>(block_sums), ticket, sums, T, B, s.nchunks,
                  (float)log1p(-(double)lambda), lambda > 0 ? (float)log((double)lambda) : -INFINITY};
  cache_combine_kernel<<<ts_cache_combine_blocks(T * B), kCombThreads, 0, st>>>(c);
  return (int)cudaGetLastError();
}

// Write a segment into the ring: h [T, B, H] packed rows of row_bytes (a multiple of 2), keys [B, Cap, row], klab int32 [B, Cap].
extern "C" int ts_cache_append(const void* h, void* keys, int* klab, const long long* labels, int T, int B, long long row_bytes, int Cap,
                               long long P0, cudaStream_t st) {
  if (row_bytes % 2 != 0 || T < 1 || B < 1 || Cap < T) return -1;
  const uintptr_t align = reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(keys) | (uintptr_t)row_bytes;
  if (align % 16 == 0) {
    cache_append_kernel<uint4><<<T * B, 128, 0, st>>>(reinterpret_cast<const uint4*>(h), reinterpret_cast<uint4*>(keys), klab, labels,
                                                      T, B, (int)(row_bytes / 16), Cap, P0);
  } else if (align % 4 == 0) {
    cache_append_kernel<uint32_t><<<T * B, 128, 0, st>>>(reinterpret_cast<const uint32_t*>(h), reinterpret_cast<uint32_t*>(keys), klab,
                                                         labels, T, B, (int)(row_bytes / 4), Cap, P0);
  } else {
    cache_append_kernel<uint16_t><<<T * B, 128, 0, st>>>(reinterpret_cast<const uint16_t*>(h), reinterpret_cast<uint16_t*>(keys), klab,
                                                         labels, T, B, (int)(row_bytes / 2), Cap, P0);
  }
  return (int)cudaGetLastError();
}

extern "C" int ts_cache_label_logprob_parts(const void* part, const float* lse, const long long* labels, float* logp, int T, int B, int C,
                                            int nt, cudaStream_t st) {
  if (nt != (C + kVocabTileClasses - 1) / kVocabTileClasses) return -1;
  const int R = T * B;
  cache_label_logprob_parts_kernel<<<(R + 255) / 256, 256, 0, st>>>(reinterpret_cast<const float4*>(part), lse, labels, logp, T, B, nt);
  return (int)cudaGetLastError();
}

extern "C" int ts_cache_label_logprob_logits(const float* logits, const long long* labels, float* logp, int T, int B, int C,
                                             cudaStream_t st) {
  const int R = T * B;
  cache_label_logprob_logits_kernel<<<(R + 7) / 8, 256, 0, st>>>(logits, labels, logp, T, B, C);
  return (int)cudaGetLastError();
}
