// Large-vocabulary per-step head (next-token language modelling): softmax cross-entropy over C >= 512 classes at every row of
// h [R = T·B, H] without ever storing the logits [R, C] or an fp32 dlogits [R, C].
//
//   logits = h [R,H] (bf16, K-major) · W [H,C] (bf16, read in place as an MN-major operand) + bias (fp32), fp32 accumulators.
//   With tied embeddings the weights are the embedding table [C,H] = W^T, read in place as a K-major operand (kBK = true
//   below): the same products in the same k order, only the shared-memory layout of the B tile differs.
//
//   * vocab_head_gemm_kernel<kFwd>: TMA + wgmma over 128-row x 256-class tiles (a cluster of two CTAs computes 256 rows and
//     shares the W tile by multicast, as gemm2_wgmma.cu).  The epilogue never writes the tile: per row it reduces the tile's
//     max, sum exp(l - max), arg-max and the label's logit from the accumulator fragments into part[R, C/256] (16 B each).
//   * vocab_head_combine_kernel: merges a row's partials in a fixed order -> lse[R]; loss, correct and N through per-block
//     partials summed by the last block (ticket): two calls on the same inputs give the same bits.
//   * vocab_head_gemm_kernel<kDlogits>: the same main loop over one chunk of rows recomputes the logits; the epilogue writes
//     dlogits = (exp(l - lse) - onehot) · dloss / N at counted rows, 0 elsewhere, as bf16 into a scratch [chunk rows, C] that
//     the caller feeds to the general GEMM (dh = dlogits · W^T, dW += h^T · dlogits).
//   * vocab_head_colsum_kernel: db (+)= column sums of the bf16 dlogits chunk, summed in a fixed order.
//   * vocab_head_gemm_kernel<kSample> (text generation, R = B rows of one step): the same main loop; the epilogue reduces each
//     row of a tile to the max and sum exp(l - max) of the logits and the max of the perturbed score (sample_score below), its
//     class and the logit there; vocab_sample_combine_kernel merges the tiles of a row in a fixed order into the sampled token
//     and its log-probability.  vocab_sample_logits_kernel makes the same partials from stored fp32 logits (the inputs this
//     GEMM does not take).
//   * Top-k / top-p sampling needs the whole row, so it stores it: vocab_head_gemm_kernel<kLogits> (the same main loop; the
//     epilogue writes acc + bias as fp32 logits [B, C]), vocab_threshold_kernel (the row's threshold tau, a radix select),
//     vocab_sample_logits_kernel<true> (the partials over the classes with l >= tau) and the same combine.
//
// Tiles are walked in bands of 16 cluster tiles (4096 rows): inside a band the class tile is the outer index, so the band's rows
// of h stay in L2 and W streams from HBM once per band.  Row r = t·B + b counts iff t < lengths[b]; lengths may be 0.
//
//   warp 0 : TMA producer     warps 1..3 : idle     warps 4..11 : two consumer warpgroups (wgmma + epilogue)
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "hopper.cuh"
#include "launchers.h"
#include "tmap.h"
#include "ts_common.cuh"

namespace {

constexpr int BM = 128;                     // rows per CTA (two m64 warpgroups)
constexpr int BN = 256;                     // classes per tile
constexpr int BK = 64;                      // 64 bf16 = 128 B = one swizzle atom
constexpr int kCtas = 2;                    // CTAs per cluster: 256 rows share one W tile
constexpr int TM = BM * kCtas;
constexpr int kBandTiles = 16;              // cluster tiles per band
constexpr int kThreads = 384;
constexpr int kConsWarp0 = 4;
constexpr int kABytes = BM * BK * 2;        // 16 KB
constexpr int kBBytes = BN * BK * 2;        // 32 KB: the whole W tile lands in both CTAs
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kStages = 4;
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 1024 /*barriers*/;

enum Mode { kFwd = 0, kDlogits = 1, kSample = 2, kLogits = 3 };

struct VocabParams {
  const float* bias;           // [C]
  const long long* labels;     // [B, T]
  const int* lengths;          // [B] or null
  // The unions overlay pointers no mode reads together, so the layout (and the code of every other mode) stays as it was.
  union {
    float4* part;              // kFwd: [R, tiles_n] {max, sum exp, arg-max (int bits), label logit or 0}
    float* logits;             // kLogits: [B, C] fp32, acc + bias
  };
  union {
    const float* lse;          // kDlogits: [R]
    const float* tau;          // vocab_sample_logits_kernel<true>: [B] the kept set's threshold, l >= tau
  };
  const float* dloss;          // kDlogits: [1]
  const int* count;            // kDlogits: [1] N
  __nv_bfloat16* dl;           // kDlogits: [rows, C]
  int R, H, C, T, B;
  int row0, rows;              // this launch covers rows [row0, row0 + rows) of h
  // kSample (T = 1): part {max, sum exp, best perturbed score, logit at it}, part_arg [R, tiles_n] the class of the best score
  int* part_arg;
  const int* step;             // decode step s (device-resident: a captured graph reads its current value)
  uint32_t seed;
  float inv_tau;               // 1 / temperature in fp32; -1 at temperature 0 (greedy: the score is the logit, no noise is drawn)
  const int* row_base;         // row word of local row 0 in the noise counter (device-resident, as step)
};

// ---- sampling -----------------------------------------------------------------------------------------------------------------
// The sampling definition, shared with ops/reference.py (sample_noise_words / sample_scores / sample_logits): change both or
// neither.  For row b at decode step s, with logits l = h W + bias:
//   temperature 0 (greedy): token = argmax_c l_c, the smallest index on a tie; no noise is drawn.
//   temperature t > 0: Gumbel-max, token = argmax_c (l_c / t + g_c), an exact draw from softmax(l / t), with
//     g_c = -log(-log u_c), u_c = ((word >> 8) + 0.5) * 2^-24 (strictly inside (0, 1), so no score is infinite), where word is word c & 3
//     of Philox4x32-10 at key (seed & 0xffffffff, 0x53414D50) and counter (c >> 2, row0 + b, s, 0).  row0 places the batch in a
//     larger set of prompts (generation in batches: the prompt's index), so no two prompts share a stream.  The second key word
//     keeps these streams apart from the dropout masks (key (seed, partition)).
//   The op also returns log p(token) = l_token - logsumexp(l), under the model's own softmax(l) whatever the temperature.
// Rounding: l is fp32 (bf16 h x bf16 W accumulated in fp32, plus the fp32 bias, or the fp32 logits of the fallback); the score
// is fmaf(l, 1/t, g) in fp32.  u has 25 significant bits at u >= 1/2, where fp32 would round 1 - 2^-25 to 1 and -log u to 0:
// below 1/2 u is exact in fp32 and -log u = -log(u); above it 1 - u is exact and -log u = -log1p(-(1 - u)) > 0.
//
// Top-k / top-p (nucleus) filtering, shared with ops/reference.py (sample_threshold / sample_logits): at temperature t > 0 the
// token is argmax over c in K of (l_c / t + g_c), with the same noise g, an exact draw from softmax(l / t) restricted to K and
// renormalised.  K = {c : l_c >= tau}:
//   top-k (0 < k < C): tau_k = the k-th largest logit counted with multiplicity; every class tied at it is kept.
//   top-p (0 < p < 1): q = softmax(l / t) over {l >= tau_k} (all classes without top-k); tau = the largest logit value v with
//     q-mass of {l >= v} at least p (ties at v are kept).  Both: top-k first, then top-p on what is left.
//   Off (k = 0 or k >= C, p = 1) or t = 0: no filter, the kernels above.  log p(token) stays under the full softmax(l).
// Coupling: the filtered path's logits are the same fp32 values kSample scores (acc + bias from the same main loop, or the same
// GEMM's logits on the fallback) and its scores are the same sample_score, so the filtered token equals the unfiltered one
// whenever that token is in K.
// Rounding of the threshold: ties and the k-th value are decided on the fp32 logits exactly.  Top-p masses are
// exp((l - max) / t) in fp32 (__expf((l - max) * (1/t))), rounded to fixed point in units of 2^-32 of the row max's mass and
// summed as u64 integers (so the sums do not depend on the order or the grid); the cut is the first value, from the top, where
// the running sum reaches ceil(p · Z) (fp64 product, Z the total).  A class below 2^-33 of the max's mass counts as 0.
constexpr uint32_t kSampleKey1 = 0x53414D50u;      // "SAMP"

TC_DEVICE uint4 sample_words(uint32_t seed, uint32_t row, uint32_t s, int c) {
  return ts::philox4x32_10(make_uint4((uint32_t)c >> 2, row, s, 0u), make_uint2(seed, kSampleKey1));
}
TC_DEVICE float sample_gumbel(uint32_t w) {
  const uint32_t k = w >> 8;
  const float u = ((float)k + 0.5f) * 0x1p-24f;
  const float e = k < (1u << 23) ? -__logf(u) : -log1pf(-(((float)((1u << 24) - 1u - k) + 0.5f) * 0x1p-24f));
  return -__logf(e);
}
TC_DEVICE float sample_score(float l, float inv_tau, uint32_t w) { return fmaf(l, inv_tau, sample_gumbel(w)); }
// best-score merge: the larger score, the smaller class on a tie
TC_DEVICE void sample_take(float& best, int& arg, float& lbest, float b2, int a2, float l2) {
  if (b2 > best || (b2 == best && a2 < arg)) { best = b2; arg = a2; lbest = l2; }
}

// tile -> (cluster tile row, class tile): bands of kBandTiles cluster tiles, class tile outer inside a band
TC_DEVICE void tile_coords(int tile, int tiles_m, int tiles_n, int& tm, int& tn) {
  const int per_band = kBandTiles * tiles_n;
  const int band = tile / per_band, rem = tile - band * per_band;
  const int gm = min(kBandTiles, tiles_m - band * kBandTiles);
  tn = rem / gm;
  tm = band * kBandTiles + rem - tn * gm;
}

// kBK: the B operand is a K-major table [C, H] (tied embeddings), else the MN-major W [H, C].  K-major: each CTA's half of the
// 256-class tile is one TMA box of 64 k (128 B, one swizzle atom) x 128 class rows, multicast to both CTAs like the W boxes.
template <int kMode, bool kBK>
__global__ void __launch_bounds__(kThreads, 1)
vocab_head_gemm_kernel(const __grid_constant__ CUtensorMap tmap_h, const __grid_constant__ CUtensorMap tmap_w, const VocabParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kABytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty = full + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t crank = tc::cluster_ctarank();
  const int tiles_n = (p.C + BN - 1) / BN;
  const int tiles_m = (p.rows + TM - 1) / TM;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = p.H / BK;
  const int cluster_id = blockIdx.x / kCtas, num_clusters = gridDim.x / kCtas;

  if (warp == 0 && lane == 0) {
    tc::prefetch_tmap(&tmap_h);
    tc::prefetch_tmap(&tmap_w);
  }
  if (warp == 1 && lane == 0) {
    // empty: every consumer warp of both CTAs (the W half this CTA loads lands in both)
    for (int s = 0; s < kStages; ++s) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], 8 * kCtas); }
    tc::fence_barrier_init();
  }
  __syncthreads();
  tc::cluster_sync();                            // the peer's barriers are initialised before anything arrives on them

  // The consumers hold 128 accumulator registers per thread and the epilogue works on all of them: setmaxnreg moves registers
  // from warpgroup 0 (producer and idle warps) to them, (168 - 56) * 128 = (224 - 168) * 256.  All four warps of a warpgroup
  // execute it at the top of the warpgroup's branch.
  if (warp < kConsWarp0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 56;" ::: "memory");
    if (warp == 0) {
      // ===================================================================== TMA producer
      const uint32_t full0 = tc::smem_u32(full), empty0 = tc::smem_u32(empty);
      const uint32_t sa0 = tc::smem_u32(smem_a), sb0 = tc::smem_u32(smem_b);
      uint32_t stage = 0, phase = 0;
      for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
        int tm, tn;
        tile_coords(tile, tiles_m, tiles_n, tm, tn);
        const int m0 = p.row0 + tm * TM + (int)crank * BM;
        const int n0 = tn * BN + (int)crank * (BN / kCtas);
        for (int kb = 0, k0 = 0; kb < num_kb; ++kb, k0 += BK) {
          const uint32_t eb = empty0 + 8 * stage, fb = full0 + 8 * stage;
          while (!tc::mbar_try_wait_u32(eb, phase ^ 1)) {}
          if (tc::elect_one()) {
            tc::mbar_expect_tx_u32(fb, kStageBytes);
            tc::tma_load_2d_u32(sa0 + stage * kABytes, &tmap_h, fb, k0, m0);
            const uint32_t sb = sb0 + stage * kBBytes + crank * (kBBytes / kCtas);     // this CTA's half of the W tile
            if (kBK) {
              tc::tma_load_2d_mc(sb, &tmap_w, fb, k0, n0, 3);                              // class rows [n0, n0 + 128)
            } else {
#pragma unroll
              for (int j = 0; j < BN / kCtas / 64; ++j) tc::tma_load_2d_mc(sb + j * 8192, &tmap_w, fb, n0 + 64 * j, k0, 3);
            }
          }
          __syncwarp();
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 224;" ::: "memory");
    // ===================================================================== consumers: wgmma main loop + epilogue
    const int wg = (warp - kConsWarp0) >> 2;             // rows [64 wg, +64) of the CTA's 128
    const int wq = warp & 3;
    const uint32_t full0 = tc::smem_u32(full), empty0 = tc::smem_u32(empty);
    const uint32_t empty0_peer = tc::mapa(empty0, crank ^ 1u);
    const uint64_t da0 = tc::desc_kmajor_sw128(tc::smem_u32(smem_a) + wg * 8192);
    const uint64_t db0 = kBK ? tc::desc_kmajor_sw128(tc::smem_u32(smem_b)) : tc::desc_mnmajor_sw128(tc::smem_u32(smem_b));
    constexpr uint32_t kBStep = kBK ? (32 >> 4) : (2048 >> 4);   // per k16: 32 B along a K-major row, 16 rows of the MN-major tile
    auto release = [&](uint32_t st) {                     // this warp has finished reading stage st (in both CTAs)
      if (lane == 0) {
        tc::mbar_arrive_u32(empty0 + 8 * st);
        tc::mbar_arrive_cluster(empty0_peer + 8 * st);
      }
    };
    float scale = 0.f;
    if (kMode == kDlogits) scale = *p.dloss / (float)*p.count;
    uint32_t stage = 0, phase = 0;
    for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
      int tm, tn;
      tile_coords(tile, tiles_m, tiles_n, tm, tn);
      const int m0 = p.row0 + tm * TM + (int)crank * BM, n0 = tn * BN;
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      uint32_t prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        while (!tc::mbar_try_wait_u32(full0 + 8 * stage, phase)) {}
        const uint64_t da = da0 + (uint64_t)(stage * (kABytes >> 4));
        const uint64_t db = db0 + (uint64_t)(stage * (kBBytes >> 4));
        tc::fence_regs(acc);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          tc::Wgmma<BN, 0, kBK ? 0 : 1>::mma(acc, da + k * (32 >> 4), db + k * kBStep, (kb > 0 || k > 0) ? 1u : 0u);
        tc::wgmma_commit();
        tc::fence_regs(acc);
        if (kb > 0) { tc::wgmma_wait<1>(); release(prev); }     // the previous stage's MMAs have retired
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      tc::wgmma_wait<0>();
      tc::fence_regs(acc);
      release(prev);                                            // the ring moves on to the next tile during this epilogue

      const int cq = n0 + 2 * (lane & 3);
      int y[2];
      bool valid[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m0 + 64 * wg + 16 * wq + (lane >> 2) + 8 * h;
        valid[h] = row < p.row0 + p.rows;
        if (kMode == kFwd || kMode == kDlogits) {
          const int t = row / p.B, b = row - t * p.B;
          const bool counted = valid[h] && (p.lengths == nullptr || t < p.lengths[b]);
          y[h] = counted ? (int)p.labels[(size_t)b * p.T + t] : -1;      // -1: an uncounted row
        }
      }
      const int row_lo = m0 + 64 * wg + 16 * wq + (lane >> 2);
      if (kMode == kFwd || kMode == kSample || kMode == kLogits) {
        // l = acc + bias; classes beyond C (C % 8 == 0: whole 8-column groups) become -inf, so the passes below skip them
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = cq + 8 * j;
          if (col < p.C) {
            const float2 b = *reinterpret_cast<const float2*>(p.bias + col);
            acc[4 * j] += b.x; acc[4 * j + 1] += b.y; acc[4 * j + 2] += b.x; acc[4 * j + 3] += b.y;
          } else {
            acc[4 * j] = acc[4 * j + 1] = acc[4 * j + 2] = acc[4 * j + 3] = -INFINITY;
          }
        }
        if (kMode == kLogits) {
          // the fp32 values kSample scores, stored (T = 1: row = batch row; rows past B are not written)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (!valid[h]) continue;
            float* lrow = p.logits + (size_t)(row_lo + 8 * h) * p.C;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const int col = cq + 8 * j;
              if (col < p.C) *reinterpret_cast<float2*>(lrow + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
          }
        } else if (kMode == kSample) {
          const bool greedy = p.inv_tau < 0.f;
          const uint32_t s = greedy ? 0u : (uint32_t)*p.step;
          const uint32_t r0 = greedy ? 0u : (uint32_t)*p.row_base;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int b = row_lo + 8 * h;                        // T = 1: row = batch row
            const bool noise = !greedy && valid[h];            // rows past B draw nothing
            float mx = -INFINITY, best = -INFINITY, lbest = 0.f;
            int arg = 0x7fffffff;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const int col = cq + 8 * j;
              const float l0 = acc[4 * j + 2 * h], l1 = acc[4 * j + 2 * h + 1];
              float s0 = l0, s1 = l1;
              if (noise && col < p.C) {
                const uint4 w = sample_words(p.seed, r0 + (uint32_t)b, s, col);   // col even: words (col & 3, col & 3 + 1)
                s0 = sample_score(l0, p.inv_tau, (col & 2) ? w.z : w.x);
                s1 = sample_score(l1, p.inv_tau, (col & 2) ? w.w : w.y);
              }
              mx = fmaxf(mx, fmaxf(l0, l1));
              if (s0 > best) { best = s0; arg = col; lbest = l0; }       // ascending columns: the smallest index wins a tie
              if (s1 > best) { best = s1; arg = col + 1; lbest = l1; }
            }
#pragma unroll
            for (int o = 1; o < 4; o <<= 1) {
              mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
              const float b2 = __shfl_xor_sync(0xffffffffu, best, o), l2 = __shfl_xor_sync(0xffffffffu, lbest, o);
              const int a2 = __shfl_xor_sync(0xffffffffu, arg, o);
              sample_take(best, arg, lbest, b2, a2, l2);
            }
            float se = 0.f;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) se += __expf(acc[4 * j + 2 * h] - mx) + __expf(acc[4 * j + 2 * h + 1] - mx);
#pragma unroll
            for (int o = 1; o < 4; o <<= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
            if (valid[h] && (lane & 3) == 0) {
              p.part[(size_t)b * tiles_n + tn] = make_float4(mx, se, best, lbest);
              p.part_arg[(size_t)b * tiles_n + tn] = arg;
            }
          }
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float mx = -INFINITY, ly = 0.f;
            int arg = 0x7fffffff;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float l = acc[4 * j + 2 * h + e];
                const int col = cq + 8 * j + e;
                if (l > mx) { mx = l; arg = col; }                // ascending columns: the smallest index wins a tie
                if (col == y[h]) ly = l;
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
            for (int j = 0; j < BN / 8; ++j) se += __expf(acc[4 * j + 2 * h] - mx) + __expf(acc[4 * j + 2 * h + 1] - mx);
#pragma unroll
            for (int o = 1; o < 4; o <<= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
            if (valid[h] && (lane & 3) == 0)
              p.part[(size_t)(row_lo + 8 * h) * tiles_n + tn] = make_float4(mx, se, __int_as_float(arg), ly);
          }
        }
      } else {
        float lse[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) lse[h] = valid[h] ? p.lse[row_lo + 8 * h] : 0.f;
        __nv_bfloat16* drow = p.dl + (size_t)(row_lo - p.row0) * p.C;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = cq + 8 * j;
          if (col < p.C) {
            const float2 b = *reinterpret_cast<const float2*>(p.bias + col);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              if (valid[h]) {
                float d0 = 0.f, d1 = 0.f;
                if (y[h] >= 0) {
                  d0 = (__expf(acc[4 * j + 2 * h] + b.x - lse[h]) - (col == y[h] ? 1.f : 0.f)) * scale;
                  d1 = (__expf(acc[4 * j + 2 * h + 1] + b.y - lse[h]) - (col + 1 == y[h] ? 1.f : 0.f)) * scale;
                }
                *reinterpret_cast<__nv_bfloat162*>(drow + (size_t)(8 * h) * p.C + col) = __floats2bfloat162_rn(d0, d1);
              }
            }
          }
        }
      }
    }
  }

  __syncthreads();
  tc::cluster_sync();                            // nobody leaves while the peer may still multicast into / arrive on its smem
}

// ---- combine ----------------------------------------------------------------------------------------------------------------
constexpr int kCombWarps = 16;                   // rows per block

struct CombineParams {
  const float4* part;          // [R, nt]
  const long long* labels;
  const int* lengths;
  float* lse;                  // [R]
  float* part_loss;            // [gridDim.x]
  int* part_ok;                // [gridDim.x]
  unsigned int* ticket;        // [1]: 0 on entry, left 0
  float* loss;
  int* correct;
  int* count;
  int R, T, B, nt;
};

// One warp per row: lane i merges class tiles i, i + 32, ... in ascending order, then the lanes merge in a fixed tree.
__global__ void __launch_bounds__(kCombWarps * 32) vocab_head_combine_kernel(const CombineParams p) {
  __shared__ float red_f[kCombWarps];
  __shared__ int red_i[kCombWarps];
  __shared__ int n_s, last_s;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // N = sum of lengths (T·B without): every block sums the B ints itself (exact, so the order does not matter)
  int N = p.T * p.B;
  if (p.lengths != nullptr) {
    if (threadIdx.x == 0) n_s = 0;
    __syncthreads();
    int s = 0;
    for (int b = threadIdx.x; b < p.B; b += blockDim.x) s += p.lengths[b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0 && s) atomicAdd(&n_s, s);
    __syncthreads();
    N = n_s;
  }
  const int row = blockIdx.x * kCombWarps + warp;
  float nll = 0.f;
  int ok = 0;
  if (row < p.R) {
    float mx = -INFINITY, se = 0.f, ly = 0.f;
    int arg = 0x7fffffff;
    for (int i = lane; i < p.nt; i += 32) {
      const float4 v = p.part[(size_t)row * p.nt + i];
      const int a = __float_as_int(v.z);
      if (v.x > mx) { se = se * __expf(mx - v.x) + v.y; mx = v.x; arg = a; }
      else se += v.y * __expf(v.x - mx);
      ly += v.w;
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, mx, o), s2 = __shfl_xor_sync(0xffffffffu, se, o);
      const int a2 = __shfl_xor_sync(0xffffffffu, arg, o);
      ly += __shfl_xor_sync(0xffffffffu, ly, o);
      const float m = fmaxf(mx, m2);
      if (m != -INFINITY) se = se * __expf(mx - m) + s2 * __expf(m2 - m);
      if (m2 > mx || (m2 == mx && a2 < arg)) arg = a2;
      mx = m;
    }
    const float lse = mx + __logf(se);
    if (lane == 0) {
      p.lse[row] = lse;
      const int t = row / p.B, b = row - t * p.B;
      if (p.lengths == nullptr || t < p.lengths[b]) {
        nll = lse - ly;
        ok = arg == (int)p.labels[(size_t)b * p.T + t] ? 1 : 0;
      }
    }
  }
  if (lane == 0) { red_f[warp] = nll; red_i[warp] = ok; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    int k = 0;
    for (int w = 0; w < kCombWarps; ++w) { s += red_f[w]; k += red_i[w]; }
    p.part_loss[blockIdx.x] = s;
    p.part_ok[blockIdx.x] = k;
    __threadfence();
    last_s = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last_s && warp == 0) {                     // the last block sums every block's partial: lane-strided, then a fixed tree
    __threadfence();
    const volatile float* pl = p.part_loss;
    const volatile int* po = p.part_ok;
    float s = 0.f;
    int k = 0;
    for (int i = lane; i < (int)gridDim.x; i += 32) { s += pl[i]; k += po[i]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); k += __shfl_xor_sync(0xffffffffu, k, o); }
    if (lane == 0) {
      *p.loss = s / (float)N;
      *p.correct = k;
      *p.count = N;
      *p.ticket = 0u;
    }
  }
}

// ---- db ---------------------------------------------------------------------------------------------------------------------
// Block (32, 8): 64 columns; thread (x, y) sums rows y, y + 8, ... of its column pair, then y = 0 adds the 8 sums in order.
__global__ void __launch_bounds__(256) vocab_head_colsum_kernel(const __nv_bfloat16* __restrict__ dl, float* __restrict__ db, int rows,
                                                                int C, int accumulate) {
  __shared__ float2 red[8][32];
  const int col = (blockIdx.x * 32 + threadIdx.x) * 2;
  float2 s = make_float2(0.f, 0.f);
  if (col < C) {
#pragma unroll 4
    for (int r = threadIdx.y; r < rows; r += 8) {
      const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dl + (size_t)r * C + col));
      s.x += v.x; s.y += v.y;
    }
  }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < C) {
    for (int y = 1; y < 8; ++y) { s.x += red[y][threadIdx.x].x; s.y += red[y][threadIdx.x].y; }
    if (accumulate) { s.x += db[col]; s.y += db[col + 1]; }
    db[col] = s.x; db[col + 1] = s.y;
  }
}

// ---- sampling: partials from stored logits, and the combine -------------------------------------------------------------
constexpr int kSampleWarps = 8;

// One warp per (row, class tile of BN): the partials of vocab_head_gemm_kernel<kSample> from fp32 logits [B, C] (bias included).
// Lane i takes the four classes 4 i + 128 k + [0, 4) of the tile, k = 0, 1: one Philox call each.
// kFilter (temperature > 0): only the classes with l >= tau[b] are scored, the others score -inf; a group of four classes with
// none kept draws no noise.  Max and sum exp still run over every class (the log-probability is under the full softmax).
template <bool kFilter>
__global__ void __launch_bounds__(kSampleWarps * 32)
vocab_sample_logits_kernel(const float* __restrict__ logits, VocabParams p) {
  const int lane = threadIdx.x & 31;
  const int tiles_n = (p.C + BN - 1) / BN;
  const int gw = blockIdx.x * kSampleWarps + (threadIdx.x >> 5);
  if (gw >= p.B * tiles_n) return;
  const int b = gw / tiles_n, tn = gw - b * tiles_n;
  const bool greedy = p.inv_tau < 0.f;
  const uint32_t s = greedy ? 0u : (uint32_t)*p.step;
  const uint32_t r0 = greedy ? 0u : (uint32_t)*p.row_base;
  float l[8], sc[8];
  if (kFilter) {
    const float tau = p.tau[b];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int c0 = tn * BN + 128 * k + 4 * lane;
      bool any = false;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        l[4 * k + i] = c0 + i < p.C ? logits[(size_t)b * p.C + c0 + i] : -INFINITY;
        any |= l[4 * k + i] >= tau;
      }
      uint4 w = make_uint4(0u, 0u, 0u, 0u);
      if (any) w = sample_words(p.seed, r0 + (uint32_t)b, s, c0);
      const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
        sc[4 * k + i] = (c0 + i < p.C && l[4 * k + i] >= tau) ? sample_score(l[4 * k + i], p.inv_tau, ws[i]) : -INFINITY;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int c0 = tn * BN + 128 * k + 4 * lane;
      uint4 w = make_uint4(0u, 0u, 0u, 0u);
      if (!greedy && c0 < p.C) w = sample_words(p.seed, r0 + (uint32_t)b, s, c0);
      const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = c0 + i;
        l[4 * k + i] = c < p.C ? logits[(size_t)b * p.C + c] : -INFINITY;
        sc[4 * k + i] = (greedy || c >= p.C) ? l[4 * k + i] : sample_score(l[4 * k + i], p.inv_tau, ws[i]);
      }
    }
  }
  float mx = -INFINITY, best = -INFINITY, lbest = 0.f;
  int arg = 0x7fffffff;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    mx = fmaxf(mx, l[i]);
    if (sc[i] > best) { best = sc[i]; arg = tn * BN + 128 * (i >> 2) + 4 * lane + (i & 3); lbest = l[i]; }
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float b2 = __shfl_xor_sync(0xffffffffu, best, o), l2 = __shfl_xor_sync(0xffffffffu, lbest, o);
    const int a2 = __shfl_xor_sync(0xffffffffu, arg, o);
    sample_take(best, arg, lbest, b2, a2, l2);
  }
  float se = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) se += __expf(l[i] - mx);
  se = ts::warp_sum(se);
  if (lane == 0) {
    p.part[(size_t)b * tiles_n + tn] = make_float4(mx, se, best, lbest);
    p.part_arg[(size_t)b * tiles_n + tn] = arg;
  }
}

// ---- the top-k / top-p threshold (definition above sample_words) --------------------------------------------------------------
// One CTA per row.  A radix select over the order-preserving u32 image of the fp32 logits, in four 8-bit passes from the top
// byte: each pass bins the candidates (the classes whose key agrees with the prefix fixed so far) by their next byte, per warp in
// shared memory with u64 integer atomics, and one warp finds the bin where the running total from the top reaches the target.
// Top-k counts classes (target k); top-p sums fixed-point masses (target ceil(p · Z), Z from the first pass) over the classes at
// or above the top-k threshold.  Integer sums: the result does not depend on the order of the atomics, the grid or the SM count.
constexpr int kSelThreads = 512;
constexpr int kSelWarps = kSelThreads / 32;

TC_DEVICE uint32_t order_key(float f) {                    // a < b <=> key(a) < key(b) for non-NaN a, b; -0 and +0 share one key
  const uint32_t u = __float_as_uint(f == 0.f ? 0.f : f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
TC_DEVICE float key_value(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }
TC_DEVICE unsigned long long mass_fixed(float l, float mx, float inv_tau) {   // exp((l - max) / t) in units of 2^-32
  return __float2ull_rn(__expf((l - mx) * inv_tau) * 0x1p32f);
}

struct SelectShared {
  unsigned long long hist[kSelWarps][256];
  unsigned long long bins[256];
  unsigned long long above, target;
  uint32_t bin, none;
};

// -> the largest key v such that the total over the candidates with key >= v (and key >= lo) reaches the target: the k-th
// largest key (mass = false, target k) or the nucleus cut (mass = true, target ceil(p · Z)).  0 if the target is out of reach.
TC_DEVICE uint32_t radix_select(const float* __restrict__ row, int C, uint32_t lo, bool mass, float mx, float inv_tau,
                                unsigned long long k, double top_p, SelectShared& sh) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t prefix = 0;
  unsigned long long above = 0, target = k;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < kSelWarps * 256; i += kSelThreads) (&sh.hist[0][0])[i] = 0ull;
    __syncthreads();
    const uint32_t hi = shift == 24 ? 0u : ~0u << (shift + 8);             // the bytes fixed by earlier passes
    for (int c = threadIdx.x; c < C; c += kSelThreads) {
      const float l = row[c];
      const uint32_t key = order_key(l);
      if (l == l && key >= lo && (key & hi) == prefix)
        atomicAdd(&sh.hist[warp][(key >> shift) & 255u], mass ? mass_fixed(l, mx, inv_tau) : 1ull);
    }
    __syncthreads();
    if (threadIdx.x < 256) {
      unsigned long long v = 0;
      for (int w = 0; w < kSelWarps; ++w) v += sh.hist[w][threadIdx.x];
      sh.bins[threadIdx.x] = v;
    }
    __syncthreads();
    if (warp == 0) {
      unsigned long long v[8], own = 0;                                    // lane i owns bins 8 i .. 8 i + 7
#pragma unroll
      for (int i = 0; i < 8; ++i) { v[i] = sh.bins[8 * lane + i]; own += v[i]; }
      unsigned long long suffix = own;                                     // the total of this lane's bins and every higher one
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_down_sync(0xffffffffu, suffix, o);
        if (lane + o < 32) suffix += t;
      }
      if (mass && shift == 24) {                                          // Z: the first pass sees every candidate
        const double z = (double)__shfl_sync(0xffffffffu, suffix, 0);
        target = (unsigned long long)ceil(top_p * z);
        if (target < 1) target = 1;
      }
      const bool mine = above + (suffix - own) < target && target <= above + suffix;
      const unsigned who = __ballot_sync(0xffffffffu, mine);
      if (who == 0u) {                                                     // out of reach (NaNs among the k): no threshold
        if (lane == 0) sh.none = 1;
      } else if (mine) {
        unsigned long long run = above + (suffix - own);
        int bin = 8 * lane;
        for (int i = 7; i >= 0; --i) {
          if (run + v[i] >= target) { bin = 8 * lane + i; break; }
          run += v[i];
        }
        sh.bin = (uint32_t)bin; sh.above = run; sh.none = 0;
      }
      if (lane == 0) sh.target = target;
    }
    __syncthreads();
    if (sh.none) return 0u;
    prefix |= sh.bin << shift;
    above = sh.above;
    target = sh.target;
  }
  return prefix;
}

// tau [B]: the kept set of row b is {c : l_c >= tau[b]} (-inf: every class).  top_k 0 or >= C and top_p >= 1 are off.
__global__ void __launch_bounds__(kSelThreads)
vocab_threshold_kernel(const float* __restrict__ logits, int C, int top_k, double top_p, float inv_tau, float* __restrict__ tau) {
  __shared__ SelectShared sh;
  __shared__ uint32_t red[kSelWarps];
  const float* row = logits + (size_t)blockIdx.x * C;
  uint32_t lo = 0;
  if (top_k > 0 && top_k < C) lo = radix_select(row, C, 0u, false, 0.f, 0.f, (unsigned long long)top_k, 1.0, sh);
  if (top_p < 1.0) {
    uint32_t m = 0;                                                       // the row's largest (non-NaN) key
    for (int c = threadIdx.x; c < C; c += kSelThreads) {
      const float l = row[c];
      if (l == l) m = max(m, order_key(l));
    }
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = 0;
    for (int w = 0; w < kSelWarps; ++w) m = max(m, red[w]);
    const float mx = key_value(m);
    if (isfinite(mx)) lo = radix_select(row, C, lo, true, mx, inv_tau, 0ull, top_p, sh);
  }
  if (threadIdx.x == 0) tau[blockIdx.x] = lo <= order_key(-INFINITY) ? -INFINITY : key_value(lo);
}

struct SampleCombineParams {
  const float4* part;          // [B, nt] {max, sum exp, best score, logit at it}
  const int* part_arg;         // [B, nt]
  int* step;                   // [1]: read by every block, advanced by the last one
  unsigned int* ticket;        // [1]: 0 on entry, left 0
  int* tokens;                 // [B]
  float* logprob;              // [B]
  int* rec_tok;                // [B, N] or null: column step - s0 gets the token
  float* rec_lp;               // [B, N] or null
  int N, s0, B, nt;
};

// One warp per row: lane i merges class tiles i, i + 32, ... in ascending order, then the lanes merge in a fixed tree (the
// smaller class wins a tie of the best score).  Two calls on the same partials give the same bits.
__global__ void __launch_bounds__(kCombWarps * 32) vocab_sample_combine_kernel(const SampleCombineParams p) {
  __shared__ int last_s;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int s = *(volatile const int*)p.step;
  const int row = blockIdx.x * kCombWarps + warp;
  if (row < p.B) {
    float mx = -INFINITY, se = 0.f, best = -INFINITY, lbest = 0.f;
    int arg = 0x7fffffff;
    for (int i = lane; i < p.nt; i += 32) {
      const float4 v = p.part[(size_t)row * p.nt + i];
      if (v.x > mx) { se = se * __expf(mx - v.x) + v.y; mx = v.x; }
      else se += v.y * __expf(v.x - mx);
      if (v.z > best) { best = v.z; arg = p.part_arg[(size_t)row * p.nt + i]; lbest = v.w; }
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, mx, o), s2 = __shfl_xor_sync(0xffffffffu, se, o);
      const float m = fmaxf(mx, m2);
      if (m != -INFINITY) se = se * __expf(mx - m) + s2 * __expf(m2 - m);
      mx = m;
      const float b2 = __shfl_xor_sync(0xffffffffu, best, o), l2 = __shfl_xor_sync(0xffffffffu, lbest, o);
      const int a2 = __shfl_xor_sync(0xffffffffu, arg, o);
      sample_take(best, arg, lbest, b2, a2, l2);
    }
    if (lane == 0) {
      // (l - max) - log(sum), the log in fp64 (one per row): lbest - (max + __logf(sum)) rounded at the magnitude of the max and
      // lost every log-probability below half an ulp of it, and __logf's absolute error near sum = 1 is ten times the rest
      // (tests/test_gpu_head_edges.py::test_sample, spread regime: log p = -1.1e-7 at max 2008 came out as 0)
      const float lp = (lbest - mx) - ts::logf_acc(se);
      p.tokens[row] = arg;
      p.logprob[row] = lp;
      const int col = s - p.s0;
      if (p.rec_tok != nullptr && col >= 0 && col < p.N) {
        p.rec_tok[(size_t)row * p.N + col] = arg;
        p.rec_lp[(size_t)row * p.N + col] = lp;
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last_s = atomicAdd(p.ticket, 1u) == gridDim.x - 1;         // every block has read the step before the last one advances it
  }
  __syncthreads();
  if (last_s && threadIdx.x == 0) {
    *p.step = s + 1;
    *p.ticket = 0u;
  }
}

int launch_sample_combine(const VocabParams& v, unsigned int* ticket, int* tokens, float* logprob, int* rec_tok, float* rec_lp,
                          int N, int s0, cudaStream_t st) {
  SampleCombineParams c{v.part, v.part_arg, const_cast<int*>(v.step), ticket, tokens, logprob, rec_tok, rec_lp, N, s0, v.B,
                        (v.C + BN - 1) / BN};
  vocab_sample_combine_kernel<<<(v.B + kCombWarps - 1) / kCombWarps, kCombWarps * 32, 0, st>>>(c);
  return (int)cudaGetLastError();
}

VocabParams sample_params(const float* bias, void* part, int* part_arg, int* step, const int* row_base, unsigned int seed,
                          float temperature, int B, int H, int C) {
  VocabParams p{};
  p.bias = bias; p.part = reinterpret_cast<float4*>(part); p.part_arg = part_arg; p.step = step; p.row_base = row_base;
  p.seed = seed; p.inv_tau = temperature > 0.f ? 1.0f / temperature : -1.f;
  p.R = B; p.H = H; p.C = C; p.T = 1; p.B = B; p.row0 = 0; p.rows = B;
  return p;
}

template <int kMode, bool kBK>
int launch_gemm_b(const void* h, const void* Wb, const VocabParams& p, int dev, cudaStream_t st) {
  if (p.H % BK != 0 || p.C % 8 != 0 || p.C < 8 || p.rows < 1) { ts::set_last_error("vocab head: needs H % 64 == 0 and C % 8 == 0"); return -2; }
  if (kBK && reinterpret_cast<uintptr_t>(Wb) % 16 != 0) { ts::set_last_error("vocab head: the K-major table must be 16-byte aligned"); return -2; }
  CUtensorMap th, tw;
  if (int rc = ts::make_tmap_2d_bf16(&th, h, (uint64_t)p.R, (uint64_t)p.H, (uint64_t)p.H, BK, BM)) return rc;
  if (kBK) { if (int rc = ts::make_tmap_2d_bf16(&tw, Wb, (uint64_t)p.C, (uint64_t)p.H, (uint64_t)p.H, BK, BN / kCtas)) return rc; }
  else     { if (int rc = ts::make_tmap_2d_bf16(&tw, Wb, (uint64_t)p.H, (uint64_t)p.C, (uint64_t)p.C, 64, BK)) return rc; }
  auto kern = vocab_head_gemm_kernel<kMode, kBK>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  const int tiles = ((p.rows + TM - 1) / TM) * ((p.C + BN - 1) / BN);
  int clusters = ts::sm_count(dev) / kCtas;
  if (clusters < 1) clusters = 1;
  if (tiles < clusters) clusters = tiles;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(clusters * kCtas); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = kSmemBytes; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = kCtas; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return (int)cudaLaunchKernelEx(&cfg, kern, th, tw, p);
}

// w_kmajor: Wb is the table [C, H] (tied embeddings), else W [H, C]
template <int kMode>
int launch_gemm(const void* h, const void* Wb, int w_kmajor, const VocabParams& p, int dev, cudaStream_t st) {
  return w_kmajor ? launch_gemm_b<kMode, true>(h, Wb, p, dev, st) : launch_gemm_b<kMode, false>(h, Wb, p, dev, st);
}

}  // namespace

// Scratch of the forward: part = float4 [R, ts_vocab_head_parts(C)]; part_loss / part_ok = [ts_vocab_head_blocks(R)]; 1 zeroed
// ticket word (left zeroed).
extern "C" int ts_vocab_head_parts(int C) { return (C + BN - 1) / BN; }
extern "C" int ts_vocab_head_blocks(int R) { return (R + kCombWarps - 1) / kCombWarps; }

// h: bf16 [R = T·B, H] packed time-major rows, Wb: bf16 [H, C] packed (w_kmajor: the table [C, H] packed, 16-byte aligned),
// labels int64 [B, T], lengths int32 [B] or null.
// -> lse [R], loss (mean NLL over the counted rows), correct, count (N) [1] each.
extern "C" int ts_vocab_head_fwd(const void* h, const void* Wb, int w_kmajor, const float* bias, const long long* labels, const int* lengths,
                                 void* part, float* lse, float* part_loss, int* part_ok, unsigned int* ticket, float* loss,
                                 int* correct, int* count, int T, int B, int H, int C, int dev, cudaStream_t st) {
  const int R = T * B;
  VocabParams p{};
  p.bias = bias; p.labels = labels; p.lengths = lengths; p.part = reinterpret_cast<float4*>(part);
  p.R = R; p.H = H; p.C = C; p.T = T; p.B = B; p.row0 = 0; p.rows = R;
  if (int rc = launch_gemm<kFwd>(h, Wb, w_kmajor, p, dev, st)) return rc;
  CombineParams c{reinterpret_cast<const float4*>(part), labels, lengths, lse, part_loss, part_ok, ticket, loss, correct, count,
                  R, T, B, ts_vocab_head_parts(C)};
  vocab_head_combine_kernel<<<ts_vocab_head_blocks(R), kCombWarps * 32, 0, st>>>(c);
  return (int)cudaGetLastError();
}

// dl [rows, C] bf16 = dlogits of rows [row0, row0 + rows) of h (see the top of the file); lse / count from the forward.
extern "C" int ts_vocab_head_dlogits(const void* h, const void* Wb, int w_kmajor, const float* bias, const long long* labels, const int* lengths,
                                     const float* lse, const float* dloss, const int* count, void* dl, int T, int B, int H, int C,
                                     int row0, int rows, int dev, cudaStream_t st) {
  VocabParams p{};
  p.bias = bias; p.labels = labels; p.lengths = lengths; p.lse = lse; p.dloss = dloss; p.count = count;
  p.dl = reinterpret_cast<__nv_bfloat16*>(dl);
  p.R = T * B; p.H = H; p.C = C; p.T = T; p.B = B; p.row0 = row0; p.rows = rows;
  if (row0 < 0 || row0 % BM != 0 || row0 + rows > p.R) { ts::set_last_error("vocab head: a chunk starts at a multiple of 128 rows inside h"); return -2; }
  return launch_gemm<kDlogits>(h, Wb, w_kmajor, p, dev, st);
}

// db [C] (+)= column sums of dl [rows, C] (bf16), C even.
extern "C" int ts_vocab_head_colsum(const void* dl, float* db, int rows, int C, int accumulate, cudaStream_t st) {
  vocab_head_colsum_kernel<<<(C + 63) / 64, dim3(32, 8), 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(dl), db, rows, C, accumulate);
  return (int)cudaGetLastError();
}

// Sampling (see sample_score above): h bf16 [B, H], Wb bf16 [H, C] (w_kmajor: [C, H]), bias fp32 [C]; part float4 [B, ts_vocab_head_parts(C)],
// part_arg int [B, ts_vocab_head_parts(C)], 1 zeroed ticket word (left zeroed); step int [1], advanced by one; row_base int [1],
// the noise counter's row word of row 0.
// -> tokens [B], logprob [B], and with rec_tok / rec_lp [B, N] column step - s0 of each.
extern "C" int ts_vocab_sample(const void* h, const void* Wb, int w_kmajor, const float* bias, float temperature, unsigned int seed, int* step,
                               const int* row_base, void* part, int* part_arg, unsigned int* ticket, int* tokens, float* logprob, int* rec_tok,
                               float* rec_lp, int N, int s0, int B, int H, int C, int dev, cudaStream_t st) {
  const VocabParams p = sample_params(bias, part, part_arg, step, row_base, seed, temperature, B, H, C);
  if (int rc = launch_gemm<kSample>(h, Wb, w_kmajor, p, dev, st)) return rc;
  return launch_sample_combine(p, ticket, tokens, logprob, rec_tok, rec_lp, N, s0, st);
}

// The same from stored fp32 logits [B, C] (bias included): the inputs vocab_head_gemm_kernel does not take, and top-k / top-p.
// tau [B] or null: with tau (temperature > 0) only the classes with l >= tau[b] are candidates.
extern "C" int ts_vocab_sample_logits(const float* logits, const float* tau, float temperature, unsigned int seed, int* step,
                                      const int* row_base, void* part, int* part_arg,
                                      unsigned int* ticket, int* tokens, float* logprob, int* rec_tok, float* rec_lp, int N, int s0,
                                      int B, int C, cudaStream_t st) {
  VocabParams p = sample_params(nullptr, part, part_arg, step, row_base, seed, temperature, B, 0, C);
  p.tau = tau;
  const int warps = B * ts_vocab_head_parts(C);
  const dim3 grid((warps + kSampleWarps - 1) / kSampleWarps);
  if (tau != nullptr) vocab_sample_logits_kernel<true><<<grid, kSampleWarps * 32, 0, st>>>(logits, p);
  else vocab_sample_logits_kernel<false><<<grid, kSampleWarps * 32, 0, st>>>(logits, p);
  if (cudaError_t e = cudaGetLastError()) return (int)e;
  return launch_sample_combine(p, ticket, tokens, logprob, rec_tok, rec_lp, N, s0, st);
}

// logits fp32 [B, C] = h [B, H] · W + bias through the sampling kernel's main loop (vocab_head_gemm_kernel<kLogits>): the same
// fp32 values ts_vocab_sample scores.  Same operand conditions as ts_vocab_sample.
extern "C" int ts_vocab_head_logits(const void* h, const void* Wb, int w_kmajor, const float* bias, float* logits, int B, int H, int C,
                                    int dev, cudaStream_t st) {
  VocabParams p = sample_params(bias, nullptr, nullptr, nullptr, nullptr, 0u, 0.f, B, H, C);
  p.logits = logits;
  return launch_gemm<kLogits>(h, Wb, w_kmajor, p, dev, st);
}

// tau [B] of the top-k / top-p filter (definition above sample_words) from fp32 logits [B, C] at temperature > 0.
extern "C" int ts_vocab_threshold(const float* logits, int B, int C, int top_k, double top_p, float temperature, float* tau,
                                  cudaStream_t st) {
  vocab_threshold_kernel<<<B, kSelThreads, 0, st>>>(logits, C, top_k, top_p, 1.0f / temperature, tau);
  return (int)cudaGetLastError();
}
