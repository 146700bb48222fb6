// General wgmma GEMM for every hoisted (non-recurrent) matrix product of the training step:
//
//     C[M,N] (=|+=)  op(A)[M,K] · op(B)[K,N]  (+ bias[N]),   bf16 operands, fp32 accumulation in registers, bf16 or fp32 output
//
//   * K-major or MN-major operands, chosen per operand: the weight-gradient products dW = dG^T · X contract over the
//     T·B rows of two row-major activations, i.e. BOTH operands are MN-major ("NT" GEMM); they are read straight out of
//     the [T·B, 4H] / [T·B, D] tensors the recurrence kernels wrote - no transposed copies.  dX = dG · W_x reads
//     W_x [4H, D] as an MN-major B operand (no W^T copy), the input projection is the plain TN case.
//   * A CTA computes a 128 x BN tile: two consumer warpgroups, 64 rows each (wgmma m64nBNk16), fed by a TMA producer warp
//     through a ring of 128B-swizzled stages.  kCtas = 2: a thread-block cluster of two CTAs computes a 256 x BN tile; each
//     CTA loads its own 128 rows of A and HALF of B, multicast into both CTAs' shared memory (half the B traffic per CTA).
//   * fp32 output can ACCUMULATE into C (beta = 1): weight gradients go straight into the flat gradient buffer.
//   * Optional dataflow gate: tile rows are only loaded once the arrival counters of their time step have reached their
//     target (the producer of A is a concurrently running persistent kernel - the layer wavefront).
//   * Optional row sums of op(A) (fp32 output): the CTAs of the first column of tiles also multiply their A stages by an
//     all-ones 64 x 8 B block (one extra m64n8k16 per k16, 1/32 of the tile's MMAs), so dW = dG^T · X brings the bias
//     gradient db = dG^T · 1 with it, summed over K in the same order - no separate column-sum pass over dG.
//
//   warp 0 : TMA producer     warps 1..3 : idle     warps 4..11 : two consumer warpgroups (wgmma + epilogue)
// Persistent, static round-robin tile schedule over min(#tiles, #SMs / kCtas) clusters.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include "hopper.cuh"
#include "tmap.h"

namespace {

constexpr int BM = 128;                     // rows per CTA (two m64 warpgroups)
constexpr int BK = 64;                      // 64 bf16 = 128 B = one swizzle atom
constexpr int kThreads = 384;
constexpr int kConsWarp0 = 4;

enum OutMode { OUT_BF16 = 0, OUT_F32 = 1, OUT_F32_ACC = 2 };

template <int kCtas, int BN> struct Cfg2 {
  static constexpr int kBNCta = BN / kCtas;                      // B columns this CTA loads (and multicasts)
  static constexpr int kABytes = BM * BK * 2;                    // 16 KB
  static constexpr int kBBytes = BN * BK * 2;                    // the whole B tile lands in every CTA
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (200 * 1024) / kStageBytes > 8 ? 8 : (200 * 1024) / kStageBytes;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 1024 /*barriers, padded to 1 KB*/
                                     + 1024 /*all-ones B block*/;
};

TC_DEVICE uint32_t cluster_ctarank2() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
TC_DEVICE void cluster_sync2() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
TC_DEVICE uint32_t mapa2(uint32_t local_smem_addr, uint32_t cta) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(cta));
  return r;
}
TC_DEVICE void mbar_arrive_cluster(uint32_t cluster_bar_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar_addr) : "memory");
}

struct Gemm2Params {
  void* C;
  const float* bias;
  int M, N, K, ldc;
  // Dataflow gate (layer wavefront): the rows of A are written by a persistent LSTM kernel that is still running.  Rows
  // [t * gate_rows_per_step, +gate_rows_per_step) belong to time step t; a tile may be loaded once ALL gate_count arrival
  // counters gate[i * gate_stride] have reached gate_base + gate_per_step * t, with t the last (gate_use_last) or first time
  // step the tile touches.  done[(row / 128) * tiles_n + tile_n]++ publishes a finished 128-row x BN output block.
  const unsigned int* gate;
  int gate_count, gate_stride, gate_base, gate_per_step, gate_rows_per_step, gate_use_last;
  long long gate_spin_limit;     // clock64 ticks before giving up (sets *gate_err)
  int* gate_err;
  unsigned int* done;
  int pdl;                       // launched as a programmatic dependent of the previous kernel (see launch2); waits for it before exiting
  int reverse_m;                 // walk the M tiles from the last to the first (the backward recurrence runs backwards in time)
  // Folded operand (a batch-major [Bsz, T, F] array read as the time-major matrix [T * Bsz, F] without a transpose pass): the
  // tensor map describes the storage as [fold = Bsz rows][T * F columns]; logical row r lives at storage row r % fold, columns
  // (r / fold) * fold_cols + [0, F).  a_fold: the K-major A operand (rows = M);  b_fold: the MN-major B operand (rows = K).
  int a_fold, b_fold, fold_cols;
  // Row sums of op(A) (see the top of the file): rowsum[m] (=|+=, rowsum_acc) sum_k op(A)[m, k]; null = none.
  float* rowsum;
  int rowsum_acc;
};

template <int kCtas, int BN, bool kAMN, bool kBMN, int kOut>
__global__ void __launch_bounds__(kThreads, 1)
gemm2_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const Gemm2Params p) {
  using C = Cfg2<kCtas, BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + C::kStages * C::kABytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::kStages * C::kStageBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + C::kStages;
  uint8_t* smem_ones = smem + C::kStages * C::kStageBytes + 1024;      // 1024-aligned: one 8 x 64 bf16 swizzle atom of 1.0

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // A kernel queued behind this one with the programmatic-dependent-launch attribute (a finished gradient bucket's fused
  // allreduce + update) may start once this grid is resident: it shares the SMs instead of waiting for the GEMM to drain.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const uint32_t crank = kCtas == 2 ? cluster_ctarank2() : 0u;
  constexpr int TM = BM * kCtas;                              // tile rows per cluster
  const int tiles_n = (p.N + BN - 1) / BN;
  const int tiles_m = (p.M + TM - 1) / TM;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = (p.K + BK - 1) / BK;
  const int cluster_id = blockIdx.x / kCtas, num_clusters = gridDim.x / kCtas;
  auto tile_m_of = [&](int tile) { const int tm = tile / tiles_n; return p.reverse_m ? tiles_m - 1 - tm : tm; };

  if (warp == 0 && lane == 0) {
    tc::prefetch_tmap(&tmap_a);
    tc::prefetch_tmap(&tmap_b);
  }
  if (warp == 1 && lane == 0) {
    // empty: every consumer warp of every CTA that reads the stage (the B half this CTA loads lands in all of them)
    for (int s = 0; s < C::kStages; ++s) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], 8 * kCtas); }
    tc::fence_barrier_init();
  }
  __syncthreads();
  if (kCtas == 2) cluster_sync2();               // the peer's barriers are initialised before anything arrives on them

  if (warp == 0) {
    // ===================================================================== TMA producer (every CTA loads its own rows)
    const uint32_t full0 = tc::smem_u32(full), empty0 = tc::smem_u32(empty);
    const uint32_t sa0 = tc::smem_u32(smem_a), sb0 = tc::smem_u32(smem_b);
    uint32_t stage = 0, phase = 0;
    bool ok = true;
    int gate_t_ok = -1;
    bool gate_dead = false;
    for (int tile = cluster_id; tile < num_tiles && ok; tile += num_clusters) {
      const int m0 = tile_m_of(tile) * TM + (int)crank * BM;
      const int n0 = (tile % tiles_n) * BN + (int)crank * C::kBNCta;
      if (p.gate != nullptr) {
        const int r0 = tile_m_of(tile) * TM, r1 = min(r0 + TM, p.M) - 1;
        const int t = (p.gate_use_last ? r1 : r0) / p.gate_rows_per_step;
        if (t != gate_t_ok && !gate_dead) {                    // tiles arrive in time order: poll once per time step and CTA
          const int target = p.gate_base + p.gate_per_step * t;
          const long long t0 = clock64();
          for (int g = lane; g < p.gate_count; g += 32) {
            const unsigned int* c = p.gate + (size_t)g * p.gate_stride;
            unsigned int v;
            while (true) {
              asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(c) : "memory");
              if ((int)v - target >= 0) break;
              if (clock64() - t0 > p.gate_spin_limit) { if (p.gate_err) atomicExch(p.gate_err, 1); ok = false; break; }
            }
          }
          ok = __all_sync(0xffffffffu, ok);
          asm volatile("fence.acq_rel.gpu;" ::: "memory");          // the producers' release -> our (TMA) reads
          asm volatile("fence.proxy.async.global;" ::: "memory");   // generic-proxy observation before async-proxy (TMA) reads
          if (!ok) { gate_dead = true; ok = true; }                 // producer died: error flag is set, finish the grid without gating
          gate_t_ok = t;
        }
      }
      // folded K-major A: the tile's 128 rows are 128 consecutive storage rows of ONE time step (fold % 128 == 0)
      const int a_col = (!kAMN && p.a_fold) ? (m0 / p.a_fold) * p.fold_cols : 0;
      const int a_row = (!kAMN && p.a_fold) ? m0 % p.a_fold : m0;
      for (int kb = 0, k0 = 0; kb < num_kb; ++kb, k0 += BK) {
        const uint32_t eb = empty0 + 8 * stage, fb = full0 + 8 * stage;
        while (!tc::mbar_try_wait_u32(eb, phase ^ 1)) {}
        if (tc::elect_one()) {
          tc::mbar_expect_tx_u32(fb, C::kStageBytes);
          const uint32_t sa = sa0 + stage * C::kABytes;
          const uint32_t sb = sb0 + stage * C::kBBytes + crank * (C::kBBytes / kCtas);   // this CTA's half of the B tile
          // folded MN-major B: the k-block's 64 rows are 64 consecutive storage rows of one time step (fold % 64 == 0)
          const int b_col = (kBMN && p.b_fold) ? (k0 / p.b_fold) * p.fold_cols : 0;
          const int b_row = (kBMN && p.b_fold) ? k0 % p.b_fold : k0;
          if (kAMN) {
#pragma unroll
            for (int j = 0; j < BM / 64; ++j) tc::tma_load_2d_u32(sa + j * 8192, &tmap_a, fb, m0 + 64 * j, k0);
          } else {
            tc::tma_load_2d_u32(sa, &tmap_a, fb, k0 + a_col, a_row);
          }
          if (kCtas == 2) {
            if (kBMN) {
#pragma unroll
              for (int j = 0; j < C::kBNCta / 64; ++j) tc::tma_load_2d_mc(sb + j * 8192, &tmap_b, fb, n0 + 64 * j + b_col, b_row, 3);
            } else {
              tc::tma_load_2d_mc(sb, &tmap_b, fb, k0, n0, 3);
            }
          } else {
            if (kBMN) {
#pragma unroll
              for (int j = 0; j < C::kBNCta / 64; ++j) tc::tma_load_2d_u32(sb + j * 8192, &tmap_b, fb, n0 + 64 * j + b_col, b_row);
            } else {
              tc::tma_load_2d_u32(sb, &tmap_b, fb, k0, n0);
            }
          }
        }
        __syncwarp();
        if (++stage == C::kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= kConsWarp0) {
    // ===================================================================== consumers: wgmma mainloop + epilogue
    const int wg = (warp - kConsWarp0) >> 2;             // rows [64 wg, +64) of the CTA's 128
    const int wq = warp & 3;                              // warp within the warpgroup
    const uint32_t full0 = tc::smem_u32(full), empty0 = tc::smem_u32(empty);
    const uint32_t empty0_peer = kCtas == 2 ? mapa2(empty0, crank ^ 1u) : 0u;
    const uint64_t da0 = kAMN ? tc::desc_mnmajor_sw128(tc::smem_u32(smem_a) + wg * 8192) : tc::desc_kmajor_sw128(tc::smem_u32(smem_a) + wg * 8192);
    const uint64_t db0 = kBMN ? tc::desc_mnmajor_sw128(tc::smem_u32(smem_b)) : tc::desc_kmajor_sw128(tc::smem_u32(smem_b));
    constexpr uint64_t kAStep = kAMN ? (2048 >> 4) : (32 >> 4);     // descriptor advance per k16
    constexpr uint64_t kBStep = kBMN ? (2048 >> 4) : (32 >> 4);
    auto release = [&](uint32_t st) {                     // this warp has finished reading stage st (in every CTA of the cluster)
      if (lane == 0) {
        tc::mbar_arrive_u32(empty0 + 8 * st);
        if (kCtas == 2) mbar_arrive_cluster(empty0_peer + 8 * st);
      }
    };
    uint32_t stage = 0, phase = 0;
    const int N = p.N, M = p.M;
    if (p.rowsum != nullptr) {                            // the all-ones B block (every byte pattern is 1.0: no swizzle to mind)
      reinterpret_cast<uint32_t*>(smem_ones)[threadIdx.x - kConsWarp0 * 32] = 0x3F803F80u;
      tc::fence_proxy_async();                            // generic-proxy stores -> wgmma (async-proxy) reads
      asm volatile("bar.sync 1, 256;" ::: "memory");
    }
    const uint64_t dones = tc::desc_kmajor_sw128(tc::smem_u32(smem_ones));
    for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
      const int m0 = tile_m_of(tile) * TM + (int)crank * BM, n0 = (tile % tiles_n) * BN;
      const bool rs = p.rowsum != nullptr && n0 == 0;     // this tile also sums its A rows
      float acc[BN / 2];
      float rsum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      uint32_t prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        while (!tc::mbar_try_wait_u32(full0 + 8 * stage, phase)) {}
        const uint64_t da = da0 + (uint64_t)(stage * (C::kABytes >> 4));
        const uint64_t db = db0 + (uint64_t)(stage * (C::kBBytes >> 4));
        tc::fence_regs(acc);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          tc::Wgmma<BN, kAMN ? 1 : 0, kBMN ? 1 : 0>::mma(acc, da + k * kAStep, db + k * kBStep, (kb > 0 || k > 0) ? 1u : 0u);
        if (rs) {
          tc::fence_regs(rsum);
#pragma unroll
          for (int k = 0; k < BK / 16; ++k)
            tc::Wgmma<8, kAMN ? 1 : 0, 0>::mma(rsum, da + k * kAStep, dones + k * (32 >> 4), (kb > 0 || k > 0) ? 1u : 0u);
        }
        tc::wgmma_commit();
        tc::fence_regs(acc);
        tc::fence_regs(rsum);
        if (kb > 0) { tc::wgmma_wait<1>(); release(prev); }     // the previous stage's MMAs have retired
        prev = stage;
        if (++stage == C::kStages) { stage = 0; phase ^= 1; }
      }
      tc::wgmma_wait<0>();
      tc::fence_regs(acc);
      tc::fence_regs(rsum);
      release(prev);
      if (rs && (lane & 3) == 0) {                        // every column of the n8 fragment holds the row sum: column 0
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m0 + 64 * wg + tc::acc_row(2 * h, wq, lane);
          if (row < M) p.rowsum[row] = rsum[2 * h] + (p.rowsum_acc ? p.rowsum[row] : 0.f);
        }
      }
      // epilogue straight from the accumulator fragments: a lane quad covers 8 consecutive columns of one row
#pragma unroll
      for (int i = 0; i < BN / 2; i += 2) {
        const int row = m0 + 64 * wg + tc::acc_row(i, wq, lane);
        const int col = n0 + tc::acc_col(i, lane);
        if (row < M && col < N) {                             // N % 8 == 0: col + 1 < N as well
          float f0 = acc[i], f1 = acc[i + 1];
          if (p.bias != nullptr) { f0 += p.bias[col]; f1 += p.bias[col + 1]; }
          if (kOut != OUT_BF16) {
            float2* dst = reinterpret_cast<float2*>(reinterpret_cast<float*>(p.C) + (size_t)row * p.ldc + col);
            if (kOut == OUT_F32_ACC) { const float2 o = *dst; f0 += o.x; f1 += o.y; }
            *dst = make_float2(f0, f1);
          } else {
            *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(p.C) + (size_t)row * p.ldc + col) =
                __floats2bfloat162_rn(f0, f1);
          }
        }
      }
      if (p.done != nullptr) {                     // publish this CTA's 128 x BN output block to the gated consumer kernel
        asm volatile("bar.sync 1, 256;" ::: "memory");           // both consumer warpgroups have issued their stores
        if (warp == kConsWarp0 && lane == 0)
          asm volatile("red.release.gpu.global.add.u32 [%0], 1;"
                       ::"l"(p.done + ((size_t)tile_m_of(tile) * kCtas + crank) * tiles_n + (tile % tiles_n)) : "memory");
      }
    }
  }

  __syncthreads();
  if (kCtas == 2) cluster_sync2();               // nobody leaves while the peer may still multicast into / arrive on its smem
  if (p.pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <int kCtas, int BN, bool kAMN, bool kBMN, int kOut>
int launch2(const void* A, const void* B, const Gemm2Params& p, int lda, int ldb, int dev, int max_ctas, cudaStream_t st) {
  using C = Cfg2<kCtas, BN>;
  CUtensorMap ta, tb;
  // K-major operand: [rows = M|N][cols = K];  MN-major operand: [rows = K][cols = M|N]
  if (kAMN) { if (int rc = ts::make_tmap_2d_bf16(&ta, A, (uint64_t)p.K, (uint64_t)p.M, (uint64_t)lda, 64, BK)) return rc; }
  else if (p.a_fold) { if (int rc = ts::make_tmap_2d_bf16(&ta, A, (uint64_t)p.a_fold, (uint64_t)(p.M / p.a_fold) * p.fold_cols, (uint64_t)lda, BK, BM)) return rc; }
  else      { if (int rc = ts::make_tmap_2d_bf16(&ta, A, (uint64_t)p.M, (uint64_t)p.K, (uint64_t)lda, BK, BM)) return rc; }
  if (kBMN && p.b_fold) { if (int rc = ts::make_tmap_2d_bf16(&tb, B, (uint64_t)p.b_fold, (uint64_t)(p.K / p.b_fold) * p.fold_cols, (uint64_t)ldb, 64, BK)) return rc; }
  else if (kBMN) { if (int rc = ts::make_tmap_2d_bf16(&tb, B, (uint64_t)p.K, (uint64_t)p.N, (uint64_t)ldb, 64, BK)) return rc; }
  else      { if (int rc = ts::make_tmap_2d_bf16(&tb, B, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)ldb, BK, C::kBNCta)) return rc; }
  auto kern = gemm2_kernel<kCtas, BN, kAMN, kBMN, kOut>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes);
    if (e != cudaSuccess) return (int)e;
    // same L1 / shared-memory split as the fused allreduce kernels: an SM only runs CTAs of two kernels at once when they
    // agree on it, and a gradient bucket's allreduce is launched (programmatic dependent) to run next to this GEMM
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    attr_set = true;
  }
  const int TM = BM * kCtas;
  const int tiles = ((p.M + TM - 1) / TM) * ((p.N + BN - 1) / BN);
  int sms = ts::sm_count(dev);
  if (max_ctas > 0 && max_ctas < sms) sms = max_ctas;
  int clusters = sms / kCtas;
  if (clusters < 1) clusters = 1;
  if (tiles < clusters) clusters = tiles;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(clusters * kCtas); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = C::kSmemBytes; cfg.stream = st;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = kCtas; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  if (p.pdl) {
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 2;
  }
  return (int)cudaLaunchKernelEx(&cfg, kern, ta, tb, p);
}

template <int kCtas, int BN, bool kAMN, bool kBMN>
int launch_out(const void* A, const void* B, const Gemm2Params& p, int lda, int ldb, int out_mode, int dev, int max_ctas, cudaStream_t st) {
  switch (out_mode) {
    case OUT_BF16: return launch2<kCtas, BN, kAMN, kBMN, OUT_BF16>(A, B, p, lda, ldb, dev, max_ctas, st);
    case OUT_F32: return launch2<kCtas, BN, kAMN, kBMN, OUT_F32>(A, B, p, lda, ldb, dev, max_ctas, st);
    case OUT_F32_ACC: return launch2<kCtas, BN, kAMN, kBMN, OUT_F32_ACC>(A, B, p, lda, ldb, dev, max_ctas, st);
  }
  return -3;
}

template <int kCtas, int BN>
int launch_major(const void* A, const void* B, const Gemm2Params& p, int lda, int ldb, int a_mn, int b_mn, int out_mode, int dev,
                 int max_ctas, cudaStream_t st) {
  if (a_mn && b_mn) return launch_out<kCtas, BN, true, true>(A, B, p, lda, ldb, out_mode, dev, max_ctas, st);
  if (a_mn) return launch_out<kCtas, BN, true, false>(A, B, p, lda, ldb, out_mode, dev, max_ctas, st);
  if (b_mn) return launch_out<kCtas, BN, false, true>(A, B, p, lda, ldb, out_mode, dev, max_ctas, st);
  return launch_out<kCtas, BN, false, false>(A, B, p, lda, ldb, out_mode, dev, max_ctas, st);
}

}  // namespace

// A: K-major [M, K] (lda = row pitch) or MN-major [K, M];  B: K-major [N, K] or MN-major [K, N];  C [M, N] row pitch ldc.
// out_mode: 0 bf16, 1 fp32, 2 fp32 accumulate (C += A·B).  ctas: 1 or 2 (cluster sharing the B tile).  bn: 128 or 256.
// gate_cfg[7] = {count, stride (u32 words), base, per_step, rows_per_step, use_last, reverse_m} (see Gemm2Params); max_ctas > 0 caps the grid.
// rowsum (fp32 [M], or null): also rowsum[m] (=|+= with rowsum_acc) the sum over K of op(A)[m, :] (fp32 output only).
extern "C" int ts_gemm2(const void* A, const void* B, void* C, const float* bias, int M, int N, int K, int lda, int ldb, int ldc,
                        int a_mn, int b_mn, int out_mode, int ctas, int bn, int dev, int max_ctas, const unsigned int* gate,
                        const int* gate_cfg, unsigned int* done, int* gate_err, int pdl, int a_fold, int b_fold, int fold_cols,
                        float* rowsum, int rowsum_acc, cudaStream_t st) {
  if (M < 1 || N < 1 || K < 1) { ts::set_last_error("gemm2: M, N and K must be positive"); return -2; }
  if (K % 8 != 0 || lda % 8 != 0 || ldb % 8 != 0) { ts::set_last_error("gemm2: K and the operand pitches must be multiples of 8"); return -2; }
  if ((a_mn && M % 8 != 0) || (b_mn && N % 8 != 0) || N % 8 != 0) { ts::set_last_error("gemm2: M (MN-major A) / N must be multiples of 8"); return -2; }
  if (out_mode != OUT_BF16 && ldc % 2 != 0) { ts::set_last_error("gemm2: fp32 output needs an even row pitch"); return -2; }
  // folded operands (see Gemm2Params): no tile / k-block may straddle two time steps or run past a time step's columns
  if (a_fold && (a_mn || gate != nullptr || a_fold % 128 != 0 || M % a_fold != 0 || K % 64 != 0 || fold_cols < K)) {
    ts::set_last_error("gemm2: folded A needs a K-major ungated operand, fold % 128 == 0, M % fold == 0, K % 64 == 0"); return -2;
  }
  if (b_fold && (!b_mn || b_fold % 64 != 0 || K % b_fold != 0 || N % bn != 0 || fold_cols < N)) {
    ts::set_last_error("gemm2: folded B needs an MN-major operand, fold % 64 == 0, K % fold == 0, N % bn == 0"); return -2;
  }
  if (rowsum != nullptr && out_mode == OUT_BF16) { ts::set_last_error("gemm2: row sums of A need an fp32 output"); return -2; }
  Gemm2Params p{};
  p.rowsum = rowsum; p.rowsum_acc = rowsum_acc;
  p.C = C; p.bias = bias; p.M = M; p.N = N; p.K = K; p.ldc = ldc;
  p.a_fold = a_fold; p.b_fold = b_fold; p.fold_cols = fold_cols;
  p.gate = gate; p.gate_err = gate_err; p.done = done; p.pdl = pdl;
  if (gate != nullptr) {
    p.gate_count = gate_cfg[0]; p.gate_stride = gate_cfg[1]; p.gate_base = gate_cfg[2]; p.gate_per_step = gate_cfg[3];
    p.gate_rows_per_step = gate_cfg[4] > 0 ? gate_cfg[4] : 1; p.gate_use_last = gate_cfg[5]; p.reverse_m = gate_cfg[6];
  }
  p.gate_spin_limit = 6000000000LL;
  if (ctas == 2) {
    if (bn == 128) return launch_major<2, 128>(A, B, p, lda, ldb, a_mn, b_mn, out_mode, dev, max_ctas, st);
    return launch_major<2, 256>(A, B, p, lda, ldb, a_mn, b_mn, out_mode, dev, max_ctas, st);
  }
  if (bn == 128) return launch_major<1, 128>(A, B, p, lda, ldb, a_mn, b_mn, out_mode, dev, max_ctas, st);
  return launch_major<1, 256>(A, B, p, lda, ldb, a_mn, b_mn, out_mode, dev, max_ctas, st);
}
