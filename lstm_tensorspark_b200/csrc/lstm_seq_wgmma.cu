// K-LSTM / K-LSTM-BWD: persistent wgmma kernels that run a whole layer's recurrence in ONE launch.
//
// What they replace (original TensorFlow model, per layer per time step): 4x matmul(ht, W_h) + bias adds + 3 sigmoid + 2 tanh +
// the c/h update, each its own op, and the mirrored autodiff backward.  The original only ever takes ONE step; these kernels
// deliver the multi-step unroll its fit_next API was built for.
//
// Design (H100, sm_90a):
//   * Every CTA keeps a bf16 slice of the recurrent weights RESIDENT in shared memory for all T steps (loaded once by
//     TMA; at H = 1024 a CTA holds 64 rows x 1024 of W_h = 128 KB).  Rows are gate-interleaved (n = 4j+g) so a CTA that
//     owns a row slice owns complete (i,f,g,o) quadruples: the gate epilogue needs no cross-CTA traffic.
//   * Per step a CTA streams a 128-row batch tile of h_{t-1} (forward) / dG_{t+1} (backward) through a bulk-copy ->
//     mbarrier ring (the operand is kept in global memory as ready-made 128B-swizzled tile images, 16 KB contiguous per
//     k-block).  Two consumer warpgroups issue wgmma (m64n64k16, bf16 -> fp32 accumulators in registers), stage the
//     accumulator through shared memory - in the ring stages they have just drained, so the ring gets that space - and do
//     the whole cell with one thread per batch row (the cell state never leaves its registers).  With one batch tile per
//     CTA the two warpgroups split its rows; with two (kTiles = 2) they PING-PONG: each warpgroup owns one tile for the whole
//     launch, so one tile's cell epilogue, exchange and dataflow signal run while the other tile's MMAs do.  At H = 1024
//     with two batch tiles per CTA the ring holds 6 stages forward, 4 backward; with one, 4 forward (pick_stages).
//   * The forward pass can split K across a cluster of 2 CTAs and the backward pass does across 4 (one gate-column quarter
//     each); the partial accumulators are reduce-scattered through DISTRIBUTED SHARED MEMORY with st.async (bytes are
//     counted on the receiver's mbarrier: no release/acquire fences).  Every member then owns 16 hidden units.
//   * Steps are not separated by a grid barrier but by DATAFLOW: every operand k-block has an arrival counter in global
//     memory (its producer CTAs: epilogue stores -> CTA barrier -> ONE red.release.gpu); the producer warp's 32 lanes poll
//     all counters of their K slice with relaxed loads and pull the blocks into the ring in arrival order (accumulation
//     order is free; the ring stage carries its k-block id to the consumers).  The consumer is the async proxy (L2),
//     so there is no acquire fence.
//   * The bookkeeping stores (h_seq / c_seq / activations for backward) are held back until the dataflow signal has left:
//     the release fence of the signal waits for every outstanding store of the SM.
//   * All CTAs are co-resident (grid <= #SMs, 1 CTA/SM, checked with cudaOccupancyMaxActiveClusters); every spin is
//     bounded and raises a sticky error flag instead of hanging the GPU.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdio.h>

#include "hopper.cuh"
#include "tmap.h"
#include "ts_common.cuh"

namespace {

constexpr int BM = 128;           // batch rows per CTA (2 x wgmma M = 64)
constexpr int BN = 64;            // accumulator columns per CTA
constexpr int BK = 64;            // K per pipeline stage (one 128 B swizzle atom of bf16)
constexpr int kMaxStages = 9;
constexpr int kEpiWarp0 = 4;
constexpr int kABytes = BM * BK * 2;          // 16 KB
constexpr int kWBlockBytes = BN * BK * 2;     // 8 KB per 64-wide K block
constexpr int kXchgBytes = 4 * BM * 16 * 2;   // backward: 4 source slots of [128 x 16] bf16 partial chunks
constexpr long long kSpinLimit = 6000000000LL;   // ~3 s of SM clocks: a bug surfaces as an error, not a hung GPU
constexpr long long kAbortGrace = 1000000000LL;  // ~0.5 s for the role loops to drain after an abort before the watchdog traps

// sync workspace (u32 words): [0,16) grid-barrier counters, [64,320) per-CTA step flags, [512 + 32 i) k-block arrival
// counters (one 128 B line each, i < tiles_m * 4H/64; seq_config rejects layouts that reach the last word), [kSyncWords-1]
// sticky error flag
constexpr int kSyncWords = 8192;
constexpr int kSyncErr = kSyncWords - 1;
constexpr int kSyncFlags = 64;
constexpr int kSyncKb = 512;

struct SeqSmem {
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
  uint64_t w_full;
  uint64_t xchg_full[2];
  uint64_t xchg_free[2];        // every cluster member has consumed its exchange buffer of the previous step (4 remote arrivals)
  uint64_t mma_turn[2];         // kTiles = 2: warpgroup h may wait for its stages of the next tile-step (4 warps of the other one)
  int abort_flag;
  int roles_done;               // role warps that have left their loops (producer, 8 consumer warps)
  uint32_t kb_idx[kMaxStages];  // which k-block sits in ring stage s (the producer fills stages in ARRIVAL order)
  float bias[64];
};

TC_DEVICE uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
TC_DEVICE void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
TC_DEVICE uint32_t mapa(uint32_t local_smem_addr, uint32_t cta) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(cta));
  return r;
}
// 16 B into a cluster member's shared memory; the bytes are accounted on ITS mbarrier (complete_tx), so the receiver needs
// no release/acquire round trip: it arms the barrier with expect_tx and waits, exactly as for a TMA load.
TC_DEVICE void st_async_u4(uint32_t remote_addr, uint4 v, uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1,%2,%3,%4}, [%5];"
               ::"r"(remote_addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(remote_bar) : "memory");
}
// "Buffer consumed" notifications carry no data: the reads they order were complete (their values used) before the CTA
// barrier that precedes the arrive.  The .release form compiles to MEMBAR.ALL.GPU + ERRBAR + CGAERRBAR - a second
// GPU-scope fence per step that competes with the one the dataflow signal needs.
TC_DEVICE void mbar_arrive_remote_relaxed(uint32_t remote_bar_addr) {
  asm volatile("mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote_bar_addr) : "memory");
}
TC_DEVICE bool mbar_try_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(tc::smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}

template <bool kClusterScope>
TC_DEVICE bool wait_bar(uint64_t* bar, uint32_t parity, volatile int* abort_flag) {
  auto probe = [&]() { return kClusterScope ? mbar_try_wait_cluster(bar, parity) : tc::mbar_try_wait(bar, parity); };
  if (probe()) return true;
  long long t0 = clock64();
  int n = 0;
  while (!probe()) {
    if ((++n & 255) == 0) {
      if (*abort_flag) return false;
      if (clock64() - t0 > kSpinLimit) { *abort_flag = 1; return false; }
    }
  }
  return true;
}

TC_DEVICE unsigned int ld_acquire_gpu(const unsigned int* ctr) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
  return v;
}
TC_DEVICE uint2 ld_relaxed_gpu_v2(const unsigned int* ctr) {
  uint2 v;
  asm volatile("ld.relaxed.gpu.global.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(ctr) : "memory");
  return v;
}
TC_DEVICE void st_release_gpu(unsigned int* ctr, unsigned int v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(ctr), "r"(v) : "memory");
}
TC_DEVICE unsigned int ld_relaxed_gpu(const unsigned int* ctr) {      // coalesces across lanes (a divergent ld.acquire does not)
  unsigned int v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
  return v;
}
TC_DEVICE void signal_counter(unsigned int* ctr) {
  asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
}
// Two-tile kernels: the second tile's per-step stamps follow the first tile's [T + 2][4] and the single-step / per-CTA stamps.
TC_DEVICE size_t dbg_tile1(int T) { return 4 * (size_t)(T + 2) + 64 + 512; }
TC_DEVICE unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

TC_DEVICE uint4 ldg_nc16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
TC_DEVICE uint4 ldg_cg16(const void* p) {          // coherent at L2: the producer is a kernel that is still running
  uint4 r;
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
// 32 contiguous bytes (one sector) as two 16 B accesses
struct alignas(32) U8 { uint32_t v[8]; };
TC_DEVICE U8 ldg_nc32(const void* p) {
  const uint4 a = ldg_nc16(p), b = ldg_nc16(reinterpret_cast<const uint8_t*>(p) + 16);
  return U8{{a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}};
}
TC_DEVICE U8 ldg_cg32(const void* p) {
  const uint4 a = ldg_cg16(p), b = ldg_cg16(reinterpret_cast<const uint8_t*>(p) + 16);
  return U8{{a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}};
}
// Wait (one lane polls, the warp follows) until the gated GEMM has published the 128 x 256 block that holds this warp's rows.
TC_DEVICE bool wait_in_gate(const unsigned int* ctr, int lane, volatile int* abort_flag) {
  int ok = 1;
  if (lane == 0) {
    long long t0 = clock64();
    int n = 0;
    while (ld_acquire_gpu(ctr) == 0u) {
      if ((++n & 63) == 0) {
        if (*abort_flag) { ok = 0; break; }
        if (clock64() - t0 > kSpinLimit) { *abort_flag = 1; ok = 0; break; }
      }
    }
  }
  ok = __shfl_sync(0xffffffffu, ok, 0);
  return ok != 0;
}
TC_DEVICE void stg16(void* p, uint4 v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
TC_DEVICE void stg32(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t e, uint32_t f, uint32_t g, uint32_t h) {
  stg16(p, make_uint4(a, b, c, d));
  stg16(reinterpret_cast<uint8_t*>(p) + 16, make_uint4(e, f, g, h));
}
TC_DEVICE void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
TC_DEVICE float bf_lo(uint32_t u) { return __uint_as_float(u << 16); }
TC_DEVICE float bf_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
TC_DEVICE uint32_t pack_bf2(float a, float b) {
  __nv_bfloat162 p = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&p);
}

struct SeqParams {
  // forward
  const __nv_bfloat16* gx;     // [T,B,4H]
  const float* bias;           // [4H]
  __nv_bfloat16* h_seq;        // [T+1,B,H]   (row 0 = h0)
  float* c_seq;                // [T+1,B,H]   (row 0 = c0)
  __nv_bfloat16* act;          // [T,B,4H]
  // backward
  const __nv_bfloat16* dh_seq; // [T,B,H] gradient into every h_t from above; null = only the final state has one (dh0 in)
  __nv_bfloat16* dpre;         // [T,B,4H]
  float* dh0;                  // [B,H] in: dL/dh_T extra, out: dL/dh_0
  float* dc0;                  // [B,H] in: dL/dc_T, out: dL/dc_0
  __nv_bfloat16* a_tiled;      // streamed operand as pre-swizzled SMEM images: [time][tiles_m][K/64][128 rows][64] (16 KB blocks)
  int tiles_m;
  int debug_mode;              // timing experiments only: 1 = skip operand loads, 2 = skip MMAs, 4 = half-size loads (garbage results), 3 = in-order stream
  unsigned int* sync;          // [63] error flag; [64 + mb * nkb + kb] arrival counter of operand k-block kb of batch tile mb
  unsigned long long* dbg;     // optional [steps][4] timestamps of CTA 0's first tile (ns); two-tile kernels: the second
                               // tile's from word dbg_tile1(T)
  int T, B, H;
  int tiles_n;                 // CTAs per batch tile
  int sync_mode;               // 0 = k-block arrival counters (dataflow), 1 = one counter per batch tile (grid barrier), 2 = per-CTA flags
  int poll_acquire;            // experiment: ld.acquire polls instead of relaxed
  // Layer wavefront (two layers' recurrences co-resident, chained through a dataflow-gated GEMM on the idle SMs):
  const unsigned int* in_gate; // completion counters of the GEMM that produces gx (fwd) / dh_seq (bwd) tile by tile while this kernel
                               // runs: [(row / 128) * in_gate_tiles_n + col / 256]; null = the operand is complete
  int in_gate_tiles_n;
  int pdl_wait;                // launched as a programmatic dependent: before exiting, wait for the grids launched before this one
                               // (completion of the chain's LAST kernel then implies completion of all of them)
  int no_trap;                 // debugging: the watchdog only records the abort (variant bit 20) instead of killing the kernel
  int extra_signal;            // one more arrival on this CTA's k-block counter after the LAST step's bookkeeping stores (a gated
                               // GEMM consumes h_seq / dpre in the natural layout, which is written after the per-step signal)
  const int* lengths;          // [B] valid steps per row (right padding, 1 <= len <= T); null = every row runs all T steps.  Read
                               // only by the kMasked instantiations: at a step t >= len the cell holds its state (h, c carried
                               // over) and the backward pass emits a zero gate gradient and passes dh / dc through unchanged.
  // Dropout between stacked layers (kDrop instantiations only): the forward pass also writes h_drop [T,B,H] (time order, mask
  // drop applied to the stored bf16 h), the backward pass applies the same mask to dh_seq as it loads it.
  __nv_bfloat16* h_drop;
  ts::DropSpec drop;
};

// Work decomposition
//   forward : CTA (mb, nb)      -> gate columns [64 nb, +64) = hidden [16 nb, +16) of batch tile mb, K = H.
//   backward: CTA (mb, nb2, ks) -> partial dh columns [64 nb2, +64) over gate-column quarter ks (K = H); the 4 ks form a
//                                 cluster; after the DSMEM reduce-scatter member ks owns hidden [64 nb2 + 16 ks, +16).
//             streamed weights (kNarrow): columns [32 nb2, +32) over gate-column half ks (K = 2H), clusters of 2; member ks
//                                 then owns hidden [32 nb2 + 16 ks, +16) - the same 16 hidden units per CTA.
// Warps: 0 = producer, 1..2 = idle, 3 = watchdog, 4..11 = two consumer warpgroups, `half` = (warp-4)/4, warp q = warp % 4.
// The producer warp runs CONVERGED and issues under elect.sync so addresses stay in uniform registers.
// kTiles = 1: warpgroup `half` computes batch rows [64 half, +64) x all accumulator columns with one wgmma per k16 (it reads
// only its half of each A tile) and stages them in shared memory; then warp q reads rows 64 half + 32 (q & 1) + lane, column
// half q >> 1: one thread = one batch row x 8 hidden units (32 accumulator columns).  The two warpgroups share the tile's
// epilogue barriers (256 threads).
// kTiles = 2 (ping-pong): the CTA serves TWO independent 128-row batch tiles with the same resident weight slice, and
// warpgroup `half` owns tile mb0 + half for the whole launch.  Per k16 it issues ONE m64n128k16 of the transposed product
// (A = the [64 gate columns x 64] weight block, B = the 128-row operand stage, 64 accumulator registers): 6 KB of shared
// memory per k16 instead of 8 KB for two m64n64k16 that each read the weight block.  It stages the whole tile (transposing
// the fragment on the way) and runs its epilogue with one thread per batch row (row
// 32 q + lane) over all 64 accumulator columns, as two passes of the 32-column body (index [column half] of the per-thread
// state).  Its barriers are its own (128 threads), so while one warpgroup is in its cell math, exchange and dataflow
// signal, the other one's MMAs keep the tensor cores busy.  The producer still fills the ring strictly in order - per step
// tile 0's k-blocks, then tile 1's - and each warpgroup waits on its own tile's stages and steps over the other's.
// setmaxnreg moves registers from warpgroup 0 (producer, idle, watchdog) to the consumers (kProducerRegs / kConsumerRegs);
// the ordered MMA turn (mma_turn, see mma_tile) keeps a warpgroup from running ahead of a stage's fills.  Half as many CTAs
// are needed (64 for B = 256, H = 1024), which leaves SMs free for the weight-gradient GEMMs that run concurrently.
//   Deadlock freedom at any ring depth >= 2: order all ring items of a CTA as the producer fills them, (step, tile, k-block).
//   Every wait an item depends on is on an EARLIER item or on other CTAs' earlier steps:
//   - the producer fills item i once items i - depth and (pairs) i + 1 - depth are released (both < i for depth >= 2), and
//     polls dataflow counters that other CTAs' epilogues of the previous step raise;
//   - a warpgroup releases an item once its MMAs have retired; the last 1-2 items of its tile-step hold the staged
//     accumulator and are released as soon as its own 4 warps have read their rows - before any wait on another CTA;
//   - backward, the warpgroup of tile m then waits for xchg_free / xchg_full of tile m: the cluster peers' MMAs of the
//     SAME (step, tile), whose items the peers' producers fill once the peers' earlier items are released;
//   - a warpgroup takes its MMA turn (mma_turn, see mma_tile) once the other warpgroup has seen its items of the preceding
//     tile-step land - earlier items again, and it holds no stage while it waits.
//   A warpgroup never holds a stage while it waits on anything outside its own 4 warps, so no cycle can form and every
//   item is eventually filled and released.  (The bounded spins and the watchdog remain as the safety net.)
// kStream = true (H too large for a resident slice, e.g. H = 2048: W_h alone is 32 MB): the weight k-block travels through
// the ring next to its operand k-block (24 KB stages, W comes out of L2 every step); everything else is unchanged.
// kFSplit (forward): a cluster of 2 CTAs splits K.  Each member contracts over HALF of h_{t-1} (8 instead of 16 operand
// k-blocks per step at H = 1024) against a [128 x H/2] weight slice, and the two partial [128 x 128] accumulators are
// reduce-scattered through DSMEM: every member ends up with the same 64 gate columns = 16 hidden units it owns in the
// unsplit kernel.  Used when the larger accumulator stage still leaves >= 3 ring stages (smaller H).
// kMasked: per-row sequence lengths (SeqParams::lengths).  A separate instantiation, so the unmasked kernels - at the register
// cap - carry no extra state; the dataflow, the exchange and the signalling are the same (a padded row still signals every step).
// kRev: the reverse-time direction of a bidirectional layer.  Forward step s processes time tau = T-1-s, the backward pass visits
// tau ascending.  The saved sequences stay in time order with the initial state in the LAST slot: h_seq / c_seq row tau < T = the
// state after processing time tau, row T = h0 / c0; act / dpre row tau = time tau.  The output is h_seq[0:T], the final state
// row 0, and dW_h pairs dpre with h_seq[1:T+1].  Only the time index of those arrays changes: the swizzled operand images
// (a_tiled), the dataflow counters and the exchange stay in processing order.  With kMasked a row's padded steps
// (tau >= len) come FIRST in the forward pass (the cell holds h0 / c0 there) and LAST in the backward pass (dh / dc carry
// through them into dh0 / dc0).  Not combined with the layer wavefront (in_gate / extra_signal; the host rejects it).
// kDrop: dropout on this layer's output sequence (SeqParams::drop).  Forward: h_drop is stored in the bookkeeping block, next to
// h_seq, so whatever gates on h_seq's natural-layout rows (the pair's gx_b GEMM, extra_signal) covers it too.  Backward: the
// dropped units of dh_seq are zeroed as it is loaded (before the MMAs of the step) and the kept ones scaled in fp32 where dh
// joins the carry.  A separate instantiation: the kernels without it are those of a build without dropout.
template <bool kBwd, int kStages, int kTiles, bool kStream, bool kFSplit = false, bool kMasked = false, bool kRev = false,
          bool kDrop = false>
__global__ void __launch_bounds__(384, 1)
lstm_seq_kernel(const __grid_constant__ CUtensorMap tmap_w, const SeqParams p) {
  static_assert(!(kFSplit && (kBwd || kStream || kTiles != 1)), "forward K-split: one tile, resident weights");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // kNarrow (streamed backward): a cluster of 2 splits K = 4H in halves, 32 accumulator columns per CTA.  Clusters of 2 pack
  // onto the GPCs where clusters of 4 do not: at H = 2048 an H100 co-schedules only 120 of the 128 CTAs in clusters of 4.
  constexpr bool kNarrow = kBwd && kStream;
  constexpr int kSplit = kBwd ? (kNarrow ? 2 : 4) : (kFSplit ? 2 : 1);     // cluster size = K-split factor
  constexpr bool kCluster = kSplit > 1;
  constexpr int kBNm = kFSplit ? 2 * BN : (kNarrow ? BN / 2 : BN);        // accumulator columns per CTA
  constexpr int kCW = kNarrow ? 16 : 32;                     // backward: accumulator columns per epilogue thread ([kCW chalf, +kCW))
  constexpr int kWBlk = kBNm * BK * 2;                       // bytes of one weight k-block
  // operand k-blocks this CTA contracts over per step (backward: K = 4H split kSplit ways)
  const int num_kb = kFSplit ? p.H / (2 * BK) : (kBwd ? 4 * p.H / (kSplit * BK) : p.H / BK);
  constexpr int kStageBytes = kStream ? kABytes + kWBlk : kABytes;
  // exchange bytes a member receives per step: backward kSplit sources x [128 rows x 16] bf16, forward K-split the peer's half
  constexpr uint32_t kXchgRecv = kBwd ? (uint32_t)(kSplit * BM * 16 * 2) : (uint32_t)kXchgBytes;
  uint8_t* smem_w = smem;                                    // resident weight slice: num_kb blocks of [kBNm x 64] (not kStream)
  uint8_t* smem_a = smem + (kStream ? 0 : (size_t)num_kb * kWBlk);    // kStages x (16 KB [+ 8 KB weight block])
  uint8_t* smem_x = smem_a + kStages * kStageBytes;          // DSMEM exchange buffer (bf16 partial sums)

  // The accumulator is staged in shared memory so that one thread can read a whole row.  One tile: a warpgroup's 64 fp32 rows
  // take kAccPieces 8 KB pieces, the A-operand halves of the ring stages it consumed last (see mma_tile).  Two tiles: a
  // warpgroup's 128 rows take whole stages, fp32 forward (2) and bf16 backward (1: every partial sum is rounded to bf16 for
  // the reduce-scatter anyway, so staging it rounded gives the same bits).  The forward K-split (32 KB per warpgroup) and a
  // tile with fewer k-blocks than pieces (H = 64) use a dedicated buffer instead (smem_bytes() sizes it for exactly these).
  constexpr bool kPP = kTiles == 2;                                           // ping-pong: warpgroup = batch tile
  constexpr int kAccRows = kPP ? BM : 64;                                     // rows a warpgroup stages
  constexpr int kAccRowBytes = kBNm * (kPP && kBwd ? 2 : 4);
  constexpr int kPieceBytes = kPP ? kABytes : kABytes / 2;
  constexpr int kAccPieces = kAccRows * kAccRowBytes / kPieceBytes;           // 2; kNarrow 1; kFSplit 4; kPP fwd 2, bwd 1
  constexpr int kAccRowsPer = kFSplit ? 64 : kPieceBytes / kAccRowBytes;      // rows per piece (kFSplit: contiguous buffer)
  const bool ring_acc = !kFSplit && num_kb >= kAccPieces;
  uint8_t* acc_s = smem_x + (kCluster ? kTiles * kXchgBytes : 0);             // dedicated staging buffer [2 x kAccRows][kBNm]
  SeqSmem* ss = reinterpret_cast<SeqSmem*>(acc_s + (ring_acc ? 0 : 2 * kAccRows * kAccRowBytes));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // Programmatic dependent launch: a kernel queued behind this one WITH the PDL attribute (the fused allreduce + update of a
  // gradient bucket that is already complete) may start once every CTA of this grid is resident - it then runs on the SMs
  // this persistent grid leaves idle instead of after it.  No effect on ordinary launches.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int mb0 = (blockIdx.x / p.tiles_n) * kTiles;          // first batch tile of this CTA
  const int in_mb = blockIdx.x % p.tiles_n;
  const uint32_t crank = kCluster ? cluster_ctarank() : 0;
  const int nb = in_mb / kSplit;                              // weight-row block of the cluster (64 rows; kFSplit: 128 rows)
  const int ks = (int)crank;                                  // K-split member
  volatile int* abort_flag = &ss->abort_flag;
  const int steps = kBwd ? p.T + 1 : p.T;                    // backward runs one extra GEMM to produce dh_0

  if (threadIdx.x == 0) {
    ss->abort_flag = 0;
    ss->roles_done = 0;
    tc::prefetch_tmap(&tmap_w);
    // a stage is consumed by 8 consumer warps, or by the 4 of the warpgroup that owns its tile (kPP)
    for (int s = 0; s < kStages; ++s) { tc::mbar_init(&ss->full[s], 1); tc::mbar_init(&ss->empty[s], kPP ? 4 : 8); }
    tc::mbar_init(&ss->w_full, 1);
    for (int i = 0; i < 2; ++i) tc::mbar_init(&ss->mma_turn[i], 4);
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&ss->xchg_full[i], 1);                   // armed locally (expect_tx = the whole 16 KB buffer), filled by st.async
      tc::mbar_init(&ss->xchg_free[i], kFSplit ? 1 : kSplit);   // remote arrivals: every writer of this buffer's readers
    }
    if (kCluster)
      for (int i = 0; i < kTiles; ++i) tc::mbar_expect_tx_u32(tc::smem_u32(&ss->xchg_full[i]), kXchgRecv);
    tc::fence_barrier_init();
  }
  if (!kBwd && threadIdx.x >= 64 && threadIdx.x < 128) ss->bias[threadIdx.x - 64] = p.bias[in_mb * BN + threadIdx.x - 64];
  __syncthreads();
  if (kCluster) cluster_sync_all();             // peers' mbarriers are initialised before anyone arrives remotely

  // The consumers of the two-tile and K-split kernels hold 64 accumulator registers per thread: setmaxnreg moves registers
  // from warpgroup 0 to them.  All four warps of a warpgroup execute it at one place (warpgroup 0: idle warps too), at the
  // top of the warpgroup's branch so that the compiler allocates the branch's registers against the new limit.
  constexpr bool kRegSplit = kPP || kFSplit;
  constexpr int kProducerRegs = kPP && !kBwd ? 64 : 56;      // (168 - kProducerRegs) * 128 = (kConsumerRegs - 168) * 256
  constexpr int kConsumerRegs = kPP && !kBwd ? 216 : 224;    // the backward consumers need the most, the forward producer more
  if (warp < kEpiWarp0) {
    if constexpr (kRegSplit) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs) : "memory");
    if (warp == 0) {
      // ======================================================================== producer
      const uint32_t w_bar = tc::smem_u32(&ss->w_full);
      if (!kStream && tc::elect_one()) {
        tc::mbar_expect_tx_u32(w_bar, (uint32_t)(num_kb * kWBlk));
        // forward: rows = gate columns [kBNm nb, +kBNm) of W_h [4H, H] (K-split: K offset = half ks).  backward: rows = hidden
        // columns [64 nb, +64) of W_h^T [H, 4H], K offset = quarter ks.
        for (int kb = 0; kb < num_kb; ++kb)
          tc::tma_load_2d_u32(tc::smem_u32(smem_w) + kb * kWBlk, &tmap_w, w_bar, ks * num_kb * BK + kb * BK, nb * kBNm);
      }
      __syncwarp();
      const uint32_t full0 = tc::smem_u32(&ss->full[0]), empty0 = tc::smem_u32(&ss->empty[0]), a0 = tc::smem_u32(smem_a);
      const int nkb_all = kSplit * num_kb;
      uint32_t stage = 0, phase = 0;
      bool ok = true;
      // one k-block: the operand is a contiguous 16 KB block = the 128B-swizzled K-major [128 x 64] tile image written by
      // the epilogues (no tensor map, no coordinates)
      const int wc0 = ks * num_kb * BK, wc1 = nb * kBNm;        // weight tensor-map coordinates of this CTA's slice
      uint32_t a_bytes = kABytes;                               // a partial batch tile only needs its first rows (8-row swizzle atoms)
      auto issue = [&](uint32_t st_, const __nv_bfloat16* src, int kb) {   // elected lane: fill ring stage st_ with k-block kb
        const uint32_t fb = full0 + 8 * st_;
        ss->kb_idx[st_] = (uint32_t)kb;                         // published by the release of the expect_tx arrive below
        if (p.debug_mode == 1) { tc::mbar_arrive(&ss->full[st_]); return; }
        tc::mbar_expect_tx_u32(fb, a_bytes + (kStream ? kWBlk : 0));
        tc::bulk_load_1d_u32(a0 + st_ * kStageBytes, src + (size_t)kb * (BM * BK), a_bytes, fb);
        if (kStream) tc::tma_load_2d_u32(a0 + st_ * kStageBytes + kABytes, &tmap_w, fb, wc0 + kb * BK, wc1);
      };
      auto load_block = [&](const __nv_bfloat16* src, int kb) -> bool {
        if (!tc::mbar_try_wait_u32(empty0 + 8 * stage, phase ^ 1)) {
          if (!wait_bar<false>(&ss->empty[stage], phase ^ 1, abort_flag)) return false;
        }
        if (tc::elect_one()) issue(stage, src, kb);
        __syncwarp();
        if (++stage == kStages) { stage = 0; phase ^= 1; }
        return true;
      };
      // two k-blocks per turn (both empty-barrier try_waits in flight together, two copies issued back to back)
      auto load_pair = [&](const __nv_bfloat16* src, int kb_a, int kb_b) -> bool {
        uint32_t s1 = stage + 1, ph1 = phase;
        if (s1 == kStages) { s1 = 0; ph1 ^= 1; }
        const bool r0 = tc::mbar_try_wait_u32(empty0 + 8 * stage, phase ^ 1);
        const bool r1 = tc::mbar_try_wait_u32(empty0 + 8 * s1, ph1 ^ 1);
        if (!r0 && !wait_bar<false>(&ss->empty[stage], phase ^ 1, abort_flag)) return false;
        if (!r1 && !wait_bar<false>(&ss->empty[s1], ph1 ^ 1, abort_flag)) return false;
        if (tc::elect_one()) {
          issue(stage, src, kb_a);
          issue(s1, src, kb_b);
        }
        __syncwarp();
        stage = s1 + 1; phase = ph1;
        if (stage == kStages) { stage = 0; phase ^= 1; }
        return true;
      };
      // Dataflow instead of a grid barrier: every operand k-block (64 columns of h_{t-1} / dG_{t+1}) has its own arrival
      // counter; the 32 lanes poll all of them at once and the blocks are pulled into the ring in the order in which their
      // producer CTAs finish, so the stream and the MMAs start under the stragglers' epilogues (accumulation order is free).
      const unsigned int per_step = kBwd ? 1u : 4u;             // arrivals per k-block and step (bwd: 1 CTA, fwd: 4 CTAs x 16 hidden)
      const uint64_t all_kb = num_kb >= 64 ? ~0ull : ((1ull << num_kb) - 1ull);
      for (int s = kBwd ? 1 : 0; s < steps && ok; ++s) {
        const int tsl = kBwd ? p.T - s : s;       // forward step s consumes h_seq[s]; backward iteration s consumes dG[T-s]
        for (int tile = 0; tile < kTiles && ok; ++tile) {
          const int mb = mb0 + tile;
          const int kb_base = ks * num_kb;
          const __nv_bfloat16* src = p.a_tiled + (((size_t)tsl * p.tiles_m + mb) * nkb_all + kb_base) * (BM * BK);
          const unsigned int* ctr = p.sync + kSyncKb + ((size_t)mb * nkb_all + kb_base) * 32;
          const unsigned int target = (unsigned)s * per_step;
          {
            const int rows = p.B - mb * BM;                     // rows beyond B are never read back from the accumulator
            a_bytes = rows >= BM ? kABytes : (uint32_t)(((rows + 7) / 8) * 8 * BK * 2);
            if (p.debug_mode == 4) a_bytes = kABytes / 2;       // experiment: half the operand traffic (results are garbage)
          }
          uint64_t pending = all_kb;
          const long long t0 = clock64();
          int spins = 0;
          bool stamped = false;
          while (pending && ok) {
            uint64_t ready = pending;
            if (s > 0) {
              if (p.sync_mode == 1) {
                const unsigned int v = p.poll_acquire ? ld_acquire_gpu(p.sync + mb) : ld_relaxed_gpu(p.sync + mb);
                ready = ((int)(v - (unsigned)s * (unsigned)p.tiles_n) >= 0) ? pending : 0ull;
              } else if (p.sync_mode == 2) {
                const unsigned int* fl = p.sync + kSyncFlags + (size_t)mb * p.tiles_n;
                if (kBwd) {                                       // k-block kb_base + lane is written by CTA kb_base + lane
                  bool r0 = false;
                  if (lane < num_kb) r0 = (int)(ld_relaxed_gpu(fl + kb_base + lane) - (unsigned)s) >= 0;
                  ready = (uint64_t)__ballot_sync(0xffffffffu, r0);
                } else {                                          // k-block j is written by CTAs 4j..4j+3; lane L reads flags 2L, 2L+1
                  bool r0 = false;
                  if (2 * lane < p.tiles_n) {
                    const uint2 v2 = ld_relaxed_gpu_v2(fl + 2 * lane);
                    r0 = ((int)(v2.x - (unsigned)s) >= 0) && ((int)(v2.y - (unsigned)s) >= 0);
                  }
                  const unsigned int b = __ballot_sync(0xffffffffu, r0);
                  unsigned int pr = b & (b >> 1) & 0x55555555u;   // bit 2j set <=> k-block j complete
                  pr = (pr | (pr >> 1)) & 0x33333333u; pr = (pr | (pr >> 2)) & 0x0f0f0f0fu;
                  pr = (pr | (pr >> 4)) & 0x00ff00ffu; pr = (pr | (pr >> 8)) & 0x0000ffffu;
                  ready = pr >> kb_base;
                }
              } else {
                bool r0 = false, r1 = false;
                if (lane < num_kb) r0 = (int)(ld_relaxed_gpu(ctr + lane * 32) - target) >= 0;
                if (lane + 32 < num_kb) r1 = (int)(ld_relaxed_gpu(ctr + (lane + 32) * 32) - target) >= 0;
                ready = (uint64_t)__ballot_sync(0xffffffffu, r0) | ((uint64_t)__ballot_sync(0xffffffffu, r1) << 32);
              }
              ready &= pending;
              if (p.debug_mode == 3) {                            // experiment: in-order issue (lowest pending block first)
                const uint64_t low = pending & (~pending + 1ull);
                ready = (ready & low) ? low : 0ull;
              }
              if (!ready) {
                if ((++spins & 63) == 0) {
                  if (*abort_flag) { ok = false; break; }
                  if (clock64() - t0 > kSpinLimit) { *abort_flag = 1; ok = false; break; }
                }
                continue;
              }
              // The producers' release made the tile image visible at L2 before the counter moved, and the only consumer is the
              // async proxy (bulk copies read L2, issued after this control dependency): a generic-proxy acquire fence here
              // costs an L2 round trip per batch of blocks and buys nothing.  The warp barrier orders polling lanes before the
              // elected lane, the proxy fence orders generic observations before the async-proxy reads.
              __syncwarp();
              asm volatile("fence.proxy.async.global;" ::: "memory");
            }
            if (p.dbg && blockIdx.x == 0 && lane == 0 && (tile == 0 || kPP) && !stamped) {
              p.dbg[(tile ? dbg_tile1(p.T) : 0) + 4 * s + 0] = gtime();
              stamped = true;
            }
            pending &= ~ready;
            while (ready && ok) {
              const int ka = __ffsll((long long)ready) - 1;
              ready &= ready - 1ull;
              if (ready) {
                const int kb2 = __ffsll((long long)ready) - 1;
                ready &= ready - 1ull;
                ok = load_pair(src, ka, kb2);
              } else {
                ok = load_block(src, ka);
              }
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) atomicAdd(&ss->roles_done, 1);
    } else if (warp == 3) {
      // ======================================================================== watchdog
      // A bounded spin that times out raises abort_flag and every role loop drains.  A thread already parked in a named
      // barrier (bar.sync cannot time out) would keep the grid alive forever: if the roles have not all left within the
      // grace period after an abort, kill the kernel (launch failure in the host process) instead of hanging the GPU.
      long long t_abort = 0;
      while (*reinterpret_cast<volatile int*>(&ss->roles_done) < 9) {
        __nanosleep(4000);
        if (*abort_flag) {
          if (t_abort == 0) t_abort = clock64();
          else if (clock64() - t_abort > kAbortGrace) {
            if (lane == 0) atomicExch(reinterpret_cast<int*>(p.sync + kSyncErr), 2);
            __threadfence_system();
            if (!p.no_trap) __trap();
            break;
          }
        }
      }
    }
  } else {
    if constexpr (kRegSplit) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs) : "memory");
    // ======================================================================== consumers (8 warps; kPP: warpgroup = batch tile)
    const int ewi = warp - kEpiWarp0;
    const int quarter = ewi & 3, half = ewi >> 2;
    // epilogue thread: row rl of the rows its warpgroup staged (= batch row rloc of the tile).  One tile: the warpgroup's 64 rows,
    // accumulator column half `chalf`.  kPP: the tile's 128 rows, both column halves (pass u = column half u).
    const int rl = kPP ? 32 * quarter + lane : 32 * (quarter & 1) + lane, chalf = kPP ? 0 : quarter >> 1;
    const int rloc = kPP ? rl : 64 * half + rl;
    const int etid = ewi * 32 + lane;
    const int gtid = kPP ? etid & 127 : etid;          // index among the threads that serve this thread's tile
    const int mb = mb0 + (kPP ? half : 0);             // this thread's batch tile
    const int row = mb * BM + rloc;
    const bool valid = row < p.B;                      // rows beyond B are computed (the operand is zero there) but never stored
    constexpr int kPass = kPP ? 2 : 1;                 // 32-column passes of the epilogue body per thread
    auto ch = [&](int u) { return kPP ? u : chalf; };  // accumulator column half of pass u
    const int H = p.H, B = p.B;
    bool ok = true;
    // wgmma over one batch tile's operand k-blocks of the current step (ring order; the stage carries its k-block id): rows
    // [64 half, +64) (kPP: all 128 rows, two m64 MMAs) x all kBNm accumulator columns, m64 x kBNm x k16, then staged in shared
    // memory so that every thread can read its own row.
    const uint32_t full0 = tc::smem_u32(&ss->full[0]), empty0 = tc::smem_u32(&ss->empty[0]);
    const uint64_t desc_a0 = tc::desc_kmajor_sw128(tc::smem_u32(smem_a));      // + stage * (kStageBytes >> 4)
    const uint64_t desc_w0 = tc::desc_kmajor_sw128(tc::smem_u32(smem_w));      // + kb * (kWBlk >> 4)
    uint32_t stage = 0, phase = 0;
    // kPP: the ring holds, per step, tile 0's num_kb k-blocks and then tile 1's.  A warpgroup steps over the other tile's.
    auto skip_tile = [&]() {
      const uint32_t adv = stage + (uint32_t)num_kb;
      stage = adv % kStages;
      phase ^= (adv / kStages) & 1u;
    };
    if (kPP && half == 1) skip_tile();
    // Ring staging: the tile's last kAccPieces stages (the ones `stage` has just moved past) hold the staged rows, piece i =
    // rows [i kAccRowsPer, +kAccRowsPer), and receive this warp's empty arrival only once it has read its row.
    auto stage_back = [&](int back) -> uint32_t { return stage >= (uint32_t)back ? stage - back : stage + kStages - back; };
    auto acc_row_ptr = [&](int r) -> uint8_t* {          // staged row r of this warpgroup's kAccRows (a warp's rows share one piece)
      uint8_t* pc = ring_acc ? smem_a + stage_back(kAccPieces - r / kAccRowsPer) * kStageBytes + (kPP ? 0 : half * (kABytes / 2))
                             : acc_s + (half * kAccRows + r / kAccRowsPer * kAccRowsPer) * kAccRowBytes;
      return pc + (r % kAccRowsPer) * kAccRowBytes;
    };
    // 16 B chunk q of a staged row r sits at q ^ (r & 7) (conflict-free row-per-thread reads); fp32 column c / bf16 pair c / 2
    auto acc_swz = [](int r, int c) { return ((((c >> 2) ^ r) & 7) | ((c >> 2) & ~7)) * 4 + (c & 3); };
    auto wg_bar = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(3 + half) : "memory"); };
    // per-step stamps of CTA 0: slot 0 first block ready (producer), 1 accumulator ready, 2 signal sent, 3 MMA start
    const bool dbg_wg = p.dbg && blockIdx.x == 0 && gtid == 0;
    auto dbg_stamp = [&](int step, int slot) { p.dbg[(kPP && half ? dbg_tile1(p.T) : 0) + 4 * step + slot] = gtime(); };
    auto mma_tile = [&](int dstep) -> bool {
      // kPP computes the TRANSPOSED product, D[64 gate columns][128 batch rows] = W_slice x tile^T: one m64n128k16 per k16 with
      // the weight block as A and the operand stage as B reads 6 KB of shared memory instead of the 8 KB of two m64n64k16 with
      // the weight block read twice.  acc[0] then holds gate column acc_row(i) x batch row acc_col(i).
      float acc[1][kPP ? kBNm : kBNm / 2];               // kPP: 64 x 128 over 128 threads
      // kPP: take the MMA turn.  A full barrier's parity only tells whether its LAST completed phase matches, so a warpgroup
      // must not wait for a stage's fill n before fill n - 1 - possibly the other warpgroup's - has landed.  Warpgroup 1's
      // tile-step n waits until warpgroup 0 has seen all its stages of step n, and warpgroup 0's step n + 1 until warpgroup 1
      // has seen those of step n: every earlier item of the ring has then landed.  (Bounded wait: mbarrier, not bar.sync.)
      const int turn = kBwd ? dstep - 1 : dstep;       // this warpgroup's tile-steps before this one
      if (kPP && (half == 1 || turn > 0) &&
          !wait_bar<false>(&ss->mma_turn[half], (uint32_t)((half ? turn : turn - 1) & 1), abort_flag))
        return false;
      // ring staging: the last kAccPieces stages of the tile stay borrowed (no empty arrival) until acc_release
      const int borrow = ring_acc ? kAccPieces : 0;
      uint32_t prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        if (!tc::mbar_try_wait_u32(full0 + 8 * stage, phase) && !wait_bar<false>(&ss->full[stage], phase, abort_flag)) {
          tc::wgmma_wait<0>();                           // no MMA may still be writing the accumulator when it goes out of scope
          return false;
        }
        if (kPP && dbg_wg && kb == 0) dbg_stamp(dstep, 3);     // (two-tile kernels only: the others are at the register cap)
        const uint32_t kbi = kStream ? 0u : (p.sync_mode == 1 ? (uint32_t)kb : ss->kb_idx[stage]);
        const uint64_t ds = desc_a0 + (uint64_t)(stage * (kStageBytes >> 4));
        const uint64_t dw = kStream ? ds + (uint64_t)(kABytes >> 4) : desc_w0 + (uint64_t)(kbi * (kWBlk >> 4));
        tc::fence_regs(acc[0]);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          if constexpr (kPP) {                           // A = weight block [64 x 64], B = the whole 128-row stage
            tc::Wgmma<BM, 0, 0>::mma(acc[0], dw + (uint64_t)(2 * k), ds + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1u : 0u);
          } else {                                       // A rows [64 half, +64)
            const uint64_t da = ds + (uint64_t)(half * ((kABytes / 2) >> 4));
            tc::Wgmma<kBNm, 0, 0>::mma(acc[0], da + (uint64_t)(2 * k), dw + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1u : 0u);
          }
        }
        tc::wgmma_commit();
        tc::fence_regs(acc[0]);
        // Hand a stage back once its MMAs have retired.  With >= 3 stages that is the previous one (its MMAs overlap this
        // stage's wait); with 2 the producer waits for both stages of a k-block pair, so each stage is released at once.
        if (kStages >= 3) {
          if (kb > 0) {
            tc::wgmma_wait<1>();
            if (lane == 0 && kb - 1 < num_kb - borrow) tc::mbar_arrive_u32(empty0 + 8 * prev);
          }
        } else {
          tc::wgmma_wait<0>();
          if (lane == 0 && kb < num_kb - borrow) tc::mbar_arrive_u32(empty0 + 8 * stage);
        }
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      if (kPP && lane == 0) tc::mbar_arrive(&ss->mma_turn[1 - half]);    // every stage of this tile-step has landed
      tc::wgmma_wait<0>();
      tc::fence_regs(acc[0]);
      // Ring staging: the MMAs that read the last stages have retired and only this warpgroup reads them (its A half; kPP: its
      // tile's stages), so the accumulator goes there.  The borrowed stages were refilled only after every warp had released
      // them the previous time: no reader of an earlier staging is left.
      if (!ring_acc) {
        if (kStages >= 3 && lane == 0) tc::mbar_arrive_u32(empty0 + 8 * prev);
        wg_bar();                                        // this warpgroup has read the previously staged accumulator
      }
      if constexpr (kPP) {
        // transposed fragment: element i = gate column g of batch row b; this warp's 16 gate columns of all 128 rows, rows
        // [8 (i / 4), +8) per group of four elements (one piece each).  Conflict-free: a warp's 32 stores of one element
        // index hit 4 rows x 8 columns, and the row swizzle puts each row's columns in different 16 B chunks.
        uint8_t* pb[kAccPieces];
#pragma unroll
        for (int pc = 0; pc < kAccPieces; ++pc) pb[pc] = acc_row_ptr(pc * kAccRowsPer);
#pragma unroll
        for (int i = 0; i < kBNm; ++i) {
          const int pc = 8 * (i >> 2) / kAccRowsPer;
          const int g = tc::acc_row(i, quarter, lane), b = tc::acc_col(i, lane);
          uint8_t* rp = pb[pc] + (b - pc * kAccRowsPer) * kAccRowBytes;
          if constexpr (kBwd)                            // bf16: 2 B of the row's 16 B chunk (g / 8) ^ (b & 7)
            *reinterpret_cast<__nv_bfloat16*>(rp + (((g >> 3) ^ b) & 7) * 16 + (g & 7) * 2) = __float2bfloat16_rn(acc[0][i]);
          else
            *reinterpret_cast<float*>(rp + acc_swz(b, g) * 4) = acc[0][i];
        }
      } else {
        uint8_t* wb = acc_row_ptr(16 * quarter);         // this warp's 16 fragment rows (one piece)
#pragma unroll
        for (int i = 0; i < kBNm / 2; i += 2) {
          const int r = tc::acc_row(i, 0, lane), c = tc::acc_col(i, lane);
          *reinterpret_cast<float2*>(wb + r * kAccRowBytes + acc_swz(r, c) * 4) = make_float2(acc[0][i], acc[0][i + 1]);
        }
      }
      wg_bar();
      return true;
    };
    auto acc_ld32 = [&](int col, uint32_t (&v)[32], bool only16 = false) {   // staged fp32 accumulator: row rl, columns [col, +32 | +16)
      const float* rb = reinterpret_cast<const float*>(acc_row_ptr(rl));
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (only16 && i >= 4) break;
        const float4 f = *reinterpret_cast<const float4*>(rb + acc_swz(rl, col + 4 * i));
        v[4 * i] = __float_as_uint(f.x); v[4 * i + 1] = __float_as_uint(f.y); v[4 * i + 2] = __float_as_uint(f.z); v[4 * i + 3] = __float_as_uint(f.w);
      }
    };
    // This warp has read its staged rows: the borrowed stages go back to the producer.  The proxy fence orders the generic
    // accesses to them before the bulk copies that refill them.  kPP: then step over the other tile's stages.
    auto acc_release = [&]() {
      if (ring_acc) {
        tc::fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
          tc::mbar_arrive_u32(empty0 + 8 * stage_back(1));
          if (kAccPieces == 2) tc::mbar_arrive_u32(empty0 + 8 * stage_back(2));
        }
      }
      if (kPP) skip_tile();
    };
    const bool dbg_thread = p.dbg && blockIdx.x == 0 && etid == 0;     // single-step stamps: CTA 0, first tile
    // The threads that serve one tile: kPP its warpgroup (the same named barrier as wg_bar), else both warpgroups.
    auto epi_bar = [&]() {
      if constexpr (kPP) wg_bar();
      else asm volatile("bar.sync 1, 256;" ::: "memory");
    };
    // exchange-buffer barriers: filled by st.async (async proxy, like a TMA load) / freed by relaxed arrives, so a CTA-scope
    // wait is enough; the cluster-scope acquire form (debug_mode 7, the earlier default) adds a CCTL.IVALL per wait
    const bool cluster_acquire = p.debug_mode == 7;
    auto xwait = [&](uint64_t* bar, uint32_t parity, volatile int* af) {
      return cluster_acquire ? wait_bar<true>(bar, parity, af) : wait_bar<false>(bar, parity, af);
    };
    // MEMBAR.ALL.GPU (the release of the dataflow signal) drains EVERY outstanding store of the SM, not just the signalling
    // thread's: if the other threads of the tile start their bookkeeping stores (h_seq / c_seq / activations) meanwhile, the
    // signal - the only thing the other CTAs wait for - is held back by 1-3 us (measured).  They wait for it instead.
    // kPP: the barrier holds back only this warpgroup.  The other warpgroup issued its bookkeeping stores right after ITS
    // signal, which comes about one MMA phase (~10 us at H = 1024) before this one's, so they have long drained by then.
    auto signal_sent_bar = [&]() {
      if constexpr (kPP) wg_bar();
      else asm volatile("bar.sync 2, 256;" ::: "memory");
    };
    // grid-barrier arrive: the CTA barrier orders every epilogue thread's writes before this thread's release
    // (same pattern as cooperative-groups grid sync).  ONE gpu-scope release: each fence is a full L2 round trip
    // (~0.8 us) and three of them used to dominate the epilogue; the generic->async proxy fence is on the consumer side.

    if (!kBwd) {
      auto j0 = [&](int u) { return in_mb * 16 + 8 * ch(u); };      // pass u's 8 hidden units
      auto n0 = [&](int u) { return in_mb * 64 + 32 * ch(u); };     // = its 32 gate columns
      uint32_t xphase = 0;
      const uint32_t xbase = tc::smem_u32(smem_x);
      const uint32_t xbar = tc::smem_u32(&ss->xchg_full[0]), fbar = tc::smem_u32(&ss->xchg_free[0]);
      const uint32_t pbar = kFSplit ? mapa(xbar, (uint32_t)(1 - ks)) : 0u;      // the peer's exchange barrier
      float cst[kPass][8];
      const size_t init_row = kRev ? (size_t)p.T * B : 0;     // the prologue wrote h0 / c0 to row 0 (forward) or row T (kRev)
#pragma unroll
      for (int u = 0; u < kPass; ++u)
#pragma unroll
        for (int i = 0; i < 8; ++i) cst[u][i] = valid ? p.c_seq[(init_row + row) * H + j0(u) + i] : 0.f;     // c_0 (written by the prologue)
      // kMasked: this thread's row length, and its last emitted h per pass (8 bf16) - a padded step re-emits it without a load.
      // Forward order: step 0 is never padded (len >= 1), so hprev needs no initial value.  kRev: the padded steps come first
      // and re-emit h0.
      int len = p.T;
      uint4 hprev[kPass];
      if constexpr (kMasked) {
        if (valid) len = p.lengths[row];
#pragma unroll
        for (int u = 0; u < kPass; ++u) {
          hprev[u] = make_uint4(0u, 0u, 0u, 0u);
          if (kRev && valid) hprev[u] = *reinterpret_cast<const uint4*>(p.h_seq + (init_row + row) * H + j0(u));
        }
      }
      for (int t = 0; t < p.T && ok; ++t) {
        const int tt = kRev ? p.T - 1 - t : t;        // the time step that processing step t handles
        // operands that do not depend on the GEMM: issue their loads before waiting on the accumulator
        U8 gxw[kPass][2];
        if (p.in_gate != nullptr) {                   // wavefront: gx[t] is produced while we run (this warp's rows: one 128-row block)
          const size_t gr = (size_t)t * B + (size_t)mb * BM;
          ok = wait_in_gate(p.in_gate + (gr >> 7) * p.in_gate_tiles_n + (n0(0) >> 8), lane, abort_flag);    // (all passes: one 256-column block)
          if (!ok) break;
          if (valid) {
#pragma unroll
            for (int u = 0; u < kPass; ++u) {
              const __nv_bfloat16* gp = p.gx + ((size_t)t * B + row) * (4 * H) + n0(u);
              gxw[u][0] = ldg_cg32(gp); gxw[u][1] = ldg_cg32(gp + 16);
            }
          }
        } else if (valid) {
#pragma unroll
          for (int u = 0; u < kPass; ++u) {
            const __nv_bfloat16* gp = p.gx + ((size_t)tt * B + row) * (4 * H) + n0(u);
            gxw[u][0] = ldg_nc32(gp); gxw[u][1] = ldg_nc32(gp + 16);
            if (t + 2 < p.T && p.debug_mode != 6)      // the x-projection comes from HBM: pull it into L2 early
              prefetch_l2(kRev ? gp - (size_t)2 * B * (4 * H) : gp + (size_t)2 * B * (4 * H));
          }
        }
        ok = mma_tile(t);
        if (!ok) break;
        unsigned long long t_acc = 0;
        if (p.dbg && t == 8 && etid == 0) t_acc = gtime();
        if (dbg_wg) dbg_stamp(t, 1);
        const bool pad = kMasked && tt >= len;        // padded step: the cell holds (the activations are computed but unused)
        float cn[kPass][8];
        uint32_t apk[kPass][16];
        uint4 h8[kPass];
#pragma unroll
        for (int u = 0; u < kPass; ++u) {
          uint32_t v[32];
          if constexpr (kFSplit) {
            // partial sums over this member's K half: columns [64 ks, +64) are mine, the other 64 go to the peer (bf16, DSMEM)
            uint32_t w32[32];
            acc_ld32(32 * chalf + 64 * (1 - ks), w32);
            acc_ld32(32 * chalf + 64 * ks, v);
            if (t > 0) {                                               // the peer has consumed last step's partial
              ok = xwait(&ss->xchg_free[0], (uint32_t)((t - 1) & 1), abort_flag);
              if (!ok) break;
            }
            const uint32_t drow = mapa(xbase + (uint32_t)(rloc * 128), (uint32_t)(1 - ks));
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              uint32_t pk[4];
#pragma unroll
              for (int k = 0; k < 4; ++k) pk[k] = pack_bf2(__uint_as_float(w32[8 * i + 2 * k]), __uint_as_float(w32[8 * i + 2 * k + 1]));
              st_async_u4(drow + (uint32_t)((((4 * chalf + i) ^ (rloc & 7))) * 16), make_uint4(pk[0], pk[1], pk[2], pk[3]), pbar);
            }
            ok = xwait(&ss->xchg_full[0], xphase, abort_flag);
            if (!ok) break;
            xphase ^= 1;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const uint4 x4 = *reinterpret_cast<const uint4*>(smem_x + (size_t)rloc * 128 + (((4 * chalf + i) ^ (rloc & 7)) * 16));
              const uint32_t w[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                v[8 * i + 2 * k] = __float_as_uint(__uint_as_float(v[8 * i + 2 * k]) + bf_lo(w[k]));
                v[8 * i + 2 * k + 1] = __float_as_uint(__uint_as_float(v[8 * i + 2 * k + 1]) + bf_hi(w[k]));
              }
            }
          } else {
            acc_ld32(32 * ch(u), v);
            if (u == kPass - 1) acc_release();          // every pass has read its columns
          }
          if (dbg_thread && t == 8 && u == 0) p.dbg[4 * (p.T + 2) + 0] = gtime();
          const float* bs = ss->bias + 32 * ch(u);
          float hv[8];
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const uint32_t ga = gxw[u][jj >> 2].v[2 * (jj & 3)], gb = gxw[u][jj >> 2].v[2 * (jj & 3) + 1];
            const float pi = __uint_as_float(v[4 * jj + 0]) + bf_lo(ga) + bs[4 * jj + 0];
            const float pf = __uint_as_float(v[4 * jj + 1]) + bf_hi(ga) + bs[4 * jj + 1];
            const float pg = __uint_as_float(v[4 * jj + 2]) + bf_lo(gb) + bs[4 * jj + 2];
            const float po = __uint_as_float(v[4 * jj + 3]) + bf_hi(gb) + bs[4 * jj + 3];
            const float ig = ts::sigmoidf_fast(pi), fg = ts::sigmoidf_fast(pf), gg = ts::tanhf_fast(pg), og = ts::sigmoidf_fast(po);
            const float c = fg * cst[u][jj] + ig * gg;
            if constexpr (kMasked) {
              if (!pad) cst[u][jj] = c;
              cn[u][jj] = cst[u][jj];
            } else {
              cst[u][jj] = c;                         // the cell state never leaves the registers of its thread
              cn[u][jj] = c;
            }
            hv[jj] = og * ts::tanhf_fast(c);
            apk[u][2 * jj] = pack_bf2(ig, fg);
            apk[u][2 * jj + 1] = pack_bf2(gg, og);
          }
          h8[u] = make_uint4(pack_bf2(hv[0], hv[1]), pack_bf2(hv[2], hv[3]), pack_bf2(hv[4], hv[5]), pack_bf2(hv[6], hv[7]));
          if constexpr (kMasked) {
            if (pad) h8[u] = hprev[u];
            hprev[u] = h8[u];
          }
          {
            // next step's operand first (the only thing other CTAs wait for): 8 values = one 16 B chunk of the swizzled
            // tile image; chunk c of row r sits at position c ^ (r & 7)
            const size_t blk = ((size_t)(t + 1) * p.tiles_m + mb) * (H / BK) + (j0(u) / BK);
            const int chunk = ((j0(u) % BK) / 8) ^ (rloc & 7);
            stg16(p.a_tiled + blk * (BM * BK) + rloc * BK + chunk * 8, h8[u]);
          }
        }
        if (!ok) break;
        if (dbg_thread && t == 8) p.dbg[4 * (p.T + 2) + 1] = gtime();
        epi_bar();
        if (gtid == 0) {
          if (dbg_thread && t == 8) p.dbg[4 * (p.T + 2) + 2] = gtime();
          if (p.dbg && t == 8 && etid == 0) {                // per-CTA stamps (skew study): accumulator ready / about to signal
            p.dbg[4 * (p.T + 2) + 64 + 2 * blockIdx.x] = t_acc;
            p.dbg[4 * (p.T + 2) + 64 + 2 * blockIdx.x + 1] = gtime();
          }
          // this CTA's 16 hidden units = a quarter of k-block nb/4
          if (p.sync_mode == 1) signal_counter(p.sync + mb);
          else if (p.sync_mode == 2) st_release_gpu(p.sync + kSyncFlags + (size_t)mb * p.tiles_n + in_mb, (unsigned)(t + 1));
          else signal_counter(p.sync + kSyncKb + ((size_t)mb * (H / BK) + (in_mb >> 2)) * 32);
          if (dbg_wg) dbg_stamp(t, 2);
        }
        // (after the CTA barrier every epilogue thread is done with this step's exchange buffer)
        if (kFSplit && etid == 32) {
          tc::mbar_expect_tx_u32(xbar, (uint32_t)kXchgBytes);        // arm the next phase, THEN let the peer overwrite the buffer
          mbar_arrive_remote_relaxed(mapa(fbar, (uint32_t)(1 - ks)));
        }
        signal_sent_bar();
        if (valid && p.debug_mode != 5) {              // everything below is off the critical path
          const size_t srow = kRev ? (size_t)tt : (size_t)(t + 1);      // state row written by this step
#pragma unroll
          for (int u = 0; u < kPass; ++u) {
            stg16(p.h_seq + (srow * B + row) * H + j0(u), h8[u]);
            if constexpr (kDrop) {                     // this thread's 8 units of row `row` are one Philox group
              const uint32_t keep = ts::dropout_keep8(p.drop, (uint32_t)__ldg(p.drop.step), row, j0(u), tt, H);
              stg16(p.h_drop + ((size_t)tt * B + row) * H + j0(u), ts::dropout_bf16x8(h8[u], keep, p.drop.scale));
            }
            float* cp = p.c_seq + (srow * B + row) * H + j0(u);
            stg32(cp, __float_as_uint(cn[u][0]), __float_as_uint(cn[u][1]), __float_as_uint(cn[u][2]), __float_as_uint(cn[u][3]),
                  __float_as_uint(cn[u][4]), __float_as_uint(cn[u][5]), __float_as_uint(cn[u][6]), __float_as_uint(cn[u][7]));
            __nv_bfloat16* ap = p.act + ((size_t)tt * B + row) * (4 * H) + n0(u);
#pragma unroll
            for (int i = 0; i < 2; ++i)
              stg32(ap + 16 * i, apk[u][8 * i], apk[u][8 * i + 1], apk[u][8 * i + 2], apk[u][8 * i + 3], apk[u][8 * i + 4], apk[u][8 * i + 5],
                    apk[u][8 * i + 6], apk[u][8 * i + 7]);
          }
        }
      }
      if (p.extra_signal && ok) {                 // the last step's h_seq rows (natural layout) are visible to the gated GEMM
        epi_bar();
        if (gtid == 0) {
          if (p.sync_mode == 1) signal_counter(p.sync + mb);
          else signal_counter(p.sync + kSyncKb + ((size_t)mb * (H / BK) + (in_mb >> 2)) * 32);
        }
      }
    } else {
      // after the reduce-scatter this cluster member owns hidden [64 nb + 16 ks, +16); pass u of this thread 8 of them
      auto j0 = [&](int u) { return nb * kBNm + ks * 16 + 8 * ch(u); };
      uint32_t xphase = 0;
      const int xt = kPP ? half : 0;                       // this tile's exchange buffer and barriers
      uint8_t* xbuf = smem_x + xt * kXchgBytes;            // [kSplit src][128 rows][16 bf16]
      const uint32_t xbase = tc::smem_u32(xbuf);
      const uint32_t xbar = tc::smem_u32(&ss->xchg_full[xt]);
      float dc[kPass][8], dh[kPass][8];
#pragma unroll
      for (int u = 0; u < kPass; ++u) {
        if (valid) {
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float4 a = *reinterpret_cast<const float4*>(p.dc0 + (size_t)row * H + j0(u) + 4 * i);
            float4 b = *reinterpret_cast<const float4*>(p.dh0 + (size_t)row * H + j0(u) + 4 * i);
            dc[u][4 * i] = a.x; dc[u][4 * i + 1] = a.y; dc[u][4 * i + 2] = a.z; dc[u][4 * i + 3] = a.w;
            dh[u][4 * i] = b.x; dh[u][4 * i + 1] = b.y; dh[u][4 * i + 2] = b.z; dh[u][4 * i + 3] = b.w;
          }
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) { dc[u][i] = 0.f; dh[u][i] = 0.f; }
        }
      }
      U8 c_carry[kPass];                        // c_t of the previous iteration = c_{t+1} of this one (one load per step, not two)
      // kMasked: right padding makes a row's padded steps the FIRST backward iterations (kRev: the LAST ones).  There dG = 0, dc
      // passes through and dh keeps the total dh (carry + dh_seq[t]): the next exchange sum adds the (exactly zero) recurrent
      // term to it.  With kRev the values carried through the trailing padded steps are dh0 / dc0.
      int len = p.T;
      if constexpr (kMasked) {
        if (valid) len = p.lengths[row];
      }
      for (int s = 0; s <= p.T && ok; ++s) {
        const int t = p.T - 1 - s;                    // operand-image slot (processing order)
        const int tt = kRev ? s : t;                  // the time step of this iteration
        const bool pad = kMasked && s < p.T && tt >= len;          // step tt is padding for this row
        // the previous iteration's step was: dh carries, c_carry is not set
        const bool prev_pad = kMasked && s > 0 && (kRev ? tt - 1 : t + 1) >= len;
        U8 avw[kPass][2], cpv[kPass], cnv[kPass];
        uint4 dhv[kPass];
        if (p.in_gate != nullptr && s < p.T) {      // wavefront: dh_seq[t] (= dX of the layer above) is produced while we run
          const size_t gr = (size_t)t * B + (size_t)mb * BM;
          ok = wait_in_gate(p.in_gate + (gr >> 7) * p.in_gate_tiles_n + (j0(0) >> 8), lane, abort_flag);    // (all passes: one 256-column block)
          if (!ok) break;
        }
        if (valid && s < p.T) {
#pragma unroll
          for (int u = 0; u < kPass; ++u) {
            const __nv_bfloat16* ap = p.act + ((size_t)tt * B + row) * (4 * H) + 4 * j0(u);
            if (!pad) { avw[u][0] = ldg_nc32(ap); avw[u][1] = ldg_nc32(ap + 16); }
            dhv[u] = p.dh_seq ? (p.in_gate ? ldg_cg16(p.dh_seq + ((size_t)t * B + row) * H + j0(u)) : ldg_nc16(p.dh_seq + ((size_t)tt * B + row) * H + j0(u)))
                              : make_uint4(0u, 0u, 0u, 0u);
            if constexpr (kDrop)                       // dropped units of dh_seq[tt] -> 0; kept ones are scaled where dh joins the carry
              dhv[u] = ts::dropout_zero_bf16x8(dhv[u], ts::dropout_keep8(p.drop, (uint32_t)__ldg(p.drop.step), row, j0(u), tt, H));
            // c_prev / c_new of step tt (kRev: rows tt + 1 / tt).  c_new is the previous iteration's c_prev in both directions.
            const float* c0p = p.c_seq + ((size_t)(kRev ? tt + 1 : t) * B + row) * H + j0(u);
            const float* c1p = p.c_seq + ((size_t)(kRev ? tt : t + 1) * B + row) * H + j0(u);
            if (!pad) {
              cpv[u] = ldg_nc32(c0p);
              cnv[u] = (s == 0 || prev_pad) ? ldg_nc32(c1p) : c_carry[u];
              c_carry[u] = cpv[u];
              if (t >= 2) {                          // saved activations come from HBM: pull the step two iterations ahead into L2
                if constexpr (kRev) {
                  prefetch_l2(ap + (size_t)2 * B * (4 * H));
                  prefetch_l2(c0p + (size_t)2 * B * H);
                  if (p.dh_seq) prefetch_l2(p.dh_seq + ((size_t)(tt + 2) * B + row) * H + j0(u));
                } else {
                  prefetch_l2(ap - (size_t)2 * B * (4 * H));
                  prefetch_l2(c0p - (size_t)2 * B * H);
                  if (p.dh_seq && !p.in_gate) prefetch_l2(p.dh_seq + ((size_t)(t - 2) * B + row) * H + j0(u));
                }
              }
            }
          }
        }
        if (s > 0) {
          ok = mma_tile(s);
          if (!ok) break;
          if (dbg_wg) dbg_stamp(s, 1);
          // this thread's partial sums, rounded to bf16 for the exchange: pass u = accumulator columns [kCW ch(u), +kCW)
          uint32_t pk[kPass][kCW / 2];
#pragma unroll
          for (int u = 0; u < kPass; ++u) {
            if constexpr (kPP) {                       // staged as bf16 (kCW = 32: 64 B of the 128 B row)
              const uint8_t* rb = acc_row_ptr(rl);
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const uint4 x4 = *reinterpret_cast<const uint4*>(rb + (((4 * ch(u) + i) ^ rl) & 7) * 16);
                pk[u][4 * i] = x4.x; pk[u][4 * i + 1] = x4.y; pk[u][4 * i + 2] = x4.z; pk[u][4 * i + 3] = x4.w;
              }
            } else {
              uint32_t v[32];
              acc_ld32(kCW * ch(u), v, kCW == 16);
#pragma unroll
              for (int i = 0; i < kCW / 2; ++i) pk[u][i] = pack_bf2(__uint_as_float(v[2 * i]), __uint_as_float(v[2 * i + 1]));
            }
          }
          acc_release();
          // A member only needs the dG blocks of ITS K-quarter, so nothing in the dataflow stops a fast member from being a
          // whole step ahead of a slow one: explicit back-pressure before overwriting anybody's exchange buffer.
          if (s > 1) {
            ok = xwait(&ss->xchg_free[xt], (uint32_t)(s & 1), abort_flag);
            if (!ok) break;
          }
          // reduce-scatter over the kSplit K parts: column chunk q (16 wide, bf16) goes to member q's slot [ks] (DSMEM)
#pragma unroll
          for (int u = 0; u < kPass; ++u) {
#pragma unroll
            for (int qq = 0; qq < kCW / 16; ++qq) {
              const uint32_t q = (uint32_t)((kCW / 16) * ch(u) + qq);
              const uint32_t dst = mapa(xbase + (uint32_t)((ks * BM + rloc) * 32), q);
              const uint32_t* a = pk[u] + 8 * qq;
              const uint32_t dbar = mapa(xbar, q);
              st_async_u4(dst, make_uint4(a[0], a[1], a[2], a[3]), dbar);
              st_async_u4(dst + 16, make_uint4(a[4], a[5], a[6], a[7]), dbar);
            }
          }
          ok = xwait(&ss->xchg_full[xt], xphase, abort_flag);
          if (!ok) break;
#pragma unroll
          for (int u = 0; u < kPass; ++u) {
            if (!prev_pad) {
#pragma unroll
              for (int i = 0; i < 8; ++i) dh[u][i] = 0.f;
            }
#pragma unroll
            for (int src = 0; src < kSplit; ++src) {
              const uint4 x4 = *reinterpret_cast<const uint4*>(xbuf + (size_t)(src * BM + rloc) * 32 + 16 * ch(u));
              const uint32_t w[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
              for (int i = 0; i < 4; ++i) { dh[u][2 * i] += bf_lo(w[i]); dh[u][2 * i + 1] += bf_hi(w[i]); }
            }
          }
        }
        if (s == p.T) {                                // the last iteration: dh_0 / dc_0 out
          if (valid) {
#pragma unroll
            for (int u = 0; u < kPass; ++u)
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                *reinterpret_cast<float4*>(p.dh0 + (size_t)row * H + j0(u) + 4 * i) = make_float4(dh[u][4 * i], dh[u][4 * i + 1], dh[u][4 * i + 2], dh[u][4 * i + 3]);
                *reinterpret_cast<float4*>(p.dc0 + (size_t)row * H + j0(u) + 4 * i) = make_float4(dc[u][4 * i], dc[u][4 * i + 1], dc[u][4 * i + 2], dc[u][4 * i + 3]);
              }
          }
          if (p.extra_signal) {                   // dpre[0] (natural layout, written after the last per-step signal) is visible to the gated GEMM
            epi_bar();
            if (gtid == 0) {
              if (p.sync_mode == 1) signal_counter(p.sync + mb);
              else signal_counter(p.sync + kSyncKb + ((size_t)mb * (4 * H / BK) + in_mb) * 32);
            }
          }
          break;
        }
        uint32_t gpk[kPass][16];
#pragma unroll
        for (int u = 0; u < kPass; ++u) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const uint32_t aa = avw[u][jj >> 2].v[2 * (jj & 3)], ab = avw[u][jj >> 2].v[2 * (jj & 3) + 1];
            const float ig = bf_lo(aa), fg = bf_hi(aa), gg = bf_lo(ab), og = bf_hi(ab);
            const uint32_t dw = (jj >> 1) == 0 ? dhv[u].x : (jj >> 1) == 1 ? dhv[u].y : (jj >> 1) == 2 ? dhv[u].z : dhv[u].w;
            const float dsj = (jj & 1) ? bf_hi(dw) : bf_lo(dw);
            const float dht = dh[u][jj] + (kDrop ? __fmul_rn(dsj, p.drop.scale) : dsj);
            const float cprev = __uint_as_float(cpv[u].v[jj]);
            const float tcn = ts::tanhf_fast(__uint_as_float(cnv[u].v[jj]));
            const float dc_in = dc[u][jj];
            const float dct = dc_in + dht * og * (1.f - tcn * tcn);
            const float d_o = dht * tcn, d_i = dct * gg, d_f = dct * cprev, d_g = dct * ig;
            dc[u][jj] = dct * fg;
            gpk[u][2 * jj] = pack_bf2(d_i * ig * (1.f - ig), d_f * fg * (1.f - fg));
            gpk[u][2 * jj + 1] = pack_bf2(d_g * (1.f - gg * gg), d_o * og * (1.f - og));
            if constexpr (kMasked) {
              if (pad) {                          // (the loads above were skipped: everything but dht is discarded)
                dc[u][jj] = dc_in;
                dh[u][jj] = dht;
                gpk[u][2 * jj] = 0u;
                gpk[u][2 * jj + 1] = 0u;
              }
            }
          }
          // next iteration's operand first: pass u's 32 gate columns = 4 chunks of row rloc of k-block j0/16
          const size_t blk = ((size_t)t * p.tiles_m + mb) * (4 * H / BK) + (j0(u) / 16);
          __nv_bfloat16* tp = p.a_tiled + blk * (BM * BK) + rloc * BK;
          // chunk c of row r sits at c ^ (r & 7): an aligned chunk pair stays an aligned pair (32 B sector p ^ ((r & 7) >> 1)),
          // swapped when r is odd -> two whole-sector 256-bit stores instead of four 16 B ones
          const bool swp = rloc & 1;
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const int sp = (2 * ch(u) + k) ^ ((rloc & 7) >> 1);
            const uint32_t* a = gpk[u] + 8 * k;
            stg32(tp + sp * 16, swp ? a[4] : a[0], swp ? a[5] : a[1], swp ? a[6] : a[2], swp ? a[7] : a[3],
                  swp ? a[0] : a[4], swp ? a[1] : a[5], swp ? a[2] : a[6], swp ? a[3] : a[7]);
          }
        }
        epi_bar();
        if (gtid == 0) {
          // this CTA's 64 gate columns = dG k-block 4 nb + ks
          if (p.sync_mode == 1) signal_counter(p.sync + mb);
          else if (p.sync_mode == 2) st_release_gpu(p.sync + kSyncFlags + (size_t)mb * p.tiles_n + in_mb, (unsigned)(s + 1));
          else signal_counter(p.sync + kSyncKb + ((size_t)mb * (4 * H / BK) + in_mb) * 32);
          if (dbg_wg) dbg_stamp(s, 2);
        }
        // (the barrier above also means every thread of the tile is done reading this step's exchange buffer)
        if (s > 0) {
          if (gtid == 32) tc::mbar_expect_tx_u32(xbar, kXchgRecv);    // arm the next phase, THEN free the buffer
          __syncwarp();
          if (gtid >= 32 && gtid < 32 + kSplit) mbar_arrive_remote_relaxed(mapa(tc::smem_u32(&ss->xchg_free[xt]), (uint32_t)(gtid - 32)));
          xphase ^= 1;
        }
        signal_sent_bar();
        if (valid) {                                   // the [T,B,4H] copy for the weight-gradient GEMMs: off the critical path
#pragma unroll
          for (int u = 0; u < kPass; ++u) {
            __nv_bfloat16* gp = p.dpre + ((size_t)tt * B + row) * (4 * H) + 4 * j0(u);
#pragma unroll
            for (int i = 0; i < 2; ++i)
              stg32(gp + 16 * i, gpk[u][8 * i], gpk[u][8 * i + 1], gpk[u][8 * i + 2], gpk[u][8 * i + 3], gpk[u][8 * i + 4], gpk[u][8 * i + 5],
                    gpk[u][8 * i + 6], gpk[u][8 * i + 7]);
          }
        }
      }
    }
  }

  if (warp >= kEpiWarp0) {
    __syncwarp();
    if (lane == 0) atomicAdd(&ss->roles_done, 1);
  }
  __syncthreads();
  if (kCluster) cluster_sync_all();              // nobody exits while a peer may still write into / arrive on its smem
  if (p.pdl_wait) asm volatile("griddepcontrol.wait;" ::: "memory");
  if (threadIdx.x == 0 && ss->abort_flag) atomicExch(reinterpret_cast<int*>(p.sync + kSyncErr), 1);
}

// One small launch instead of ~12 framework ops: h_seq[0] <- h0, c_seq[0] <- c0 (the reverse direction passes row T), the
// swizzled tile image of h0 (slot 0 of the streamed operand, zero rows beyond B), and the step counters <- 0.
__global__ void seq_prologue_kernel(const __nv_bfloat16* __restrict__ h0, const float* __restrict__ c0,
                                    __nv_bfloat16* __restrict__ h_seq0, float* __restrict__ c_seq0,
                                    __nv_bfloat16* __restrict__ tiled0, unsigned int* __restrict__ sync, int B, int H, int tiles_m) {
  const int nchunk = H / 8, nkb = H / BK;
  const int total = tiles_m * BM * nchunk;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int r = i / nchunk, c = i % nchunk;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r < B) {
      v = *reinterpret_cast<const uint4*>(h0 + (size_t)r * H + 8 * c);
      *reinterpret_cast<uint4*>(h_seq0 + (size_t)r * H + 8 * c) = v;
    }
    const int mb = r / BM, rloc = r % BM, kb = c / 8, pos = (c % 8) ^ (rloc & 7);
    *reinterpret_cast<uint4*>(tiled0 + (((size_t)mb * nkb + kb) * BM + rloc) * BK + pos * 8) = v;
  }
  const int n4 = B * H / 4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x)
    reinterpret_cast<float4*>(c_seq0)[i] = reinterpret_cast<const float4*>(c0)[i];
  if (blockIdx.x == 0)
    for (int i = threadIdx.x; i < kSyncErr; i += blockDim.x) sync[i] = 0u;
}

size_t smem_bytes(int H, bool bwd, int stages, int tiles, bool stream = false, bool fsplit = false) {
  const bool narrow = bwd && stream;                       // streamed backward: 32 accumulator columns per CTA (kNarrow)
  const size_t ring = (size_t)stages * (stream ? kABytes + (narrow ? kWBlockBytes / 2 : kWBlockBytes) : kABytes);
  // resident weights: H/64 blocks of [64 x 64] (forward K-split: H/128 blocks of [128 x 64] = the same bytes)
  // The staged accumulator lives in drained ring stages, except for the forward K-split and H = 64 (one k-block per tile,
  // two 8 KB pieces per warpgroup; two tiles: two whole fp32 stages forward, one bf16 stage backward): those keep a
  // dedicated fp32 buffer of [128 x columns] per tile being staged at once (lstm_seq_kernel, ring_acc).
  const bool dedicated = fsplit || (!narrow && H / BK < 2 && !(tiles == 2 && bwd));
  const size_t acc_stage = dedicated ? (size_t)tiles * BM * (fsplit ? 2 * BN : BN) * sizeof(float) : 0;
  return (stream ? 0 : (size_t)(H / BK) * kWBlockBytes) + ring + ((bwd || fsplit) ? tiles * kXchgBytes : 0) + acc_stage + sizeof(SeqSmem) + 1024;
}

template <bool kBwd, int kStages, int kTiles, bool kStream = false, bool kFSplit = false, bool kMasked = false, bool kRev = false,
          bool kDrop = false>
int launch_cfg(const CUtensorMap& tw, const SeqParams& p, int grid, cudaStream_t st) {
  auto kern = lstm_seq_kernel<kBwd, kStages, kTiles, kStream, kFSplit, kMasked, kRev, kDrop>;
  const size_t smem = smem_bytes(p.H, kBwd, kStages, kTiles, kStream, kFSplit);
  constexpr int kClusterDim = kBwd ? (kStream ? 2 : 4) : (kFSplit ? 2 : 1);
  if (smem > 227 * 1024) return -4;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(384); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = kClusterDim; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  if (kClusterDim > 1) {
    int nclusters = 0;
    e = cudaOccupancyMaxActiveClusters(&nclusters, kern, &cfg);
    if (e != cudaSuccess) { cudaGetLastError(); return -20; }
    if (nclusters * kClusterDim < grid) return -21;    // not co-resident
  }
  if (p.pdl_wait) {                                    // start as soon as the previous kernel of the stream is fully resident
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 2;
  }
  e = cudaLaunchKernelEx(&cfg, kern, tw, p);
  return (int)e;
}

template <bool kBwd, bool kMasked, bool kRev, bool kDrop>
int dispatch(const CUtensorMap& tw, const SeqParams& p, int grid, int stages, int tiles, bool stream, bool fsplit, cudaStream_t st) {
  if constexpr (!kBwd) {
    if (fsplit) {                                  // forward K-split (cluster of 2), one batch tile per CTA
      switch (stages) {
        case 3: return launch_cfg<false, 3, 1, false, true, kMasked, kRev, kDrop>(tw, p, grid, st);
        case 4: return launch_cfg<false, 4, 1, false, true, kMasked, kRev, kDrop>(tw, p, grid, st);
        case 5: return launch_cfg<false, 5, 1, false, true, kMasked, kRev, kDrop>(tw, p, grid, st);
        case 6: return launch_cfg<false, 6, 1, false, true, kMasked, kRev, kDrop>(tw, p, grid, st);
      }
      return -5;
    }
  }
  if (stream) {                                    // streamed weights: 24 KB stages, one batch tile per CTA
    switch (stages) {
      case 4: return launch_cfg<kBwd, 4, 1, true, false, kMasked, kRev, kDrop>(tw, p, grid, st);
      case 6: return launch_cfg<kBwd, 6, 1, true, false, kMasked, kRev, kDrop>(tw, p, grid, st);
      case 8: return launch_cfg<kBwd, 8, 1, true, false, kMasked, kRev, kDrop>(tw, p, grid, st);
    }
    return -5;
  }
  if (tiles == 2) {
    switch (stages) {
      case 2: return launch_cfg<kBwd, 2, 2, false, false, kMasked, kRev, kDrop>(tw, p, grid, st);
      case 3: return launch_cfg<kBwd, 3, 2, false, false, kMasked, kRev, kDrop>(tw, p, grid, st);
      case 4: return launch_cfg<kBwd, 4, 2, false, false, kMasked, kRev, kDrop>(tw, p, grid, st);
      case 5: return launch_cfg<kBwd, 5, 2, false, false, kMasked, kRev, kDrop>(tw, p, grid, st);
      case 6: return launch_cfg<kBwd, 6, 2, false, false, kMasked, kRev, kDrop>(tw, p, grid, st);
    }
  } else {
    switch (stages) {
      case 2: return launch_cfg<kBwd, 2, 1, false, false, kMasked, kRev, kDrop>(tw, p, grid, st);
      case 3: return launch_cfg<kBwd, 3, 1, false, false, kMasked, kRev, kDrop>(tw, p, grid, st);
      case 4: return launch_cfg<kBwd, 4, 1, false, false, kMasked, kRev, kDrop>(tw, p, grid, st);
      case 5: return launch_cfg<kBwd, 5, 1, false, false, kMasked, kRev, kDrop>(tw, p, grid, st);
      case 6: return launch_cfg<kBwd, 6, 1, false, false, kMasked, kRev, kDrop>(tw, p, grid, st);
    }
  }
  return -5;
}

template <bool kBwd, bool kDrop>
int dispatch_dir(const CUtensorMap& tw, const SeqParams& p, int grid, int stages, int tiles, bool stream, bool fsplit, cudaStream_t st,
                 bool reverse) {
  return reverse ? (p.lengths ? dispatch<kBwd, true, true, kDrop>(tw, p, grid, stages, tiles, stream, fsplit, st)
                              : dispatch<kBwd, false, true, kDrop>(tw, p, grid, stages, tiles, stream, fsplit, st))
                 : (p.lengths ? dispatch<kBwd, true, false, kDrop>(tw, p, grid, stages, tiles, stream, fsplit, st)
                              : dispatch<kBwd, false, false, kDrop>(tw, p, grid, stages, tiles, stream, fsplit, st));
}

int pick_stages(int H, bool bwd, int tiles) {
  // One tile per CTA forward with H >= 1024 (>= 16 k-blocks per step, the resident slice takes >= 128 KB): 4 stages, not the
  // deepest ring that fits.  At B = 256, H = 1024 on an H100 80GB HBM3 (700 W) a step took 10.9-11.5 us with 4 stages against
  // 11.3-12.1 us with 6 (11.3-11.8 with 5, 12.1-12.4 with 3), eight runs each; 4 was the fastest within every set of runs.
  if (!bwd && tiles == 1 && H / BK >= 16 && smem_bytes(H, false, 4, 1) <= 227 * 1024) return 4;
  for (int s = 6; s >= 2; --s)
    if (smem_bytes(H, bwd, s, tiles) <= 227 * 1024) return s;
  return 0;
}

}  // namespace

// sync_ws: kSyncWords u32 (layout above); everything but the sticky error flag in the last word is zeroed before every launch.
// variant (tuning knob, 0 = defaults) = tiles_per_cta + 16*stages + 4096*debug_mode:  tiles_per_cta 0 -> 1 (set 2 to let a
// CTA alternate two batch tiles);  stages 0 -> deepest ring that fits next to the resident weight slice.
struct SeqCfg {
  int stages, tiles;
  bool stream, fsplit;
};

// The launch configuration seq_common() uses for H, B and variant (no device needed): 0, or a negative code with the error
// message set.
static int seq_config(bool bwd, int H, int B, int variant, SeqCfg& c) {
  if (H % 64 != 0) { ts::set_last_error("lstm_seq: H must be a multiple of 64"); return -2; }
  const int tiles_m = (B + BM - 1) / BM;
  int stages = (variant >> 4) & 15, tiles = variant & 15;
  if (tiles != 2 || tiles_m % 2 != 0) tiles = 1;
  // resident weight slice up to H = 1152 (forward) / 1024 (backward; cuda_lstm._bwd_cluster and _tiles_per_cta assume this
  // boundary), else stream the weights through the ring
  const bool stream = H > (bwd ? 1024 : 1152) || ((variant >> 8) & 1);
  if (stream) tiles = 1;
  if (bwd && stream && 4 * H / (2 * BK) > 64) { ts::set_last_error("lstm_seq: streamed backward needs H <= 2048"); return -2; }
  // one arrival counter per operand k-block of every batch tile, at word kSyncKb + 32 i: the last one must stay below the
  // sticky error word (a layout with more counters would count its arrivals into the error flag)
  const int counters = tiles_m * (bwd ? 4 * H : H) / BK;
  if (kSyncKb + 32 * (counters - 1) >= kSyncErr) {
    ts::set_last_error("lstm_seq: the k-block arrival counters of this layout do not fit in the sync workspace");
    return -2;
  }
  // forward: 2-way K split (cluster of 2) unless disabled by variant bit 19
  const bool fsplit = !bwd && !stream && tiles == 1 && H % 128 == 0 && !((variant >> 19) & 1) &&
                      smem_bytes(H, false, 3, 1, false, true) <= 227 * 1024;
  if (stream) {
    if (stages != 4 && stages != 6 && stages != 8) stages = smem_bytes(H, bwd, 8, 1, true) <= 227 * 1024 ? 8 : 6;
  } else if (fsplit) {
    if (stages < 3 || stages > 6 || smem_bytes(H, false, stages, 1, false, true) > 227 * 1024) {
      stages = 6;
      while (stages > 3 && smem_bytes(H, false, stages, 1, false, true) > 227 * 1024) --stages;
    }
  } else {
    if (stages == 0) stages = pick_stages(H, bwd, tiles);
    if (stages < 2 || smem_bytes(H, bwd, stages, tiles) > 227 * 1024) { ts::set_last_error("lstm_seq: weight slice does not fit in shared memory"); return -4; }
  }
  c = SeqCfg{stages, tiles, stream, fsplit};
  return 0;
}

template <bool kBwd>
static int seq_common(SeqParams& p, const void* w_base, int variant, cudaStream_t st, bool reverse) {
  const int H = p.H, B = p.B;
  if (reverse && (p.in_gate != nullptr || p.extra_signal)) {
    ts::set_last_error("lstm_seq: the reverse direction does not run in the layer wavefront (in_gate / extra_signal)");
    return -2;
  }
  SeqCfg cfg;
  if (int rc = seq_config(kBwd, H, B, variant, cfg)) return rc;
  const int stages = cfg.stages, tiles = cfg.tiles;
  const bool stream = cfg.stream, fsplit = cfg.fsplit;
  const int tiles_m = (B + BM - 1) / BM, tiles_n = kBwd ? (H / BN) * 4 : 4 * H / BN;
  p.debug_mode = (variant >> 12) & 7;
  p.sync_mode = (variant >> 16) & 3;
  p.poll_acquire = (variant >> 18) & 1;
  p.no_trap = (variant >> 20) & 1;
  int dev = 0;
  cudaGetDevice(&dev);
  const int grid = (tiles_m / tiles) * tiles_n;
  if (grid > ts::sm_count(dev)) { ts::set_last_error("lstm_seq: grid exceeds SM count (not co-resident)"); return -3; }
  const int K = kBwd ? 4 * H : H, N = kBwd ? H : 4 * H;
  CUtensorMap tw;
  if (int rc = ts::make_tmap_2d_bf16(&tw, w_base, (uint64_t)N, (uint64_t)K, (uint64_t)K, BK, fsplit ? 2 * BN : ((kBwd && stream) ? BN / 2 : BN))) return rc;
  p.tiles_n = tiles_n;
  p.tiles_m = tiles_m;
  int rc = p.drop.step ? dispatch_dir<kBwd, true>(tw, p, grid, stages, tiles, stream, fsplit, st, reverse)
                       : dispatch_dir<kBwd, false>(tw, p, grid, stages, tiles, stream, fsplit, st, reverse);
  if (rc == -21) ts::set_last_error("lstm_seq: the thread-block clusters are not co-resident on this device");
  return rc;
}

extern "C" int ts_lstm_seq_fwd(const void* gx, const void* w_h, const float* bias, const void* h_seq, const float* c_seq,
                               void* act, const float* c0, void* dbg, void* a_tiled, int T, int B, int H, unsigned int* sync_ws, int variant,
                               cudaStream_t st, const void* h0, const unsigned int* in_gate, int in_gate_tiles_n, int extra_signal, int launch_flags,
                               const int* lengths, int reverse, void* h_drop, const int* drop_step, const unsigned int* drop_desc) {
  if (!(launch_flags & 1)) {           // bit 0: the caller has run ts_lstm_seq_prologue itself (wavefront: all prologues precede the chain)
    const int tiles_m = (B + BM - 1) / BM;
    const int total = tiles_m * BM * (H / 8);
    int blocks = (total + 255) / 256;
    if (blocks > 592) blocks = 592;
    const size_t init_off = reverse ? (size_t)T * B * H : 0;      // h0 / c0 go to row T of the reverse direction
    seq_prologue_kernel<<<blocks, 256, 0, st>>>((const __nv_bfloat16*)h0, c0, (__nv_bfloat16*)h_seq + init_off, (float*)c_seq + init_off,
                                                (__nv_bfloat16*)a_tiled, sync_ws, B, H, tiles_m);
  }
  SeqParams p{};
  p.a_tiled = (__nv_bfloat16*)a_tiled;
  p.gx = (const __nv_bfloat16*)gx; p.bias = bias; p.h_seq = (__nv_bfloat16*)h_seq; p.c_seq = (float*)c_seq;
  p.act = (__nv_bfloat16*)act; p.sync = sync_ws; p.T = T; p.B = B; p.H = H; p.dbg = (unsigned long long*)dbg;
  p.in_gate = in_gate; p.in_gate_tiles_n = in_gate_tiles_n; p.extra_signal = extra_signal;
  p.pdl_wait = (launch_flags >> 1) & 1;
  p.lengths = lengths;
  p.h_drop = (__nv_bfloat16*)h_drop;
  p.drop = ts::make_drop_spec(drop_step, drop_desc);
  return seq_common<false>(p, w_h, variant, st, reverse != 0);
}

// The launch configuration ts_lstm_seq_fwd / _bwd choose for H, B and variant, without a device: out = {ring stages, batch
// tiles per CTA, streamed weights, forward K-split}.  0, or a negative code with ts_last_error set.
extern "C" int ts_lstm_seq_config(int bwd, int H, int B, int variant, int* out) {
  SeqCfg c;
  if (int rc = seq_config(bwd != 0, H, B, variant, c)) return rc;
  out[0] = c.stages; out[1] = c.tiles; out[2] = c.stream; out[3] = c.fsplit;
  return 0;
}

extern "C" int ts_lstm_seq_prologue(const void* h0, const float* c0, void* h_seq, float* c_seq, void* a_tiled, unsigned int* sync_ws,
                                    int B, int H, cudaStream_t st) {
  const int tiles_m = (B + BM - 1) / BM;
  const int total = tiles_m * BM * (H / 8);
  int blocks = (total + 255) / 256;
  if (blocks > 592) blocks = 592;
  seq_prologue_kernel<<<blocks, 256, 0, st>>>((const __nv_bfloat16*)h0, c0, (__nv_bfloat16*)h_seq, c_seq, (__nv_bfloat16*)a_tiled, sync_ws, B, H, tiles_m);
  return (int)cudaGetLastError();
}

extern "C" int ts_lstm_seq_bwd(const void* dh_seq, const void* w_hT, const void* act, const float* c_seq, const void* dpre,
                               float* dh0, float* dc0, void* dbg, void* a_tiled, int T, int B, int H, unsigned int* sync_ws, int variant,
                               cudaStream_t st, const unsigned int* in_gate, int in_gate_tiles_n, int extra_signal, int launch_flags,
                               const int* lengths, int reverse, const int* drop_step, const unsigned int* drop_desc) {
  if (!(launch_flags & 1)) cudaMemsetAsync(sync_ws, 0, kSyncErr * sizeof(unsigned int), st);      // arrival counters restart at 0 every launch
  SeqParams p{};
  p.a_tiled = (__nv_bfloat16*)a_tiled;
  p.dh_seq = (const __nv_bfloat16*)dh_seq; p.act = (__nv_bfloat16*)act; p.c_seq = (float*)c_seq; p.dpre = (__nv_bfloat16*)dpre;
  p.dh0 = dh0; p.dc0 = dc0; p.sync = sync_ws; p.T = T; p.B = B; p.H = H; p.dbg = (unsigned long long*)dbg;
  p.in_gate = in_gate; p.in_gate_tiles_n = in_gate_tiles_n; p.extra_signal = extra_signal;
  p.pdl_wait = (launch_flags >> 1) & 1;
  p.lengths = lengths;
  p.drop = ts::make_drop_spec(drop_step, drop_desc);
  return seq_common<true>(p, w_hT, variant, st, reverse != 0);
}


// Feasibility probe: how many clusters of `cluster` CTAs of the backward kernel (1 CTA/SM, ~226 KB smem) can be co-resident.
// The fast path needs every CTA of the backward kernel co-resident, in clusters of 4 (cuda_lstm.py asks this once per device).
extern "C" int ts_lstm_seq_cluster_probe(int cluster) {
  auto kern = lstm_seq_kernel<true, 4, 1, false, false>;
  const size_t smem = 226 * 1024;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { cudaGetLastError(); return -1; }
  if (cluster > 8 && cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) { cudaGetLastError(); return -2; }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(128 / cluster * cluster); cfg.blockDim = dim3(384); cfg.dynamicSmemBytes = smem; cfg.stream = 0;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) { cudaGetLastError(); return -3; }
  return n;
}
