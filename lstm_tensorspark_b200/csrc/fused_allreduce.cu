// K-AR: the cross-replica parameter average / gradient allreduce, FUSED with the update, in one kernel that
// moves the data itself over NVLink 5 / NVSwitch (peer-pointer loads/stores, or NVLS multimem ld_reduce / st).
// No NCCL call and no separate elementwise kernel on this path.
//
// Replaces: Spark reduceByKey(mean) + collect of the 8 gate-keyed weight records, once per job
// (original src/rnn.py:393-407) — and, for per-step gradient sync, the
// allreduce + ApplyAdam pair a NCCL build would run.
//
// Buffers are NVLink-symmetric (same offset on every rank); the host passes every rank's base pointer.
//   mode AVG  : w  <- (sum_r w_r)/N                       (reference semantics; input == output buffer)
//   mode SGD  : g  =  (sum_r g_r)/N ; w <- w - lr*(g + wd*w)
//   mode ADAM : g  =  (sum_r g_r)/N ; TF-Adam on (w, m, v)
// every mode also refreshes the bf16 shadow of w that the tensor-core kernels read.
//   one-shot : every rank reads all N peers for the whole message and updates its own replica
//              (2 barriers + 1 NVLink round trip; small messages).  AVG stages w in a symmetric scratch
//              first so nobody reads a half-updated peer.
//   two-shot : rank r owns slice r: reduce it (peer loads in fixed rank order, or ONE multimem.ld_reduce —
//              the switch adds), update it, and write the result into all N replicas (peer stores, or ONE
//              multimem.st — the switch fans out).  In-place safe (only the owner touches a slice), replicas
//              end bit-identical, optimizer state is touched for 1/N of the elements per rank.
// Cross-GPU barrier: per-CTA flag slots in a symmetric pad, monotonically increasing epochs (never reset),
// st.release.sys / ld.acquire.sys, bounded spin -> error flag instead of a hang if a peer died.
#include "ts_common.cuh"

namespace {

constexpr int kMaxRanks = 16;
constexpr int kMaxBlocks = 256;
constexpr int kThreads = 512;

enum Mode { MODE_AVG = 0, MODE_SGD = 1, MODE_ADAM = 2 };

struct ARArgs {
  float* in[kMaxRanks];        // symmetric input  (grads for SGD/ADAM; params for AVG two-shot; staging for AVG one-shot)
  float* param[kMaxRanks];     // symmetric fp32 params (two-shot writes all; one-shot writes [rank] only)
  __nv_bfloat16* shadow[kMaxRanks];  // symmetric bf16 shadow (entries may be null)
  uint32_t* flags[kMaxRanks];  // symmetric flag pads: [kMaxBlocks][kMaxRanks] u32
  float* mc_in;                // multicast alias of in   (null -> peer loads)
  float* mc_param;             // multicast alias of param
  __nv_bfloat16* mc_shadow;    // multicast alias of shadow
  float* m;                    // local Adam slots
  float* v;
  uint32_t* epochs;            // local [kMaxBlocks] barrier epochs
  int* err;                    // local error flag (1 = barrier timeout)
  int* step_dev;               // Adam: device-resident step counter (graph-replay safe); null -> lr is already corrected
  long long n4;                // message length in float4
  long long wd_n4;             // weight decay applies to float4 indices below this (the LSTM variables)
  int rank, world;
  float inv_world, lr, b1, b2, eps, wd;
  unsigned long long timeout_ns;
  int pdl;                     // launched as a programmatic dependent: wait for the previous kernel of the stream before exiting
};

TS_DEVICE float4 ld_f4(const float* p) {
  float4 r;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
TS_DEVICE void st_f4(float* p, float4 v) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
TS_DEVICE void st_u2(void* p, uint2 v) {
  asm volatile("st.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
TS_DEVICE float4 mc_ld_reduce_f4(const float* p) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
  return r;
}
TS_DEVICE void mc_st_f4(float* p, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
TS_DEVICE void mc_st_bf16x4(void* p, uint2 v) {
  asm volatile("multimem.st.relaxed.sys.global.v2.bf16x2 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
TS_DEVICE uint2 pack_bf16x4(float4 v) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y);
  __nv_bfloat162 hi = __floats2bfloat162_rn(v.z, v.w);
  uint2 r;
  r.x = *reinterpret_cast<uint32_t*>(&lo);
  r.y = *reinterpret_cast<uint32_t*>(&hi);
  return r;
}
TS_DEVICE unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// All CTAs with the same blockIdx on every rank meet here.  Writes made by any thread of this CTA before the
// call are visible to the peers after their wait returns (bar.sync + cumulative release / acquire, sys scope).
TS_DEVICE void cross_rank_barrier(const ARArgs& a, uint32_t epoch) {
  __syncthreads();
  int t = threadIdx.x;
  if (t < a.world) {
    uint32_t* remote = a.flags[t] + blockIdx.x * kMaxRanks + a.rank;
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(remote), "r"(epoch) : "memory");
    const uint32_t* mine = a.flags[a.rank] + blockIdx.x * kMaxRanks + t;
    unsigned long long t0 = globaltimer_ns();
    uint32_t seen;
    int spins = 0;
    while (true) {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(mine) : "memory");
      if ((int32_t)(seen - epoch) >= 0) break;
      if ((++spins & 1023) == 0 && globaltimer_ns() - t0 > a.timeout_ns) {
        atomicExch(a.err, 1);
        break;
      }
    }
  }
  __syncthreads();
}

template <int kMode>
TS_DEVICE float4 apply_update(const ARArgs& a, float4 sum, long long i, float4 w, float lr) {
  float4 g;
  g.x = sum.x * a.inv_world; g.y = sum.y * a.inv_world; g.z = sum.z * a.inv_world; g.w = sum.w * a.inv_world;
  if (kMode == MODE_AVG) return g;
  float* wp = &w.x; float* gp = &g.x;
  const float wd = i < a.wd_n4 ? a.wd : 0.f;
  if (kMode == MODE_SGD) {
#pragma unroll
    for (int k = 0; k < 4; ++k) wp[k] -= lr * (gp[k] + wd * wp[k]);
    return w;
  }
  float4 mv = reinterpret_cast<float4*>(a.m)[i], vv = reinterpret_cast<float4*>(a.v)[i];
  float* mp = &mv.x; float* vp = &vv.x;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float gg = gp[k] + wd * wp[k];
    mp[k] = a.b1 * mp[k] + (1.f - a.b1) * gg;
    vp[k] = a.b2 * vp[k] + (1.f - a.b2) * gg * gg;
    wp[k] -= lr * mp[k] / (sqrtf(vp[k]) + a.eps);        // lr is the bias-corrected lr_t
  }
  reinterpret_cast<float4*>(a.m)[i] = mv;
  reinterpret_cast<float4*>(a.v)[i] = vv;
  return w;
}

// ---------------------------------------------------------------------------------------------------------
// two-shot
// ---------------------------------------------------------------------------------------------------------
TS_DEVICE float effective_lr(const ARArgs& a) {
  if (a.step_dev == nullptr) return a.lr;
  const float t = (float)(*a.step_dev);
  return a.lr * sqrtf(1.f - powf(a.b2, t)) / (1.f - powf(a.b1, t));
}
__global__ void ar_inc_step_kernel(int* step) { *step += 1; }

template <int kMode, bool kMulticast>
__global__ void __launch_bounds__(kThreads) ar_two_shot_kernel(const __grid_constant__ ARArgs a) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");      // the next bucket may start next to this one
  const float lr = kMode == MODE_ADAM ? effective_lr(a) : a.lr;
  uint32_t epoch = a.epochs[blockIdx.x];
  cross_rank_barrier(a, ++epoch);              // every rank's inputs are final

  long long per = (a.n4 + a.world - 1) / a.world;
  long long lo = per * a.rank, hi = lo + per < a.n4 ? lo + per : a.n4;
  long long stride = (long long)gridDim.x * kThreads;
  long long i = lo + (long long)blockIdx.x * kThreads + threadIdx.x;
  for (; i < hi; i += stride) {
    float4 sum;
    if (kMulticast) {
      sum = mc_ld_reduce_f4(a.mc_in + 4 * i);
    } else {
      float4 part[kMaxRanks];
#pragma unroll
      for (int r = 0; r < kMaxRanks; ++r)
        if (r < a.world) part[r] = ld_f4(a.in[r] + 4 * i);           // all loads in flight first
      sum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int r = 0; r < kMaxRanks; ++r)
        if (r < a.world) { sum.x += part[r].x; sum.y += part[r].y; sum.z += part[r].z; sum.w += part[r].w; }
    }
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    if (kMode != MODE_AVG) w = reinterpret_cast<const float4*>(a.param[a.rank])[i];
    float4 nw = apply_update<kMode>(a, sum, i, w, lr);
    uint2 sh = pack_bf16x4(nw);
    if (kMulticast) {
      mc_st_f4(a.mc_param + 4 * i, nw);
      if (a.mc_shadow) mc_st_bf16x4(a.mc_shadow + 4 * i, sh);
    } else {
#pragma unroll
      for (int r = 0; r < kMaxRanks; ++r)
        if (r < a.world) {
          st_f4(a.param[r] + 4 * i, nw);
          if (a.shadow[r]) st_u2(a.shadow[r] + 4 * i, sh);
        }
    }
  }
  cross_rank_barrier(a, ++epoch);              // every replica holds every slice
  if (threadIdx.x == 0) a.epochs[blockIdx.x] = epoch;
  if (a.pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------------------
// one-shot
// ---------------------------------------------------------------------------------------------------------
template <int kMode>
__global__ void __launch_bounds__(kThreads) ar_one_shot_kernel(const __grid_constant__ ARArgs a) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const float lr = kMode == MODE_ADAM ? effective_lr(a) : a.lr;
  uint32_t epoch = a.epochs[blockIdx.x];
  long long stride = (long long)gridDim.x * kThreads;
  long long first = (long long)blockIdx.x * kThreads + threadIdx.x;
  float* my_param = a.param[a.rank];
  if (kMode == MODE_AVG) {                     // stage w so peers never read a half-averaged replica
    for (long long i = first; i < a.n4; i += stride)
      reinterpret_cast<float4*>(a.in[a.rank])[i] = reinterpret_cast<const float4*>(my_param)[i];
  }
  cross_rank_barrier(a, ++epoch);
  for (long long i = first; i < a.n4; i += stride) {
    float4 part[kMaxRanks];
#pragma unroll
    for (int r = 0; r < kMaxRanks; ++r)
      if (r < a.world) part[r] = ld_f4(a.in[r] + 4 * i);
    float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < kMaxRanks; ++r)        // fixed order -> bit-identical on every rank
      if (r < a.world) { sum.x += part[r].x; sum.y += part[r].y; sum.z += part[r].z; sum.w += part[r].w; }
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    if (kMode != MODE_AVG) w = reinterpret_cast<const float4*>(my_param)[i];
    float4 nw = apply_update<kMode>(a, sum, i, w, lr);
    reinterpret_cast<float4*>(my_param)[i] = nw;
    if (a.shadow[a.rank]) reinterpret_cast<uint2*>(a.shadow[a.rank])[i] = pack_bf16x4(nw);
  }
  cross_rank_barrier(a, ++epoch);              // peers are done reading my input: it may be overwritten
  if (threadIdx.x == 0) a.epochs[blockIdx.x] = epoch;
  if (a.pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
}

// pdl: programmatic dependent launch - the kernel may start while the PREVIOUS kernel of the stream is still running (as soon
// as all of that kernel's CTAs are resident and have executed griddepcontrol.launch_dependents).  Used to run a gradient
// bucket's allreduce + update on the ~20 SMs a persistent LSTM recurrence kernel leaves idle; it does not read anything the
// previous kernel writes, so it never executes griddepcontrol.wait.
template <typename K>
int launch_k(K kern, const ARArgs& a, int blocks, int pdl, cudaStream_t st) {
  // no shared memory of our own, but ask for the max-shared L1 split: the split the tensor-core kernels run with, so that
  // these CTAs can be co-resident with a weight-gradient GEMM on the same SMs (see gemm2_wgmma.cu)
  cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
  return (int)cudaLaunchKernelEx(&cfg, kern, a);
}

template <int kMode>
int launch_mode(const ARArgs& a, int two_shot, int multicast, int blocks, int pdl, cudaStream_t st) {
  if (two_shot) {
    if (multicast) return launch_k(ar_two_shot_kernel<kMode, true>, a, blocks, pdl, st);
    return launch_k(ar_two_shot_kernel<kMode, false>, a, blocks, pdl, st);
  }
  return launch_k(ar_one_shot_kernel<kMode>, a, blocks, pdl, st);
}

}  // namespace

// ptrs: [4][world] = in, param, shadow, flags base pointers of every rank.
extern "C" int ts_fused_allreduce(const unsigned long long* ptrs, unsigned long long mc_in, unsigned long long mc_param,
                                  unsigned long long mc_shadow, float* m, float* v, unsigned int* epochs, int* err,
                                  long long n, int rank, int world, int mode, int two_shot, int multicast, int blocks,
                                  float lr, float b1, float b2, float eps, float wd, double timeout_s,
                                  cudaStream_t st, int* step_dev, long long wd_n, int bump_step, int pdl) {
  // the decay is chosen per float4: a cut inside one would decay a different range than [0, wd_n)
  if (world > kMaxRanks || world < 1 || n % 4 != 0 || (wd_n >= 0 && wd_n % 4 != 0)) return -2;
  if (blocks > kMaxBlocks) blocks = kMaxBlocks;
  if (blocks < 1) blocks = 1;
  ARArgs a;
  for (int r = 0; r < kMaxRanks; ++r) {
    a.in[r] = r < world ? (float*)ptrs[0 * world + r] : nullptr;
    a.param[r] = r < world ? (float*)ptrs[1 * world + r] : nullptr;
    a.shadow[r] = r < world ? (__nv_bfloat16*)ptrs[2 * world + r] : nullptr;
    a.flags[r] = r < world ? (uint32_t*)ptrs[3 * world + r] : nullptr;
  }
  a.mc_in = (float*)mc_in; a.mc_param = (float*)mc_param; a.mc_shadow = (__nv_bfloat16*)mc_shadow;
  a.m = m; a.v = v; a.epochs = epochs; a.err = err; a.step_dev = (mode == MODE_ADAM) ? step_dev : nullptr;
  if (a.step_dev && bump_step) ar_inc_step_kernel<<<1, 1, 0, st>>>(a.step_dev);     // once per optimizer step, not per bucket
  a.wd_n4 = wd_n < 0 ? n / 4 : wd_n / 4;
  a.n4 = n / 4; a.rank = rank; a.world = world; a.inv_world = 1.0f / (float)world;
  a.lr = lr; a.b1 = b1; a.b2 = b2; a.eps = eps; a.wd = wd;
  a.timeout_ns = (unsigned long long)(timeout_s * 1e9);
  a.pdl = pdl;
  if (multicast && (!mc_in || !mc_param)) multicast = 0;
  switch (mode) {
    case MODE_AVG: return launch_mode<MODE_AVG>(a, two_shot, multicast, blocks, pdl, st);
    case MODE_SGD: return launch_mode<MODE_SGD>(a, two_shot, multicast, blocks, pdl, st);
    case MODE_ADAM: return launch_mode<MODE_ADAM>(a, two_shot, multicast, blocks, pdl, st);
  }
  return -3;
}

// Adam's device-resident step counter += 1 (once per optimizer step, BEFORE backward: a launch of its own between a
// weight-gradient GEMM and a bucket's allreduce would serialise the two)
extern "C" int ts_ar_bump_step(int* step_dev, cudaStream_t st) {
  ar_inc_step_kernel<<<1, 1, 0, st>>>(step_dev);
  return (int)cudaGetLastError();
}

extern "C" int ts_ar_max_blocks() { return kMaxBlocks; }
// Flag pads / epoch counters come in kSlots independent sets: two buckets whose kernels are in flight at the same time (the
// second one is a programmatic dependent of the first) must not share barrier state.
constexpr int kSlots = 8;
extern "C" int ts_ar_flag_words() { return kMaxBlocks * kMaxRanks * kSlots; }
extern "C" int ts_ar_slots() { return kSlots; }
