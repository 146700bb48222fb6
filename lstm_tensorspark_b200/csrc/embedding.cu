// Token embedding in front of the first LSTM layer (--vocab_size V): x_t = Embedding[tok_t], nn.Embedding(V, E).
//
// Tokens are int32 [B,T] (batch-major, as the loaders hold them); lengths (int32 [B], device, optional) mark the counted steps
// t < len_b.  Row r = t·B + b of the time-major output / gradient is position (t, b).  A position is counted when t < len_b and
// its id lies in [0, V): anything else reads a zero row and gets no gradient, so no kernel ever reads outside the table.  Nothing
// is read back to the host, so a captured graph holds across token batches and lengths.
//
//   forward   one launch: x [T·B, E] = table[tok] (the bf16 shadow on the bf16 path), one warp per row, 16-byte vector copies
//             when a row is a whole number of 16 B, element copies otherwise.
//   backward  dW [V, E] fp32 (the table's flat gradient sink: overwrite writes every row, zeros included; accumulate adds only
//             to the rows of ids present).  Three launches, bitwise reproducible and independent of the grid and the SM count:
//     1. rank    one CTA per chunk of kChunk rows: a bitonic sort of (id, row) in shared memory gives each counted row its rank
//                among the chunk's rows of the same id (rows stay in increasing order) and the chunk's runs (id, count); the
//                counts are added to a per-id histogram (integer atomics: order-independent).
//     2. plan    one CTA: exclusive scans of the histogram (segment offsets, the number of kSeg-row pieces of each id), then the
//                chunks in order hand every run its base within its id's segment, then every row is scattered to its place.
//                The result is a stable counting sort: the rows of one id in increasing row order t·B + b.
//     3. sum     one CTA per id plus one per further piece of a long segment: sums its rows of dx in fp32 in row order.  An id
//                with several pieces writes per-piece partials, and the last piece to take the id's ticket sums them in piece
//                order (and leaves the ticket 0).  A single id at every position costs T·B / kSeg CTAs, not one.
#include "ts_common.cuh"

namespace {

constexpr int kChunk = 1024;           // rows per CTA of the rank kernel (= its threads)
constexpr int kSeg = 64;               // rows per piece of an id's segment in the sum kernel
constexpr int kSumThreads = 256;
constexpr int kFwdThreads = 256;       // 8 rows (one warp each) per CTA
constexpr unsigned kNone = 0xFFFFFFFFu;

// Exclusive prefix sum over the CTA (blockDim.x a multiple of 32, at most 1024); `total` = the sum over all threads.
TS_DEVICE int block_excl_scan(int v, int* wt, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) wt[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int s = lane < nw ? wt[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    wt[lane] = s;                                              // inclusive; lanes >= nw hold the total
  }
  __syncthreads();
  const int base = warp ? wt[warp - 1] : 0;
  total = wt[31];
  __syncthreads();                                             // wt is reused by the next call
  return base + x - v;
}

template <typename TT>
__global__ void __launch_bounds__(kFwdThreads) embed_fwd_kernel(const TT* __restrict__ table, const int* __restrict__ tok,
                                                                const int* __restrict__ lengths, int T, int B, int E, int V,
                                                                long long N, int vec, TT* __restrict__ x) {
  const long long r = (long long)blockIdx.x * (kFwdThreads / 32) + (threadIdx.x >> 5);
  if (r >= N) return;
  const int lane = threadIdx.x & 31;
  const int t = (int)(r / B), b = (int)(r - (long long)t * B);
  const int len = lengths ? lengths[b] : T;
  int id = -1;
  if (t < len) {
    const int v = tok[(size_t)b * T + t];
    if (v >= 0 && v < V) id = v;
  }
  TT* dst = x + r * E;
  if (vec) {
    const int nv = (int)(E * sizeof(TT) / 16);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    if (id < 0) {
      for (int k = lane; k < nv; k += 32) d4[k] = make_uint4(0u, 0u, 0u, 0u);
    } else {
      const uint4* s4 = reinterpret_cast<const uint4*>(table + (size_t)id * E);
      for (int k = lane; k < nv; k += 32) d4[k] = __ldg(s4 + k);
    }
    return;
  }
  const TT* src = table + (size_t)(id < 0 ? 0 : id) * E;
  for (int k = lane; k < E; k += 32) dst[k] = id < 0 ? ts::Cvt<TT>::from_f(0.f) : src[k];
}

// elem_run[r]: the global run slot of row r (-1 = not counted), elem_rank[r]: its rank within the run; run_id / run_cnt per slot
// k·kChunk + i; nruns[k]; counts[id] += run counts.
__global__ void __launch_bounds__(kChunk) embed_rank_kernel(const int* __restrict__ tok, const int* __restrict__ lengths, int T,
                                                            int B, int V, int N, int* __restrict__ counts, int* __restrict__ elem_run,
                                                            int* __restrict__ elem_rank, int* __restrict__ run_id,
                                                            int* __restrict__ run_cnt, int* __restrict__ nruns) {
  __shared__ unsigned long long key[kChunk];
  __shared__ int start[kChunk + 1];
  __shared__ int wt[32];
  const int k = blockIdx.x, i = threadIdx.x;
  const int r = k * kChunk + i;
  unsigned id = kNone;
  if (r < N) {
    const int t = r / B, b = r - t * B;
    const int len = lengths ? lengths[b] : T;
    if (t < len) {
      const int v = tok[(size_t)b * T + t];
      if (v >= 0 && v < V) id = (unsigned)v;
    }
    elem_run[r] = -1;
  }
  key[i] = ((unsigned long long)id << 32) | (unsigned)i;      // unique keys: the sorted order is the (id, row) order
  __syncthreads();
  for (int size = 2; size <= kChunk; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const int j = i ^ stride;
      if (j > i) {
        const unsigned long long a = key[i], c = key[j];
        if ((a > c) == ((i & size) == 0)) { key[i] = c; key[j] = a; }
      }
      __syncthreads();
    }
  }
  const unsigned long long me = key[i];
  const unsigned sid = (unsigned)(me >> 32);
  const bool valid = sid != kNone;
  const bool head = valid && (i == 0 || (unsigned)(key[i - 1] >> 32) != sid);
  int total;
  const int before = block_excl_scan(head ? 1 : 0, wt, total);  // heads at sorted positions < i
  if (head) start[before] = i;
  if (valid && (i == kChunk - 1 || (unsigned)(key[i + 1] >> 32) == kNone)) start[total] = i + 1;
  __syncthreads();
  if (valid) {
    const int run = head ? before : before - 1;
    const int row = k * kChunk + (int)(me & 0xFFFFFFFFu);
    elem_run[row] = k * kChunk + run;
    elem_rank[row] = i - start[run];
    if (head) {
      const int cnt = start[run + 1] - i;
      run_id[k * kChunk + run] = (int)sid;
      run_cnt[k * kChunk + run] = cnt;
      atomicAdd(counts + sid, cnt);
    }
  }
  if (i == 0) nruns[k] = total;
}

// One CTA of kChunk threads.  counts -> offs / xoff / poff (exclusive scans, entry V = the total) and back to 0; cursor = offs;
// run_base per run slot (chunks in order); sorted[offs[id] + rank] = row.
__global__ void __launch_bounds__(kChunk) embed_plan_kernel(int V, int N, int nchunks, int* __restrict__ counts,
                                                            int* __restrict__ offs, int* __restrict__ xoff, int* __restrict__ poff,
                                                            int* __restrict__ cursor, const int* __restrict__ elem_run,
                                                            const int* __restrict__ elem_rank, const int* __restrict__ run_id,
                                                            const int* __restrict__ run_cnt, int* __restrict__ run_base,
                                                            const int* __restrict__ nruns, int* __restrict__ sorted) {
  __shared__ int wt[32];
  int c0 = 0, c1 = 0, c2 = 0;
  for (int base = 0; base < V; base += kChunk) {
    const int v = base + threadIdx.x;
    int c = 0;
    if (v < V) { c = counts[v]; counts[v] = 0; }
    const int pieces = (c + kSeg - 1) / kSeg;
    int t0, t1, t2;
    const int e0 = block_excl_scan(c, wt, t0);
    const int e1 = block_excl_scan(pieces > 1 ? pieces - 1 : 0, wt, t1);   // CTAs beyond the first of an id
    const int e2 = block_excl_scan(pieces > 1 ? pieces : 0, wt, t2);       // partial slots
    if (v < V) { offs[v] = c0 + e0; cursor[v] = c0 + e0; xoff[v] = c1 + e1; poff[v] = c2 + e2; }
    c0 += t0; c1 += t1; c2 += t2;
  }
  if (threadIdx.x == 0) { offs[V] = c0; xoff[V] = c1; poff[V] = c2; }
  __syncthreads();
  for (int k = 0; k < nchunks; ++k) {                          // a chunk's runs have distinct ids: one thread each, no conflict
    const int i = threadIdx.x;
    if (i < nruns[k]) {
      const int s = k * kChunk + i, id = run_id[s];
      const int b0 = cursor[id];
      run_base[s] = b0;
      cursor[id] = b0 + run_cnt[s];
    }
    __syncthreads();
  }
  for (int r = threadIdx.x; r < N; r += kChunk) {
    const int er = elem_run[r];
    if (er >= 0) sorted[run_base[er] + elem_rank[r]] = r;
  }
}

template <typename TD>
__global__ void __launch_bounds__(kSumThreads) embed_sum_kernel(const TD* __restrict__ dx, int E, int V, const int* __restrict__ offs,
                                                                const int* __restrict__ xoff, const int* __restrict__ poff,
                                                                const int* __restrict__ sorted, float* __restrict__ partial,
                                                                unsigned int* __restrict__ tickets, float* __restrict__ dW,
                                                                int accumulate) {
  __shared__ int rows[kSeg];
  __shared__ bool last_s;
  int v, j;
  if ((int)blockIdx.x < V) {
    v = blockIdx.x;
    j = 0;
  } else {
    const int e = (int)blockIdx.x - V;
    if (e >= xoff[V]) return;
    int lo = 0, hi = V;                                        // xoff[lo] <= e < xoff[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (xoff[mid] <= e) lo = mid; else hi = mid;
    }
    v = lo;
    j = e - xoff[v] + 1;
  }
  const int beg = offs[v], c = offs[v + 1] - beg;
  float* out = dW + (size_t)v * E;
  if (c == 0) {
    if (!accumulate)
      for (int col = threadIdx.x; col < E; col += kSumThreads) out[col] = 0.f;
    return;
  }
  const int pieces = (c + kSeg - 1) / kSeg;
  const int r0 = j * kSeg, nr = min(kSeg, c - r0);
  if ((int)threadIdx.x < nr) rows[threadIdx.x] = sorted[beg + r0 + threadIdx.x];
  __syncthreads();
  float* dst = pieces == 1 ? nullptr : partial + (size_t)(poff[v] + j) * E;
  for (int col = threadIdx.x; col < E; col += kSumThreads) {
    float acc = 0.f;
#pragma unroll 4
    for (int q = 0; q < nr; ++q) acc += ts::Cvt<TD>::to_f(dx[(size_t)rows[q] * E + col]);
    if (pieces == 1) out[col] = accumulate ? out[col] + acc : acc;
    else dst[col] = acc;
  }
  if (pieces == 1) return;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last_s = atomicAdd(tickets + v, 1u) == (unsigned)(pieces - 1);
  __syncthreads();
  if (!last_s) return;
  __threadfence();
  const float* p = partial + (size_t)poff[v] * E;
  for (int col = threadIdx.x; col < E; col += kSumThreads) {
    float acc = 0.f;
    for (int q = 0; q < pieces; ++q) acc += __ldcg(p + (size_t)q * E + col);
    out[col] = accumulate ? out[col] + acc : acc;
  }
  if (threadIdx.x == 0) tickets[v] = 0u;
}

// int32 scratch layout of the backward pass (see ts_embed_scratch_numel)
struct Scratch {
  int *cursor, *offs, *xoff, *poff, *elem_run, *elem_rank, *run_id, *run_cnt, *run_base, *sorted, *nruns;
};

Scratch carve(int* s, int N, int V) {
  const int nchunks = (N + kChunk - 1) / kChunk;
  const size_t NC = (size_t)nchunks * kChunk;
  Scratch p;
  p.cursor = s;  s += V;
  p.offs = s;    s += V + 1;
  p.xoff = s;    s += V + 1;
  p.poff = s;    s += V + 1;
  p.elem_run = s;  s += N;
  p.elem_rank = s; s += N;
  p.run_id = s;    s += NC;
  p.run_cnt = s;   s += NC;
  p.run_base = s;  s += NC;
  p.sorted = s;    s += N;
  p.nruns = s;
  return p;
}

}  // namespace

// Scratch of ts_embed_bwd for N = T·B rows, V ids and width E: ints[0] int32 words of working space, ints[1] fp32 words of piece
// partials.  Besides these the call takes `zeroed`, 2 V int32 words (per-id counts, then per-id tickets) that must be zero when it
// starts; it leaves every word it touches zero again, so one zeroed buffer serves calls of any V up to its size.
extern "C" void ts_embed_scratch_numel(long long N, long long V, long long E, long long* ints) {
  const long long nchunks = (N + kChunk - 1) / kChunk;
  ints[0] = 4 * V + 3 + 3 * N + 3 * nchunks * kChunk + nchunks;
  ints[1] = (2 * (N / kSeg) + 2) * E;        // pieces of multi-piece ids: sum ceil(c / kSeg) over c > kSeg <= 2 N / kSeg
}

// table [V, E] (bf16 iff bf16), tok int32 [B, T], lengths int32 [B] or null -> x [T·B, E] of the table's type.
extern "C" int ts_embed_fwd(const void* table, int bf16, const int* tok, const int* lengths, int T, int B, int E, int V, void* x,
                            cudaStream_t st) {
  if (T < 1 || B < 1 || E < 1 || V < 1) return -2;
  const long long N = (long long)T * B;
  const size_t elt = bf16 ? 2 : 4;
  const int vec = ((size_t)E * elt) % 16 == 0 && ((uintptr_t)table % 16) == 0 && ((uintptr_t)x % 16) == 0;
  const unsigned grid = (unsigned)((N + kFwdThreads / 32 - 1) / (kFwdThreads / 32));
  if (bf16)
    embed_fwd_kernel<__nv_bfloat16><<<grid, kFwdThreads, 0, st>>>((const __nv_bfloat16*)table, tok, lengths, T, B, E, V, N, vec,
                                                                  (__nv_bfloat16*)x);
  else
    embed_fwd_kernel<float><<<grid, kFwdThreads, 0, st>>>((const float*)table, tok, lengths, T, B, E, V, N, vec, (float*)x);
  return (int)cudaGetLastError();
}

// dx [T·B, E] (bf16 iff dx_bf16) -> dW fp32 [V, E]: overwrite every row (accumulate = 0) or add to the rows of ids present.
extern "C" int ts_embed_bwd(const void* dx, int dx_bf16, const int* tok, const int* lengths, int T, int B, int E, int V, float* dW,
                            int accumulate, int* zeroed, int* scratch, float* partial, cudaStream_t st) {
  if (T < 1 || B < 1 || E < 1 || V < 1) return -2;
  const long long N64 = (long long)T * B;
  if (N64 > (1LL << 30) || (long long)V > (1LL << 30)) return -3;
  const int N = (int)N64;
  const int nchunks = (N + kChunk - 1) / kChunk;
  Scratch s = carve(scratch, N, V);
  int* counts = zeroed;                                        // reset by the plan kernel
  unsigned int* tickets = (unsigned int*)(zeroed + V);         // reset by the last piece of each id
  embed_rank_kernel<<<nchunks, kChunk, 0, st>>>(tok, lengths, T, B, V, N, counts, s.elem_run, s.elem_rank, s.run_id, s.run_cnt,
                                                s.nruns);
  embed_plan_kernel<<<1, kChunk, 0, st>>>(V, N, nchunks, counts, s.offs, s.xoff, s.poff, s.cursor, s.elem_run, s.elem_rank,
                                          s.run_id, s.run_cnt, s.run_base, s.nruns, s.sorted);
  const unsigned grid = (unsigned)(V + N / kSeg + 1);          // one CTA per id + at most N / kSeg further pieces
  if (dx_bf16)
    embed_sum_kernel<__nv_bfloat16><<<grid, kSumThreads, 0, st>>>((const __nv_bfloat16*)dx, E, V, s.offs, s.xoff, s.poff, s.sorted,
                                                                  partial, tickets, dW, accumulate);
  else
    embed_sum_kernel<float><<<grid, kSumThreads, 0, st>>>((const float*)dx, E, V, s.offs, s.xoff, s.poff, s.sorted, partial,
                                                          tickets, dW, accumulate);
  return (int)cudaGetLastError();
}

extern "C" int ts_embed_bwd_launches() { return 3; }
