// K-HEAD, generic half: sparse softmax cross-entropy + accuracy + dlogits over logits that are already computed (the shapes
// the tensor-core head of head_wgmma.cu does not take: fp32 activations, more than 256 classes).  One warp per batch row.
// Reference: sparse_softmax_cross_entropy_with_logits -> reduce_mean -> argmax/equal/cast/reduce_mean
// (original src/rnn.py:55-63, 84-92).
#include "launchers.h"
#include "ts_common.cuh"

namespace {

// kExact (fp32 activations): exp / log in fp64 rounded once, and log-probabilities as (l - max) - log(sum) so that no fp32
// rounding at the magnitude of the logits enters them (tests/test_gpu_head_edges.py::test_last_state_head, fp32 rows of the
// negative regime, where l - (max + log(sum)) at l ~ -990 was off by up to half an ulp of 990 in every probability).  The bf16
// instantiation keeps the fast intrinsics and l - (max + log(sum)).  Each row's NLL goes to nll[row]; sum_rows_kernel adds them.
template <bool kExact>
__global__ void xent_rows_kernel(const float* __restrict__ logits, const long long* __restrict__ labels,
                                 float* __restrict__ dlogits, float* __restrict__ nll, int* __restrict__ correct,
                                 int B, int C) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (warp >= B) return;
  const float* r = logits + (size_t)warp * C;
  float mx = -INFINITY;
  int arg = 0x7fffffff;
  for (int c = lane; c < C; c += 32)
    if (r[c] > mx) { mx = r[c]; arg = c; }
  for (int o = 16; o > 0; o >>= 1) {
    float om = __shfl_xor_sync(0xffffffffu, mx, o);
    int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
  }
  float se = 0.f;
  for (int c = lane; c < C; c += 32) se += kExact ? ts::expf_acc(r[c] - mx) : expf(r[c] - mx);
  se = ts::warp_sum(se);
  const float ls = kExact ? ts::logf_acc(se) : logf(se);
  float lse = mx + ls;
  int y = (int)labels[warp];
  float invB = 1.0f / (float)B;
  for (int c = lane; c < C; c += 32)
    dlogits[(size_t)warp * C + c] = ((kExact ? ts::expf_acc((r[c] - mx) - ls) : expf(r[c] - lse)) - (c == y ? 1.f : 0.f)) * invB;
  if (lane == 0) {
    nll[warp] = kExact ? (mx - r[y]) + ls : lse - r[y];
    if (arg == y) atomicAdd(correct, 1);
  }
}

// loss_sum = the sum of nll [B] in a fixed order: thread t adds rows t, t + 256, ..., then a tree over the threads.  (One fp32
// atomicAdd per row summed in whatever order the warps arrived: not reproducible, and up to 2x the fp32 budget of the loss over
// 200 rows, tests/test_gpu_head_edges.py::test_last_state_head, fp32 rows.)
constexpr int kSumThreads = 256;
__global__ void __launch_bounds__(kSumThreads) sum_rows_kernel(const float* __restrict__ nll, float* __restrict__ loss_sum, int B) {
  __shared__ float red[kSumThreads];
  float s = 0.f;
  for (int i = threadIdx.x; i < B; i += kSumThreads) s += nll[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = kSumThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss_sum = red[0];
}

}  // namespace

// exact: the fp32 path's accurate softmax (xent_rows_kernel<true>).  nll: scratch [B].  loss_sum is overwritten.
extern "C" int ts_xent_rows(const float* logits, const long long* labels, float* dlogits, float* nll, float* loss_sum, int* correct,
                            int B, int C, int exact, cudaStream_t st) {
  int thr = 128, blk = (B * 32 + thr - 1) / thr;
  if (exact) xent_rows_kernel<true><<<blk, thr, 0, st>>>(logits, labels, dlogits, nll, correct, B, C);
  else xent_rows_kernel<false><<<blk, thr, 0, st>>>(logits, labels, dlogits, nll, correct, B, C);
  sum_rows_kernel<<<1, kSumThreads, 0, st>>>(nll, loss_sum, B);
  return (int)cudaGetLastError();
}
