// K-HEAD, generic half: sparse softmax cross-entropy + accuracy + dlogits over logits that are already computed (the shapes
// the tensor-core head of head_wgmma.cu does not take: fp32 activations, more than 256 classes).  One warp per batch row.
// Reference: sparse_softmax_cross_entropy_with_logits -> reduce_mean -> argmax/equal/cast/reduce_mean
// (original src/rnn.py:55-63, 84-92).
#include "ts_common.cuh"

namespace {

__global__ void xent_rows_kernel(const float* __restrict__ logits, const long long* __restrict__ labels,
                                 float* __restrict__ dlogits, float* __restrict__ loss_sum, int* __restrict__ correct,
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
  for (int c = lane; c < C; c += 32) se += expf(r[c] - mx);
  se = ts::warp_sum(se);
  float lse = mx + logf(se);
  int y = (int)labels[warp];
  float invB = 1.0f / (float)B;
  for (int c = lane; c < C; c += 32)
    dlogits[(size_t)warp * C + c] = (expf(r[c] - lse) - (c == y ? 1.f : 0.f)) * invB;
  if (lane == 0) {
    atomicAdd(loss_sum, lse - r[y]);
    if (arg == y) atomicAdd(correct, 1);
  }
}

}  // namespace

extern "C" int ts_xent_rows(const float* logits, const long long* labels, float* dlogits, float* loss_sum, int* correct,
                            int B, int C, cudaStream_t st) {
  int thr = 128, blk = (B * 32 + thr - 1) / thr;
  xent_rows_kernel<<<blk, thr, 0, st>>>(logits, labels, dlogits, loss_sum, correct, B, C);
  return (int)cudaGetLastError();
}
