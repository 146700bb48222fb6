// Any-shape GEMM on the CUDA cores:  C[M,N] = beta * C + A[M,K] · B[K,N]  with arbitrary element strides (so every
// transpose is free), bf16 or fp32 operands, fp32 accumulation.  It serves the shapes the tensor-core kernels cannot take
// (TMA needs 16 B-aligned pitches and the tensor-core tiles 64-wide K blocks): the reference's own configuration - iris,
// in_features = 4, hidden 16, batch 10, ONE time step (original src/rnn.py:312-321, lstm.py:88-91) - and the fp32
// parity path.  Performance target: none; these products are a few kFLOP.  Keeping them on our own kernel means the
// product path never calls a library GEMM.
#include "launchers.h"
#include "ts_common.cuh"

namespace {

constexpr int GT = 32;     // output tile
constexpr int GK = 16;     // k tile
constexpr int GCHUNK = 64; // k tiles per partial sum

template <typename TA, typename TB, typename TC>
__global__ void __launch_bounds__(256) gemm_generic_kernel(const TA* __restrict__ A, const TB* __restrict__ B, TC* __restrict__ C,
                                                           const float* __restrict__ bias, int M, int N, int K, long long a_rs, long long a_cs,
                                                           long long b_rs, long long b_cs, long long c_rs, float beta) {
  __shared__ float sa[GK][GT + 1];
  __shared__ float sb[GK][GT + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;          // 16 x 16 threads, 2 x 2 outputs each
  const int m0 = blockIdx.x * GT, n0 = blockIdx.y * GT;          // M on grid x (up to 2^31 - 1 blocks): M = T·B rows
  // Long contractions (the weight gradients, K = T·B rows) are summed in three levels - GK products per k tile, GCHUNK k tiles
  // per chunk, the chunks - so that the fp32 rounding error grows with about GK + GCHUNK + K / (GK·GCHUNK) terms instead of K.
  // With K <= GK it is the plain fma chain.
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, chunk[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  int tiles = 0;
  for (int k0 = 0; k0 < K; k0 += GK) {
    for (int i = threadIdx.x; i < GK * GT; i += 256) {
      const int kk = i / GT, mm = i % GT;
      const int m = m0 + mm, k = k0 + kk;
      sa[kk][mm] = (m < M && k < K) ? ts::Cvt<TA>::to_f(A[(long long)m * a_rs + (long long)k * a_cs]) : 0.f;
      const int n = n0 + mm;
      sb[kk][mm] = (n < N && k < K) ? ts::Cvt<TB>::to_f(B[(long long)k * b_rs + (long long)n * b_cs]) : 0.f;
    }
    __syncthreads();
    float part[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
    for (int kk = 0; kk < GK; ++kk) {
      const float a0 = sa[kk][ty], a1 = sa[kk][ty + 16], b0 = sb[kk][tx], b1 = sb[kk][tx + 16];
      part[0][0] = fmaf(a0, b0, part[0][0]); part[0][1] = fmaf(a0, b1, part[0][1]);
      part[1][0] = fmaf(a1, b0, part[1][0]); part[1][1] = fmaf(a1, b1, part[1][1]);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) chunk[i][j] += part[i][j];
    if (++tiles == GCHUNK) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) { acc[i][j] += chunk[i][j]; chunk[i][j] = 0.f; }
      tiles = 0;
    }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) acc[i][j] += chunk[i][j];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int m = m0 + ty + 16 * i, n = n0 + tx + 16 * j;
      if (m < M && n < N) {
        TC* c = C + (long long)m * c_rs + n;
        float v = acc[i][j] + (bias ? bias[n] : 0.f);
        if (beta != 0.f) v += beta * ts::Cvt<TC>::to_f(*c);
        *c = ts::Cvt<TC>::from_f(v);
      }
    }
}

template <typename TA, typename TB, typename TC>
int launch_g(const void* A, const void* B, void* C, const float* bias, int M, int N, int K, long long a_rs, long long a_cs, long long b_rs,
             long long b_cs, long long c_rs, float beta, cudaStream_t st) {
  dim3 grid((M + GT - 1) / GT, (N + GT - 1) / GT);
  gemm_generic_kernel<TA, TB, TC><<<grid, 256, 0, st>>>((const TA*)A, (const TB*)B, (TC*)C, bias, M, N, K, a_rs, a_cs, b_rs, b_cs, c_rs, beta);
  return (int)cudaGetLastError();
}

}  // namespace

// dtype codes: 0 = fp32, 1 = bf16.  A element (m,k) at A[m*a_rs + k*a_cs], B element (k,n) at B[k*b_rs + n*b_cs], C row pitch c_rs.
extern "C" int ts_gemm_generic(const void* A, const void* B, void* C, const float* bias, int M, int N, int K, long long a_rs, long long a_cs,
                               long long b_rs, long long b_cs, long long c_rs, int a_bf16, int b_bf16, int c_bf16, float beta, cudaStream_t st) {
  if (M <= 0 || N <= 0) return 0;
  using bf = __nv_bfloat16;
#define GO(TA, TB, TC) return launch_g<TA, TB, TC>(A, B, C, bias, M, N, K, a_rs, a_cs, b_rs, b_cs, c_rs, beta, st)
  if (a_bf16 && b_bf16) { if (c_bf16) GO(bf, bf, bf); else GO(bf, bf, float); }
  if (a_bf16 && !b_bf16) { if (c_bf16) GO(bf, float, bf); else GO(bf, float, float); }
  if (!a_bf16 && b_bf16) { if (c_bf16) GO(float, bf, bf); else GO(float, bf, float); }
  if (c_bf16) GO(float, float, bf); else GO(float, float, float);
#undef GO
}
