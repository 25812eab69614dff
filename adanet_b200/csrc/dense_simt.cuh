// CUDA-core fp32 GEMM used (a) as the always-available exact-fp32 dense path for
// shapes the tcgen05 path does not take (skinny logits layers, ragged K) and
// (b) as the on-device cross-check of the tensor path.
//
//   C[M,N] = op(A) * op(B)     A_T=0: A[m*lda+k]   A_T=1: A[k*lda+m]
//                              B_T=0: B[k*ldb+n]   B_T=1: B[n*ldb+k]
//
// Epilogues: bias+activation (dense fwd), ReLU mask (dX), split-K partial (dW).
#pragma once
#include "common.cuh"

namespace adn {
namespace simt {

enum { EPI_BIAS_ACT = 0, EPI_MASK = 1, EPI_PARTIAL = 2 };

struct GemmArgs {
  const float* A;
  const float* B;
  float* C;
  int M, N, K;
  int lda, ldb, ldc;
  const float* bias;  // EPI_BIAS_ACT (nullable)
  int act;
  const float* mask;  // EPI_MASK (nullable): C *= (mask[m*ldmask+n] > 0)
  int ldmask;
  int k_per_split;    // EPI_PARTIAL: blockIdx.z covers K range [z*kps, (z+1)*kps); C += z*M*N
};

template <int BM, int BN, int BK, int TM, int TN, bool A_T, bool B_T, int EPI>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
sgemm_kernel(GemmArgs g) {
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int VM = TM < 4 ? TM : 4;
  constexpr int VN = TN < 4 ? TN : 4;
  constexpr int TX = BN / TN;  // threads across N
  constexpr int TY = BM / TM;
  constexpr int PAD = 4;
  constexpr int A_PER = BM * BK / NT;
  constexpr int B_PER = BN * BK / NT;
  static_assert(BM * BK % NT == 0 && BN * BK % NT == 0, "tile/threads mismatch");

  __shared__ float As[BK][BM + PAD];
  __shared__ float Bs[BK][BN + PAD];

  const int tid = threadIdx.x;
  const int tx = tid % TX, ty = tid / TX;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  int k_begin = 0, k_end = g.K;
  float* C = g.C;
  if (EPI == EPI_PARTIAL) {
    k_begin = blockIdx.z * g.k_per_split;
    k_end = min(g.K, k_begin + g.k_per_split);
    C += (size_t)blockIdx.z * g.M * g.N;
  }

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float ra[A_PER], rb[B_PER];

  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int idx = tid + i * NT;
      int mm, kk;
      if (A_T) { mm = idx % BM; kk = idx / BM; } else { kk = idx % BK; mm = idx / BK; }
      int m = m0 + mm, k = k0 + kk;
      float v = 0.f;
      if (m < g.M && k < k_end) v = A_T ? __ldg(g.A + (size_t)k * g.lda + m) : __ldg(g.A + (size_t)m * g.lda + k);
      ra[i] = v;
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int idx = tid + i * NT;
      int nn, kk;
      if (B_T) { kk = idx % BK; nn = idx / BK; } else { nn = idx % BN; kk = idx / BN; }
      int n = n0 + nn, k = k0 + kk;
      float v = 0.f;
      if (n < g.N && k < k_end) v = B_T ? __ldg(g.B + (size_t)n * g.ldb + k) : __ldg(g.B + (size_t)k * g.ldb + n);
      rb[i] = v;
    }
  };
  auto store_tiles = [&]() {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int idx = tid + i * NT;
      int mm, kk;
      if (A_T) { mm = idx % BM; kk = idx / BM; } else { kk = idx % BK; mm = idx / BK; }
      As[kk][mm] = ra[i];
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int idx = tid + i * NT;
      int nn, kk;
      if (B_T) { kk = idx % BK; nn = idx / BK; } else { nn = idx % BN; kk = idx / BN; }
      Bs[kk][nn] = rb[i];
    }
  };

  if (k_begin < k_end) load_tiles(k_begin);
  for (int k0 = k_begin; k0 < k_end; k0 += BK) {
    store_tiles();
    __syncthreads();
    if (k0 + BK < k_end) load_tiles(k0 + BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[kk][(i / VM) * (TY * VM) + ty * VM + (i % VM)];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[kk][(j / VN) * (TX * VN) + tx * VN + (j % VN)];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + (i / VM) * (TY * VM) + ty * VM + (i % VM);
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n = n0 + (j / VN) * (TX * VN) + tx * VN + (j % VN);
      if (n >= g.N) continue;
      float v = acc[i][j];
      if (EPI == EPI_BIAS_ACT) {
        if (g.bias) v += __ldg(g.bias + n);
        if (g.act == ADN_ACT_RELU) v = fmaxf(v, 0.f);
      } else if (EPI == EPI_MASK) {
        if (g.mask && !(__ldg(g.mask + (size_t)m * g.ldmask + n) > 0.f)) v = 0.f;
      }
      C[(size_t)m * g.ldc + n] = v;
    }
  }
}

// out[i] = scale * sum_{s<S} part[s*stride + i] (fixed order -> deterministic) for several jobs in one launch
struct ReduceJob { const float* part; float* out; int64_t n; int S; int64_t stride; float scale = 1.0f; };   // out = scale * sum
int reduce_partials_group(const ReduceJob* jobs, int n, cudaStream_t st);
// column sums out[c] = scale * sum_r x[r, c] via fixed-order partials for several jobs in one launch (+ one reduce
// launch); part = 64 * cols floats of scratch per job
struct ColsumJob { const float* x; float* out; int64_t rows, cols; float* part; float scale = 1.0f; };
int colsum_group(const ColsumJob* jobs, int n, cudaStream_t st);

int dense_fwd(const float* x, const float* w, const float* b, float* y, int64_t batch, int64_t in,
              int64_t out, int act, cudaStream_t st);
int dense_bwd(const float* x, const float* w, const float* dz, float* dx, float* dw, float* db,
              int64_t batch, int64_t in, int64_t out, int x_relu_mask, void* ws, int64_t ws_bytes,
              cudaStream_t st);
int64_t dense_bwd_workspace_bytes(int64_t batch, int64_t in, int64_t out);
int dw_splits(int64_t batch, int64_t in, int64_t out);

}  // namespace simt
}  // namespace adn
