// Launchers for the CUDA-core fp32 dense path.  See dense_simt.cuh.
#include <algorithm>

#include "dense_simt.cuh"

namespace adn {
namespace simt {

// rows per first-level slice: at most 64 slices, at least 64 rows each (each thread then adds >= 8 rows)
static inline int colsum_slice_rows(int64_t rows) {
  int64_t r = ceil_div(rows, 64);
  r = ceil_div(r, 8) * 8;
  return (int)(r < 64 ? 64 : r);
}

// ---- one launch for the same reduction of several jobs (blockIdx.z = job) ----
static constexpr int kMaxJobs = 16;
struct ReduceJobs { ReduceJob j[kMaxJobs]; };
struct ColsumJobs { ColsumJob j[kMaxJobs]; int rps[kMaxJobs]; };

static __global__ void reduce_partials_group_kernel(const __grid_constant__ ReduceJobs jobs) {
  const ReduceJob& jb = jobs.j[blockIdx.z];
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= jb.n) return;
  float acc = 0.f;
  for (int s = 0; s < jb.S; ++s) acc += jb.part[(size_t)s * jb.stride + i];
  jb.out[i] = acc * jb.scale;     // scale is a power of two (gradient planes carry 2^k): exact
}

static __global__ void __launch_bounds__(256)
colsum_partial_group_kernel(const __grid_constant__ ColsumJobs jobs) {
  __shared__ float sm[8][33];
  const ColsumJob& jb = jobs.j[blockIdx.z];
  const int rows_per_slice = jobs.rps[blockIdx.z];
  const int N = (int)jb.cols, rows = (int)jb.rows;
  const int cx = threadIdx.x % 32, ry = threadIdx.x / 32;
  const int n = blockIdx.x * 32 + cx;
  const int r0 = blockIdx.y * rows_per_slice;
  if (r0 >= rows || blockIdx.x * 32 >= N) return;       // uniform per block
  const int r1 = min(rows, r0 + rows_per_slice);
  float acc = 0.f;
  if (n < N)
    for (int r = r0 + ry; r < r1; r += 8) acc += jb.x[(size_t)r * N + n];
  sm[ry][cx] = acc;
  __syncthreads();
  if (ry == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][cx];
    jb.part[(size_t)blockIdx.y * N + n] = t;
  }
}

int reduce_partials_group(const ReduceJob* jobs, int n, cudaStream_t st) {
  for (int i0 = 0; i0 < n; i0 += kMaxJobs) {
    const int m = std::min(kMaxJobs, n - i0);
    ReduceJobs rj{};
    int64_t max_n = 0;
    for (int i = 0; i < m; ++i) { rj.j[i] = jobs[i0 + i]; max_n = std::max(max_n, jobs[i0 + i].n); }
    dim3 grid((unsigned)ceil_div(max_n, 256), 1, (unsigned)m);
    reduce_partials_group_kernel<<<grid, 256, 0, st>>>(rj);
    ADN_CHECK_LAUNCH("reduce_partials_group");
  }
  return ADN_OK;
}

int colsum_group(const ColsumJob* jobs, int n, cudaStream_t st) {
  for (int i0 = 0; i0 < n; i0 += kMaxJobs) {
    const int m = std::min(kMaxJobs, n - i0);
    ColsumJobs cj{};
    ReduceJobs rj{};
    int64_t max_cols = 0;
    int max_s2 = 0;
    for (int i = 0; i < m; ++i) {
      cj.j[i] = jobs[i0 + i];
      cj.rps[i] = colsum_slice_rows(jobs[i0 + i].rows);
      const int s2 = (int)ceil_div(jobs[i0 + i].rows, cj.rps[i]);
      max_s2 = std::max(max_s2, s2);
      max_cols = std::max(max_cols, jobs[i0 + i].cols);
      rj.j[i] = ReduceJob{jobs[i0 + i].part, jobs[i0 + i].out, jobs[i0 + i].cols, s2, jobs[i0 + i].cols, jobs[i0 + i].scale};
    }
    dim3 grid((unsigned)ceil_div(max_cols, 32), (unsigned)max_s2, (unsigned)m);
    colsum_partial_group_kernel<<<grid, 256, 0, st>>>(cj);
    ADN_CHECK_LAUNCH("colsum_group");
    dim3 grid2((unsigned)ceil_div(max_cols, 256), 1, (unsigned)m);
    reduce_partials_group_kernel<<<grid2, 256, 0, st>>>(rj);
    ADN_CHECK_LAUNCH("colsum_group reduce");
  }
  return ADN_OK;
}

// Tile configs: BIG for wide N, SKINNY for N <= 32 (logits layers).
#define ADN_BIG 128, 128, 16, 8, 8
#define ADN_SKINNY 128, 16, 16, 4, 2

template <bool A_T, bool B_T, int EPI>
static int launch_gemm(const GemmArgs& g, int splits, cudaStream_t st, const char* what) {
  if (g.N <= 32) {
    dim3 grid((unsigned)ceil_div(g.N, 16), (unsigned)ceil_div(g.M, 128), (unsigned)splits);
    sgemm_kernel<ADN_SKINNY, A_T, B_T, EPI><<<grid, 256, 0, st>>>(g);
  } else {
    dim3 grid((unsigned)ceil_div(g.N, 128), (unsigned)ceil_div(g.M, 128), (unsigned)splits);
    sgemm_kernel<ADN_BIG, A_T, B_T, EPI><<<grid, 256, 0, st>>>(g);
  }
  ADN_CHECK_LAUNCH(what);
  return ADN_OK;
}

int dense_fwd(const float* x, const float* w, const float* b, float* y, int64_t batch, int64_t in,
              int64_t out, int act, cudaStream_t st) {
  GemmArgs g{};
  g.A = x; g.B = w; g.C = y;
  g.M = (int)batch; g.N = (int)out; g.K = (int)in;
  g.lda = (int)in; g.ldb = (int)out; g.ldc = (int)out;
  g.bias = b; g.act = act;
  return launch_gemm<false, false, EPI_BIAS_ACT>(g, 1, st, "simt dense_fwd");
}

int dw_splits(int64_t batch, int64_t in, int64_t out) {
  int64_t bn = out <= 32 ? 16 : 128;
  int64_t tiles = ceil_div(in, 128) * ceil_div(out, bn);
  int64_t target = 2 * (int64_t)sm_count();
  int64_t s = ceil_div(target, tiles);
  int64_t max_s = ceil_div(batch, 256);
  if (s > max_s) s = max_s;
  if (s > 64) s = 64;
  if (s < 1) s = 1;
  return (int)s;
}

static int64_t max_splits(int64_t batch) {
  int64_t s = ceil_div(batch, 256);
  if (s > 64) s = 64;
  if (s < 1) s = 1;
  return s;
}

int64_t dense_bwd_workspace_bytes(int64_t batch, int64_t in, int64_t out) {
  // dW partials sized for the worst-case split count (64) so every dense path
  // (SIMT or tcgen05) can share the buffer regardless of its own split choice.
  int64_t s = max_splits(batch);
  int64_t s2 = 64;   // colsum_slice_rows(): at most 64 first-level slices
  return align_up((s * in * out + s2 * out) * (int64_t)sizeof(float), 256);
}

int dense_bwd(const float* x, const float* w, const float* dz, float* dx, float* dw, float* db,
              int64_t batch, int64_t in, int64_t out, int x_relu_mask, void* ws, int64_t ws_bytes,
              cudaStream_t st) {
  if (ws_bytes < dense_bwd_workspace_bytes(batch, in, out))
    return fail(ADN_ERR_WORKSPACE, "dense_bwd: workspace %lld < %lld bytes", (long long)ws_bytes,
                (long long)dense_bwd_workspace_bytes(batch, in, out));
  float* wsf = reinterpret_cast<float*>(ws);
  // ---- dW = x^T @ dz  (split-K over the batch, fixed-order reduction) ----
  const int S = dw_splits(batch, in, out);
  {
    GemmArgs g{};
    g.A = x; g.B = dz;
    g.M = (int)in; g.N = (int)out; g.K = (int)batch;
    g.lda = (int)in; g.ldb = (int)out; g.ldc = (int)out;
    g.k_per_split = (int)align_up(ceil_div(batch, S), 16);
    g.C = (S == 1) ? dw : wsf;
    int rc = launch_gemm<true, false, EPI_PARTIAL>(g, S, st, "simt dense_bwd dW");
    if (rc) return rc;
    const ReduceJob red{wsf, dw, in * out, S, in * out};
    if (S > 1 && (rc = reduce_partials_group(&red, 1, st))) return rc;
  }
  // ---- db = colsum(dz) ----
  if (db) {
    const ColsumJob job{dz, db, batch, out, wsf + (size_t)max_splits(batch) * in * out};
    int rc = colsum_group(&job, 1, st);
    if (rc) return rc;
  }
  // ---- dx = (dz @ w^T) * relu_mask(x) ----
  if (dx) {
    GemmArgs g{};
    g.A = dz; g.B = w; g.C = dx;
    g.M = (int)batch; g.N = (int)in; g.K = (int)out;
    g.lda = (int)out; g.ldb = (int)out; g.ldc = (int)in;
    g.mask = x_relu_mask ? x : nullptr; g.ldmask = (int)in;
    int rc = launch_gemm<false, true, EPI_MASK>(g, 1, st, "simt dense_bwd dX");
    if (rc) return rc;
  }
  return ADN_OK;
}

}  // namespace simt
}  // namespace adn
