// Streaming evaluation metrics of the binary and regression heads (include/adanet_b200.h adn_metrics_group): one
// launch (+ one finalize launch) per kOpsPerLaunch ensembles adds an evaluation batch to each ensemble's threshold
// histograms, class-id counts and fp64 sums.
#include "common.cuh"

namespace adn {
namespace metrics {

constexpr int kOpsPerLaunch = 32;
constexpr int kThreads = 256;
constexpr int kMaxCtasPerOp = 128;
constexpr int64_t kElemsPerCta = 1024;   // 32 CTAs per op at 32768 rows of one logit
constexpr int kBuckets = ADN_METRICS_THRESHOLDS + 1;
// a CTA counts its slice in 32-bit shared-memory histograms (native shared atomics); a call whose op slices could
// overflow them is refused
constexpr int64_t kMaxElemsPerCta = (int64_t)1 << 31;
static_assert(ADN_METRICS_COUNTS == 2 * kBuckets + 2, "counts layout");

struct Op {
  const float* logits;
  const float* labels_f;
  int64_t* counts;
  double* sums;
  int64_t dim;
  int kind;
};
struct Params {
  Op op[kOpsPerLaunch];
  int n;
};

// CTAs per op: a function of (rows, max dim) only, so the per-CTA partials and their fixed-order finalize add the
// same values in the same order on every run and device
int ctas_per_op(int64_t rows, int64_t dim) {
  const int64_t c = ceil_div(rows * dim, kElemsPerCta);
  return (int)(c < 1 ? 1 : (c > kMaxCtasPerOp ? kMaxCtasPerOp : c));
}

// fixed-order block sum (warp shuffle tree, then the warps in order); the result is valid in thread 0
__device__ __forceinline__ double block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < kThreads / 32; ++i) s += red[i];
  return s;
}

// grid (ctas, ops): CTA blockIdx.x of op blockIdx.y takes a contiguous slice of the op's rows * dim elements and
// writes partial[(blockIdx.y * ctas + blockIdx.x) * 3 + k] = that slice's {sum of p or logits, sum of labels, count}
__global__ void __launch_bounds__(kThreads) metrics_kernel(const __grid_constant__ Params P, int64_t rows,
                                                          double* partial) {
  __shared__ float thr[ADN_METRICS_THRESHOLDS];
  __shared__ unsigned int hist[ADN_METRICS_COUNTS];   // < 2^32 per CTA: see kMaxElemsPerCta
  __shared__ double red[kThreads / 32];
  const Op& o = P.op[blockIdx.y];
  const bool binary = o.kind == ADN_METRICS_BINARY;
  // Keras AUC(num_thresholds=200): [0 - 1e-7, 1/199, ..., 198/199, 1 + 1e-7] computed in double, rounded to fp32
  for (int i = threadIdx.x; i < ADN_METRICS_THRESHOLDS; i += kThreads)
    thr[i] = i == 0 ? (float)(0.0 - 1e-7)
                    : (i == ADN_METRICS_THRESHOLDS - 1 ? (float)(1.0 + 1e-7)
                                                       : (float)((double)i / (double)(ADN_METRICS_THRESHOLDS - 1)));
  for (int i = threadIdx.x; i < ADN_METRICS_COUNTS; i += kThreads) hist[i] = 0u;
  __syncthreads();
  const int64_t total = rows * o.dim;
  const int64_t per = (total + gridDim.x - 1) / gridDim.x;
  const int64_t lo = (int64_t)blockIdx.x * per < total ? (int64_t)blockIdx.x * per : total;
  const int64_t hi = lo + per < total ? lo + per : total;
  double sp = 0.0, sl = 0.0;
  for (int64_t e = lo + threadIdx.x; e < hi; e += kThreads) {
    const float x = o.logits[e], y = o.labels_f[e];
    sl += (double)y;
    if (!binary) {
      sp += (double)x;
      continue;
    }
    const float p = 1.f / (1.f + expf(-x));
    sp += (double)p;
    // bucket = #{i : thr[i] < p}: start at p's grid point and step to the boundary (thresholds ascend); a NaN p is
    // below no threshold, bucket 0
    int b = 0;
    if (p == p) {
      b = __float2int_rd(p * (float)(ADN_METRICS_THRESHOLDS - 1));
      b = b < 0 ? 0 : (b > ADN_METRICS_THRESHOLDS ? ADN_METRICS_THRESHOLDS : b);
      while (b < ADN_METRICS_THRESHOLDS && thr[b] < p) ++b;
      while (b > 0 && !(thr[b - 1] < p)) --b;
    }
    const int pos = y > 0.5f ? 1 : 0;
    atomicAdd(&hist[pos * kBuckets + b], 1u);
    if (x > 0.f) atomicAdd(&hist[2 * kBuckets + pos], 1u);   // class_ids = argmax([0, logit])
  }
  const double s0 = block_sum(sp, red);
  const double s1 = block_sum(sl, red);
  if (threadIdx.x == 0) {
    double* w = partial + ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * 3;
    w[0] = s0;
    w[1] = s1;
    w[2] = (double)(hi - lo);
  }
  if (binary) {
    __syncthreads();
    for (int i = threadIdx.x; i < ADN_METRICS_COUNTS; i += kThreads)
      if (hist[i]) atomicAdd(reinterpret_cast<unsigned long long*>(o.counts + i), (unsigned long long)hist[i]);
  }
}

// thread j: op j's sums[k] += its CTA partials, in CTA order
__global__ void metrics_finalize_kernel(const __grid_constant__ Params P, const double* partial, int ctas) {
  const int j = threadIdx.x;
  if (j >= P.n) return;
  double s[3] = {0.0, 0.0, 0.0};
  for (int c = 0; c < ctas; ++c)
    for (int k = 0; k < 3; ++k) s[k] += partial[((int64_t)j * ctas + c) * 3 + k];
  for (int k = 0; k < 3; ++k) P.op[j].sums[k] += s[k];
}

int64_t workspace_bytes(int64_t rows, int64_t dim, int64_t n) {
  if (rows < 1 || dim < 1 || n < 1) return 256;
  return n * ctas_per_op(rows, dim) * 3 * (int64_t)sizeof(double) + 256;
}

}  // namespace metrics
}  // namespace adn

using namespace adn;

extern "C" int adn_metrics_group(const adn_metrics_op* ops, int n, int64_t rows, void* workspace,
                                 int64_t workspace_bytes, void* stream) {
  if (!ops || n < 1 || n > ADN_METRICS_MAX_OPS)
    return fail(ADN_ERR_INVALID, "adn_metrics_group: %d ops (1..%d)", n, ADN_METRICS_MAX_OPS);
  if (rows < 1) return fail(ADN_ERR_INVALID, "adn_metrics_group: rows %lld < 1", (long long)rows);
  if (!workspace) return fail(ADN_ERR_INVALID, "adn_metrics_group: null workspace");
  int64_t dim = 0;
  for (int i = 0; i < n; ++i) {
    const adn_metrics_op& o = ops[i];
    if (o.kind != ADN_METRICS_BINARY && o.kind != ADN_METRICS_MEANS)
      return fail(ADN_ERR_INVALID, "adn_metrics_group: op %d has bad kind %d", i, o.kind);
    if (!o.logits || !o.labels_f || !o.sums || (o.kind == ADN_METRICS_BINARY && !o.counts))
      return fail(ADN_ERR_INVALID, "adn_metrics_group: op %d has a null pointer", i);
    if (o.dim < 1) return fail(ADN_ERR_INVALID, "adn_metrics_group: op %d has dim %lld < 1", i, (long long)o.dim);
    if (o.kind == ADN_METRICS_BINARY && o.dim != 1)
      return fail(ADN_ERR_UNSUPPORTED, "adn_metrics_group: op %d is BINARY with dim %lld != 1", i, (long long)o.dim);
    if (o.dim > ((metrics::kMaxElemsPerCta * metrics::kMaxCtasPerOp) / rows))
      return fail(ADN_ERR_UNSUPPORTED, "adn_metrics_group: op %d has more than %lld elements", i,
                  (long long)(metrics::kMaxElemsPerCta * metrics::kMaxCtasPerOp));
    for (int j = 0; j < i; ++j)
      if (ops[j].sums == o.sums) return fail(ADN_ERR_INVALID, "adn_metrics_group: ops %d and %d share sums", j, i);
    dim = o.dim > dim ? o.dim : dim;
  }
  if (workspace_bytes < metrics::workspace_bytes(rows, dim, n))
    return fail(ADN_ERR_WORKSPACE, "adn_metrics_group: workspace %lld < %lld bytes", (long long)workspace_bytes,
                (long long)metrics::workspace_bytes(rows, dim, n));
  const int ctas = metrics::ctas_per_op(rows, dim);
  double* partial = reinterpret_cast<double*>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
  cudaStream_t s = as_stream(stream);
  for (int base = 0; base < n; base += metrics::kOpsPerLaunch) {
    metrics::Params P{};
    P.n = n - base < metrics::kOpsPerLaunch ? n - base : metrics::kOpsPerLaunch;
    for (int j = 0; j < P.n; ++j) {
      const adn_metrics_op& o = ops[base + j];
      P.op[j] = metrics::Op{o.logits, o.labels_f, o.counts, o.sums, o.dim, o.kind};
    }
    double* part = partial + (int64_t)base * ctas * 3;
    metrics::metrics_kernel<<<dim3(ctas, P.n), metrics::kThreads, 0, s>>>(P, rows, part);
    ADN_CHECK_LAUNCH("metrics_kernel");
    metrics::metrics_finalize_kernel<<<1, 32, 0, s>>>(P, part, ctas);
    ADN_CHECK_LAUNCH("metrics_finalize_kernel");
  }
  return ADN_OK;
}
