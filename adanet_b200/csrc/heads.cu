// Fused AdaNet ensemble head (K4), plain head loss (K3), zero-debiased EMA (K6)
// and L1 norm.  HBM-bound: every member-logit element is read from DRAM once
// (pass 1), re-read from L2 for the mixture-weight gradient (pass 2), with
// coalesced float4 loads over the flat [rows*dim] tile of each member.
//
// Reference arithmetic being replaced (file:line in tensorflow/adanet v0.9.0):
//   weighted logits / sum    adanet/ensemble/weighted.py:433-453,545-561
//   head loss                adanet/core/ensemble_builder.py:416-420,571-583
//   complexity regulariser   adanet/ensemble/weighted.py:351-358,563-604
//   adanet_loss              adanet/core/ensemble_builder.py:423-426
//   mixture-weight gradient  adanet/ensemble/weighted.py:606-617
//   EMA                      adanet/core/candidate.py:117-129
#include <algorithm>

#include "common.cuh"
#include "plane_fmt.cuh"

namespace adn {

static constexpr int kRows = 128;       // rows (examples) per CTA == threads per CTA
static constexpr int kMaxMembers = 64;
static constexpr int kMaxDim = 64;

struct HeadParams {
  const float* members[kMaxMembers];
  float gammas[kMaxMembers];
  int n_members;
  int head, mixture;
  const float* w;        // SCALAR [N] / VECTOR [N,dim] / MATRIX l1 norms [N]; null => 1.0
  const float* bias;     // [dim] or null
  const int64_t* labels;
  const float* labels_f;
  float* dens;           // [B,dim] or null
  pl::PlaneView densp;   // split planes of dens * dens_scale (csrc/plane_fmt.cuh) or hi == null
  float dens_scale;      // power of two
  int dens_nkb;          // k-blocks of the plane tensor
  unsigned int* ovf;
  int colsum_only;       // want_grads without the mixture-weight pass: only column sums of dens -> dbias
  float* ens_out;        // [B,dim] or null
  float* part;           // workspace: per-CTA partials, output-major [n_out][n_cta] (coalesced for the finalize)
  int n_cta;
  int64_t batch;
  int dim;
  int n_out;             // 1 + dim + N*wdim
  int want_grads;
  int reg_is_zero;
  float reg_multiplier;
  float* out3;
  float* dw;
  float* dbias;
};

__device__ __forceinline__ float weight_of(const HeadParams& p, int k, int c) {
  if (p.mixture == ADN_MIX_MATRIX || p.w == nullptr) return 1.f;
  return p.mixture == ADN_MIX_SCALAR ? __ldg(p.w + k) : __ldg(p.w + (size_t)k * p.dim + c);
}

// Block-wide sum of one value per thread in a FIXED order (shuffle tree inside each warp, then warp 0..W-1 in
// sequence): run-to-run deterministic.  `wred` holds kRows/32 floats; the result is returned on thread 0 only.
__device__ __forceinline__ float block_sum(float v, float* wred, int tid) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((tid & 31) == 0) wred[tid >> 5] = v;
  __syncthreads();
  float t = 0.f;
  if (tid == 0) {
#pragma unroll
    for (int w = 0; w < kRows / 32; ++w) t += wred[w];
  }
  __syncthreads();
  return t;
}

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gsrc, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc),
               "r"(bytes)
               : "memory");
}

// One CTA = kRows examples, one thread per example.  The CTA's contiguous [kRows*dim] slab of EVERY member is
// brought into shared memory with one burst of 16-byte cp.async copies (all members in flight at once: the
// kernel is a pure HBM stream, SURVEY.md 8d: N*C*4 + 8 bytes per example), then each thread works on its row:
// weighted sum, head loss and gradient, and the mixture-weight gradient from the SAME smem copy (no second
// read).  All reductions are shuffle trees in a fixed order (no serial loops over rows, no atomics).
// smem layout (floats): mem[n_members][kRows*dim] | ens[kRows*dim] | wred[kRows/32 * max(dim, n_members)]
template <int CT>   // CT > 0: logits dimension known at compile time (loops unroll, row offsets fold); 0: runtime
__device__ __forceinline__ void head_body(const HeadParams& p, float* smem, const int cta) {
  const int C = CT > 0 ? CT : p.dim, N = p.n_members;
  float* mem = smem;
  float* ens = smem + (size_t)N * kRows * C;
  float* wred = ens + kRows * C;        // [kRows/32][max(C, N)] warp partials
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = (int64_t)cta * kRows;
  const int rows = (int)min((int64_t)kRows, p.batch - r0);
  const int valid = rows * C;           // flat elements of this CTA's slab
  const size_t base = (size_t)r0 * C;
  const int nvec = (kRows * C) / 4;     // kRows*C is a multiple of 4

  // ---- stream every member's slab into smem (zero-filled past `valid`) ----
  for (int k = 0; k < N; ++k) {
    const float* m = p.members[k] + base;
    float* dst = mem + (size_t)k * kRows * C;
    if ((reinterpret_cast<uintptr_t>(m) & 15) == 0) {
      for (int v = tid; v < nvec; v += kRows) {
        const int i = v * 4;
        const int bytes = max(0, min(16, (valid - i) * 4));
        cp_async16(dst + i, bytes > 0 ? m + i : m, bytes);
      }
    } else {
      for (int i = tid; i < kRows * C; i += kRows) dst[i] = (i < valid) ? __ldg(m + i) : 0.f;
    }
  }
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  // ---- per-row: ens = bias + sum_k w_k (.) member_k (sequential over members like tf.add, weighted.py:558-561),
  //      loss_r, g[r,:] = dLoss/d ens (kept in the thread's smem row) ----
  float* e = ens + tid * C;
  float loss_r = 0.f;
  if (tid < rows) {
    for (int c = 0; c < C; ++c) {
      float v = p.bias ? __ldg(p.bias + c) : 0.f;
      for (int k = 0; k < N; ++k) v += weight_of(p, k, c) * mem[(size_t)k * kRows * C + tid * C + c];
      e[c] = v;
    }
    if (p.ens_out) {
      for (int c = 0; c < C; ++c) p.ens_out[base + (size_t)tid * C + c] = e[c];
    }
    if (p.head == ADN_HEAD_SOFTMAX_XENT) {
      const int y = (int)p.labels[r0 + tid];
      float mx = e[0];
      for (int c = 1; c < C; ++c) mx = fmaxf(mx, e[c]);
      const float zy = e[y] - mx;
      float s = 0.f;
      for (int c = 0; c < C; ++c) {          // one expf per class: the exponentials are kept in the row
        const float ex = expf(e[c] - mx);
        e[c] = ex;
        s += ex;
      }
      const float logs = logf(s);
      loss_r = -(zy - logs);
      const float inv = 1.f / s, invb = 1.f / (float)p.batch;
      for (int c = 0; c < C; ++c) e[c] = (e[c] * inv - (c == y ? 1.f : 0.f)) * invb;
    } else if (p.head == ADN_HEAD_MSE) {
      const float invn = 1.f / ((float)p.batch * (float)C);
      for (int c = 0; c < C; ++c) {
        float d = e[c] - p.labels_f[(size_t)(r0 + tid) * C + c];
        loss_r += d * d;
        e[c] = 2.f * d * invn;
      }
    } else {  // sigmoid cross-entropy, max(x,0) - x z + log1p(exp(-|x|))
      const float invn = 1.f / ((float)p.batch * (float)C);
      for (int c = 0; c < C; ++c) {
        float x = e[c], z = p.labels_f[(size_t)(r0 + tid) * C + c];
        loss_r += fmaxf(x, 0.f) - x * z + log1pf(expf(-fabsf(x)));
        e[c] = (1.f / (1.f + expf(-x)) - z) * invn;
      }
    }
  } else {
    for (int c = 0; c < C; ++c) e[c] = 0.f;
  }
  float* part = p.part + cta;                          // output j of this CTA lives at part[j * n_cta]
  const size_t ps = (size_t)p.n_cta;
  {
    const float t = block_sum(loss_r, wred, tid);     // (contains the barrier that publishes every row's g)
    if (tid == 0) part[0] = t;
  }
  if (p.dens) {
    for (int i = tid; i < valid; i += kRows) p.dens[base + i] = ens[i];
  }
  if (p.densp.hi) {
    // same gradient (times the power-of-two plane scale) as hi/lo planes: the A / B operand of the subnetwork's
    // backward GEMMs; padding columns of the last k-block are rewritten as zeros
    const int bk = pl::fmt_bk(p.densp.fmt);
    const int pc = p.dens_nkb * bk;
    // 8 columns per thread and store (16 B of each fp16 plane): consecutive threads fill one row's k-block line
    const int pc8 = pc >> 3;               // pc is a multiple of the k-block width (32 or 64 columns)
    for (int i = tid; i < kRows * pc8; i += kRows) {
      const int c8 = i % pc8, r = i / pc8;
      if (r0 + r >= p.batch) continue;
      float m8[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int c = c8 * 8 + q;
        m8[q] = (c < C) ? ens[r * C + c] * p.dens_scale : 0.f;
      }
      pl::plane_store8(p.densp, r0 + r, (int64_t)c8 * 8, m8, p.ovf);
    }
    // sign bits are not consumed for gradient tensors
  }
  if (!p.want_grads) return;

  // ---- column sums of g -> dbias partial: warp trees per column, then the warps in sequence ----
  const int wr = (C > N) ? C : N;          // row stride of the warp-partial scratch
  // thread (w, c) adds column c over the 32 rows of row-group w straight from the smem rows (fixed order)
  for (int j = tid; j < (kRows / 32) * C; j += kRows) {
    const int w = j / C, c = j - w * C;
    const float* col = ens + (size_t)(w * 32) * C + c;
    float v = 0.f;
#pragma unroll 8
    for (int r = 0; r < 32; ++r) v += col[r * C];
    wred[w * wr + c] = v;
  }
  __syncthreads();
  if (tid < C) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kRows / 32; ++w) t += wred[w * wr + tid];
    part[(1 + tid) * ps] = t;
  }
  if (p.mixture == ADN_MIX_MATRIX || p.colsum_only) return;

  // ---- dw_k partials = sum_b g (.) member_k from the smem copy of the members ----
  if (p.mixture == ADN_MIX_SCALAR) {
    __syncthreads();                       // dbias readers done with wred
    for (int k = 0; k < N; ++k) {
      const float* mrow = mem + (size_t)k * kRows * C + tid * C;
      float d = 0.f;
      for (int c = 0; c < C; ++c) d += e[c] * mrow[c];       // row dot product, then the block tree
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) d += __shfl_down_sync(0xffffffffu, d, o);
      if (lane == 0) wred[warp * wr + k] = d;
    }
    __syncthreads();
    if (tid < N) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kRows / 32; ++w) t += wred[w * wr + tid];
      part[(1 + C + tid) * ps] = t;
    }
  } else {
    for (int k = 0; k < N; ++k) {
      const float* mrow = mem + (size_t)k * kRows * C + tid * C;
      __syncthreads();                     // previous readers done with wred
      for (int c = 0; c < C; ++c) {
        float v = e[c] * mrow[c];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) wred[warp * wr + c] = v;
      }
      __syncthreads();
      if (tid < C) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < kRows / 32; ++w) t += wred[w * wr + tid];
        part[(1 + C + k * C + tid) * ps] = t;
      }
    }
  }
}

template <int CT>
__global__ void __launch_bounds__(kRows)
ensemble_head_kernel(const __grid_constant__ HeadParams p) {
  extern __shared__ __align__(16) float smem[];
  head_body<CT>(p, smem, blockIdx.x);
}

// Grouped form: blockIdx.y selects one of up to kMaxGroup independent heads over the same minibatch -- the
// subnetwork losses and the candidate-ensemble heads of every candidate of the GPU in ONE launch (they only read
// logits the forward waves have produced), instead of two launches per candidate on side streams.
static constexpr int kMaxGroup = 24;
struct HeadGroup {
  HeadParams p[kMaxGroup];
  int n;
};
template <int CT>
__global__ void __launch_bounds__(kRows)
ensemble_head_group_kernel(const __grid_constant__ HeadGroup g) {
  extern __shared__ __align__(16) float smem[];
  head_body<CT>(g.p[blockIdx.y], smem, blockIdx.x);
}

// Fixed-order reduction of the per-CTA partials + regulariser + adanet loss.
// First level for many CTAs: block j sums the n_cta partials of output j (coalesced, fixed order) into out[j].
__global__ void __launch_bounds__(256)
head_partials_kernel(const float* __restrict__ part, float* __restrict__ out, int n_cta) {
  __shared__ float wsum[8];
  const float* src = part + (size_t)blockIdx.x * n_cta;
  float t = 0.f;
  for (int b = threadIdx.x; b < n_cta; b += 256) t += src[b];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    float r = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) r += wsum[w];
    out[blockIdx.x] = r;
  }
}

__device__ __forceinline__ void finalize_body(const HeadParams& p, const float* __restrict__ part, int n_cta) {
  __shared__ float s_loss, s_reg;
  const int C = p.dim;
  const int wdim = (p.mixture == ADN_MIX_SCALAR) ? 1 : C;
  const int n_w = (p.mixture == ADN_MIX_MATRIX || p.colsum_only) ? 0 : p.n_members * wdim;
  const int n_red = p.want_grads ? (1 + C + n_w) : 1;
  // one warp per output: lanes stride over the CTA partials, then a fixed-order shuffle tree
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int j = wid; j < n_red; j += nwarps) {
    float t = 0.f;
    for (int b = lane; b < n_cta; b += 32) t += part[(size_t)j * n_cta + b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
    if (lane != 0) continue;
    if (j == 0) {
      float denom = (p.head == ADN_HEAD_SOFTMAX_XENT) ? (float)p.batch : (float)p.batch * (float)C;
      s_loss = t / denom;
    } else if (j < 1 + C) {
      if (p.dbias) p.dbias[j - 1] = t;
    } else if (p.dw) {
      const int idx = j - 1 - C;
      const int k = idx / wdim;
      float g = t;
      if (!p.reg_is_zero) {
        const float w = p.w ? p.w[idx] : 1.f;
        const float sgn = (w > 0.f) ? 1.f : ((w < 0.f) ? -1.f : 0.f);
        g += p.reg_multiplier * p.gammas[k] * sgn;
      }
      p.dw[idx] = g;
    }
  }
  if (threadIdx.x == 0) {
    float reg = 0.f;
    if (!p.reg_is_zero) {
      for (int k = 0; k < p.n_members; ++k) {
        float l1 = 0.f;
        if (p.mixture == ADN_MIX_MATRIX) {
          l1 = p.w[k];
        } else if (p.w == nullptr) {
          l1 = (float)wdim;
        } else {
          for (int c = 0; c < wdim; ++c) l1 += fabsf(p.w[k * wdim + c]);
        }
        reg += p.gammas[k] * l1;
      }
    }
    s_reg = reg;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    p.out3[0] = s_loss;
    p.out3[1] = s_reg;
    p.out3[2] = s_loss + s_reg;
  }
}

__global__ void __launch_bounds__(256)
ensemble_finalize_kernel(const __grid_constant__ HeadParams p, const float* __restrict__ part, int n_cta) {
  finalize_body(p, part, n_cta);
}
__global__ void __launch_bounds__(256)
ensemble_finalize_group_kernel(const __grid_constant__ HeadGroup g) {
  const HeadParams& p = g.p[blockIdx.x];
  finalize_body(p, p.part, p.n_cta);
}

__device__ __forceinline__ void ema_update(float* state, const float* loss, float decay);
// Per-step bookkeeping of every candidate ensemble in one launch (thread j = head j): zero-debiased EMA of its
// adanet loss (candidate.py:117-129) and its row of the loss trace {sub_loss, ens_loss, adanet_loss, ema}
// (iteration.py:961-996 reports the same scalars through hooks).
struct BookEntry {
  float* ema_state;        // {biased, n, value}
  const float* out3;       // {loss, reg, adanet_loss} of the head
  const float* sub_loss;   // subnetwork loss (or a NaN constant)
  float* trace;            // [capacity][4]
  float decay;
  int capacity;
};
struct BookGroup {
  BookEntry e[64];
  int n;
};
__global__ void head_bookkeeping_kernel(const __grid_constant__ BookGroup g, const int64_t* step) {
  const int j = threadIdx.x;
  if (j >= g.n) return;
  const BookEntry& e = g.e[j];
  ema_update(e.ema_state, e.out3 + 2, e.decay);
  float* row = e.trace + (size_t)(*step % e.capacity) * 4;
  row[0] = *e.sub_loss;
  row[1] = e.out3[0];
  row[2] = e.out3[2];
  row[3] = e.ema_state[2];
}

__device__ __forceinline__ void ema_update(float* state, const float* loss, float decay) {
  // candidate.py:117-129 -> assign_moving_average(zero_debias=True) [TF]
  float biased = state[0], n = state[1];
  const float x = *loss;
  biased = biased - (biased - x) * (1.f - decay);
  n += 1.f;
  const float factor = 1.f - powf(decay, n);
  state[0] = biased;
  state[1] = n;
  state[2] = biased / factor;
}
__global__ void ema_update_kernel(float* state, const float* loss, float decay) { ema_update(state, loss, decay); }

__global__ void __launch_bounds__(1024) l1_norm_kernel(const float* x, int64_t n, float* out) {
  __shared__ float sm[1024];
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += 1024) acc += fabsf(x[i]);
  sm[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 512; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sm[0];
}

static int64_t head_workspace_bytes(int64_t batch, int64_t dim, int64_t members) {
  int64_t n_cta = ceil_div(batch, kRows);
  int64_t n_out = 1 + dim + members * dim;
  return align_up((n_cta + 1) * n_out * (int64_t)sizeof(float), 256);   // + one row for the two-level finalize
}

static size_t head_smem_bytes(int dim, int members) {
  const int wr = dim > members ? dim : members;
  return ((size_t)(members + 1) * kRows * dim + (size_t)(kRows / 32) * wr) * sizeof(float);
}

static int run_head(HeadParams& p, void* ws, int64_t ws_bytes, cudaStream_t st) {
  if (p.batch <= 0 || p.dim <= 0) return fail(ADN_ERR_INVALID, "head: empty batch/dim");
  if (p.dim > kMaxDim) return fail(ADN_ERR_UNSUPPORTED, "head: dim %d > %d", p.dim, kMaxDim);
  if (p.n_members < 1 || p.n_members > kMaxMembers)
    return fail(ADN_ERR_UNSUPPORTED, "head: n_members %d not in [1,%d]", p.n_members, kMaxMembers);
  if (p.head == ADN_HEAD_SOFTMAX_XENT ? p.labels == nullptr : p.labels_f == nullptr)
    return fail(ADN_ERR_INVALID, "head: labels missing for head kind %d", p.head);
  const int wdim = (p.mixture == ADN_MIX_SCALAR) ? 1 : p.dim;
  p.n_out = 1 + p.dim + p.n_members * wdim;
  if (ws_bytes < head_workspace_bytes(p.batch, p.dim, p.n_members))
    return fail(ADN_ERR_WORKSPACE, "head: workspace %lld < %lld bytes", (long long)ws_bytes,
                (long long)head_workspace_bytes(p.batch, p.dim, p.n_members));
  p.part = reinterpret_cast<float*>(ws);
  const int n_cta = (int)ceil_div(p.batch, kRows);
  p.n_cta = n_cta;
  const size_t smem = head_smem_bytes(p.dim, p.n_members);
  if (smem > 227 * 1024)
    return fail(ADN_ERR_UNSUPPORTED, "head: n_members*dim = %d*%d does not fit shared memory", p.n_members, p.dim);
  switch (p.dim) {
    case 1: ensemble_head_kernel<1><<<n_cta, kRows, smem, st>>>(p); break;
    case 2: ensemble_head_kernel<2><<<n_cta, kRows, smem, st>>>(p); break;
    case 3: ensemble_head_kernel<3><<<n_cta, kRows, smem, st>>>(p); break;
    case 4: ensemble_head_kernel<4><<<n_cta, kRows, smem, st>>>(p); break;
    case 10: ensemble_head_kernel<10><<<n_cta, kRows, smem, st>>>(p); break;
    case 16: ensemble_head_kernel<16><<<n_cta, kRows, smem, st>>>(p); break;
    default: ensemble_head_kernel<0><<<n_cta, kRows, smem, st>>>(p); break;
  }
  ADN_CHECK_LAUNCH("ensemble_head");
  if (n_cta > 512) {
    // many CTAs (large batches): one block per output sums its partials first, the finalize then sees one row
    const int n_red = p.want_grads ? (1 + p.dim + ((p.mixture == ADN_MIX_MATRIX || p.colsum_only) ? 0 : p.n_members * wdim)) : 1;
    float* red = p.part + (size_t)n_cta * p.n_out;
    head_partials_kernel<<<n_red, 256, 0, st>>>(p.part, red, n_cta);
    ADN_CHECK_LAUNCH("head_partials");
    ensemble_finalize_kernel<<<1, 256, 0, st>>>(p, red, 1);
  } else {
    ensemble_finalize_kernel<<<1, 256, 0, st>>>(p, p.part, n_cta);
  }
  ADN_CHECK_LAUNCH("ensemble_finalize");
  return ADN_OK;
}

int heads_init() {
#define ADN_HEAD_ATTR(CT) \
  ADN_CUDA(cudaFuncSetAttribute(ensemble_head_kernel<CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024))
  ADN_HEAD_ATTR(0); ADN_HEAD_ATTR(1); ADN_HEAD_ATTR(2); ADN_HEAD_ATTR(3); ADN_HEAD_ATTR(4); ADN_HEAD_ATTR(10);
  ADN_HEAD_ATTR(16);
#undef ADN_HEAD_ATTR
  return ADN_OK;
}

int64_t head_workspace_bytes_public(int64_t batch, int64_t dim, int64_t members) {
  return head_workspace_bytes(batch, dim, members < 1 ? 1 : members);
}

}  // namespace adn

using namespace adn;


extern "C" int adn_head_loss(int head, const float* logits, const int64_t* labels, const float* labels_f,
                             float* loss_out, float* dlogits, int64_t batch, int64_t dim,
                             void* workspace, int64_t workspace_bytes, void* stream) {
  return adn_head_loss_p(head, logits, labels, labels_f, loss_out, dlogits, nullptr, nullptr, 0, batch, dim, workspace,
                         workspace_bytes, stream);
}

extern "C" int adn_head_loss_p(int head, const float* logits, const int64_t* labels, const float* labels_f,
                               float* loss_out, float* dlogits, void* dlogits_planes, float* dlogits_colsum,
                               int dz_log2_scale, int64_t batch, int64_t dim, void* workspace, int64_t workspace_bytes,
                               void* stream) {
  if (!logits || !loss_out) return fail(ADN_ERR_INVALID, "adn_head_loss: null pointer");
  if (head < 0 || head > 2) return fail(ADN_ERR_INVALID, "adn_head_loss: bad head %d", head);
  // out3 needs 3 floats; the public contract is loss_out[0], so stage through workspace tail.
  HeadParams p{};
  p.members[0] = logits;
  p.n_members = 1;
  p.head = head;
  p.mixture = ADN_MIX_SCALAR;
  p.labels = labels;
  p.labels_f = labels_f;
  p.dens = dlogits;
  if (dz_log2_scale < -60 || dz_log2_scale > 60) return fail(ADN_ERR_INVALID, "adn_head_loss_p: bad dz_log2_scale");
  if (dlogits_planes) {
    const int fmt = pl::format();
    p.densp = pl::plane_view(fmt, dlogits_planes, batch, dim);
    p.dens_scale = ldexpf(1.0f, dz_log2_scale);
    p.dens_nkb = (int)ceil_div(dim, pl::fmt_bk(fmt));
    p.ovf = pl::overflow_flag();
  }
  p.batch = batch;
  p.dim = (int)dim;
  p.want_grads = dlogits_colsum ? 1 : 0;
  p.colsum_only = 1;
  p.dbias = dlogits_colsum;
  p.reg_is_zero = 1;
  const int64_t need = head_workspace_bytes_public(batch, dim, 1);
  if (workspace_bytes < need + 16)
    return fail(ADN_ERR_WORKSPACE, "adn_head_loss: workspace %lld < %lld bytes", (long long)workspace_bytes,
                (long long)(need + 16));
  float* out3 = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + need);
  p.out3 = out3;
  int rc = run_head(p, workspace, need, as_stream(stream));
  if (rc) return rc;
  ADN_CUDA(cudaMemcpyAsync(loss_out, out3, sizeof(float), cudaMemcpyDeviceToDevice, as_stream(stream)));
  return ADN_OK;
}

extern "C" int adn_ensemble_head(int head, int mixture_type, const float* const* members_host, int n_members,
                                 const float* w, const float* bias, const float* gammas_host, int reg_is_zero,
                                 float reg_multiplier, const int64_t* labels, const float* labels_f,
                                 float* out3, float* dw, float* dbias, float* dens, float* ens_out,
                                 int64_t batch, int64_t dim, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
  if (!members_host || !out3) return fail(ADN_ERR_INVALID, "adn_ensemble_head: null pointer");
  if (head < 0 || head > 2) return fail(ADN_ERR_INVALID, "adn_ensemble_head: bad head %d", head);
  if (mixture_type < 0 || mixture_type > 2)
    return fail(ADN_ERR_INVALID, "adn_ensemble_head: bad mixture type %d", mixture_type);
  if (n_members < 1 || n_members > kMaxMembers)
    return fail(ADN_ERR_UNSUPPORTED, "adn_ensemble_head: n_members %d not in [1,%d]", n_members, kMaxMembers);
  if (mixture_type == ADN_MIX_MATRIX && dw)
    return fail(ADN_ERR_INVALID, "adn_ensemble_head: dw must be NULL for MATRIX mixture weights");
  if (!reg_is_zero && !gammas_host) return fail(ADN_ERR_INVALID, "adn_ensemble_head: gammas missing");
  HeadParams p{};
  for (int k = 0; k < n_members; ++k) {
    if (!members_host[k]) return fail(ADN_ERR_INVALID, "adn_ensemble_head: member %d is null", k);
    p.members[k] = members_host[k];
    p.gammas[k] = gammas_host ? gammas_host[k] : 0.f;
  }
  p.n_members = n_members;
  p.head = head;
  p.mixture = mixture_type;
  p.w = w;
  p.bias = bias;
  p.labels = labels;
  p.labels_f = labels_f;
  p.dens = dens;
  p.ens_out = ens_out;
  p.batch = batch;
  p.dim = (int)dim;
  p.want_grads = (dw || dbias) ? 1 : 0;
  p.reg_is_zero = reg_is_zero;
  p.reg_multiplier = reg_multiplier;
  p.out3 = out3;
  p.dw = dw;
  p.dbias = dbias;
  return run_head(p, workspace, workspace_bytes, as_stream(stream));
}

extern "C" int adn_ema_update(float* state, const float* loss, float decay, void* stream) {
  if (!state || !loss) return fail(ADN_ERR_INVALID, "adn_ema_update: null pointer");
  ema_update_kernel<<<1, 1, 0, as_stream(stream)>>>(state, loss, decay);
  ADN_CHECK_LAUNCH("ema_update");
  return ADN_OK;
}

extern "C" int adn_l1_norm(const float* x, int64_t n, float* out, void* stream) {
  if (!x || !out || n < 0) return fail(ADN_ERR_INVALID, "adn_l1_norm: bad argument");
  l1_norm_kernel<<<1, 1024, 0, as_stream(stream)>>>(x, n, out);
  ADN_CHECK_LAUNCH("l1_norm");
  return ADN_OK;
}


// ---- grouped heads (include/adanet_b200.h: adn_head_group / adn_head_bookkeeping) ----
namespace adn {
template <int CT>
static void launch_head_group(const HeadGroup& g, int n_cta, size_t smem, cudaStream_t st) {
  ensemble_head_group_kernel<CT><<<dim3((unsigned)n_cta, (unsigned)g.n), kRows, smem, st>>>(g);
}
int heads_group_init() {
#define ADN_HEADG_ATTR(CT) \
  ADN_CUDA(cudaFuncSetAttribute(ensemble_head_group_kernel<CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024))
  ADN_HEADG_ATTR(0); ADN_HEADG_ATTR(1); ADN_HEADG_ATTR(2); ADN_HEADG_ATTR(3); ADN_HEADG_ATTR(4); ADN_HEADG_ATTR(10);
  ADN_HEADG_ATTR(16);
#undef ADN_HEADG_ATTR
  return ADN_OK;
}
}  // namespace adn

namespace adn {
// Checks op `idx` of adn_head_group and fills its launch parameters; touches no device memory.
static int head_group_op(const adn_head_op& o, int idx, int64_t batch, int64_t dim, int fmt, int n_cta, HeadParams& p) {
  if (!o.members_host || !o.out3 || !o.workspace) return fail(ADN_ERR_INVALID, "adn_head_group: op %d: null pointer", idx);
  if (o.head < 0 || o.head > 2 || o.mixture_type < 0 || o.mixture_type > 2)
    return fail(ADN_ERR_INVALID, "adn_head_group: op %d: bad head / mixture type", idx);
  if (o.n_members < 1 || o.n_members > kMaxMembers)
    return fail(ADN_ERR_UNSUPPORTED, "adn_head_group: op %d: n_members %d not in [1,%d]", idx, o.n_members, kMaxMembers);
  if (o.mixture_type == ADN_MIX_MATRIX && o.dw) return fail(ADN_ERR_INVALID, "adn_head_group: op %d: dw must be NULL for MATRIX", idx);
  if (!o.reg_is_zero && !o.gammas_host) return fail(ADN_ERR_INVALID, "adn_head_group: op %d: gammas missing", idx);
  if (o.head == ADN_HEAD_SOFTMAX_XENT ? o.labels == nullptr : o.labels_f == nullptr)
    return fail(ADN_ERR_INVALID, "adn_head_group: op %d: labels missing", idx);
  if (o.dz_log2_scale < -60 || o.dz_log2_scale > 60) return fail(ADN_ERR_INVALID, "adn_head_group: op %d: bad dz_log2_scale", idx);
  for (int k = 0; k < o.n_members; ++k) {
    if (!o.members_host[k]) return fail(ADN_ERR_INVALID, "adn_head_group: op %d: member %d is null", idx, k);
    p.members[k] = o.members_host[k];
    p.gammas[k] = o.gammas_host ? o.gammas_host[k] : 0.f;
  }
  p.n_members = o.n_members;
  p.head = o.head;
  p.mixture = o.mixture_type;
  p.w = o.w;
  p.bias = o.bias;
  p.labels = o.labels;
  p.labels_f = o.labels_f;
  p.dens = o.dens;
  p.ens_out = o.ens_out;
  if (o.dens_planes) {
    p.densp = pl::plane_view(fmt, o.dens_planes, batch, dim);
    p.dens_scale = ldexpf(1.0f, o.dz_log2_scale);
    p.dens_nkb = (int)ceil_div(dim, pl::fmt_bk(fmt));
    p.ovf = pl::overflow_flag();
  }
  p.batch = batch;
  p.dim = (int)dim;
  p.colsum_only = o.colsum_only ? 1 : 0;
  p.want_grads = (o.dw || o.dbias) ? 1 : 0;
  p.reg_is_zero = o.colsum_only ? 1 : o.reg_is_zero;
  p.reg_multiplier = o.reg_multiplier;
  p.out3 = o.out3;
  p.dw = o.colsum_only ? nullptr : o.dw;
  p.dbias = o.dbias;
  const int wdim = (p.mixture == ADN_MIX_SCALAR) ? 1 : p.dim;
  p.n_out = 1 + p.dim + p.n_members * wdim;
  if (o.workspace_bytes < head_workspace_bytes(batch, dim, o.n_members))
    return fail(ADN_ERR_WORKSPACE, "adn_head_group: op %d: workspace %lld < %lld bytes", idx, (long long)o.workspace_bytes,
                (long long)head_workspace_bytes(batch, dim, o.n_members));
  p.part = reinterpret_cast<float*>(o.workspace);
  p.n_cta = n_cta;
  return ADN_OK;
}

// Fills the launch of ops [i0, i0 + g.n) and the shared memory it needs.
static int head_group_chunk(const adn_head_op* ops, int i0, int m, int64_t batch, int64_t dim, int fmt, int n_cta,
                            HeadGroup& g, size_t& smem) {
  g = HeadGroup{};
  g.n = m;
  smem = 0;
  for (int i = 0; i < m; ++i) {
    const int rc = head_group_op(ops[i0 + i], i0 + i, batch, dim, fmt, n_cta, g.p[i]);
    if (rc) return rc;
    smem = std::max(smem, head_smem_bytes(g.p[i].dim, g.p[i].n_members));
  }
  if (smem > 227 * 1024) return fail(ADN_ERR_UNSUPPORTED, "adn_head_group: members x dim does not fit shared memory");
  return ADN_OK;
}
}  // namespace adn

extern "C" int adn_head_group(const adn_head_op* ops, int n, int64_t batch, int64_t dim, void* stream) {
  if (n < 0 || (n > 0 && !ops)) return fail(ADN_ERR_INVALID, "adn_head_group: bad ops");
  if (batch <= 0 || dim <= 0 || dim > kMaxDim) return fail(ADN_ERR_INVALID, "adn_head_group: bad batch/dim");
  const int n_cta = (int)ceil_div(batch, kRows);
  const int fmt = pl::format();
  const bool single_path = n_cta > 512;      // very large batches: two-level finalize of the single-head path
  HeadGroup g;
  size_t smem;
  int rc;
  // every op is checked before the first launch, so a rejected call writes nothing
  for (int i0 = 0; i0 < n; i0 += kMaxGroup)
    if ((rc = head_group_chunk(ops, i0, std::min(kMaxGroup, n - i0), batch, dim, fmt, n_cta, g, smem))) return rc;
  for (int i0 = 0; i0 < n; i0 += kMaxGroup) {
    const int m = std::min(kMaxGroup, n - i0);
    if ((rc = head_group_chunk(ops, i0, m, batch, dim, fmt, n_cta, g, smem))) return rc;
    if (single_path) {
      for (int i = 0; i < m; ++i) {
        const adn_head_op& o = ops[i0 + i];
        if ((rc = run_head(g.p[i], o.workspace, o.workspace_bytes, as_stream(stream)))) return rc;
      }
      continue;
    }
    cudaStream_t st = as_stream(stream);
    switch ((int)dim) {
      case 1: launch_head_group<1>(g, n_cta, smem, st); break;
      case 2: launch_head_group<2>(g, n_cta, smem, st); break;
      case 3: launch_head_group<3>(g, n_cta, smem, st); break;
      case 4: launch_head_group<4>(g, n_cta, smem, st); break;
      case 10: launch_head_group<10>(g, n_cta, smem, st); break;
      case 16: launch_head_group<16>(g, n_cta, smem, st); break;
      default: launch_head_group<0>(g, n_cta, smem, st); break;
    }
    ADN_CHECK_LAUNCH("ensemble_head_group");
    ensemble_finalize_group_kernel<<<m, 256, 0, st>>>(g);
    ADN_CHECK_LAUNCH("ensemble_finalize_group");
  }
  return ADN_OK;
}

extern "C" int adn_head_bookkeeping(const adn_head_book* books, int n, const int64_t* step_dev, void* stream) {
  if (n < 0 || (n > 0 && !books) || !step_dev) return fail(ADN_ERR_INVALID, "adn_head_bookkeeping: bad argument");
  // every entry is checked before the first launch, so a rejected call writes nothing
  for (int i = 0; i < n; ++i) {
    const adn_head_book& b = books[i];
    if (!b.ema_state || !b.out3 || !b.sub_loss || !b.trace || b.capacity < 1)
      return fail(ADN_ERR_INVALID, "adn_head_bookkeeping: entry %d: bad argument", i);
  }
  for (int i0 = 0; i0 < n; i0 += 64) {
    const int m = std::min(64, n - i0);
    BookGroup g{};
    g.n = m;
    for (int i = 0; i < m; ++i) {
      const adn_head_book& b = books[i0 + i];
      g.e[i] = BookEntry{b.ema_state, b.out3, b.sub_loss, b.trace, b.decay, b.capacity};
    }
    head_bookkeeping_kernel<<<1, 64, 0, as_stream(stream)>>>(g, step_dev);
    ADN_CHECK_LAUNCH("head_bookkeeping");
  }
  return ADN_OK;
}
