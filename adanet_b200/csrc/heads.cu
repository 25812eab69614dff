// Fused AdaNet ensemble head (K4), plain head loss (K3), zero-debiased EMA (K6)
// and L1 norm.  HBM-bound: every member-logit element is read from DRAM once
// (pass 1), re-read from L2 for the mixture-weight gradient (pass 2), with
// coalesced float4 loads over the flat [rows*dim] tile of each member.
// Every head entry point (adn_head_group, adn_ensemble_head, adn_head_loss(_p))
// goes through one validator (head_group_op) and one launcher (run_heads) of one
// kernel family: a single head is a one-op group.  adn_head_group_wide runs the
// same ops through the same validator on a second kernel that keeps no copy of
// the members in shared memory, for heads the first one cannot hold (dim > 64,
// or members x dim past its slab); both share the finalize.
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
static constexpr size_t kHeadSmemMax = 227 * 1024;
// wide kernel (adn_head_group_wide)
static constexpr int kWThreads = 256;
static constexpr int kWMaxDim = 16384;
static constexpr int kWMaxRows = 32;              // rows per row block
static constexpr int kWRowBytes = 96 * 1024;      // smem for the row block's gradient rows: two CTAs per SM
static constexpr int kWMaxCta = 512;

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
  // wide kernel only (wide_geom): rows per row block, row blocks per CTA, smem row stride, 16 B loads allowed
  int rb, bpc, ld, vec;
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

// blockIdx.y selects one of up to kMaxGroup independent heads over the same minibatch -- the subnetwork losses and
// the candidate-ensemble heads of every candidate of the GPU in ONE launch (they only read logits the forward waves
// have produced), instead of two launches per candidate on side streams.
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
ensemble_finalize_group_kernel(const __grid_constant__ HeadGroup g) {
  const HeadParams& p = g.p[blockIdx.x];
  finalize_body(p, p.part, p.n_cta);
}

// ---- wide heads: any dim up to kWMaxDim, no per-member smem slab ----
// Four consecutive columns [c, c + nv) of a row: one 16 B load when `vec` (dim % 4 == 0 and aligned bases), else scalar
// loads of the nv <= 4 valid columns.  Either way the same elements land in the same lanes, so the arithmetic below
// does not depend on the alignment.
__device__ __forceinline__ float4 wide_ld4(const float* p, int nv, int vec) {
  if (vec) return __ldg(reinterpret_cast<const float4*>(p));
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  v.x = __ldg(p);
  if (nv > 1) v.y = __ldg(p + 1);
  if (nv > 2) v.z = __ldg(p + 2);
  if (nv > 3) v.w = __ldg(p + 3);
  return v;
}
__device__ __forceinline__ void wide_st4(float* p, float4 v, int nv, int vec) {
  if (vec) {
    *reinterpret_cast<float4*>(p) = v;
    return;
  }
  p[0] = v.x;
  if (nv > 1) p[1] = v.y;
  if (nv > 2) p[2] = v.z;
  if (nv > 3) p[3] = v.w;
}
__device__ __forceinline__ float warp_sum_xor(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One CTA = p.bpc consecutive row blocks of p.rb rows (the last CTA may own fewer; p.n_cta of them per op).
// Row phase: warp w takes rows w, w + 8, ... of the block; lane l owns the 4-column chunks l, l + 32, ... of the row:
// ens = bias + sum_k w_k (.) m_k in member order (one read of each member element from DRAM), then the head's loss
// and dLoss/d(ens) = g into the block's smem row (softmax: row max, then the sum of exponentials).  Per-row sums are a
// lane-sequential sum and a fixed xor tree.  Column phase: thread t owns columns t, t + 256, ... and adds the block's g
// rows in row order into the CTA's accumulators (dbias, VECTOR dw from an L2 re-read of the member rows; SCALAR dw from
// per-row dot products the row phase left in smem).  The accumulators live in the CTA's own contiguous slice of the
// workspace and are moved to the output-major partials the finalize reads once the CTA is done.  Every order depends
// only on (batch, dim, n_members).
// smem: g[rb][ld] | rowdot[rb][kMaxMembers] | wloss[kWThreads / 32]
__global__ void __launch_bounds__(kWThreads, 2)
ensemble_head_wide_kernel(const __grid_constant__ HeadGroup grp) {
  extern __shared__ __align__(16) float smem[];
  const HeadParams& p = grp.p[blockIdx.y];
  const int cta = blockIdx.x;
  if (cta >= p.n_cta) return;
  const int C = p.dim, N = p.n_members, ld = p.ld, rb = p.rb, vec = p.vec;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int kWarps = kWThreads / 32;
  float* grow = smem;
  float* rowdot = grow + (size_t)rb * ld;
  float* wloss = rowdot + (size_t)rb * kMaxMembers;
  const bool want_dw = p.want_grads && !(p.mixture == ADN_MIX_MATRIX || p.colsum_only);
  const bool scalar_dw = want_dw && p.mixture == ADN_MIX_SCALAR;
  const bool vector_dw = want_dw && p.mixture == ADN_MIX_VECTOR;
  const bool unit_w = p.mixture == ADN_MIX_MATRIX || p.w == nullptr;
  const int nch = (C + 3) >> 2;
  const float invb = 1.f / (float)p.batch, invn = 1.f / ((float)p.batch * (float)C);
  float* acc = p.part + (size_t)p.n_out * p.n_cta + (size_t)cta * p.n_out;   // this CTA's accumulators [n_out]
  const int64_t n_blocks = (p.batch + rb - 1) / rb;
  const int64_t b0 = (int64_t)cta * p.bpc, b1 = min(b0 + p.bpc, n_blocks);
  float wl = 0.f;                    // this warp's loss over its rows, row order

  for (int64_t blk = b0; blk < b1; ++blk) {
    const int64_t row0 = blk * rb;
    const int nrows = (int)min((int64_t)rb, p.batch - row0);
    // ---- row phase ----
    for (int s = warp; s < nrows; s += kWarps) {
      const int64_t r = row0 + s;
      const size_t roff = (size_t)r * C;
      float* e = grow + (size_t)s * ld;
      float mx = -INFINITY, lsum = 0.f;
      for (int i = lane; i < nch; i += 32) {
        const int c = i * 4, nv = min(4, C - c);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p.bias) v = wide_ld4(p.bias + c, nv, 0);
#pragma unroll 4
        for (int k = 0; k < N; ++k) {
          const float4 m = wide_ld4(p.members[k] + roff + c, nv, vec);
          float4 wk = make_float4(1.f, 1.f, 1.f, 1.f);
          if (!unit_w) {
            if (p.mixture == ADN_MIX_SCALAR) {
              const float ws = __ldg(p.w + k);
              wk = make_float4(ws, ws, ws, ws);
            } else {
              wk = wide_ld4(p.w + (size_t)k * C + c, nv, vec);
            }
          }
          v.x += wk.x * m.x;
          v.y += wk.y * m.y;
          v.z += wk.z * m.z;
          v.w += wk.w * m.w;
        }
        if (p.ens_out) wide_st4(p.ens_out + roff + c, v, nv, vec);
        float a[4] = {v.x, v.y, v.z, v.w};
        if (p.head == ADN_HEAD_SOFTMAX_XENT) {
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (q < nv) mx = fmaxf(mx, a[q]);
        } else {
          const float4 z4 = wide_ld4(p.labels_f + roff + c, nv, vec);
          const float z[4] = {z4.x, z4.y, z4.z, z4.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (q >= nv) {
              a[q] = 0.f;
              continue;
            }
            if (p.head == ADN_HEAD_MSE) {
              const float d = a[q] - z[q];
              lsum += d * d;
              a[q] = 2.f * d * invn;
            } else {
              const float x = a[q];
              lsum += fmaxf(x, 0.f) - x * z[q] + log1pf(expf(-fabsf(x)));
              a[q] = (1.f / (1.f + expf(-x)) - z[q]) * invn;
            }
          }
        }
        *reinterpret_cast<float4*>(e + c) = make_float4(a[0], a[1], a[2], a[3]);
      }
      if (p.head == ADN_HEAD_SOFTMAX_XENT) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        const int y = (int)p.labels[r];
        __syncwarp();
        const float zy = e[y] - mx;
        __syncwarp();
        float sx = 0.f;
        for (int i = lane; i < nch; i += 32) {
          const int c = i * 4, nv = min(4, C - c);
          float4 v = *reinterpret_cast<float4*>(e + c);
          v.x = expf(v.x - mx);
          v.y = nv > 1 ? expf(v.y - mx) : 0.f;
          v.z = nv > 2 ? expf(v.z - mx) : 0.f;
          v.w = nv > 3 ? expf(v.w - mx) : 0.f;
          sx += v.x;
          sx += v.y;
          sx += v.z;
          sx += v.w;
          *reinterpret_cast<float4*>(e + c) = v;
        }
        sx = warp_sum_xor(sx);
        lsum = -(zy - logf(sx));
        const float inv = 1.f / sx;
        for (int i = lane; i < nch; i += 32) {
          const int c = i * 4, nv = min(4, C - c);
          float4 v = *reinterpret_cast<float4*>(e + c);
          v.x = (v.x * inv - (c == y ? 1.f : 0.f)) * invb;
          v.y = nv > 1 ? (v.y * inv - (c + 1 == y ? 1.f : 0.f)) * invb : 0.f;
          v.z = nv > 2 ? (v.z * inv - (c + 2 == y ? 1.f : 0.f)) * invb : 0.f;
          v.w = nv > 3 ? (v.w * inv - (c + 3 == y ? 1.f : 0.f)) * invb : 0.f;
          *reinterpret_cast<float4*>(e + c) = v;
        }
      } else {
        lsum = warp_sum_xor(lsum);
      }
      wl += lsum;
      if (p.dens) {
        for (int i = lane; i < nch; i += 32) {
          const int c = i * 4, nv = min(4, C - c);
          wide_st4(p.dens + roff + c, *reinterpret_cast<const float4*>(e + c), nv, vec);
        }
      }
      if (scalar_dw) {
        // g_r . m_k per member (member row re-read from L2)
        for (int k = 0; k < N; ++k) {
          float d = 0.f;
          for (int i = lane; i < nch; i += 32) {
            const int c = i * 4, nv = min(4, C - c);
            const float4 m = wide_ld4(p.members[k] + roff + c, nv, vec);
            const float4 g = *reinterpret_cast<const float4*>(e + c);
            d += g.x * m.x;
            d += g.y * m.y;
            d += g.z * m.z;
            d += g.w * m.w;
          }
          d = warp_sum_xor(d);
          if (lane == 0) rowdot[s * kMaxMembers + k] = d;
        }
      }
    }
    __syncthreads();
    // ---- planes of g * dens_scale, zero padding columns up to the last k-block ----
    if (p.densp.hi) {
      const int pc8 = (p.dens_nkb * pl::fmt_bk(p.densp.fmt)) >> 3;
      for (int i = tid; i < nrows * pc8; i += kWThreads) {
        const int s = i / pc8, c8 = i - s * pc8;
        const float* e = grow + (size_t)s * ld;
        float m8[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int c = c8 * 8 + q;
          m8[q] = (c < C) ? e[c] * p.dens_scale : 0.f;
        }
        pl::plane_store8(p.densp, row0 + s, (int64_t)c8 * 8, m8, p.ovf);
      }
    }
    // ---- column phase: block sums in row order, added to the CTA's accumulators ----
    if (p.want_grads) {
      const bool first = blk == b0;
      for (int c = tid; c < C; c += kWThreads) {
        float t = 0.f;
        for (int s = 0; s < nrows; ++s) t += grow[(size_t)s * ld + c];
        acc[1 + c] = first ? t : acc[1 + c] + t;
        if (vector_dw) {
          for (int k = 0; k < N; ++k) {
            const float* mk = p.members[k] + (size_t)row0 * C + c;
            float d = 0.f;
            for (int s = 0; s < nrows; ++s) d += grow[(size_t)s * ld + c] * __ldg(mk + (size_t)s * C);
            float* a = acc + 1 + C + (size_t)k * C + c;
            *a = first ? d : *a + d;
          }
        }
      }
      if (scalar_dw) {
        for (int k = tid; k < N; k += kWThreads) {
          float d = 0.f;
          for (int s = 0; s < nrows; ++s) d += rowdot[s * kMaxMembers + k];
          acc[1 + C + k] = first ? d : acc[1 + C + k] + d;
        }
      }
    }
    __syncthreads();                 // the next block rewrites the smem rows
  }

  // ---- this CTA's partials, output-major (part[j * n_cta + cta]); each thread moves the accumulators it wrote ----
  float* part = p.part + cta;
  const size_t ps = (size_t)p.n_cta;
  if (lane == 0) wloss[warp] = wl;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += wloss[w];
    part[0] = t;
  }
  if (!p.want_grads) return;
  for (int c = tid; c < C; c += kWThreads) {
    part[(1 + c) * ps] = acc[1 + c];
    if (vector_dw)
      for (int k = 0; k < N; ++k) part[(1 + C + (size_t)k * C + c) * ps] = acc[1 + C + (size_t)k * C + c];
  }
  if (scalar_dw)
    for (int k = tid; k < N; k += kWThreads) part[(1 + C + k) * ps] = acc[1 + C + k];
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

// 0: the op runs on adn_head_group (dim <= 64 and its member slab fits shared memory), 1: on adn_head_group_wide
int head_path(int64_t dim, int64_t members) {
  return (dim >= 1 && dim <= kMaxDim && members >= 1 && members <= kMaxMembers &&
          head_smem_bytes((int)dim, (int)members) <= kHeadSmemMax) ? 0 : 1;
}

// Wide kernel geometry, a function of (batch, dim, members) alone: row blocks of rb rows (as many as kWRowBytes of
// gradient rows hold, up to kWMaxRows), split into n_cta runs of bpc consecutive blocks.  The CTA cap keeps the
// workspace (2 x n_out floats per CTA) near 32 MB for the widest heads and the finalize on one level.
struct WideGeom {
  int rb, ld, bpc, n_cta;
  int64_t cta_cap;       // n_cta never exceeds it, for this batch or any smaller one
};
static WideGeom wide_geom(int64_t batch, int64_t dim, int64_t members) {
  WideGeom g;
  g.ld = (int)align_up(dim, 4);
  g.rb = (int)std::max<int64_t>(1, std::min<int64_t>(kWMaxRows, kWRowBytes / (g.ld * (int64_t)sizeof(float))));
  const int64_t n_blocks = ceil_div(batch, g.rb);
  const int64_t n_out = 1 + dim + members * dim;
  const int64_t cap = std::max<int64_t>(64, std::min<int64_t>(kWMaxCta, (int64_t(1) << 22) / n_out));
  g.cta_cap = std::min(n_blocks, cap);
  g.bpc = (int)ceil_div(n_blocks, g.cta_cap);
  g.n_cta = (int)ceil_div(n_blocks, g.bpc);
  return g;
}
// partials [n_out][n_cta] | per-CTA accumulators [n_cta][n_out]
static int64_t head_wide_workspace_bytes(int64_t batch, int64_t dim, int64_t members) {
  const int64_t n_out = 1 + dim + members * dim;
  return align_up(2 * wide_geom(batch, dim, members).cta_cap * n_out * (int64_t)sizeof(float), 256);
}
static size_t head_wide_smem_bytes(int64_t dim) {
  const WideGeom g = wide_geom(1, dim, 1);
  return ((size_t)g.rb * g.ld + (size_t)g.rb * kMaxMembers + kWThreads / 32) * sizeof(float);
}

static void launch_head_group(const HeadGroup& g, int n_cta, size_t smem, cudaStream_t st) {
  const dim3 grid((unsigned)n_cta, (unsigned)g.n);
  switch (g.p[0].dim) {    // every op of a call shares dim
    case 1: ensemble_head_group_kernel<1><<<grid, kRows, smem, st>>>(g); break;
    case 2: ensemble_head_group_kernel<2><<<grid, kRows, smem, st>>>(g); break;
    case 3: ensemble_head_group_kernel<3><<<grid, kRows, smem, st>>>(g); break;
    case 4: ensemble_head_group_kernel<4><<<grid, kRows, smem, st>>>(g); break;
    case 10: ensemble_head_group_kernel<10><<<grid, kRows, smem, st>>>(g); break;
    case 16: ensemble_head_group_kernel<16><<<grid, kRows, smem, st>>>(g); break;
    default: ensemble_head_group_kernel<0><<<grid, kRows, smem, st>>>(g); break;
  }
}

int heads_init() {
#define ADN_HEAD_ATTR(CT) \
  ADN_CUDA(cudaFuncSetAttribute(ensemble_head_group_kernel<CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024))
  ADN_HEAD_ATTR(0); ADN_HEAD_ATTR(1); ADN_HEAD_ATTR(2); ADN_HEAD_ATTR(3); ADN_HEAD_ATTR(4); ADN_HEAD_ATTR(10);
  ADN_HEAD_ATTR(16);
#undef ADN_HEAD_ATTR
  ADN_CUDA(cudaFuncSetAttribute(ensemble_head_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  return ADN_OK;
}

int64_t head_workspace_bytes_public(int64_t batch, int64_t dim, int64_t members) {
  return head_workspace_bytes(batch, dim, members < 1 ? 1 : members);
}

int64_t head_wide_workspace_bytes_public(int64_t batch, int64_t dim, int64_t members) {
  return head_wide_workspace_bytes(batch < 1 ? 1 : batch, dim < 1 ? 1 : dim, members < 1 ? 1 : members);
}

// Checks one op (`what` names it in messages) and fills its launch parameters; touches no device memory.
static int head_group_op(const adn_head_op& o, const char* what, int64_t batch, int64_t dim, int fmt, int n_cta,
                         bool wide, HeadParams& p) {
  if (!o.members_host || !o.out3 || !o.workspace) return fail(ADN_ERR_INVALID, "%s: null pointer", what);
  if (o.head < 0 || o.head > 2 || o.mixture_type < 0 || o.mixture_type > 2)
    return fail(ADN_ERR_INVALID, "%s: bad head / mixture type (%d, %d)", what, o.head, o.mixture_type);
  if (o.n_members < 1 || o.n_members > kMaxMembers)
    return fail(ADN_ERR_UNSUPPORTED, "%s: n_members %d not in [1,%d]", what, o.n_members, kMaxMembers);
  if (o.mixture_type == ADN_MIX_MATRIX && o.dw) return fail(ADN_ERR_INVALID, "%s: dw must be NULL for MATRIX", what);
  if (!o.reg_is_zero && !o.gammas_host) return fail(ADN_ERR_INVALID, "%s: gammas missing", what);
  if (o.head == ADN_HEAD_SOFTMAX_XENT ? o.labels == nullptr : o.labels_f == nullptr)
    return fail(ADN_ERR_INVALID, "%s: labels missing", what);
  if (o.dz_log2_scale < -60 || o.dz_log2_scale > 60) return fail(ADN_ERR_INVALID, "%s: bad dz_log2_scale", what);
  for (int k = 0; k < o.n_members; ++k) {
    if (!o.members_host[k]) return fail(ADN_ERR_INVALID, "%s: member %d is null", what, k);
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
  const int64_t need = wide ? head_wide_workspace_bytes(batch, dim, o.n_members) : head_workspace_bytes(batch, dim, o.n_members);
  if (o.workspace_bytes < need)
    return fail(ADN_ERR_WORKSPACE, "%s: workspace %lld < %lld bytes", what, (long long)o.workspace_bytes, (long long)need);
  p.part = reinterpret_cast<float*>(o.workspace);
  p.n_cta = n_cta;
  if (wide) {
    const WideGeom g = wide_geom(batch, dim, o.n_members);
    p.n_cta = g.n_cta;
    p.rb = g.rb;
    p.bpc = g.bpc;
    p.ld = g.ld;
    // 16 B loads and stores of every row the kernel streams, when all of them are 16 B aligned
    bool al = dim % 4 == 0;
    auto a16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    for (int k = 0; k < o.n_members; ++k) al = al && a16(o.members_host[k]);
    if (o.head != ADN_HEAD_SOFTMAX_XENT) al = al && a16(o.labels_f);
    if (o.mixture_type == ADN_MIX_VECTOR && o.w) al = al && a16(o.w);
    if (o.dens) al = al && a16(o.dens);
    if (o.ens_out) al = al && a16(o.ens_out);
    p.vec = al ? 1 : 0;
  }
  return ADN_OK;
}

// Fills the launch of ops [i0, i0 + m) and the shared memory it needs.  A grouped call (`per_op`) names each op by
// its index after `what`.
static int head_group_chunk(const adn_head_op* ops, int i0, int m, int64_t batch, int64_t dim, int fmt, int n_cta,
                            const char* what, bool per_op, bool wide, HeadGroup& g, size_t& smem) {
  g = HeadGroup{};
  g.n = m;
  smem = 0;
  for (int i = 0; i < m; ++i) {
    char name[64];
    if (per_op) snprintf(name, sizeof(name), "%s: op %d", what, i0 + i);
    const int rc = head_group_op(ops[i0 + i], per_op ? name : what, batch, dim, fmt, n_cta, wide, g.p[i]);
    if (rc) return rc;
    smem = std::max(smem, wide ? head_wide_smem_bytes(dim) : head_smem_bytes(g.p[i].dim, g.p[i].n_members));
  }
  if (!wide && smem > kHeadSmemMax) return fail(ADN_ERR_UNSUPPORTED, "%s: members x dim does not fit shared memory", what);
  return ADN_OK;
}

// Every head entry point: ops over one minibatch, all checked before the first launch, so a rejected call writes
// nothing.  Up to 512 CTAs per op: one head launch and one finalize launch per kMaxGroup ops.  Beyond (very large
// batches), op by op: its head launch, one block per output summing the CTA partials of that output, and a finalize
// that sees the reduced row alone.
static int run_heads(const adn_head_op* ops, int n, int64_t batch, int64_t dim, const char* what, bool per_op,
                     cudaStream_t st) {
  if (batch <= 0 || dim <= 0 || dim > kMaxDim) return fail(ADN_ERR_INVALID, "%s: bad batch/dim", what);
  const int n_cta = (int)ceil_div(batch, kRows);
  const int fmt = pl::format();
  HeadGroup g;
  size_t smem;
  int rc;
  for (int i0 = 0; i0 < n; i0 += kMaxGroup)
    if ((rc = head_group_chunk(ops, i0, std::min(kMaxGroup, n - i0), batch, dim, fmt, n_cta, what, per_op, false, g,
                               smem)))
      return rc;
  for (int i0 = 0; i0 < n; i0 += kMaxGroup) {
    const int m = std::min(kMaxGroup, n - i0);
    if ((rc = head_group_chunk(ops, i0, m, batch, dim, fmt, n_cta, what, per_op, false, g, smem))) return rc;
    if (n_cta <= 512) {
      launch_head_group(g, n_cta, smem, st);
      ADN_CHECK_LAUNCH("ensemble_head_group");
      ensemble_finalize_group_kernel<<<m, 256, 0, st>>>(g);
      ADN_CHECK_LAUNCH("ensemble_finalize_group");
      continue;
    }
    for (int i = 0; i < m; ++i) {
      HeadGroup one{};
      one.n = 1;
      HeadParams& p = one.p[0];
      p = g.p[i];
      launch_head_group(one, n_cta, head_smem_bytes(p.dim, p.n_members), st);
      ADN_CHECK_LAUNCH("ensemble_head_group");
      const int n_red = !p.want_grads ? 1 : (p.mixture == ADN_MIX_MATRIX || p.colsum_only) ? 1 + p.dim : p.n_out;
      float* red = p.part + (size_t)n_cta * p.n_out;
      head_partials_kernel<<<n_red, 256, 0, st>>>(p.part, red, n_cta);
      ADN_CHECK_LAUNCH("head_partials");
      p.part = red;
      p.n_cta = 1;
      ensemble_finalize_group_kernel<<<1, 256, 0, st>>>(one);
      ADN_CHECK_LAUNCH("ensemble_finalize_group");
    }
  }
  return ADN_OK;
}

// adn_head_group_wide: the same ops, validation and partials as run_heads, on the wide kernel (no shared-memory fit,
// dim up to kWMaxDim).  At most kWMaxCta CTAs per op, so one head launch and one finalize launch per kMaxGroup ops.
static int run_heads_wide(const adn_head_op* ops, int n, int64_t batch, int64_t dim, cudaStream_t st) {
  const char* what = "adn_head_group_wide";
  if (n < 0 || (n > 0 && !ops)) return fail(ADN_ERR_INVALID, "%s: bad ops", what);
  if (batch <= 0) return fail(ADN_ERR_INVALID, "%s: bad batch %lld", what, (long long)batch);
  if (dim < 1 || dim > kWMaxDim)
    return fail(ADN_ERR_UNSUPPORTED, "%s: dim %lld not in [1,%d]", what, (long long)dim, kWMaxDim);
  const int fmt = pl::format();
  HeadGroup g;
  size_t smem;
  int rc;
  for (int i0 = 0; i0 < n; i0 += kMaxGroup)
    if ((rc = head_group_chunk(ops, i0, std::min(kMaxGroup, n - i0), batch, dim, fmt, 0, what, true, true, g, smem)))
      return rc;
  for (int i0 = 0; i0 < n; i0 += kMaxGroup) {
    const int m = std::min(kMaxGroup, n - i0);
    if ((rc = head_group_chunk(ops, i0, m, batch, dim, fmt, 0, what, true, true, g, smem))) return rc;
    int n_cta = 1;
    for (int i = 0; i < m; ++i) n_cta = std::max(n_cta, g.p[i].n_cta);
    ensemble_head_wide_kernel<<<dim3((unsigned)n_cta, (unsigned)m), kWThreads, smem, st>>>(g);
    ADN_CHECK_LAUNCH("ensemble_head_wide");
    ensemble_finalize_group_kernel<<<m, 256, 0, st>>>(g);
    ADN_CHECK_LAUNCH("ensemble_finalize_group");
  }
  return ADN_OK;
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
  if (!logits || !loss_out) return fail(ADN_ERR_INVALID, "adn_head_loss_p: null pointer");
  // out3 needs 3 floats; the public contract is loss_out[0], so stage through workspace tail.
  const int64_t need = head_workspace_bytes_public(batch, dim, 1);
  if (workspace_bytes < need + 16)
    return fail(ADN_ERR_WORKSPACE, "adn_head_loss_p: workspace %lld < %lld bytes", (long long)workspace_bytes,
                (long long)(need + 16));
  if (dim > kMaxDim) return fail(ADN_ERR_UNSUPPORTED, "adn_head_loss_p: dim %lld > %d", (long long)dim, kMaxDim);
  float* out3 = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + need);
  adn_head_op o{};
  o.head = head;
  o.mixture_type = ADN_MIX_SCALAR;
  o.members_host = &logits;
  o.n_members = 1;
  o.reg_is_zero = 1;
  o.dz_log2_scale = dz_log2_scale;
  o.labels = labels;
  o.labels_f = labels_f;
  o.out3 = out3;
  o.dbias = dlogits_colsum;
  o.dens = dlogits;
  o.dens_planes = dlogits_planes;
  o.colsum_only = 1;
  o.workspace = workspace;
  o.workspace_bytes = need;
  const int rc = run_heads(&o, 1, batch, dim, "adn_head_loss_p", false, as_stream(stream));
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
  if (dim > kMaxDim) return fail(ADN_ERR_UNSUPPORTED, "adn_ensemble_head: dim %lld > %d", (long long)dim, kMaxDim);
  adn_head_op o{};
  o.head = head;
  o.mixture_type = mixture_type;
  o.members_host = members_host;
  o.n_members = n_members;
  o.reg_is_zero = reg_is_zero;
  o.w = w;
  o.bias = bias;
  o.gammas_host = gammas_host;
  o.reg_multiplier = reg_multiplier;
  o.labels = labels;
  o.labels_f = labels_f;
  o.out3 = out3;
  o.dw = dw;
  o.dbias = dbias;
  o.dens = dens;
  o.ens_out = ens_out;
  o.workspace = workspace;
  o.workspace_bytes = workspace_bytes;
  return run_heads(&o, 1, batch, dim, "adn_ensemble_head", false, as_stream(stream));
}

extern "C" int adn_head_group(const adn_head_op* ops, int n, int64_t batch, int64_t dim, void* stream) {
  if (n < 0 || (n > 0 && !ops)) return fail(ADN_ERR_INVALID, "adn_head_group: bad ops");
  return run_heads(ops, n, batch, dim, "adn_head_group", true, as_stream(stream));
}

extern "C" int adn_head_group_wide(const adn_head_op* ops, int n, int64_t batch, int64_t dim, void* stream) {
  return run_heads_wide(ops, n, batch, dim, as_stream(stream));
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
