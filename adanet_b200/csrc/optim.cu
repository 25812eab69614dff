// K5: TF1 optimizer update rules, one launch for all parameter tensors of a
// candidate (multi-tensor apply).  HBM-bound elementwise work: float4 where
// the tensors are 16B-aligned, grid sized to the work.
//
// Replaces the apply half of optimizer.minimize at
//   adanet/examples/simple_dnn.py:110 and adanet/ensemble/weighted.py:616.
// Update rules are TensorFlow 1.x's (not vendored by the reference):
//   GradientDescent  v -= lr*g
//   Momentum         acc = m*acc + g ; v -= lr*acc
//   RMSProp          ms = rho*ms + (1-rho) g^2 ; mom = mu*mom + lr*g/sqrt(ms+eps) ; v -= mom   (ms init 1)
//   Adam             lr_t = lr*sqrt(1-b2^t)/(1-b1^t) ; m += (1-b1)(g-m) ; v += (1-b2)(g^2-v) ;
//                    var -= lr_t*m/(sqrt(v)+eps)
//   Momentum+cosine  Momentum with lr_t = tf.train.cosine_decay(lr, step, decay_steps, alpha) read from the
//                    device step counter (customizing_adanet.ipynb SimpleCNNBuilder.build_subnetwork_train_op)
#include "common.cuh"
#include "plane_fmt.cuh"

namespace adn {

static constexpr int kMaxTensors = 32;     // per optimizer (ABI)
static constexpr int kMaxGroupTensors = 96; // per launch
static constexpr int kMaxGroupOpts = 32;    // optimizers per launch
static constexpr int kChunk = 4096;         // elements per CTA

// One launch applies several optimizers (adn_opt_step_group): tensor t belongs to optimizer opt[t].
struct OptParams {
  float* p[kMaxGroupTensors];
  const float* g[kMaxGroupTensors];
  float* s0[kMaxGroupTensors];
  float* s1[kMaxGroupTensors];
  // optional split planes of 2-D parameters, refreshed with the update (plane_fmt.cuh layout)
  void* plane_hi[kMaxGroupTensors];    // hi plane base (nullable per tensor)
  void* plane_lo[kMaxGroupTensors];
  int64_t size[kMaxGroupTensors];
  int chunk_start[kMaxGroupTensors + 1];  // prefix sum of chunks per tensor
  int cols[kMaxGroupTensors];
  unsigned char opt[kMaxGroupTensors];
  int n;
  int kind[kMaxGroupOpts];
  float h0[kMaxGroupOpts], h1[kMaxGroupOpts], h2[kMaxGroupOpts], h3[kMaxGroupOpts];
  const int64_t* step_dev[kMaxGroupOpts];
  int fmt;
  unsigned int* ovf;
};

__device__ __forceinline__ void store_planes(const OptParams& o, int t, int64_t j, float v) {
  if (!o.plane_hi[t]) return;
  const int cols = o.cols[t];
  const int64_t rows = o.size[t] / cols;
  const int64_t r = j / cols;
  const int c = (int)(j - r * cols);
  pl::plane_store(pl::PlaneView{o.plane_hi[t], o.plane_lo[t], nullptr, rows, o.fmt}, r, c, v, o.ovf);
}

// four consecutive elements j..j+3 (j a multiple of 4): when the row length is a multiple of 4 they share a row and a
// k-block, so one 32-bit division locates them and each plane takes one 8 B (fp16) / 16 B (TF32) store
__device__ __forceinline__ void store_planes4(const OptParams& o, int t, int64_t j, const float4& v) {
  if (!o.plane_hi[t]) return;
  const int cols = o.cols[t];
  if ((cols & 3) != 0 || o.size[t] > 0x7fffffffLL) {
    store_planes(o, t, j, v.x); store_planes(o, t, j + 1, v.y);
    store_planes(o, t, j + 2, v.z); store_planes(o, t, j + 3, v.w);
    return;
  }
  const int ji = (int)j, r = ji / cols, c = ji - r * cols;
  const int64_t rows = (int)o.size[t] / cols;
  if (o.fmt == pl::FMT_F16) {
    __half h[4], l[4];
    pl::split_f16(v.x, h[0], l[0]); pl::split_f16(v.y, h[1], l[1]);
    pl::split_f16(v.z, h[2], l[2]); pl::split_f16(v.w, h[3], l[3]);
    if (pl::f16_overflows(v.x) | pl::f16_overflows(v.y) | pl::f16_overflows(v.z) | pl::f16_overflows(v.w)) pl::raise_overflow(o.ovf);
    const int64_t dst = ((int64_t)(c >> 6) * rows + r) * 64 + (c & 63);
    const uint2 hw = make_uint2((uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16),
                                (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16));
    const uint2 lw = make_uint2((uint32_t)__half_as_ushort(l[0]) | ((uint32_t)__half_as_ushort(l[1]) << 16),
                                (uint32_t)__half_as_ushort(l[2]) | ((uint32_t)__half_as_ushort(l[3]) << 16));
    *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(o.plane_hi[t]) + dst) = hw;
    *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(o.plane_lo[t]) + dst) = lw;
  } else {
    float4 h, l;
    pl::split_tf32(v.x, h.x, l.x); pl::split_tf32(v.y, h.y, l.y);
    pl::split_tf32(v.z, h.z, l.z); pl::split_tf32(v.w, h.w, l.w);
    const int64_t dst = ((int64_t)(c >> 5) * rows + r) * 32 + (c & 31);
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(o.plane_hi[t]) + dst) = h;
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(o.plane_lo[t]) + dst) = l;
  }
}

__device__ __forceinline__ void apply_one(int kind, float& p, float g, float& s0, float& s1, float h0, float h1,
                                          float h2, float h3, float lr_t) {
  switch (kind) {
    case ADN_OPT_SGD:
      p -= h0 * g;
      break;
    case ADN_OPT_MOMENTUM:
      s0 = h1 * s0 + g;
      p -= h0 * s0;
      break;
    case ADN_OPT_MOMENTUM_COSINE:
      s0 = h1 * s0 + g;
      p -= lr_t * s0;
      break;
    case ADN_OPT_RMSPROP:
      s0 = h1 * s0 + (1.f - h1) * g * g;
      s1 = h2 * s1 + h0 * g / sqrtf(s0 + h3);
      p -= s1;
      break;
    default:  // ADAM
      s0 += (1.f - h1) * (g - s0);
      s1 += (1.f - h2) * (g * g - s1);
      p -= lr_t * s0 / (sqrtf(s1) + h3);
      break;
  }
}

__global__ void __launch_bounds__(256) opt_step_kernel(const __grid_constant__ OptParams o) {
  // locate the tensor of this CTA (binary search over the chunk prefix sums)
  int lo = 0, hi = o.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((int)blockIdx.x >= o.chunk_start[mid]) lo = mid; else hi = mid - 1;
  }
  const int t = lo;
  const int q = o.opt[t];
  const int kind = o.kind[q];
  const float h0 = o.h0[q], h1 = o.h1[q], h2 = o.h2[q], h3 = o.h3[q];
  const int64_t off = (int64_t)(blockIdx.x - o.chunk_start[t]) * kChunk;
  const int64_t end = min(o.size[t], off + kChunk);
  float* p = o.p[t];
  const float* g = o.g[t];
  float* s0 = o.s0[t];
  float* s1 = o.s1[t];
  float lr_t = h0;
  if (kind == ADN_OPT_ADAM) {
    const float tt = (float)(*o.step_dev[q] + 1);
    lr_t = h0 * sqrtf(1.f - powf(h2, tt)) / (1.f - powf(h1, tt));
  } else if (kind == ADN_OPT_MOMENTUM_COSINE) {
    // tf.train.cosine_decay [TF]: step clipped to decay_steps, fp32 arithmetic
    const float st = fminf((float)(*o.step_dev[q]), h2);
    const float cosine = 0.5f * (1.f + cosf(3.14159265358979323846f * (st / h2)));
    lr_t = h0 * ((1.f - h3) * cosine + h3);
  }
  const bool vec = (((uintptr_t)p | (uintptr_t)g | (uintptr_t)s0 | (uintptr_t)s1) & 15) == 0;
  if (vec) {
    for (int64_t i = off + threadIdx.x * 4; i < end; i += 256 * 4) {
      if (i + 3 < end) {
        float4 pv = *reinterpret_cast<float4*>(p + i);
        float4 gv = __ldg(reinterpret_cast<const float4*>(g + i));
        float4 a = s0 ? *reinterpret_cast<float4*>(s0 + i) : make_float4(0, 0, 0, 0);
        float4 b = s1 ? *reinterpret_cast<float4*>(s1 + i) : make_float4(0, 0, 0, 0);
        apply_one(kind, pv.x, gv.x, a.x, b.x, h0, h1, h2, h3, lr_t);
        apply_one(kind, pv.y, gv.y, a.y, b.y, h0, h1, h2, h3, lr_t);
        apply_one(kind, pv.z, gv.z, a.z, b.z, h0, h1, h2, h3, lr_t);
        apply_one(kind, pv.w, gv.w, a.w, b.w, h0, h1, h2, h3, lr_t);
        *reinterpret_cast<float4*>(p + i) = pv;
        store_planes4(o, t, i, pv);
        if (s0) *reinterpret_cast<float4*>(s0 + i) = a;
        if (s1) *reinterpret_cast<float4*>(s1 + i) = b;
      } else {
        for (int64_t j = i; j < end; ++j) {
          float pv = p[j], a = s0 ? s0[j] : 0.f, b = s1 ? s1[j] : 0.f;
          apply_one(kind, pv, g[j], a, b, h0, h1, h2, h3, lr_t);
          p[j] = pv;
          store_planes(o, t, j, pv);
          if (s0) s0[j] = a;
          if (s1) s1[j] = b;
        }
      }
    }
  } else {
    for (int64_t j = off + threadIdx.x; j < end; j += 256) {
      float pv = p[j], a = s0 ? s0[j] : 0.f, b = s1 ? s1[j] : 0.f;
      apply_one(kind, pv, g[j], a, b, h0, h1, h2, h3, lr_t);
      p[j] = pv;
      store_planes(o, t, j, pv);
      if (s0) s0[j] = a;
      if (s1) s1[j] = b;
    }
  }
}

struct StepPtrs {
  int64_t* p[kMaxGroupOpts];
  int n;
};
__global__ void step_increment_group_kernel(const __grid_constant__ StepPtrs s) {
  if ((int)threadIdx.x < s.n) *s.p[threadIdx.x] += 1;
}
__global__ void step_increment_kernel(int64_t* step) { *step += 1; }

}  // namespace adn

using namespace adn;


extern "C" int adn_opt_step(int kind, float* const* params_host, const float* const* grads_host,
                            float* const* slot0_host, float* const* slot1_host, const int64_t* sizes_host,
                            int n_tensors, const float* hyper_host, int64_t* step_dev, void* stream) {
  return adn_opt_step_p(kind, params_host, grads_host, slot0_host, slot1_host, sizes_host, n_tensors, hyper_host,
                        step_dev, nullptr, nullptr, stream);
}

namespace adn {
static int n_slots(int kind) {
  return kind == ADN_OPT_SGD ? 0 : ((kind == ADN_OPT_MOMENTUM || kind == ADN_OPT_MOMENTUM_COSINE) ? 1 : 2);
}

// checks one optimizer of a call; returns 0 or an error
static int check_optimizer(const adn_opt_op& op, const char* what) {
  const int kind = op.kind;
  if (kind < ADN_OPT_SGD || kind > ADN_OPT_MOMENTUM_COSINE) return fail(ADN_ERR_INVALID, "%s: bad kind %d", what, kind);
  if (op.n_tensors < 1 || op.n_tensors > kMaxTensors)
    return fail(ADN_ERR_UNSUPPORTED, "%s: n_tensors %d not in [1,%d]", what, op.n_tensors, kMaxTensors);
  if (!op.params_host || !op.grads_host || !op.sizes_host || !op.hyper_host) return fail(ADN_ERR_INVALID, "%s: null pointer", what);
  const int need_slots = n_slots(kind);
  if (need_slots >= 1 && !op.slot0_host) return fail(ADN_ERR_INVALID, "%s: slot0 required", what);
  if (need_slots >= 2 && !op.slot1_host) return fail(ADN_ERR_INVALID, "%s: slot1 required", what);
  if ((kind == ADN_OPT_ADAM || kind == ADN_OPT_MOMENTUM_COSINE) && !op.step_dev)
    return fail(ADN_ERR_INVALID, "%s: Adam / cosine-decay Momentum need step_dev", what);
  if (kind == ADN_OPT_MOMENTUM_COSINE && !(op.hyper_host[2] > 0.f))
    return fail(ADN_ERR_INVALID, "%s: cosine decay needs decay_steps > 0", what);
  for (int i = 0; i < op.n_tensors; ++i) {
    if (!op.params_host[i] || !op.grads_host[i] || op.sizes_host[i] <= 0)
      return fail(ADN_ERR_INVALID, "%s: tensor %d null or empty", what, i);
    if ((need_slots >= 1 && !op.slot0_host[i]) || (need_slots >= 2 && !op.slot1_host[i]))
      return fail(ADN_ERR_INVALID, "%s: slot for tensor %d is null", what, i);
    if (op.planes_host && op.planes_host[i] &&
        (!op.cols_host || op.cols_host[i] <= 0 || op.sizes_host[i] % op.cols_host[i] != 0 || op.cols_host[i] > INT32_MAX))
      return fail(ADN_ERR_INVALID, "%s: tensor %d: cols must divide its size", what, i);
  }
  return ADN_OK;
}

// appends one checked optimizer's tensors to the launch description
static void add_optimizer(OptParams& o, StepPtrs& steps, int& chunks, int q, const adn_opt_op& op) {
  const int kind = op.kind;
  const int need_slots = n_slots(kind);
  for (int i = 0; i < op.n_tensors; ++i) {
    const int t = o.n;
    o.p[t] = op.params_host[i];
    o.g[t] = op.grads_host[i];
    o.s0[t] = need_slots >= 1 ? op.slot0_host[i] : nullptr;
    o.s1[t] = need_slots >= 2 ? op.slot1_host[i] : nullptr;
    o.size[t] = op.sizes_host[i];
    o.plane_hi[t] = nullptr;
    if (op.planes_host && op.planes_host[i]) {
      const pl::PlaneView v = pl::plane_view(pl::format(), op.planes_host[i], op.sizes_host[i] / op.cols_host[i], op.cols_host[i]);
      o.plane_hi[t] = v.hi;
      o.plane_lo[t] = v.lo;
      o.cols[t] = (int)op.cols_host[i];
    }
    o.opt[t] = (unsigned char)q;
    o.chunk_start[t] = chunks;
    chunks += (int)ceil_div(op.sizes_host[i], kChunk);
    o.n = t + 1;
  }
  o.kind[q] = kind;
  o.h0[q] = op.hyper_host[0];
  o.h1[q] = kind >= ADN_OPT_MOMENTUM ? op.hyper_host[1] : 0.f;
  o.h2[q] = kind >= ADN_OPT_RMSPROP ? op.hyper_host[2] : 0.f;
  o.h3[q] = kind >= ADN_OPT_RMSPROP ? op.hyper_host[3] : 0.f;   // MOMENTUM_COSINE (4): {lr, momentum, decay_steps, alpha}
  o.step_dev[q] = op.step_dev;
  if (op.step_dev) steps.p[steps.n++] = op.step_dev;
}

static int flush(OptParams& o, StepPtrs& steps, int& chunks, cudaStream_t st) {
  if (o.n == 0) return ADN_OK;
  o.chunk_start[o.n] = chunks;
  o.fmt = pl::format();
  o.ovf = pl::overflow_flag();
  opt_step_kernel<<<chunks, 256, 0, st>>>(o);
  ADN_CHECK_LAUNCH("opt_step");
  if (steps.n > 0) {
    step_increment_group_kernel<<<1, kMaxGroupOpts, 0, st>>>(steps);
    ADN_CHECK_LAUNCH("step_increment");
  }
  o.n = 0;
  steps.n = 0;
  chunks = 0;
  return ADN_OK;
}
}  // namespace adn

extern "C" int adn_opt_step_group(const adn_opt_op* ops, int n, void* stream) {
  if (n < 0 || (n > 0 && !ops)) return fail(ADN_ERR_INVALID, "adn_opt_step_group: bad ops");
  static thread_local OptParams o;          // ~8 KB: keep it off the stack of deep Python call chains
  static thread_local StepPtrs steps;
  o.n = 0;
  steps.n = 0;
  int chunks = 0, q = 0, rc;
  // every op is checked before the first launch, so a rejected call changes no parameter, slot, plane or step counter
  for (int i = 0; i < n; ++i) {
    if (ops[i].n_tensors > kMaxTensors || ops[i].n_tensors < 1)
      return fail(ADN_ERR_UNSUPPORTED, "adn_opt_step_group: op %d: n_tensors %d not in [1,%d]", i, ops[i].n_tensors, kMaxTensors);
    char what[48];
    snprintf(what, sizeof(what), "adn_opt_step_group: op %d", i);
    if ((rc = check_optimizer(ops[i], what))) return rc;
  }
  for (int i = 0; i < n; ++i) {
    if (o.n + ops[i].n_tensors > kMaxGroupTensors || q == kMaxGroupOpts) {
      if ((rc = flush(o, steps, chunks, as_stream(stream)))) return rc;
      q = 0;
    }
    add_optimizer(o, steps, chunks, q, ops[i]);
    ++q;
  }
  return flush(o, steps, chunks, as_stream(stream));
}

extern "C" int adn_opt_step_p(int kind, float* const* params_host, const float* const* grads_host,
                              float* const* slot0_host, float* const* slot1_host, const int64_t* sizes_host,
                              int n_tensors, const float* hyper_host, int64_t* step_dev,
                              void* const* planes_host, const int64_t* cols_host, void* stream) {
  adn_opt_op op{};
  op.kind = kind;
  op.n_tensors = n_tensors;
  op.params_host = params_host;
  op.grads_host = grads_host;
  op.slot0_host = slot0_host;
  op.slot1_host = slot1_host;
  op.sizes_host = sizes_host;
  op.hyper_host = hyper_host;
  op.step_dev = step_dev;
  op.planes_host = planes_host;
  op.cols_host = cols_host;
  return adn_opt_step_group(&op, 1, stream);
}
