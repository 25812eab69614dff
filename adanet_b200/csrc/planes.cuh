// Plane-native tensor-core dense pipeline (see planes.cu for the design, plane_fmt.cuh for the formats).
#pragma once
#include "common.cuh"
#include "plane_fmt.cuh"

namespace adn {
namespace pl {

int init();
int set_format(int fmt);
int read_overflow(int* out_host, int reset, cudaStream_t st);
long long map_cache_hits();
long long map_cache_misses();
int64_t dense_bwd_workspace_bytes(int64_t batch, int64_t in, int64_t out);

// src * 2^log2_scale -> planes (+ sign bits)
int split(int fmt, const float* src, int64_t rows, int64_t cols, void* planes, int log2_scale, cudaStream_t st);
int merge(int fmt, const void* planes, int64_t rows, int64_t cols, float* dst, cudaStream_t st);
// one dense layer of one subnetwork; groups = the same layer wave of several subnetworks in one launch
struct FwdSrc {         // one more input piece of a multi-source forward (include/adanet_b200.h adn_fwd_src)
  const void* xp;       // planes [batch, in]
  const void* wp;       // planes [in, out]
  int64_t in;
};
struct FwdOp {
  const void* xp;       // planes [batch, in]
  const void* wp;       // planes [in, out]
  const float* bias;    // [out] or null
  void* yp;             // planes [batch, out] (exactly one of yp / y)
  float* y;             // dense  [batch, out]
  int64_t in, out;
  int act;
  float dropout_rate = 0.f;          // tf.layers.dropout on the output (planes out), see include/adanet_b200.h
  uint32_t dropout_seed = 0;
  int dropout_layer = 0;
  int64_t dropout_row0 = 0;          // first minibatch row of a row slice: the mask is the full batch's
  const int64_t* dropout_step = nullptr;
  const FwdSrc* srcs = nullptr;      // y = act(x w + sum_q srcs[q].x srcs[q].w + b), n_srcs <= ADN_FWD_MAX_SRCS
  int n_srcs = 0;
};
struct BwdOp {
  const void* xp;       // planes [batch, in]
  const void* wp;       // planes [in, out] (needed when dx is requested)
  const void* dzp;      // planes [batch, out], holding dz * 2^dz_log2_scale
  void* dxp;            // planes [batch, in] or null (keeps the scale of dzp)
  float* dx;            // dense  [batch, in] or null (at most one of dxp / dx; un-scaled)
  float* dx_colsum;     // [in] or null (un-scaled)
  float* dw;            // dense [in, out] or null (un-scaled)
  int64_t in, out;
  int x_relu_mask;
  int dz_log2_scale;
  void* ws;             // dense_bwd_workspace_bytes(batch, in, out), one per op
  int64_t ws_bytes;
  float dx_mul = 1.f;   // dx (planes or dense) is multiplied by this: 1 / (1 - rate) below a dropped-out activation
};
// The alignment every GEMM operand plane is checked against (include/adanet_b200.h asks callers for 256 B; the TMA
// descriptors need 128 B).
inline bool planes_aligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 127) == 0; }
int dense_fwd_group(int fmt, const FwdOp* ops, int n, int64_t batch, cudaStream_t st);
int dense_bwd_group(int fmt, const BwdOp* ops, int n, int64_t batch, cudaStream_t st);
// exactly one of yp (planes out) / y (dense fp32 out) is non-null
int dense_fwd(int fmt, const void* xp, const void* wp, const float* bias, void* yp, float* y, int64_t batch, int64_t in,
              int64_t out, int act, cudaStream_t st);
// dw nullable; at most one of dxp (planes) / dx (dense); dx_colsum[in] = column sums of dx (nullable)
int dense_bwd(int fmt, const void* xp, const void* wp, const void* dzp, void* dxp, float* dx, float* dx_colsum, float* dw,
              int64_t batch, int64_t in, int64_t out, int x_relu_mask, int dz_log2_scale, void* ws, int64_t ws_bytes,
              cudaStream_t st);

}  // namespace pl
}  // namespace adn
