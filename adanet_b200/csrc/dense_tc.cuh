// Tensor-core split-plane dense path (planes.cu): TMA-fed wgmma / mma.sync, register accumulators.
// See dense_tc.cu for the design.  Entry points mirror dense_simt.cuh.
#pragma once
#include "common.cuh"

namespace adn {
namespace tc {

int init();
bool fwd_supported(int64_t batch, int64_t in, int64_t out);
bool bwd_supported(int64_t batch, int64_t in, int64_t out);
int64_t dense_bwd_workspace_bytes(int64_t batch, int64_t in, int64_t out);
int64_t dense_fwd_workspace_bytes(int64_t batch, int64_t in, int64_t out);
int dense_fwd(const float* x, const float* w, const float* b, float* y, int64_t batch, int64_t in,
              int64_t out, int act, void* ws, int64_t ws_bytes, cudaStream_t st);
int dense_bwd(const float* x, const float* w, const float* dz, float* dx, float* dw, float* db,
              int64_t batch, int64_t in, int64_t out, int x_relu_mask, void* ws, int64_t ws_bytes,
              cudaStream_t st);

}  // namespace tc
}  // namespace adn
