// fp32-in / fp32-out entry points of the tcgen05 dense path (adn_dense_fwd / adn_dense_bwd with
// ADN_PATH_TCGEN05 or AUTO): the operands are split into TF32 hi/lo planes (always TF32 here: the caller's
// gradient magnitudes are unknown, so no fp16 scale can be chosen for it) in the caller's
// workspace and the plane-native GEMM of planes.cu does the rest.  A subnetwork that keeps its
// activations in plane format (adn_dense_fwd_p / adn_dense_bwd_p, what core/engine.py runs) never
// pays these conversion passes; this file exists so that the row-major fp32 ABI stays a drop-in.
//
// Reference arithmetic being replaced: tf.layers.dense / tf.matmul and their gradients,
//   adanet/examples/simple_dnn.py:72-86,103-110.
#include "dense_simt.cuh"
#include "dense_tc.cuh"
#include "planes.cuh"

namespace adn {
namespace tc {

int init() { return pl::init(); }

// the tensor path pays a split pre-pass per call: skinny layers stay on CUDA cores in AUTO mode
bool fwd_supported(int64_t batch, int64_t in, int64_t out) { return batch >= 128 && in >= 32 && out >= 64; }
bool bwd_supported(int64_t batch, int64_t in, int64_t out) { return batch >= 128 && in >= 32 && out >= 64; }

static inline int64_t pbytes(int64_t rows, int64_t cols) { return align_up(pl::planes_bytes(pl::FMT_TF32, rows, cols), 256); }

int64_t dense_fwd_workspace_bytes(int64_t batch, int64_t in, int64_t out) {
  if (!fwd_supported(batch, in, out)) return 0;
  return pbytes(batch, in) + pbytes(in, out) + 512;
}

int64_t dense_bwd_workspace_bytes(int64_t batch, int64_t in, int64_t out) {
  if (!bwd_supported(batch, in, out)) return 0;
  return pbytes(batch, in) + pbytes(in, out) + pbytes(batch, out) + align_up(pl::dense_bwd_workspace_bytes(batch, in, out), 256) +
         align_up(64 * out * (int64_t)sizeof(float), 256) + 512;
}

struct Carver {
  char* p;
  char* end;
  bool ok = true;
  void* take(int64_t bytes) {
    bytes = align_up(bytes, 256);
    if (p + bytes > end) { ok = false; return nullptr; }
    void* r = p;
    p += bytes;
    return r;
  }
};

static Carver carver(void* ws, int64_t ws_bytes) {
  return Carver{reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255),
                reinterpret_cast<char*>(ws) + ws_bytes};
}

int dense_fwd(const float* x, const float* w, const float* b, float* y, int64_t batch, int64_t in, int64_t out,
              int act, void* ws, int64_t ws_bytes, cudaStream_t st) {
  if (!ws || ws_bytes < dense_fwd_workspace_bytes(batch, in, out))
    return fail(ADN_ERR_WORKSPACE, "tc dense_fwd: workspace %lld < %lld bytes", (long long)ws_bytes,
                (long long)dense_fwd_workspace_bytes(batch, in, out));
  Carver c = carver(ws, ws_bytes);
  void* xp = c.take(pl::planes_bytes(pl::FMT_TF32, batch, in));
  void* wp = c.take(pl::planes_bytes(pl::FMT_TF32, in, out));
  if (!c.ok) return fail(ADN_ERR_WORKSPACE, "tc dense_fwd: workspace carve failed");
  int rc;
  if ((rc = pl::split(pl::FMT_TF32, x, batch, in, xp, 0, st))) return rc;
  if ((rc = pl::split(pl::FMT_TF32, w, in, out, wp, 0, st))) return rc;
  return pl::dense_fwd(pl::FMT_TF32, xp, wp, b, nullptr, y, batch, in, out, act, st);
}

int dense_bwd(const float* x, const float* w, const float* dz, float* dx, float* dw, float* db, int64_t batch,
              int64_t in, int64_t out, int x_relu_mask, void* ws, int64_t ws_bytes, cudaStream_t st) {
  if (!ws || ws_bytes < dense_bwd_workspace_bytes(batch, in, out))
    return fail(ADN_ERR_WORKSPACE, "tc dense_bwd: workspace %lld < %lld bytes", (long long)ws_bytes,
                (long long)dense_bwd_workspace_bytes(batch, in, out));
  Carver c = carver(ws, ws_bytes);
  void* xp = c.take(pl::planes_bytes(pl::FMT_TF32, batch, in));
  void* wp = c.take(pl::planes_bytes(pl::FMT_TF32, in, out));
  void* dzp = c.take(pl::planes_bytes(pl::FMT_TF32, batch, out));
  const int64_t inner = pl::dense_bwd_workspace_bytes(batch, in, out);
  void* inner_ws = c.take(inner);
  float* dbpart = reinterpret_cast<float*>(c.take(64 * out * (int64_t)sizeof(float)));
  if (!c.ok) return fail(ADN_ERR_WORKSPACE, "tc dense_bwd: workspace carve failed");
  int rc;
  if ((rc = pl::split(pl::FMT_TF32, x, batch, in, xp, 0, st))) return rc;     // also yields the sign bits used as the ReLU mask
  if ((rc = pl::split(pl::FMT_TF32, dz, batch, out, dzp, 0, st))) return rc;
  if (dx && (rc = pl::split(pl::FMT_TF32, w, in, out, wp, 0, st))) return rc;
  const simt::ColsumJob db_job{dz, db, batch, out, dbpart};
  if (db && (rc = simt::colsum_group(&db_job, 1, st))) return rc;
  return pl::dense_bwd(pl::FMT_TF32, xp, wp, dzp, nullptr, dx, nullptr, dw, batch, in, out, x_relu_mask, 0, inner_ws, inner, st);
}

}  // namespace tc
}  // namespace adn
