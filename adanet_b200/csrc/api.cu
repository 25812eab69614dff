// C-ABI glue: error state, queries, dense path dispatch (SIMT fp32 vs tensor-core split planes).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "dense_simt.cuh"
#include "dense_tc.cuh"
#include "planes.cuh"

namespace adn {
namespace conv { int64_t bwd_workspace_bytes(int64_t batch, int cin, int f); int init(); }
namespace convtc { int init(); }

thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};
static std::atomic<int> g_path{ADN_PATH_AUTO};
static std::atomic<int> g_sm_count{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int sm_count() {
  int v = g_sm_count.load();
  if (v > 0) return v;
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
    (void)cudaGetLastError();
    n = 132;  // H100 SXM
  }
  g_sm_count.store(n);
  return n;
}

int dense_path() {
  static bool env_read = false;
  if (!env_read) {
    env_read = true;
    const char* e = getenv("ADN_DENSE_PATH");
    if (e) {
      if (!strcmp(e, "simt")) g_path.store(ADN_PATH_SIMT);
      else if (!strcmp(e, "tcgen05")) g_path.store(ADN_PATH_TCGEN05);
      else if (!strcmp(e, "auto")) g_path.store(ADN_PATH_AUTO);
    }
  }
  return g_path.load();
}

int64_t head_workspace_bytes_public(int64_t batch, int64_t dim, int64_t members);
int heads_init();
int heads_group_init();

}  // namespace adn

using namespace adn;

extern "C" const char* adn_last_error(void) { return g_err; }

extern "C" int adn_init(void) {
  static std::atomic<int> done{0};
  if (done.load()) return ADN_OK;
  int rc = heads_init();
  if (rc) return rc;
  rc = heads_group_init();
  if (rc) return rc;
  rc = pl::init();
  if (rc) return rc;
  rc = conv::init();
  if (rc) return rc;
  rc = convtc::init();
  if (rc) return rc;
  (void)sm_count();
  done.store(1);
  return ADN_OK;
}

extern "C" int adn_set_dense_path(int path) {
  if (path < ADN_PATH_AUTO || path > ADN_PATH_TCGEN05) return fail(ADN_ERR_INVALID, "adn_set_dense_path: bad path %d", path);
  (void)dense_path();  // consume env first so an explicit call wins
  g_path.store(path);
  return ADN_OK;
}

static int pick_fwd_path(int64_t batch, int64_t in, int64_t out) {
  const int p = dense_path();
  if (p == ADN_PATH_SIMT) return ADN_PATH_SIMT;
  return tc::fwd_supported(batch, in, out) ? ADN_PATH_TCGEN05 : (p == ADN_PATH_TCGEN05 ? -1 : ADN_PATH_SIMT);
}

static int pick_bwd_path(int64_t batch, int64_t in, int64_t out) {
  const int p = dense_path();
  if (p == ADN_PATH_SIMT) return ADN_PATH_SIMT;
  return tc::bwd_supported(batch, in, out) ? ADN_PATH_TCGEN05 : (p == ADN_PATH_TCGEN05 ? -1 : ADN_PATH_SIMT);
}

extern "C" int adn_query(int key, int64_t a, int64_t b, int64_t c, int64_t* out_host) {
  if (!out_host) return fail(ADN_ERR_INVALID, "adn_query: null out");
  switch (key) {
    case ADN_Q_VERSION: *out_host = 100; return ADN_OK;
    case ADN_Q_DENSE_BWD_WORKSPACE_BYTES: {
      int64_t s = simt::dense_bwd_workspace_bytes(a, b, c);
      int64_t t = tc::dense_bwd_workspace_bytes(a, b, c);
      *out_host = s > t ? s : t;
      return ADN_OK;
    }
    case ADN_Q_DENSE_FWD_WORKSPACE_BYTES:
      *out_host = (pick_fwd_path(a, b, c) == ADN_PATH_TCGEN05) ? tc::dense_fwd_workspace_bytes(a, b, c) : 0;
      return ADN_OK;
    case ADN_Q_HEAD_WORKSPACE_BYTES: *out_host = head_workspace_bytes_public(a, b, c) + 256; return ADN_OK;
    case ADN_Q_DENSE_FWD_PATH: *out_host = pick_fwd_path(a, b, c); return ADN_OK;
    case ADN_Q_DENSE_BWD_PATH: *out_host = pick_bwd_path(a, b, c); return ADN_OK;
    case ADN_Q_SM_COUNT: *out_host = sm_count(); return ADN_OK;
    case ADN_Q_PLANES_BYTES: *out_host = pl::planes_bytes(pl::format(), a, b); return ADN_OK;
    case ADN_Q_PLANE_FORMAT: *out_host = pl::format(); return ADN_OK;
    case ADN_Q_TMA_MAP_CACHE_HITS: *out_host = pl::map_cache_hits(); return ADN_OK;
    case ADN_Q_TMA_MAP_CACHE_MISSES: *out_host = pl::map_cache_misses(); return ADN_OK;
    case ADN_Q_DENSE_BWD_P_WORKSPACE_BYTES: *out_host = pl::dense_bwd_workspace_bytes(a, b, c); return ADN_OK;
    case ADN_Q_COLSUM_WORKSPACE_BYTES: *out_host = 64 * b * (int64_t)sizeof(float) + 256; return ADN_OK;
    case ADN_Q_CONV_STEM_BWD_WORKSPACE_BYTES: *out_host = conv::bwd_workspace_bytes(a, (int)b, (int)c); return ADN_OK;
    case ADN_Q_LAUNCH_COUNT: *out_host = g_launches.load(); return ADN_OK;
    default: return fail(ADN_ERR_INVALID, "adn_query: unknown key %d", key);
  }
}

extern "C" int adn_dense_fwd(const float* x, const float* w, const float* b, float* y, int64_t batch, int64_t in,
                             int64_t out, int act, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!x || !w || !y) return fail(ADN_ERR_INVALID, "adn_dense_fwd: null pointer");
  if (batch <= 0 || in <= 0 || out <= 0 || batch > INT32_MAX || in > INT32_MAX || out > INT32_MAX)
    return fail(ADN_ERR_INVALID, "adn_dense_fwd: bad shape [%lld,%lld]x[%lld,%lld]", (long long)batch,
                (long long)in, (long long)in, (long long)out);
  if (act != ADN_ACT_NONE && act != ADN_ACT_RELU) return fail(ADN_ERR_INVALID, "adn_dense_fwd: bad act %d", act);
  const int path = pick_fwd_path(batch, in, out);
  if (path < 0)
    return fail(ADN_ERR_UNSUPPORTED, "adn_dense_fwd: tcgen05 path forced but shape [%lld,%lld,%lld] unsupported",
                (long long)batch, (long long)in, (long long)out);
  if (path == ADN_PATH_TCGEN05)
    return tc::dense_fwd(x, w, b, y, batch, in, out, act, workspace, workspace_bytes, as_stream(stream));
  return simt::dense_fwd(x, w, b, y, batch, in, out, act, as_stream(stream));
}

extern "C" int adn_dense_bwd(const float* x, const float* w, const float* dz, float* dx, float* dw, float* db,
                             int64_t batch, int64_t in, int64_t out, int x_relu_mask, void* workspace,
                             int64_t workspace_bytes, void* stream) {
  if (!x || !dz || !dw || !workspace) return fail(ADN_ERR_INVALID, "adn_dense_bwd: null pointer");
  if (dx && !w) return fail(ADN_ERR_INVALID, "adn_dense_bwd: w required when dx requested");
  if (batch <= 0 || in <= 0 || out <= 0 || batch > INT32_MAX || in > INT32_MAX || out > INT32_MAX)
    return fail(ADN_ERR_INVALID, "adn_dense_bwd: bad shape");
  const int path = pick_bwd_path(batch, in, out);
  if (path < 0)
    return fail(ADN_ERR_UNSUPPORTED, "adn_dense_bwd: tcgen05 path forced but shape [%lld,%lld,%lld] unsupported",
                (long long)batch, (long long)in, (long long)out);
  if (path == ADN_PATH_TCGEN05)
    return tc::dense_bwd(x, w, dz, dx, dw, db, batch, in, out, x_relu_mask, workspace, workspace_bytes,
                         as_stream(stream));
  return simt::dense_bwd(x, w, dz, dx, dw, db, batch, in, out, x_relu_mask, workspace, workspace_bytes,
                         as_stream(stream));
}

static bool bad_shape(int64_t a, int64_t b, int64_t c) {
  return a <= 0 || b <= 0 || c <= 0 || a > INT32_MAX || b > INT32_MAX || c > INT32_MAX;
}

extern "C" int adn_set_plane_format(int fmt) { return pl::set_format(fmt); }

extern "C" int adn_plane_overflow(int* flag_host, int reset, void* stream) {
  if (!flag_host) return fail(ADN_ERR_INVALID, "adn_plane_overflow: null pointer");
  return pl::read_overflow(flag_host, reset, as_stream(stream));
}

extern "C" int adn_planes_split_scaled(const float* src, int64_t rows, int64_t cols, void* planes, int log2_scale,
                                       void* stream) {
  if (!src || !planes) return fail(ADN_ERR_INVALID, "adn_planes_split: null pointer");
  if (bad_shape(rows, cols, 1)) return fail(ADN_ERR_INVALID, "adn_planes_split: bad shape");
  if (log2_scale < -60 || log2_scale > 60) return fail(ADN_ERR_INVALID, "adn_planes_split: bad log2_scale %d", log2_scale);
  return pl::split(pl::format(), src, rows, cols, planes, log2_scale, as_stream(stream));
}

extern "C" int adn_planes_split(const float* src, int64_t rows, int64_t cols, void* planes, void* stream) {
  return adn_planes_split_scaled(src, rows, cols, planes, 0, stream);
}

extern "C" int adn_planes_merge(const void* planes, int64_t rows, int64_t cols, float* dst, void* stream) {
  if (!planes || !dst) return fail(ADN_ERR_INVALID, "adn_planes_merge: null pointer");
  if (bad_shape(rows, cols, 1)) return fail(ADN_ERR_INVALID, "adn_planes_merge: bad shape");
  return pl::merge(pl::format(), planes, rows, cols, dst, as_stream(stream));
}

extern "C" int adn_dense_fwd_p(const void* xp, const void* wp, const float* b, void* yp, float* y, int64_t batch,
                               int64_t in, int64_t out, int act, void* stream) {
  if (!xp || !wp) return fail(ADN_ERR_INVALID, "adn_dense_fwd_p: null pointer");
  if ((yp == nullptr) == (y == nullptr)) return fail(ADN_ERR_INVALID, "adn_dense_fwd_p: exactly one of yp / y");
  if (bad_shape(batch, in, out)) return fail(ADN_ERR_INVALID, "adn_dense_fwd_p: bad shape");
  if (act != ADN_ACT_NONE && act != ADN_ACT_RELU) return fail(ADN_ERR_INVALID, "adn_dense_fwd_p: bad act %d", act);
  return pl::dense_fwd(pl::format(), xp, wp, b, yp, y, batch, in, out, act, as_stream(stream));
}

extern "C" int adn_dense_bwd_p(const void* xp, const void* wp, const void* dzp, void* dxp, float* dx,
                               float* dx_colsum, float* dw, int64_t batch, int64_t in, int64_t out, int x_relu_mask,
                               int dz_log2_scale, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!xp || !dzp || !workspace) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p: null pointer");
  if ((dxp || dx) && !wp) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p: wp required when dx requested");
  if (dxp && dx) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p: at most one of dxp / dx");
  if (dx_colsum && !(dxp || dx)) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p: dx_colsum needs dx");
  if (bad_shape(batch, in, out)) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p: bad shape");
  if (dz_log2_scale < -60 || dz_log2_scale > 60) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p: bad dz_log2_scale");
  return pl::dense_bwd(pl::format(), xp, wp, dzp, dxp, dx, dx_colsum, dw, batch, in, out, x_relu_mask, dz_log2_scale,
                       workspace, workspace_bytes, as_stream(stream));
}

extern "C" int adn_colsum(const float* x, int64_t rows, int64_t cols, float* out, void* workspace,
                          int64_t workspace_bytes, void* stream) {
  if (!x || !out || !workspace) return fail(ADN_ERR_INVALID, "adn_colsum: null pointer");
  if (bad_shape(rows, cols, 1)) return fail(ADN_ERR_INVALID, "adn_colsum: bad shape");
  if (workspace_bytes < 64 * cols * (int64_t)sizeof(float))
    return fail(ADN_ERR_WORKSPACE, "adn_colsum: workspace too small");
  return simt::colsum(x, out, rows, cols, reinterpret_cast<float*>(workspace), as_stream(stream));
}

extern "C" int adn_dense_fwd_p_group(const adn_fwd_op* ops, int n, int64_t batch, void* stream) {
  if (n < 0 || (n > 0 && !ops)) return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: bad ops");
  if (n > 256) return fail(ADN_ERR_UNSUPPORTED, "adn_dense_fwd_p_group: n %d > 256", n);
  pl::FwdOp o[256];
  pl::FwdSrc srcs[256][ADN_FWD_MAX_SRCS];
  for (int i = 0; i < n; ++i) {
    if (!ops[i].xp || !ops[i].wp) return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: null pointer", i);
    const int ns = ops[i].n_srcs;
    if (ns < 0 || ns > ADN_FWD_MAX_SRCS || (ns > 0 && !ops[i].srcs))
      return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: n_srcs %d (0..%d, srcs non-NULL)", i, ns, ADN_FWD_MAX_SRCS);
    int64_t k_total = ops[i].in;
    for (int q = 0; q < ns; ++q) {
      const adn_fwd_src& s = ops[i].srcs[q];
      if (!s.xp || !s.wp) return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: piece %d: null pointer", i, q);
      if (bad_shape(batch, s.in, ops[i].out))
        return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: piece %d: bad shape (in %lld)", i, q, (long long)s.in);
      if (!pl::planes_aligned(s.xp) || !pl::planes_aligned(s.wp))
        return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: piece %d: plane buffers must be 256 B aligned", i, q);
      srcs[i][q] = pl::FwdSrc{s.xp, s.wp, s.in};
      k_total += s.in;
    }
    if (ns > 0 && k_total > INT32_MAX) return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: total K too large", i);
    if ((ops[i].yp == nullptr) == (ops[i].y == nullptr))
      return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: exactly one of yp / y", i);
    if (bad_shape(batch, ops[i].in, ops[i].out)) return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: bad shape", i);
    if (ops[i].act != ADN_ACT_NONE && ops[i].act != ADN_ACT_RELU)
      return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: bad act %d", i, ops[i].act);
    o[i] = pl::FwdOp{ops[i].xp, ops[i].wp, ops[i].bias, ops[i].yp, ops[i].y, ops[i].in, ops[i].out, ops[i].act};
    if (ns > 0) {
      o[i].srcs = srcs[i];
      o[i].n_srcs = ns;
    }
    if (ops[i].dropout_rate != 0.f) {
      if (!(ops[i].dropout_rate > 0.f && ops[i].dropout_rate < 1.f) || !ops[i].yp || !ops[i].dropout_step_dev)
        return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: dropout needs 0 < rate < 1, planes out and a step counter", i);
      if (ops[i].dropout_row0 < 0) return fail(ADN_ERR_INVALID, "adn_dense_fwd_p_group: op %d: dropout_row0 < 0", i);
      o[i].dropout_row0 = ops[i].dropout_row0;
      o[i].dropout_rate = ops[i].dropout_rate;
      o[i].dropout_seed = ops[i].dropout_seed;
      o[i].dropout_layer = ops[i].dropout_layer;
      o[i].dropout_step = ops[i].dropout_step_dev;
    }
  }
  return pl::dense_fwd_group(pl::format(), o, n, batch, as_stream(stream));
}

extern "C" int adn_dense_bwd_p_group(const adn_bwd_op* ops, int n, int64_t batch, void* stream) {
  if (n < 0 || (n > 0 && !ops)) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p_group: bad ops");
  if (n > 256) return fail(ADN_ERR_UNSUPPORTED, "adn_dense_bwd_p_group: n %d > 256", n);
  pl::BwdOp o[256];
  for (int i = 0; i < n; ++i) {
    const adn_bwd_op& p = ops[i];
    if (!p.xp || !p.dzp || !p.workspace) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p_group: op %d: null pointer", i);
    if ((p.dxp || p.dx) && !p.wp) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p_group: op %d: wp required for dx", i);
    if (p.dxp && p.dx) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p_group: op %d: at most one of dxp / dx", i);
    if (p.dx_colsum && !(p.dxp || p.dx)) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p_group: op %d: dx_colsum needs dx", i);
    if (bad_shape(batch, p.in, p.out)) return fail(ADN_ERR_INVALID, "adn_dense_bwd_p_group: op %d: bad shape", i);
    if (p.dz_log2_scale < -60 || p.dz_log2_scale > 60)
      return fail(ADN_ERR_INVALID, "adn_dense_bwd_p_group: op %d: bad dz_log2_scale", i);
    o[i] = pl::BwdOp{p.xp, p.wp, p.dzp, p.dxp, p.dx, p.dx_colsum, p.dw, p.in, p.out, p.x_relu_mask, p.dz_log2_scale,
                     p.workspace, p.workspace_bytes};
    if (p.dx_mul != 0.f) o[i].dx_mul = p.dx_mul;
  }
  return pl::dense_bwd_group(pl::format(), o, n, batch, as_stream(stream));
}
