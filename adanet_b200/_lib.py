"""ctypes binding of the C-ABI in include/adanet_b200.h.

No torch types cross this boundary: tensors are passed as ``data_ptr()``
integers and the CUDA stream as its raw handle.  The shared library is built
in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a); if it is missing the
import of any compute entry point fails loudly -- there is no CPU fallback.
"""

from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libadanet_b200.so")

# constants mirrored from include/adanet_b200.h
ACT_NONE, ACT_RELU = 0, 1
HEAD_SOFTMAX_XENT, HEAD_MSE, HEAD_SIGMOID_XENT = 0, 1, 2
MIX_SCALAR, MIX_VECTOR, MIX_MATRIX = 0, 1, 2
OPT_SGD, OPT_MOMENTUM, OPT_RMSPROP, OPT_ADAM, OPT_MOMENTUM_COSINE = 0, 1, 2, 3, 4
PATH_AUTO, PATH_SIMT, PATH_TCGEN05 = 0, 1, 2
PLANES_TF32, PLANES_F16 = 0, 1
(Q_VERSION, Q_DENSE_BWD_WS, Q_HEAD_WS, Q_DENSE_FWD_PATH, Q_SM_COUNT, Q_LAUNCH_COUNT, Q_DENSE_BWD_PATH,
 Q_DENSE_FWD_WS, Q_PLANES_BYTES, Q_DENSE_BWD_P_WS, Q_COLSUM_WS, Q_CONV_STEM_BWD_WS, Q_PLANE_FORMAT,
 Q_TMA_MAP_CACHE_HITS, Q_TMA_MAP_CACHE_MISSES) = range(15)

EXPORTS = (
    "adn_last_error", "adn_init", "adn_query", "adn_set_dense_path", "adn_dense_fwd", "adn_dense_bwd", "adn_head_loss",
    "adn_ensemble_head", "adn_opt_step", "adn_l1_norm", "adn_ema_update", "adn_record_scalars",
    "adn_counter_add", "adn_planes_split", "adn_planes_merge", "adn_dense_fwd_p", "adn_dense_bwd_p", "adn_colsum",
    "adn_opt_step_p", "adn_head_loss_p", "adn_dense_fwd_p_group", "adn_dense_bwd_p_group",
    "adn_l1_grad_add", "adn_conv_stem_fwd", "adn_conv_stem_bwd", "adn_set_plane_format", "adn_plane_overflow",
    "adn_planes_split_scaled", "adn_head_group", "adn_head_bookkeeping", "adn_opt_step_group",
)


FWD_MAX_SRCS = 3      # ADN_FWD_MAX_SRCS


class FwdSrc(ctypes.Structure):
  """adn_fwd_src (include/adanet_b200.h): one more input piece of a multi-source forward op"""
  _fields_ = [("xp", c_void_p), ("wp", c_void_p), ("in_", c_int64)]


class FwdOp(ctypes.Structure):
  """adn_fwd_op (include/adanet_b200.h)"""
  _fields_ = [("xp", c_void_p), ("wp", c_void_p), ("bias", c_void_p), ("yp", c_void_p), ("y", c_void_p),
              ("in_", c_int64), ("out", c_int64), ("act", ctypes.c_int32), ("reserved", ctypes.c_int32),
              ("dropout_rate", c_float), ("dropout_seed", ctypes.c_uint32), ("dropout_layer", ctypes.c_int32),
              ("dropout_row0", ctypes.c_int32), ("dropout_step_dev", c_void_p),
              ("srcs", POINTER(FwdSrc)), ("n_srcs", ctypes.c_int32), ("reserved3", ctypes.c_int32)]


class BwdOp(ctypes.Structure):
  """adn_bwd_op (include/adanet_b200.h)"""
  _fields_ = [("xp", c_void_p), ("wp", c_void_p), ("dzp", c_void_p), ("dxp", c_void_p), ("dx", c_void_p),
              ("dx_colsum", c_void_p), ("dw", c_void_p), ("in_", c_int64), ("out", c_int64),
              ("x_relu_mask", ctypes.c_int32), ("dz_log2_scale", ctypes.c_int32), ("workspace", c_void_p),
              ("workspace_bytes", c_int64), ("dx_mul", c_float), ("reserved2", c_float)]


class HeadOp(ctypes.Structure):
  """adn_head_op (include/adanet_b200.h)"""
  _fields_ = [("head", ctypes.c_int32), ("mixture_type", ctypes.c_int32), ("members_host", POINTER(c_void_p)),
              ("n_members", ctypes.c_int32), ("reg_is_zero", ctypes.c_int32), ("w", c_void_p), ("bias", c_void_p),
              ("gammas_host", POINTER(c_float)), ("reg_multiplier", c_float), ("dz_log2_scale", ctypes.c_int32),
              ("labels", c_void_p), ("labels_f", c_void_p), ("out3", c_void_p), ("dw", c_void_p), ("dbias", c_void_p),
              ("dens", c_void_p), ("ens_out", c_void_p), ("dens_planes", c_void_p), ("colsum_only", ctypes.c_int32),
              ("reserved", ctypes.c_int32), ("workspace", c_void_p), ("workspace_bytes", c_int64)]


class HeadBook(ctypes.Structure):
  """adn_head_book (include/adanet_b200.h)"""
  _fields_ = [("ema_state", c_void_p), ("out3", c_void_p), ("sub_loss", c_void_p), ("trace", c_void_p),
              ("decay", c_float), ("capacity", ctypes.c_int32)]


class OptOp(ctypes.Structure):
  """adn_opt_op (include/adanet_b200.h)"""
  _fields_ = [("kind", ctypes.c_int32), ("n_tensors", ctypes.c_int32), ("params_host", POINTER(c_void_p)),
              ("grads_host", POINTER(c_void_p)), ("slot0_host", POINTER(c_void_p)), ("slot1_host", POINTER(c_void_p)),
              ("sizes_host", POINTER(c_int64)), ("hyper_host", POINTER(c_float)), ("step_dev", c_void_p),
              ("planes_host", POINTER(c_void_p)), ("cols_host", POINTER(c_int64))]


class AdnError(RuntimeError):
  pass


_lib = None


def load():
  """Loads (once) and returns the ctypes library, with prototypes set."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise AdnError(
        "adanet_b200 CUDA extension not built: %s is missing. Run `python -c 'import __graft_entry__ as g; "
        "g.build()'` at the repo root (needs nvcc). There is no CPU fallback." % LIB_PATH)
  lib = ctypes.CDLL(LIB_PATH)
  p, i64, f32 = c_void_p, c_int64, c_float
  lib.adn_last_error.restype = c_char_p
  lib.adn_last_error.argtypes = []
  lib.adn_init.argtypes = []
  lib.adn_query.argtypes = [c_int, i64, i64, i64, POINTER(i64)]
  lib.adn_set_dense_path.argtypes = [c_int]
  lib.adn_dense_fwd.argtypes = [p, p, p, p, i64, i64, i64, c_int, p, i64, p]
  lib.adn_dense_bwd.argtypes = [p, p, p, p, p, p, i64, i64, i64, c_int, p, i64, p]
  lib.adn_head_loss.argtypes = [c_int, p, p, p, p, p, i64, i64, p, i64, p]
  lib.adn_ensemble_head.argtypes = [c_int, c_int, POINTER(p), c_int, p, p, POINTER(f32), c_int, f32, p, p,
                                    p, p, p, p, p, i64, i64, p, i64, p]
  lib.adn_opt_step.argtypes = [c_int, POINTER(p), POINTER(p), POINTER(p), POINTER(p), POINTER(i64), c_int,
                               POINTER(f32), p, p]
  lib.adn_l1_norm.argtypes = [p, i64, p, p]
  lib.adn_ema_update.argtypes = [p, p, f32, p]
  lib.adn_record_scalars.argtypes = [POINTER(p), c_int, p, i64, p, i64, p]
  lib.adn_counter_add.argtypes = [p, i64, p]
  lib.adn_planes_split.argtypes = [p, i64, i64, p, p]
  lib.adn_planes_split_scaled.argtypes = [p, i64, i64, p, c_int, p]
  lib.adn_planes_merge.argtypes = [p, i64, i64, p, p]
  lib.adn_set_plane_format.argtypes = [c_int]
  lib.adn_plane_overflow.argtypes = [POINTER(c_int), c_int, p]
  lib.adn_dense_fwd_p.argtypes = [p, p, p, p, p, i64, i64, i64, c_int, p]
  lib.adn_dense_bwd_p.argtypes = [p, p, p, p, p, p, p, i64, i64, i64, c_int, c_int, p, i64, p]
  lib.adn_colsum.argtypes = [p, i64, i64, p, p, i64, p]
  lib.adn_head_loss_p.argtypes = [c_int, p, p, p, p, p, p, p, c_int, i64, i64, p, i64, p]
  lib.adn_l1_grad_add.argtypes = [p, p, i64, f32, p]
  lib.adn_conv_stem_fwd.argtypes = [p, p, p, p, p, i64, c_int, c_int, c_int, c_int, p]
  lib.adn_conv_stem_bwd.argtypes = [p, p, p, p, p, i64, c_int, c_int, c_int, c_int, p, i64, p]
  lib.adn_dense_fwd_p_group.argtypes = [POINTER(FwdOp), c_int, i64, p]
  lib.adn_dense_bwd_p_group.argtypes = [POINTER(BwdOp), c_int, i64, p]
  lib.adn_opt_step_p.argtypes = [c_int, POINTER(p), POINTER(p), POINTER(p), POINTER(p), POINTER(i64), c_int,
                                 POINTER(f32), p, POINTER(p), POINTER(i64), p]
  lib.adn_head_group.argtypes = [POINTER(HeadOp), c_int, i64, i64, p]
  lib.adn_head_bookkeeping.argtypes = [POINTER(HeadBook), c_int, p, p]
  lib.adn_opt_step_group.argtypes = [POINTER(OptOp), c_int, p]
  for name in EXPORTS:
    if name != "adn_last_error":
      getattr(lib, name).restype = c_int
  _lib = lib
  return lib


def check(rc: int, what: str = ""):
  if rc != 0:
    msg = load().adn_last_error().decode("utf-8", "replace")
    raise AdnError("%s failed (%d): %s" % (what or "adanet_b200 call", rc, msg))


def query(key: int, a: int = 0, b: int = 0, c: int = 0) -> int:
  out = c_int64(0)
  check(load().adn_query(key, a, b, c, ctypes.byref(out)), "adn_query")
  return int(out.value)


def launch_count() -> int:
  return query(Q_LAUNCH_COUNT)


def set_dense_path(path: int):
  check(load().adn_set_dense_path(path), "adn_set_dense_path")


def plane_format() -> int:
  """Current split-plane format of the *_p entry points (PLANES_F16 unless ADN_PLANES=tf32 / set_plane_format)."""
  return query(Q_PLANE_FORMAT)


def set_plane_format(fmt: int):
  check(load().adn_set_plane_format(fmt), "adn_set_plane_format")


def plane_overflow(stream_ptr: int = 0, reset: bool = True) -> bool:
  """Reads (and by default clears) the sticky "a finite value did not fit fp16 planes" flag; synchronises the stream."""
  out = c_int(0)
  check(load().adn_plane_overflow(ctypes.byref(out), 1 if reset else 0, stream_ptr), "adn_plane_overflow")
  return bool(out.value)


def ptr_array(ptrs):
  arr = (c_void_p * len(ptrs))()
  for i, v in enumerate(ptrs):
    arr[i] = v
  return arr


def f32_array(vals):
  arr = (c_float * len(vals))()
  for i, v in enumerate(vals):
    arr[i] = float(v)
  return arr


def i64_array(vals):
  arr = (c_int64 * len(vals))()
  for i, v in enumerate(vals):
    arr[i] = int(v)
  return arr
